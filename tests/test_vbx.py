"""VBx x-vector path: CPU host-logic tests + GPU parity tests (K4 features, K5 ResNet101)."""
import ctypes
import os

import numpy as np
import pytest

torch = pytest.importorskip('torch')


# ------------------------------------------------------------------ CPU
def test_vbx_oracle_features_golden(golden, media):
    """oracle restatement == real features_vbx.py (goldens made by make_golden.py)."""
    import hashlib
    from oracle import segmenter_oracle as so, vbx_oracle as vx
    sig = so.read_wav_16k_mono(os.path.join(media, 'lamartine.wav'), dtype='float64')
    cases = {'lamartine': sig, 'synth': golden['synth_sig'].astype(np.float64),
             'short': golden['synth_sig'][:16000 * 2 + 77].astype(np.float64)}
    for name, s in cases.items():
        fea = vx.get_features(s)
        assert len(fea) == int(golden['vbx_%s_M' % name])
        assert np.array_equal(fea[golden['vbx_%s_rows' % name]], golden['vbx_%s_fea' % name])
        assert hashlib.sha256(np.ascontiguousarray(fea).tobytes()).hexdigest() == str(golden['vbx_%s_sha' % name])


def test_vbx_host_tables_and_plan():
    from inaspeechsegmenter_b200 import vbx_segmenter as vb
    from oracle import vbx_oracle as vx
    assert np.array_equal(vb.mel_fbank_htk64(), vx.mel_bank()) and np.count_nonzero(vx.mel_bank()) == 475   # SURVEY V3
    assert np.array_equal(vb.povey_window(), vx.povey_window())
    d = vb.DitherCache('cpu').get(1000).numpy()[:1000]
    assert np.array_equal(d, vx.dither_stream(1000))
    for M in (5, 9, 10, 33, 34, 35, 143, 144, 145, 167, 168, 169, 170, 200, 1464):
        assert vb.window_plan(M) == vx.window_plan(M)


def test_resnet_oracle_golden(golden):
    """functional ResNet101 restatement == real resnet.py output stored in the golden file."""
    from oracle import vbx_oracle as vx
    net = vx.ResNet101Oracle(vx.synthetic_resnet101_state(seed=5), threads=4)
    y = net.forward(torch.from_numpy(golden['resnet_x'][:1]))
    assert np.allclose(y.numpy(), golden['resnet_y'][:1], rtol=0, atol=1e-4 * np.abs(golden['resnet_y']).max())


def test_resnet_blob_layout():
    from inaspeechsegmenter_b200 import _lib, vbx_segmenter as vb
    from oracle import vbx_oracle as vx
    sd = vx.synthetic_resnet101_state(seed=5)
    blob = vb.resnet_blob_from_state(sd)
    nb = (ctypes.c_int * 4)(*vb.NUM_BLOCKS)
    need = _lib.load().iss_resnet_blob_len(32, 64, 256, ctypes.cast(nb, ctypes.c_void_p))
    assert blob.size == need
    nparam = sum(v.numel() for k, v in sd.items() if 'running' not in k)
    assert abs(nparam - 14.84e6) < 0.05e6            # SURVEY fact 9: 14.84 M parameters


# ------------------------------------------------------------------ GPU
gpu = pytest.mark.gpu


def _lib_mod():
    from inaspeechsegmenter_b200 import _lib
    return _lib


@pytest.fixture(scope='module')
def vctx():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from inaspeechsegmenter_b200 import engine
    return engine.Context(0)


@gpu
def test_k4_features_vs_reference_golden(vctx, golden, media):
    from inaspeechsegmenter_b200 import vbx_segmenter as vb
    from oracle import segmenter_oracle as so, vbx_oracle as vx
    fe = vb.VbxFrontEnd(vctx)
    sig = so.read_wav_16k_mono(os.path.join(media, 'lamartine.wav'), dtype='float32')
    cases = {'lamartine': sig, 'synth': golden['synth_sig'], 'short': golden['synth_sig'][:16000 * 2 + 77]}
    for name, s in cases.items():
        ref = vx.get_features(s.astype(np.float64))
        got = fe(torch.from_numpy(np.ascontiguousarray(s, dtype=np.float32)).cuda()).cpu().numpy()
        assert got.shape == ref.shape == (int(golden['vbx_%s_M' % name]), 64)
        err = np.abs(got - ref).max()
        exact = float((got == ref).mean())
        assert err <= 2e-6, (name, err)                 # float64 pipeline, float32 output: <= 1-2 ulp
        assert exact > 0.98, (name, exact)
        assert np.abs(got[golden['vbx_%s_rows' % name]] - golden['vbx_%s_fea' % name]).max() <= 2e-6
    # int16 PCM input == the same samples as float
    s16 = np.round(golden['synth_sig'] * 32768).astype(np.int16)
    a = fe(torch.from_numpy(s16).cuda())
    b = fe(torch.from_numpy(golden['synth_sig']).cuda())
    assert torch.equal(a, b)
    # the public helper
    assert np.abs(vb.get_features(golden['synth_sig'].astype(np.float64)) - vx.get_features(golden['synth_sig'].astype(np.float64))).max() <= 2e-6


@gpu
def test_k5_resnet_vs_oracle(vctx, golden):
    from inaspeechsegmenter_b200 import vbx_segmenter as vb
    from oracle import vbx_oracle as vx
    sd = vx.synthetic_resnet101_state(seed=5)
    ext = vb.B200BackendExtractor(state_dict=sd, ctx=vctx)
    assert abs(ext.flops_per_window - 11.30e9) < 0.05e9       # SURVEY fact 9: 5.65 GMAC per 64x144 window
    x, y = golden['resnet_x'], golden['resnet_y']              # produced by the REAL resnet.py
    scale = np.abs(y).max()
    lib = _lib_mod().load()
    prev = lib.iss_get_gemm_mode()
    # tolerance relative to max|y| after 104 convolution layers: fp32 CUDA-core engine 2e-5;
    # tensor-core engines 1e-4 (their 3-product split drops the lo . lo term, ~2^-22 per product).
    # The reference's own check of this network is 4 decimals (run_test.py:189-195); the layer-level
    # float64 bound is test_resnet_probes_gpu.py's.
    try:
        for mode, tol in ((0, 2e-5), (2, 1e-4), (3, 1e-4)):
            lib.iss_set_gemm_mode(mode)
            for i in range(len(x)):
                got = ext.get_embedding(x[i].T)                    # get_embedding takes [T, 64]
                assert np.abs(got - y[i]).max() <= tol * scale, (mode, np.abs(got - y[i]).max() / scale)
            got = ext.get_embedding(golden['resnet_xs'][0].T)      # tail-window length 131
            assert np.abs(got - golden['resnet_ys'][0]).max() <= tol * np.abs(golden['resnet_ys']).max(), mode
    finally:
        lib.iss_set_gemm_mode(prev)


@gpu
def test_k5_residual_layer_modes_are_bit_identical(vctx):
    """ResNet101 x-vectors on window counts that leave a partial 128-row tile at the end of every stage: the default engine
    (fp16 split, split-half words between layers) gives the same x-vectors bit for bit when run again, and agrees with the
    3xTF32 engine and the fp32 CUDA-core engine within the tensor-core tolerance."""
    from inaspeechsegmenter_b200 import vbx_segmenter as vb
    from oracle import vbx_oracle as vx
    ext = vb.B200BackendExtractor(state_dict=vx.synthetic_resnet101_state(seed=5), ctx=vctx)
    lib = _lib_mod().load()
    prev = lib.iss_get_gemm_mode()
    g = torch.Generator(device='cpu').manual_seed(3)
    try:
        for nwin in (37, 256 + 5, 700):                               # partial tiles / one sweep + a remainder / several sweeps
            fea = torch.randn(24 * nwin + 144, 64, generator=g).cuda()
            starts = np.arange(nwin) * 24
            out = {}
            for mode in (3, 2, 0):
                lib.iss_set_gemm_mode(mode)
                out[mode] = ext.embed_windows(fea, starts, 144).cpu().numpy()
            lib.iss_set_gemm_mode(3)
            again = ext.embed_windows(fea, starts, 144).cpu().numpy()
            ref = out[3]
            assert np.isfinite(ref).all() and np.abs(ref).max() > 0
            assert np.array_equal(again, ref), nwin
            for mode in (2, 0):
                assert np.abs(out[mode] - ref).max() <= 2e-4 * np.abs(ref).max(), (nwin, mode, float(np.abs(out[mode] - ref).max()))
    finally:
        lib.iss_set_gemm_mode(prev)


@gpu
def test_vbx_extractor_call_vs_oracle(vctx, golden):
    """B200BackendExtractor.__call__ (batched) == the reference windowing loop with the oracle network."""
    from inaspeechsegmenter_b200 import vbx_segmenter as vb
    from oracle import vbx_oracle as vx
    sd = vx.synthetic_resnet101_state(seed=5)
    ext = vb.B200BackendExtractor(state_dict=sd, ctx=vctx)
    fea = vx.get_features(golden['synth_sig'].astype(np.float64))[:330]     # 8 regular windows + a tail
    ref = vx.extract_xvectors(fea, vx.ResNet101Oracle(sd), 'clip', 3.3)
    got = ext('clip', fea, 3.3)
    assert [(k, s) for k, s, _ in got] == [(k, s) for k, s, _ in ref]
    scale = max(np.abs(x).max() for _, _, x in ref)
    for (_, _, a), (_, _, b) in zip(got, ref):
        assert np.abs(a - b).max() <= 2e-4 * scale


def _synthetic_mlp(seed=3):
    rng = np.random.default_rng(seed)
    L, W = [{'class_name': 'InputLayer', 'config': {'name': 'in', 'batch_input_shape': [None, 256]}}], {}
    dims = [256, 128, 64, 1]
    for i in range(3):
        n = 'dense_%d' % i
        W[n + '/kernel'] = (rng.standard_normal((dims[i], dims[i + 1])) * np.sqrt(1.0 / dims[i])).astype(np.float32)
        W[n + '/bias'] = rng.normal(0, 0.1, dims[i + 1]).astype(np.float32)
        L.append({'class_name': 'Dense', 'config': {'name': n, 'units': dims[i + 1], 'use_bias': True,
                                                    'activation': 'sigmoid' if i == 2 else 'relu'}})
        if i == 0:
            b = 'bn_0'
            W[b + '/gamma'] = rng.uniform(0.8, 1.2, 128).astype(np.float32); W[b + '/beta'] = rng.normal(0, 0.1, 128).astype(np.float32)
            W[b + '/moving_mean'] = rng.normal(0, 0.1, 128).astype(np.float32); W[b + '/moving_variance'] = rng.uniform(0.5, 1.5, 128).astype(np.float32)
            L.append({'class_name': 'BatchNormalization', 'config': {'name': b, 'axis': -1, 'epsilon': 1e-3}})
        if i < 2:
            L.append({'class_name': 'Dropout', 'config': {'name': 'do_%d' % i, 'rate': 0.3}})
    return {'class_name': 'Sequential', 'config': {'name': 'mlp', 'layers': L}}, W


def test_vfs_glue_matches_oracle_cpu():
    """Interval bookkeeping of VoiceFemininityScoring (no GPU): product helpers vs the oracle restatement."""
    from inaspeechsegmenter_b200 import vbx_segmenter as vb
    from oracle import vfs_oracle
    rng = np.random.default_rng(5)
    vad = [('noEnergy', 0.0, 1.0), ('speech', 1.0, 4.2), ('music', 4.2, 6.0), ('speech', 6.0, 6.9), ('noise', 6.9, 9.0), ('speech', 9.0, 12.0)]
    xv = [('k%d' % i, (round(i * 0.24, 3), round(i * 0.24 + 1.44, 3)), rng.standard_normal(256).astype(np.float32)) for i in range(44)]
    cfg, w = _synthetic_mlp()
    mlp = lambda x: vfs_oracle.mlp_numpy(cfg, w, x)                       # noqa: E731
    for thresh in (0.62, 0.7, 0.99):
        ref = vfs_oracle.femininity(vad, xv, mlp, thresh)

        class Fake:
            vad_thresh = thresh
        speech = [(b, e) for lab, b, e in vad if lab == 'speech']
        kept = vb.VoiceFemininityScoring.apply_vad(Fake, list(xv), speech)
        p = mlp(np.asarray([x for _, _, x in kept]))
        p = np.squeeze(p) if len(p) > 1 else p
        got = (vb.get_femininity_score([(s[0], s[1], pi) for (_, s, _), pi in zip(kept, p)]), sum(e - b for b, e in speech), len(kept))
        assert got[0] == ref[0] and abs(got[1] - ref[1]) < 1e-12 and got[2] == ref[2], (thresh, got, ref)


@gpu
def test_vfs_end_to_end_vs_oracle(vctx, synth_models):
    """VoiceFemininityScoring on a synthetic clip: VAD + K4 + K5 + device MLP + glue == oracle pipeline."""
    import sys
    sys.path.insert(0, os.path.dirname(__file__))
    from conftest import synth_audio
    from inaspeechsegmenter_b200 import vbx_segmenter as vb
    from oracle import cnn_oracle, segmenter_oracle as so, vbx_oracle as vx, vfs_oracle
    import warnings
    sd = vx.synthetic_resnet101_state(seed=5)
    cfg, w = _synthetic_mlp()
    s16 = synth_audio(30, seed=42)
    vfs = vb.VoiceFemininityScoring('vfp', ffmpeg=None, models={'vad': synth_models['smn'], 'mlp': (cfg, w), 'resnet': sd})
    got = vfs.score_signal(s16, 'clip')
    # oracle pipeline
    mspec, loge, difflen = so.media2feats(s16.astype(np.float32) / np.float32(32768))
    v = so.DnnSegmenterOracle(cnn_oracle.KerasLikeModel(*synth_models['smn']), **so.VAD_SMN)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        vad_seg = so.segment_feats(mspec, loge, difflen, 0, v, None)
    fea = vx.get_features(s16.astype(np.float64) / 32768.0)
    xv = vx.extract_xvectors(fea, vx.ResNet101Oracle(sd, threads=8), 'clip', len(s16) / 16000)
    ref = vfs_oracle.femininity(vad_seg, xv, lambda x: vfs_oracle.mlp_numpy(cfg, w, x), 0.62)
    assert got[2] == ref[2] and abs(got[1] - ref[1]) < 1e-9, (got, ref)
    assert got[0] == ref[0] or (got[0] is not None and abs(got[0] - ref[0]) <= 1.0 / max(ref[2], 1)), (got, ref)
    # device MLP vs numpy on the same inputs
    x = np.asarray([x for _, _, x in xv])
    assert np.abs(vfs.gender_detection_mlp_model.predict(x) - vfs_oracle.mlp_numpy(cfg, w, x)).max() <= 1e-5
