"""GPU parity tests (run with -m gpu on an H100): every CUDA kernel, called
through the C ABI, against the CPU oracle on the same seeded inputs and against
the committed reference goldens.  Nothing here reads /root/reference."""
import json
import os

import numpy as np
import pytest

from conftest import synth_audio

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REPORT = {}


@pytest.fixture(scope='module')
def rt():
    """Runtime handles shared by the module."""
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from inaspeechsegmenter_b200 import _lib, engine
    from inaspeechsegmenter_b200.sidekit_mfcc import SidekitFrontEnd
    ctx = engine.Context(0)
    return dict(ctx=ctx, fe=SidekitFrontEnd(ctx), lib=_lib, engine=engine)


@pytest.fixture(scope='module', autouse=True)
def _dump_report():
    yield
    os.makedirs(os.path.join(ROOT, 'gpurun_out'), exist_ok=True)
    with open(os.path.join(ROOT, 'gpurun_out', 'parity_report.json'), 'w') as f:
        json.dump(REPORT, f, indent=1, sort_keys=True)


def _signals(golden, media):
    from oracle import segmenter_oracle as so
    return {
        'musanmix': so.read_wav_16k_mono(os.path.join(media, 'musanmix.wav')),
        'silence2sec': so.read_wav_16k_mono(os.path.join(media, 'silence2sec.wav')),
        'lamartine': so.read_wav_16k_mono(os.path.join(media, 'lamartine.wav')),
        'synth': golden['synth_sig'],
        'gen60': synth_audio(60).astype(np.float32) / np.float32(32768),
    }


# ------------------------------------------------------------------ K1
@pytest.mark.parametrize('prec', ['fp64', 'fp32'])
def test_k1_features_vs_oracle(rt, golden, media, prec):
    from oracle import sidekit_oracle as sk
    lib = rt['lib']
    mode = lib.FFT_FP64 if prec == 'fp64' else lib.FFT_FP32
    # tolerance on log-mel (log units).  fp64 mode follows the reference's own
    # precision recipe, fp32 mode is bounded by single-precision FFT round-off.
    tol_mspec = 2e-5 if prec == 'fp64' else 5e-2
    for name, sig in _signals(golden, media).items():
        mspec_o, loge_o = sk.logmel_loge(sig)
        pcm = torch.from_numpy(np.ascontiguousarray(sig, dtype=np.float32)).cuda()
        mspec, loge, stats = rt['fe'](pcm, mode)
        torch.cuda.synchronize()
        mspec, loge, stats = mspec.cpu().numpy(), loge.cpu().numpy(), stats.cpu().numpy()
        assert mspec.shape == mspec_o.shape and loge.shape == loge_o.shape
        # -inf pattern (silent frames) must match exactly
        assert np.array_equal(np.isfinite(mspec), np.isfinite(mspec_o)), name
        assert np.array_equal(np.isfinite(loge), np.isfinite(loge_o)), name
        fin = np.isfinite(mspec_o)
        err = np.abs(mspec[fin] - mspec_o[fin]).max() if fin.any() else 0.0
        finl = np.isfinite(loge_o)
        errl = np.abs(loge[finl] - loge_o[finl]).max() if finl.any() else 0.0
        REPORT['k1_%s_%s' % (prec, name)] = dict(mspec_max_abs=float(err), loge_max_abs=float(errl),
                                                 exact_frac=float((mspec[fin] == mspec_o[fin]).mean()) if fin.any() else 1.0)
        assert err <= tol_mspec, (name, err)
        assert errl <= 2e-6 * max(1.0, np.abs(loge_o[finl]).max() if finl.any() else 1.0), (name, errl)
        assert stats[1] == finl.sum()
        if finl.any():
            assert abs(stats[0] - loge_o[finl].astype(np.float64).sum()) <= 1e-5 * finl.sum()


def test_k1_int16_equals_float32_input(rt):
    s16 = synth_audio(20, seed=5)
    f32 = s16.astype(np.float32) / np.float32(32768)
    a = rt['fe'](torch.from_numpy(s16).cuda(), rt['lib'].FFT_FP64)
    b = rt['fe'](torch.from_numpy(f32).cuda(), rt['lib'].FFT_FP64)
    torch.cuda.synchronize()
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])


def test_k1_unaligned_and_tiny_inputs(rt):
    from oracle import sidekit_oracle as sk
    s16 = synth_audio(3, seed=9)
    base = torch.from_numpy(np.concatenate((np.zeros(1, np.int16), s16))).cuda()
    for n in (400, 401, 559, 560, 719, 720, 10479, 10480, 10481, 16000 * 3):
        view = base[1:1 + n]                       # 2-byte aligned only
        mspec, loge, stats = rt['fe'](view, rt['lib'].FFT_FP64)
        torch.cuda.synchronize()
        mo, lo = sk.logmel_loge(s16[:n].astype(np.float32) / np.float32(32768))
        assert mspec.shape[0] == len(lo) == sk.num_frames(n)
        fin = np.isfinite(mo)
        assert np.abs(mspec.cpu().numpy()[fin] - mo[fin]).max() <= 2e-5
    m, l, st = rt['fe'](torch.zeros(399, dtype=torch.int16, device='cuda'), rt['lib'].FFT_FP64)
    assert m.shape == (0, 24) and l.shape == (0,)


# ------------------------------------------------------------------ K3
def test_k3_energy_viterbi_golden(rt, golden, media):
    """Energy activity through K1 + reduction + K3 == reference-derived goldens
    (both FFT precisions), incl. the musanmix noEnergy rows and silence."""
    eng, lib = rt['engine'], rt['lib']
    for prec in (lib.FFT_FP64, lib.FFT_FP32):
        for name, sig in _signals(golden, media).items():
            if name == 'gen60':
                continue
            pcm = torch.from_numpy(np.ascontiguousarray(sig, dtype=np.float32)).cuda()
            mspec, loge, stats = rt['fe'](pcm, prec)
            track = eng.energy_viterbi(rt['ctx'], loge, stats, 0.03, out_stride=2).cpu().numpy()
            from inaspeechsegmenter_b200.segmenter import _rle
            segs = np.array([(lab, a, b) for lab, a, b in _rle(track)], dtype=np.int64)
            assert np.array_equal(segs, golden[name + '_energy_segs']), (name, prec)


def test_k3_energy_viterbi_full_track_vs_oracle(rt):
    from oracle import segmenter_oracle as so
    from oracle import sidekit_oracle as sk
    sig = synth_audio(300, seed=77).astype(np.float32) / np.float32(32768)
    mo, lo = sk.logmel_loge(sig)
    ref = so.energy_activity(lo, 0.03)
    loge = torch.from_numpy(lo).cuda()
    fin = np.isfinite(lo)
    stats = torch.tensor([lo[fin].astype(np.float64).sum(), float(fin.sum())], dtype=torch.float64).cuda()
    for stride in (1, 2):
        got = rt['engine'].energy_viterbi(rt['ctx'], loge, stats, 0.03, out_stride=stride).cpu().numpy()
        assert np.array_equal(got, ref[::stride].astype(np.uint8))


@pytest.mark.parametrize('L,seed', [(70001, 1), (16384 * 5, 2), (16384 * 5 + 1, 3), (3600037, 4)])
def test_k3_energy_viterbi_chunk_parallel_equals_serial_chain(rt, L, seed):
    """The chunk-parallel energy decode (16384-frame chunks, max-plus transfer matrices) against the serial
    chain kernel on tracks up to 10 h (3.6 M frames), and against the reference-pinned C oracle on the shorter ones:
    activity bursts of every length, frames sitting within a few ulps of the threshold, -inf (silent) frames."""
    from oracle import segmenter_oracle as so
    rng = np.random.default_rng(seed)
    lo = np.empty(L, dtype=np.float32)
    pos = 0
    while pos < L:                                              # alternating quiet / active runs, 1 frame .. 40 s
        n = int(min(L - pos, rng.choice([1, 2, 3, 7, 40, 300, 4000]) * (1 + rng.integers(0, 3))))
        level = rng.choice([-14.0, -9.0, -3.0, 1.5])
        lo[pos:pos + n] = level + rng.normal(0, 1.0, n)
        pos += n
    fin_mean = float(np.mean(lo))
    thr = np.float32(fin_mean + np.log(0.03))
    near = rng.integers(0, L, 2000)
    lo[near] = np.nextafter(np.full(2000, thr, dtype=np.float32), (np.inf * rng.choice([-1.0, 1.0], 2000)).astype(np.float32))   # +-1 ulp around the threshold
    lo[rng.integers(0, L, 500)] = -np.inf
    loge = torch.from_numpy(lo).cuda()
    eng, lib = rt['engine'], rt['lib'].load()
    stats = eng.loge_stats(rt['ctx'], loge)
    try:
        lib.iss_set_energy_viterbi_serial(1)
        serial = eng.energy_viterbi(rt['ctx'], loge, stats, 0.03, out_stride=1).cpu().numpy()
        lib.iss_set_energy_viterbi_serial(0)
        chunked = eng.energy_viterbi(rt['ctx'], loge, stats, 0.03, out_stride=1).cpu().numpy()
        chunked2 = eng.energy_viterbi(rt['ctx'], loge, stats, 0.03, out_stride=2).cpu().numpy()
    finally:
        lib.iss_set_energy_viterbi_serial(0)
    assert np.array_equal(chunked, serial)
    assert np.array_equal(chunked2, serial[::2])
    assert 0 < serial.mean() < 1
    if L < 200000:
        ref = so.energy_activity(lo, 0.03)
        assert np.array_equal(serial, ref.astype(np.uint8))
    REPORT['k3_energy_chunked_L%d' % L] = dict(identical_to_serial=True, frames=int(L), active=float(serial.mean()))


def test_k3_segments_golden_and_random(rt, golden):
    from oracle import viterbi_oracle as vo
    eng = rt['engine']
    # golden cases with float32 emissions = log(p): feed p = exp(em) is lossy, so rebuild p from seeds instead:
    rng = np.random.default_rng(123)
    for K, arg in ((2, 150), (3, 80), (2, 80), (4, 80)):
        lens = [1, 2, 3, 31, 32, 33, 255, 256, 257, 700, 5000, 20011]
        probs = []
        for T in lens:
            p = rng.random((T, K)).astype(np.float32) ** 3 + 1e-7
            dom = np.repeat(rng.integers(0, K, T // 40 + 1), 40)[:T]
            p[np.arange(T), dom] += rng.uniform(0.2, 2.0)
            p = (p / p.sum(1, keepdims=True)).astype(np.float32)
            if T > 10:
                p[T // 2] = 0.5                      # the override rows (all-equal emissions)
                p[T // 3, 0] = 0.0                   # an exact zero -> -inf emission
            probs.append(p)
        allp = np.concatenate(probs)
        off = np.concatenate(([0], np.cumsum(lens)))
        tr = vo.diag_trans_exp(arg, K)
        got = eng.viterbi_segments(rt['ctx'], torch.from_numpy(allp).cuda(), off, tr).cpu().numpy()
        for i, T in enumerate(lens):
            ref = vo.viterbi_c(vo.emissions_kernel(probs[i]), tr)
            assert np.array_equal(got[off[i]:off[i + 1]], ref.astype(np.uint8)), (K, T)


# ------------------------------------------------------------------ K2
def _oracle_probs(cfg, w, mspec, nmel, ranges):
    from oracle import cnn_oracle, segmenter_oracle as so
    model = cnn_oracle.KerasLikeModel(cfg, w)
    patches, finite = so.get_patches(mspec[:, :nmel].copy())
    idx = np.concatenate([np.arange(a, b) for a, b in ranges])
    p = model.predict(np.expand_dims(patches[idx], 3).astype(np.float32))
    p[~finite[idx]] = 0.5
    return p


@pytest.mark.parametrize('which,nmel', [('smn', 21), ('sm', 21), ('gender', 24)])
def test_k2_cnn_softmax_vs_oracle(rt, synth_models, which, nmel):
    """Per-frame softmax within 1e-4 (north-star tolerance) of the fp32 torch-CPU oracle."""
    from oracle import sidekit_oracle as sk
    cfg, w = synth_models[which]
    sig = synth_audio(40, seed=3).astype(np.float32) / np.float32(32768)
    mspec, loge = sk.logmel_loge(sig)
    L = len(loge)
    P = (L + 1) // 2
    ranges = [(0, 40), (40, 41), (100, 777), (P - 60, P)]
    ref = _oracle_probs(cfg, w, mspec, nmel, ranges)
    net = rt['engine'].CnnModel.from_keras(rt['ctx'], cfg, w, nmel)
    got = net.forward(torch.from_numpy(mspec).cuda(), ranges).cpu().numpy()
    assert got.shape == ref.shape
    err = np.abs(got - ref).max()
    REPORT['k2_%s' % which] = dict(softmax_max_abs=float(err), n=int(len(ref)), nonfinite_rows=int((ref == 0.5).all(1).sum()),
                                   flops_per_patch=net.flops_per_patch)
    assert (ref == 0.5).all(1).sum() > 0            # the silent span exercises the override
    assert err <= 1e-4, err


@pytest.mark.parametrize('mode', [0, 2, 3])
def test_k2_all_gemm_engines_vs_oracle(rt, synth_models, mode):
    """fp32 CUDA-core kernel, wgmma 3xTF32 and the default fp16-split wgmma engine against the fp32 oracle (1e-4)."""
    from oracle import sidekit_oracle as sk
    lib = rt['lib'].load()
    prev = lib.iss_get_gemm_mode()
    try:
        rt['lib'].check(lib.iss_set_gemm_mode(mode), 'set mode')
        cfg, w = synth_models['gender']
        sig = synth_audio(30, seed=17).astype(np.float32) / np.float32(32768)
        mspec, loge = sk.logmel_loge(sig)
        P = (len(loge) + 1) // 2
        ranges = [(0, 300), (P - 257, P)]
        ref = _oracle_probs(cfg, w, mspec, 24, ranges)
        net = rt['engine'].CnnModel.from_keras(rt['ctx'], cfg, w, 24)
        got = net.forward(torch.from_numpy(mspec).cuda(), ranges).cpu().numpy()
        err = np.abs(got - ref).max()
        REPORT['k2_gender_gemm_mode%d' % mode] = dict(softmax_max_abs=float(err))
        assert err <= 1e-4, err
    finally:
        lib.iss_set_gemm_mode(prev)


def test_k2_first_layer_fused_vs_standalone_and_fallback(rt, synth_models, monkeypatch):
    """The first layer evaluated inside the second convolution's operand fill (float64 map Y, FirstFuse) against the
    stand-alone first-layer kernel and the oracle; a batch whose patches are far apart must take the un-fused path
    (the map would not fit) and still be right."""
    from oracle import sidekit_oracle as sk
    cfg, w = synth_models['smn']
    sig = synth_audio(120, seed=5).astype(np.float32) / np.float32(32768)
    mspec, loge = sk.logmel_loge(sig)
    P = (len(loge) + 1) // 2
    net = rt['engine'].CnnModel.from_keras(rt['ctx'], cfg, w, 21)
    dm = torch.from_numpy(mspec).cuda()
    lib = rt['lib'].load()
    for ranges in ([(0, 700), (900, 1400)], [(3, 23), (P - 30, P)]):        # contiguous-ish (fused) / far apart (fallback)
        ref = _oracle_probs(cfg, w, mspec, 21, ranges)
        monkeypatch.setenv('ISS_B200_FUSE_FIRST', '1')
        l0 = lib.iss_launch_count()
        fused = net.forward(dm, ranges).cpu().numpy()
        n_fused = lib.iss_launch_count() - l0
        monkeypatch.setenv('ISS_B200_FUSE_FIRST', '0')
        l0 = lib.iss_launch_count()
        plain = net.forward(dm, ranges).cpu().numpy()
        n_plain = lib.iss_launch_count() - l0
        assert np.abs(fused - ref).max() <= 1e-4 and np.abs(plain - ref).max() <= 1e-4
        assert np.abs(fused - plain).max() <= 2e-5
        REPORT['k2_first_fused_%d_patches' % len(ref)] = dict(vs_oracle=float(np.abs(fused - ref).max()), vs_standalone=float(np.abs(fused - plain).max()),
                                                              launches_fused=int(n_fused), launches_standalone=int(n_plain))
    monkeypatch.delenv('ISS_B200_FUSE_FIRST', raising=False)


@pytest.mark.parametrize('which,nmel', [('smn', 21), ('gender', 24)])
def test_k2_direct_kernel_variants_vs_oracle(rt, synth_models, monkeypatch, which, nmel):
    """The fp16-split engine with the 2x2 max-pooling folded into its operand fill against its fall-backs -- pooling as its
    own kernel, and the 3xTF32 engine (fp32 activations, nothing folded) -- and the oracle, on ranges that make tiles
    straddle patches and end in a partial tile."""
    from oracle import sidekit_oracle as sk
    cfg, w = synth_models[which]
    sig = synth_audio(100, seed=9).astype(np.float32) / np.float32(32768)
    mspec, loge = sk.logmel_loge(sig)
    P = (len(loge) + 1) // 2
    net = rt['engine'].CnnModel.from_keras(rt['ctx'], cfg, w, nmel)
    dm = torch.from_numpy(mspec).cuda()
    lib = rt['lib'].load()
    prev = lib.iss_get_gemm_mode()
    ranges = [(0, 1), (5, 612), (700, P)]
    ref = _oracle_probs(cfg, w, mspec, nmel, ranges)
    out, launches = {}, {}
    try:
        for name, mode, env in (('folded', 3, {}), ('pool_kernel', 3, {'ISS_B200_FUSE_POOL': '0'}), ('engine2', 2, {})):
            monkeypatch.delenv('ISS_B200_FUSE_POOL', raising=False)
            for k, v in env.items():
                monkeypatch.setenv(k, v)
            rt['lib'].check(lib.iss_set_gemm_mode(mode), 'set mode')
            l0 = lib.iss_launch_count()
            out[name] = net.forward(dm, ranges).cpu().numpy()
            launches[name] = lib.iss_launch_count() - l0
    finally:
        lib.iss_set_gemm_mode(prev)
        monkeypatch.delenv('ISS_B200_FUSE_POOL', raising=False)
    for name, got in out.items():
        assert np.abs(got - ref).max() <= 1e-4, name
    assert np.abs(out['folded'] - out['pool_kernel']).max() == 0.0          # the folded pooling keeps the same words
    assert np.abs(out['folded'] - out['engine2']).max() <= 2e-5
    assert launches['folded'] < launches['pool_kernel']
    REPORT['k2_folded_pooling_%s' % which] = dict(vs_oracle={k: float(np.abs(v - ref).max()) for k, v in out.items()}, launches=launches)


@pytest.mark.parametrize('L', [68, 69, 70, 101, 135, 136])
def test_k2_edge_replication(rt, synth_models, L):
    cfg, w = synth_models['sm']
    rng = np.random.default_rng(L)
    mspec = (rng.standard_normal((L, 24)) * 3 - 5).astype(np.float32)
    P = (L + 1) // 2
    ref = _oracle_probs(cfg, w, mspec, 21, [(0, P)])
    net = rt['engine'].CnnModel.from_keras(rt['ctx'], cfg, w, 21)
    got = net.forward(torch.from_numpy(mspec).cuda(), [(0, P)]).cpu().numpy()
    assert got.shape == (P, 2) and np.abs(got - ref).max() <= 1e-4


# ------------------------------------------------------------------ end to end
def _oracle_segmentation(sig_f32, synth_models, vad='smn', gender=True):
    from oracle import cnn_oracle, segmenter_oracle as so
    mspec, loge, difflen = so.media2feats(sig_f32)
    vspec = so.VAD_SMN if vad == 'smn' else so.VAD_SM
    v = so.DnnSegmenterOracle(cnn_oracle.KerasLikeModel(*synth_models[vad]), **vspec)
    g = so.DnnSegmenterOracle(cnn_oracle.KerasLikeModel(*synth_models['gender']), **so.GENDER) if gender else None
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        return so.segment_feats(mspec, loge, difflen, 0, v, g), v, g


@pytest.mark.parametrize('vad,gender', [('smn', True), ('sm', True), ('smn', False)])
def test_e2e_segmentation_identical_to_oracle(rt, synth_models, vad, gender):
    from inaspeechsegmenter_b200 import Segmenter
    s16 = synth_audio(90, seed=42)
    ref, v, g = _oracle_segmentation(s16.astype(np.float32) / np.float32(32768), synth_models, vad, gender)
    seg = Segmenter(vad_engine=vad, detect_gender=gender, ffmpeg=None,
                    models={'vad': synth_models[vad], 'gender': synth_models['gender']})
    got = seg.segment_signal(s16)
    assert got == ref, (got[:5], ref[:5])
    # per-frame softmax of the VAD network on every evaluated patch
    err = np.abs(seg.vad.last_probs.cpu().numpy() - v.last_probs).max()
    REPORT['e2e_%s_%s' % (vad, gender)] = dict(vad_softmax_max_abs=float(err), n_segments=len(ref))
    assert err <= 1e-4


def test_e2e_file_api_and_exports(rt, synth_models, media, tmp_path):
    """Segmenter(media) and batch_process on the reference WAV fixtures: the
    weights-free rows/boundaries of the golden CSV are reproduced, files are written."""
    from inaspeechsegmenter_b200 import Segmenter
    seg = Segmenter(vad_engine='smn', detect_gender=True, ffmpeg=None,
                    models={'vad': synth_models['smn'], 'gender': synth_models['gender']})
    wav = os.path.join(media, 'musanmix.wav')
    got = seg(wav)
    rows = []
    with open(os.path.join(media, 'musanmix-smn-gender.csv')) as f:
        next(f)
        for line in f:
            lab, a, b = line.rstrip('\n').split('\t')
            rows.append((lab, float(a), float(b)))
    assert [s for s in got if s[0] == 'noEnergy'] == [r for r in rows if r[0] == 'noEnergy']
    for i in range(len(got) - 1):
        assert got[i][2] == got[i + 1][1]                  # run_test.py:68-88 (test_boundaries)
    assert seg(os.path.join(media, 'silence2sec.wav')) == [('noEnergy', 0.0, 1.98)]
    outs = [str(tmp_path / 'a.csv'), str(tmp_path / 'sub' / 'b.csv'), str(tmp_path / 'c.csv')]
    dur, nb, avg, lmsg = seg.batch_process([wav, '/nonexistent.wav', os.path.join(media, 'silence2sec.wav')], outs)
    assert nb == 2 and [m[1] for m in lmsg] == [0, 2, 0]     # run_test.py:129-134 (missing input does not abort)
    assert open(outs[2]).read() == open(os.path.join(media, 'silence2sec-smn-gender.csv')).read()
    dur, nb, avg, lmsg = seg.batch_process([wav], [outs[0]], skipifexist=True, output_format='textgrid')
    assert lmsg[0][1] == 1
    with pytest.raises(NotImplementedError):
        seg.batch_process([wav], [outs[0]], output_format='json')


def test_e2e_short_media(rt, synth_models):
    """< 68 frames: the padding path of segmenter.py:60-65,150-152 (0021.mp3 case)."""
    import warnings
    from inaspeechsegmenter_b200 import Segmenter
    s16 = synth_audio(1.5, seed=8)[:59 * 160 + 400]             # 60 frames -> difflen 8
    seg = Segmenter(vad_engine='sm', detect_gender=True, ffmpeg=None,
                    models={'vad': synth_models['sm'], 'gender': synth_models['gender']})
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        got = seg.segment_signal(s16)
        ref, _, _ = _oracle_segmentation(s16.astype(np.float32) / np.float32(32768), synth_models, 'sm', True)
    assert got == ref


def test_cli_with_hdf5_models(rt, synth_models, media, tmp_path, monkeypatch):
    """CLI (reference flags) + Keras .hdf5 model lookup: models are read through the pure-Python
    HDF5 reader from $ISS_B200_MODEL_DIR, outputs are the reference's CSV format."""
    from inaspeechsegmenter_b200 import cli, keras_hdf5, models as M
    mdir = tmp_path / 'models'
    mdir.mkdir()
    keras_hdf5.write_keras_hdf5(str(mdir / 'keras_speech_music_noise_cnn.hdf5'), *synth_models['smn'])
    keras_hdf5.write_keras_hdf5(str(mdir / 'keras_male_female_cnn.hdf5'), *synth_models['gender'])
    monkeypatch.setenv(M.MODEL_DIR_ENV, str(mdir))
    out = tmp_path / 'out'
    out.mkdir()
    cli.main(['-i', os.path.join(media, 'silence2sec.wav'), os.path.join(media, 'musanmix.wav'), '-o', str(out), '-b', 'None'])
    assert (out / 'silence2sec.csv').read_bytes() == open(os.path.join(media, 'silence2sec-smn-gender.csv'), 'rb').read()
    got = (out / 'musanmix.csv').read_text().splitlines()
    ref = open(os.path.join(media, 'musanmix-smn-gender.csv')).read().splitlines()
    assert got[0] == ref[0] and [l for l in got if l.startswith('noEnergy')] == [l for l in ref if l.startswith('noEnergy')]


def test_cli_devices_spawns_one_worker_per_device(rt, synth_models, media, tmp_path, monkeypatch):
    """`--devices a,b` (cli.py: files dealt round-robin to one spawned process per device -- the role of the reference's
    Pyro farm, scripts/ina_speech_segmenter_pyro_client.py:64-74, on one host): the outputs are byte-identical to the
    single-process run.  On a one-GPU box both workers share device 0."""
    import torch
    from inaspeechsegmenter_b200 import cli, keras_hdf5, models as M
    mdir = tmp_path / 'models'
    mdir.mkdir()
    keras_hdf5.write_keras_hdf5(str(mdir / 'keras_speech_music_noise_cnn.hdf5'), *synth_models['smn'])
    keras_hdf5.write_keras_hdf5(str(mdir / 'keras_male_female_cnn.hdf5'), *synth_models['gender'])
    monkeypatch.setenv(M.MODEL_DIR_ENV, str(mdir))
    files = [os.path.join(media, f) for f in ('silence2sec.wav', 'musanmix.wav', 'lamartine.wav')]
    one, two = tmp_path / 'one', tmp_path / 'two'
    one.mkdir(); two.mkdir()
    cli.main(['-i'] + files + ['-o', str(one), '-b', 'None'])
    devs = '0,1' if torch.cuda.device_count() > 1 else '0,0'
    cli.main(['-i'] + files + ['-o', str(two), '-b', 'None', '--devices', devs])
    for f in ('silence2sec.csv', 'musanmix.csv', 'lamartine.csv'):
        assert (two / f).read_bytes() == (one / f).read_bytes(), f


def _alt_keras_cnn(nmel, n_classes, seed):
    """A second architecture exercising the rest of the layer interpreter: 'same' padding, strides,
    'same' max-pooling with odd sizes, activation fused in the Conv2D config, Dense -> ReLU -> BatchNorm
    (affine AFTER the activation), bias-free convolution, BatchNorm without scale."""
    rng = np.random.default_rng(seed)
    L, W = [], {}

    def conv(name, kh, kw, cin, cout, strides, padding, act, bias=True):
        W[name + '/kernel'] = (rng.standard_normal((kh, kw, cin, cout)) * np.sqrt(2.0 / (kh * kw * cin))).astype(np.float32)
        if bias:
            W[name + '/bias'] = rng.normal(0, 0.05, cout).astype(np.float32)
        L.append({'class_name': 'Conv2D', 'config': {'name': name, 'filters': cout, 'kernel_size': [kh, kw], 'strides': strides,
                                                      'padding': padding, 'use_bias': bias, 'activation': act}})

    def bn(name, ch, scale=True):
        if scale:
            W[name + '/gamma'] = rng.uniform(0.8, 1.2, ch).astype(np.float32)
        W[name + '/beta'] = rng.normal(0, 0.1, ch).astype(np.float32)
        W[name + '/moving_mean'] = rng.normal(0, 0.2, ch).astype(np.float32)
        W[name + '/moving_variance'] = rng.uniform(0.5, 1.5, ch).astype(np.float32)
        L.append({'class_name': 'BatchNormalization', 'config': {'name': name, 'axis': -1, 'epsilon': 1e-3, 'center': True, 'scale': scale}})

    L.append({'class_name': 'InputLayer', 'config': {'name': 'in', 'batch_input_shape': [None, 68, nmel, 1]}})
    conv('c1', 3, 3, 1, 32, [1, 1], 'same', 'relu')                       # first layer with padding (first-layer kernel, padded)
    conv('c2', 3, 3, 32, 64, [2, 1], 'same', 'linear', bias=False)        # stride 2 in time, asymmetric 'same' padding, TC path
    bn('b2', 64, scale=False)
    L.append({'class_name': 'Activation', 'config': {'name': 'a2', 'activation': 'relu'}})
    L.append({'class_name': 'MaxPooling2D', 'config': {'name': 'p2', 'pool_size': [3, 2], 'strides': [2, 2], 'padding': 'same'}})
    conv('c3', 1, 1, 64, 96, [1, 1], 'valid', 'relu')                     # 1x1, N = 96 (32-wide TC tiles)
    L.append({'class_name': 'MaxPooling2D', 'config': {'name': 'p3', 'pool_size': [2, 2], 'strides': None, 'padding': 'valid'}})
    L.append({'class_name': 'Flatten', 'config': {'name': 'f'}})
    h, w = 68, nmel
    h, w = -(-h // 2), w                    # c2 stride (2,1) same
    h, w = -(-h // 2), -(-w // 2)           # p2 same
    h, w = h // 2, w // 2                   # p3 valid
    fin = h * w * 96
    W['d1/kernel'] = (rng.standard_normal((fin, 64)) * np.sqrt(2.0 / fin)).astype(np.float32)
    W['d1/bias'] = rng.normal(0, 0.05, 64).astype(np.float32)
    L.append({'class_name': 'Dense', 'config': {'name': 'd1', 'units': 64, 'use_bias': True, 'activation': 'relu'}})
    bn('bd1', 64)                                                          # BatchNorm AFTER the activation
    L.append({'class_name': 'Dropout', 'config': {'name': 'do', 'rate': 0.5}})
    W['d2/kernel'] = (rng.standard_normal((64, n_classes)) * np.sqrt(1.0 / 64)).astype(np.float32)
    W['d2/bias'] = rng.normal(0, 0.05, n_classes).astype(np.float32)
    L.append({'class_name': 'Dense', 'config': {'name': 'd2', 'units': n_classes, 'use_bias': True, 'activation': 'linear'}})
    L.append({'class_name': 'Activation', 'config': {'name': 'sm', 'activation': 'softmax'}})
    return {'class_name': 'Sequential', 'config': {'name': 'alt', 'layers': L}}, W


@pytest.mark.parametrize('mode', [0, 2, 3])
@pytest.mark.parametrize('nmel', [21, 24])
def test_k2_layer_interpreter_alt_architecture(rt, nmel, mode):
    """The release networks' architecture is unknown here, so the generic layer interpreter is
    checked on a second, deliberately different Keras config (padding/stride/pool/BN-order variants)."""
    from oracle import sidekit_oracle as sk
    lib = rt['lib'].load()
    prev = lib.iss_get_gemm_mode()
    try:
        lib.iss_set_gemm_mode(mode)
        cfg, w = _alt_keras_cnn(nmel, 3, seed=nmel)
        sig = synth_audio(25, seed=29).astype(np.float32) / np.float32(32768)
        mspec, loge = sk.logmel_loge(sig)
        P = (len(loge) + 1) // 2
        ranges = [(0, 50), (200, 460), (P - 40, P)]
        ref = _oracle_probs(cfg, w, mspec, nmel, ranges)
        net = rt['engine'].CnnModel.from_keras(rt['ctx'], cfg, w, nmel)
        got = net.forward(torch.from_numpy(mspec).cuda(), ranges).cpu().numpy()
        err = np.abs(got - ref).max()
        REPORT['k2_alt_arch_nmel%d_mode%d' % (nmel, mode)] = dict(softmax_max_abs=float(err))
        assert got.shape == ref.shape and err <= 1e-4, err
    finally:
        lib.iss_set_gemm_mode(prev)
