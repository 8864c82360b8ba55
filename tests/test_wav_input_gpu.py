"""WAV files of any rate, channel count and PCM encoding without ffmpeg, on the device (run with -m gpu on an H100):
the resampler's reading of the stored WAV encodings against oracle/resample_ref.py, and Segmenter /
VoiceFemininityScoring / batch_process on such files against the in-memory APIs."""
import os
import warnings

import numpy as np
import pytest

from conftest import synth_audio
from resample_fixtures import reference
from wav_fixtures import decode, encode, fixtures, write_wav

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')


@pytest.fixture(scope='module')
def rt():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from inaspeechsegmenter_b200 import _lib, engine, io, resample, segmenter
    return dict(lib=_lib, engine=engine, io=io, resample=resample, segmenter=segmenter, ctx=engine.Context(0))


@pytest.fixture(scope='module')
def wavs(tmp_path_factory):
    return fixtures(str(tmp_path_factory.mktemp('wavs')))


def _stored(w):
    with open(w.path, 'rb') as f:
        f.seek(w.start)
        return f.read(w.nbytes)


def _check(got, x, rate, what):
    q, tie, _, _ = reference(x, rate)
    got = got.cpu().numpy() if isinstance(got, torch.Tensor) else got
    assert got.shape == q.shape, what
    assert not tie.any(), (what, int(tie.sum()))
    bad = got != q
    assert not bad.any(), (what, int(bad.sum()), np.flatnonzero(bad)[:5], got[bad][:5], q[bad][:5])


def test_kernel_equals_reference_on_every_fixture(rt, wavs):
    """Each fixture's file route (pinned read, one upload, resample) equals the oracle at every sample; so do its
    stored bytes at a device address that is not 16-byte aligned (scalar loads), and one packed call over all
    fixtures (one launch per group) equals the calls on each alone."""
    io, resample, segmenter, ctx = rt['io'], rt['resample'], rt['segmenter'], rt['ctx']
    ws = {name: io.wav_data(path) for name, (path, _, _, _) in wavs.items()}
    singles = {}
    for name, w in ws.items():
        x = decode(_stored(w), w.encoding, w.channels)
        singles[name] = segmenter._wav_to16k(ctx, w)
        _check(singles[name], x, w.rate, (name, 'file'))
        shift = io.BYTES[w.encoding]                        # 1, 2, 3, 4 or 8 bytes past a 16-byte boundary
        buf = torch.empty(w.nbytes + shift + 16, dtype=torch.uint8, device='cuda')
        view = buf[shift:shift + w.nbytes]
        view.copy_(torch.frombuffer(bytearray(_stored(w)), dtype=torch.uint8))
        out = torch.empty(resample.num_frames(w.frames, w.rate), dtype=torch.int16, device='cuda')
        resample.to16k_multi(ctx, [view.view(w.shape)], w.rate, out, [0], encoding=w.encoding)
        _check(out, x, w.rate, (name, 'misaligned'))
    names = list(ws)
    pcms = segmenter._stage_pass([ws[n] for n in names], ctx.device)
    packed = resample.resample_pass(ctx, pcms, [ws[n].rate for n in names], [ws[n].encoding for n in names])
    for n, p in zip(names, packed):
        assert torch.equal(p, singles[n]), n


def test_other_pcm_consumers_refuse_the_wav_encodings(rt):
    """K1 and K4 take int16 and float32 only: every other pcm_format is ISS_ERR_INVALID before any launch."""
    from inaspeechsegmenter_b200.sidekit_mfcc import SidekitFrontEnd
    from inaspeechsegmenter_b200.vbx_segmenter import VbxFrontEnd
    L, ctx = rt['lib'], rt['engine'].Context(0)
    SidekitFrontEnd(ctx)
    VbxFrontEnd(ctx)
    lib, p = L.load(), L.ptr
    x = torch.zeros(16000, dtype=torch.int16, device='cuda')
    work = torch.zeros(1 << 22, dtype=torch.uint8, device='cuda')
    ptrs = (L._c.c_void_p * 1)(x.data_ptr())
    n = np.array([16000], dtype=np.int64)
    zero = np.zeros(8, dtype=np.int64)
    c0 = lib.iss_launch_count()
    for fmt in (L.PCM_U8, L.PCM_S24, L.PCM_S32, L.PCM_F64):
        rcs = [lib.iss_sidekit_features(ctx.handle, p(x), fmt, 16000, L.FFT_FP64, p(work), p(work), p(work), None),
               lib.iss_sidekit_features_multi(ctx.handle, 1, ptrs, p(n), fmt, L.FFT_FP64, p(work), p(zero), p(work),
                                              p(zero), p(work), None),
               lib.iss_vbx_features(ctx.handle, p(x), fmt, 16000, p(work), p(work), p(work), None),
               lib.iss_vbx_features_multi(ctx.handle, 1, ptrs, p(n), fmt, p(work), p(work), p(zero), p(work), None),
               lib.iss_vbx_fbank_window_multi(ctx.handle, 1, ptrs, ptrs, p(zero), fmt, p(work), None)]
        assert rcs == [-1] * 5, (fmt, rcs)
        assert b'pcm_format' in lib.iss_last_error()
    assert lib.iss_launch_count() == c0
    torch.cuda.synchronize()
    ctx.close()


# ------------------------------------------------------------------ end to end
E2E = [('u8', 1, 8000), ('s16', 2, 16000), ('s24', 2, 48000), ('s32', 6, 44100), ('f32', 1, 192000),
       ('f64', 2, 48000)]


def _audio(seconds, C, rate, seed):
    """float64 [frames, C]: synthetic speech / music / noise per channel, with a little noise below int16's step so
    that int32 and float64 files hold more than 16 bits."""
    rng = np.random.default_rng(seed)
    x = np.stack([synth_audio(seconds, seed=seed + c, sr=rate) / 32768.0 for c in range(C)], axis=1)
    return np.clip(x + rng.standard_normal(x.shape) * 2e-6, -1, 1)


def _e2e_file(directory, enc, C, rate, seconds=12, seed=0, **kw):
    path = os.path.join(directory, 'e2e_%s_%dch_%d.wav' % (enc, C, rate))
    return write_wav(path, encode(_audio(seconds, C, rate, seed), enc), enc, C, rate, **kw)


def _expected_pcm(rt, path):
    """The samples segment_signal is compared with: read_wav's float32 signal where that conversion is exact (u8,
    s16, s24, f32), else the oracle's 16 kHz int16 output (s32, f64)."""
    w = rt['io'].wav_data(path)
    if w.encoding in ('s32', 'f64'):
        q, tie, _, _ = reference(decode(_stored(w), w.encoding, w.channels), w.rate)
        assert not tie.any()
        return q, 16000
    x, sr = rt['io'].read_wav(path, 'float32')
    return x, sr


def _segmenter(rt, synth_models):
    return rt['segmenter'].Segmenter(vad_engine='smn', detect_gender=True, ffmpeg=None,
                                     models={'vad': synth_models['smn'], 'gender': synth_models['gender']})


def test_segmenter_call_equals_segment_signal(rt, synth_models, tmp_path):
    seg = _segmenter(rt, synth_models)
    lib = rt['lib'].load()
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        for i, (enc, C, rate) in enumerate(E2E):
            path = _e2e_file(str(tmp_path), enc, C, rate, seed=10 * i)
            x, sr = _expected_pcm(rt, path)
            got = seg(path)
            assert got == seg.segment_signal(x, sample_rate=sr), (enc, C, rate)
            assert got[-1][2] == pytest.approx(12.0, abs=0.03)
        ext = _e2e_file(str(tmp_path), 's24', 2, 48000, seed=99, extensible=True, pre_chunks=((b'bext', b'abc'),))
        x, sr = _expected_pcm(rt, ext)
        assert seg(ext) == seg.segment_signal(x, sample_rate=sr)
        # 16 kHz mono of any encoding keeps the host conversion: no resampler launch, media2sig16kmono's signal
        for enc in ('u8', 's24', 'f64'):
            path = _e2e_file(str(tmp_path), enc, 1, 16000, seed=7)
            sig = rt['io'].media2sig16kmono(path, ffmpeg=None, dtype='float32', return_int16=True)
            ref = seg.segment_signal(sig)
            c0 = lib.iss_launch_count()
            got = seg(path)
            c1 = lib.iss_launch_count()
            seg.segment_signal(sig)
            assert got == ref and c1 - c0 == lib.iss_launch_count() - c1, enc


def test_batch_process_equals_call(rt, synth_models, tmp_path):
    from inaspeechsegmenter_b200.export_funcs import seg2csv
    seg = _segmenter(rt, synth_models)
    src = tmp_path / 'in'
    src.mkdir()
    files = [_e2e_file(str(src), enc, C, rate, seconds=8, seed=20 + i) for i, (enc, C, rate) in enumerate(E2E)]
    files.insert(2, _e2e_file(str(src), 's16', 1, 16000, seconds=8, seed=40))
    bad = str(src / 'broken.wav')
    with open(bad, 'wb') as f:
        f.write(b'RIFF....not a wave file')
    files.insert(4, bad)
    outs = [str(tmp_path / 'out' / (os.path.basename(f)[:-4] + '.csv')) for f in files]
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        _, n_ok, _, msgs = seg.batch_process(files, outs)
        assert n_ok == len(files) - 1
        assert [(d, c) for d, c, _ in msgs] == [(o, 2 if f == bad else 0) for f, o in zip(files, outs)]
        for f, o, (_, code, text) in zip(files, outs, msgs):
            if f == bad:
                with pytest.raises(ValueError):
                    seg(f)
                assert text == 'error: ' + str(ValueError)
                continue
            assert text.startswith('ok ')
            with open(o, 'rb') as fh:
                assert fh.read() == seg2csv(seg(f)).encode(), f


def test_vfs_call_equals_score_signal(rt, synth_models, tmp_path):
    from inaspeechsegmenter_b200 import vbx_segmenter as vb
    from test_vfs_pack_gpu import vfs_models
    vfs = vb.VoiceFemininityScoring(ffmpeg=None, models=vfs_models(synth_models))

    def score(fn):
        try:
            return fn()
        except ZeroDivisionError as e:          # score_signal's own error when no window is kept
            return type(e)

    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        scored = 0
        for i, (enc, C, rate) in enumerate([('s24', 2, 48000), ('f64', 2, 44100), ('u8', 1, 22050)]):
            path = _e2e_file(str(tmp_path), enc, C, rate, seconds=30, seed=70 + i)
            x, sr = _expected_pcm(rt, path)
            got = score(lambda: vfs(path))
            assert got == score(lambda: vfs.score_signal(x, sample_rate=sr)), (enc, C, rate)
            scored += isinstance(got, tuple) and got[2] > 0
        assert scored >= 2
