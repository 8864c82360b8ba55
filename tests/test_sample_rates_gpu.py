"""The resampler (resample.cu) against the float64 reference of oracle/resample_ref.py, and the sample_rate /
sample_rates arguments of Segmenter and VoiceFemininityScoring end to end (run with -m gpu on an H100)."""
import warnings

import numpy as np
import pytest

from conftest import synth_audio
from oracle import resample_ref as rr
from resample_fixtures import reference

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')

RATES = [8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000, 96000, 192000]


@pytest.fixture(scope='module')
def rt():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from inaspeechsegmenter_b200 import _lib, engine, resample, segmenter
    return dict(lib=_lib, engine=engine, resample=resample, segmenter=segmenter, ctx=engine.Context(0))


def _lengths(rate):
    up, down = rr.factors(rate)
    span = (20 * max(up, down) + 1) // up + 1
    return sorted({1, 2, max(down - 1, 1), down, down + 1, span - 1, span, span + 1, 3 * rate + 17})


def _recording(rate, n, C, fmt, seed):
    """Noise, a tone and impulses per channel, with channel 0 a full-scale square over its second half (clipping)."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / rate
    x = rng.standard_normal((n, C)) * 0.2 + 0.3 * np.sin(2 * np.pi * (440 + 97 * np.arange(C)) * t[:, None])
    x[::max(n // 5, 1)] = 0.95
    x[n // 2:, 0] = np.where(np.sin(2 * np.pi * 1234 * t[n // 2:]) >= 0, 1.0, -1.0)
    x = np.clip(x, -1, 1)
    if fmt == 'int16':
        return np.clip(np.round(x * 32768), -32768, 32767).astype(np.int16)
    return x.astype(np.float32)


def _check(got, x, rate, what):
    q, tie, _, _ = reference(x, rate)
    got = got.cpu().numpy() if isinstance(got, torch.Tensor) else got
    assert got.shape == q.shape, what
    bad = (got != q) & ~tie
    assert not bad.any(), (what, int(bad.sum()), np.flatnonzero(bad)[:5], got[bad][:5], q[bad][:5])
    return int(tie.sum())


@pytest.mark.parametrize('rate', RATES)
@pytest.mark.parametrize('fmt', ['int16', 'float32'])
def test_kernel_equals_reference(rt, rate, fmt):
    """Every rate, mono / stereo / 6 channels, the boundary lengths, as host arrays (one call each), CUDA tensors (one
    packed call) and views at an odd frame offset (not 16-byte aligned: scalar loads); packed equals single."""
    resample = rt['resample']
    ctx = rt['ctx']
    ties = {}
    for C in (1, 2, 6):
        if rate == 16000 and C == 1:
            continue                        # 16 kHz mono is never resampled
        xs = [_recording(rate, n, C, fmt, seed=rate + 7 * n + C) for n in _lengths(rate)]
        singles = [resample.to16k(ctx, x if C > 1 else x[:, 0], rate) for x in xs]
        for x, s in zip(xs, singles):
            ties[(C, len(x), 'host')] = _check(s, x, rate, (rate, fmt, C, len(x), 'host'))
        dev = [torch.from_numpy(np.concatenate([x[:1], x])).cuda()[1:] for x in xs]      # odd offset
        for x, d in zip(xs, dev):
            ties[(C, len(x), 'view')] = _check(resample.to16k(ctx, d, rate), x, rate, (rate, fmt, C, len(x), 'view'))
        packed = resample.resample_pass(ctx, [torch.from_numpy(x).cuda() for x in xs], [rate] * len(xs))
        for s, p in zip(singles, packed):
            assert torch.equal(s, p), (rate, fmt, C)
    print('%d Hz %s: %d near ties over %d recordings' % (rate, fmt, sum(ties.values()), len(ties)))
    assert sum(ties.values()) == 0


def test_packed_groups_equal_single_calls(rt):
    """One pass with several (rate, channels, dtype) groups, 16 kHz mono passed through, in input order."""
    resample = rt['resample']
    ctx = rt['ctx']
    spec = [(48000, 2, 'int16'), (44100, 1, 'float32'), (16000, 1, 'int16'), (48000, 2, 'int16'), (22050, 6, 'int16'),
            (44100, 1, 'float32'), (16000, 2, 'float32'), (8000, 1, 'int16')]
    xs = [_recording(r, 3 * r + 11 * i, C, f, seed=i) for i, (r, C, f) in enumerate(spec)]
    xs = [x[:, 0] if C == 1 else x for x, (_, C, _) in zip(xs, spec)]
    rates = [r for r, _, _ in spec]
    pcms = rt['segmenter']._stage_pass(xs, ctx.device)
    out = resample.resample_pass(ctx, pcms, rates)
    for x, o, p, r in zip(xs, out, pcms, rates):
        if r == 16000 and x.ndim == 1:
            assert o is p
        else:
            assert o.dtype == torch.int16 and o.data_ptr() % 16 == 0
            assert torch.equal(o, resample.to16k(ctx, x, r))


def test_ties_round_to_even_at_16k_stereo(rt):
    x = np.array([[1, 2], [2, 3], [-1, -2], [-2, -3], [32767, 32767], [-32768, -32767]] * 100, dtype=np.int16)
    got = rt['resample'].to16k(rt['ctx'], x, 16000).cpu().numpy()
    assert list(got[:6]) == [2, 2, -2, -2, 32767, -32768]
    _check(got, x, 16000, '16k stereo ties')


def test_c_abi_errors(rt):
    lib, ctx, resample = rt['lib'].load(), rt['ctx'], rt['resample']
    assert lib.iss_resample_num_frames(48000, 48000) == 16000
    assert lib.iss_resample_num_frames(441, 44100) == 160 and lib.iss_resample_num_frames(442, 44100) == 161
    assert lib.iss_resample_num_frames(10, 7999) == -1
    h = np.ascontiguousarray(resample.lowpass(1, 3))
    assert lib.iss_resample_upload_taps(ctx.handle, 48000, rt['lib'].ptr(h), h.size - 1) == -1
    c2 = rt['engine'].Context(0)
    x = torch.zeros(4800, dtype=torch.int16, device='cuda')
    out = torch.empty(1600, dtype=torch.int16, device='cuda')
    ptrs = (rt['lib']._c.c_void_p * 1)(x.data_ptr())
    n = np.array([4800], dtype=np.int64)
    off = np.zeros(1, dtype=np.int64)
    rc = lib.iss_resample_to16k_multi(c2.handle, 1, ptrs, rt['lib'].ptr(n), 1, 48000, 1, rt['lib'].ptr(out),
                                      rt['lib'].ptr(off), None)
    assert rc == -5 and b'no taps' in lib.iss_last_error()
    assert lib.iss_resample_upload_taps(c2.handle, 48000, rt['lib'].ptr(h), h.size) == 0
    assert lib.iss_resample_to16k_multi(c2.handle, 1, ptrs, rt['lib'].ptr(n), 1, 48000, 1, rt['lib'].ptr(out),
                                        rt['lib'].ptr(off), None) == 0
    assert lib.iss_resample_release_taps(c2.handle, 48000) == 0
    assert lib.iss_resample_to16k_multi(c2.handle, 1, ptrs, rt['lib'].ptr(n), 1, 48000, 1, rt['lib'].ptr(out),
                                        rt['lib'].ptr(off), None) == -5
    assert lib.iss_resample_to16k_multi(c2.handle, 1, ptrs, rt['lib'].ptr(n), 9, 48000, 1, rt['lib'].ptr(out),
                                        rt['lib'].ptr(off), None) == -1
    torch.cuda.synchronize()
    c2.close()


# ------------------------------------------------------------------ end to end
def _segmenter(rt, synth_models):
    return rt['segmenter'].Segmenter(vad_engine='smn', detect_gender=True, ffmpeg=None,
                                     models={'vad': synth_models['smn'], 'gender': synth_models['gender']})


def _stereo(seconds, sr, seed):
    return np.stack([synth_audio(seconds, seed=seed, sr=sr), synth_audio(seconds, seed=seed + 1, sr=sr)], axis=1)


def test_default_rate_path_is_untouched(rt, synth_models):
    """With the default sample_rate nothing is resampled: the launches and results of the 16 kHz pipeline
    (feats_from_signal + segment_feats, what segment_signal ran before sample_rate existed)."""
    seg = _segmenter(rt, synth_models)
    lib = rt['lib'].load()
    s16 = synth_audio(30, seed=3)
    f32 = s16.astype(np.float32) / np.float32(32768) * np.float32(0.7)          # not a multiple of 1/32768
    for sig in (s16, f32, torch.from_numpy(f32).cuda()):
        seg.segment_signal(sig)
        c0 = lib.iss_launch_count()
        m, l, d = rt['segmenter'].feats_from_signal(sig, 0, seg.fft_precision, 'main')
        ref = seg.segment_feats(m, l, d, 0)
        c1 = lib.iss_launch_count()
        a = seg.segment_signal(sig)
        c2 = lib.iss_launch_count()
        b = seg.segment_signal(sig, sample_rate=16000)
        c3 = lib.iss_launch_count()
        assert a == b == ref
        assert c1 - c0 == c2 - c1 == c3 - c2
    clips = [s16[i * 32000:(i + 1) * 32000] for i in range(10)] + [f32[:48000]]
    c0 = lib.iss_launch_count()
    a = seg.segment_signals(clips)
    c1 = lib.iss_launch_count()
    b = seg.segment_signals(clips, sample_rates=[16000] * len(clips))
    c2 = lib.iss_launch_count()
    assert a == b and c1 - c0 == c2 - c1


def test_segment_signal_resampled_equals_reference_pcm(rt, synth_models):
    seg = _segmenter(rt, synth_models)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        for x, rate in ((synth_audio(60, sr=48000), 48000), (_stereo(60, 44100, 31), 44100)):
            q, tie, _, _ = reference(x, rate)
            assert not tie.any()
            got = seg.segment_signal(x, sample_rate=rate)
            assert got == seg.segment_signal(q)
            assert got[-1][2] == pytest.approx(len(q) / 16000, abs=0.03)
            assert seg.segment_signal(torch.from_numpy(x).cuda(), 1.5, sample_rate=rate) == seg.segment_signal(q, 1.5)


def _mixed_list():
    x48 = _stereo(20, 48000, 41)
    x44 = synth_audio(15, seed=43, sr=44100)
    x22 = synth_audio(12, seed=44, sr=22050).astype(np.float32) / np.float32(32768)
    s16 = synth_audio(10, seed=45)
    sigs = [s16, x48, torch.from_numpy(x44).cuda(), x22, torch.from_numpy(_stereo(8, 48000, 46)).cuda(),
            s16.astype(np.float32) / np.float32(32768), x44[:44100 * 3], torch.from_numpy(s16[:40000]).cuda()]
    rates = [16000, 48000, 44100, 22050, 48000, 16000, 44100, 16000]
    return sigs, rates


def test_segment_signals_mixed_rates_equals_segment_signal(rt, synth_models):
    seg = _segmenter(rt, synth_models)
    sigs, rates = _mixed_list()
    starts = [0.25 * i for i in range(len(sigs))]
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        got = seg.segment_signals(sigs, starts, rates)
        assert got == [seg.segment_signal(s, t, r) for s, t, r in zip(sigs, starts, rates)]


def test_segment_signals_long_resampled_recording(rt, synth_models):
    """A 48 kHz recording of LONG_FRAMES frames at 16 kHz goes through segment_signal, one frame fewer is packed."""
    from inaspeechsegmenter_b200 import pack
    seg = _segmenter(rt, synth_models)
    n16 = (pack.LONG_FRAMES - 1) * 160 + 400
    x = synth_audio(n16 * 3 / 48000, seed=50, sr=48000)
    sigs, rates = [x, x[:-3], synth_audio(5, seed=51, sr=48000)], [48000] * 3
    passes, long_ = rt['resample'].plan(sigs, rates)
    assert long_ == [0] and passes == [[1, 2]]
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        assert seg.segment_signals(sigs, sample_rates=rates) == [seg.segment_signal(s, 0, r) for s, r in zip(sigs, rates)]


def test_errors_before_any_launch(rt, synth_models):
    seg = _segmenter(rt, synth_models)
    lib = rt['lib'].load()
    x = synth_audio(2, seed=60, sr=48000)
    c0 = lib.iss_launch_count()
    for bad in (7999, 192001, 44100.5, None):
        with pytest.raises(ValueError):
            seg.segment_signal(x, sample_rate=bad)
        with pytest.raises(ValueError):
            seg.segment_signals([x, x], sample_rates=[48000, bad])
    with pytest.raises(ValueError, match='channels'):
        seg.segment_signal(np.zeros((48000, 9), np.int16), sample_rate=48000)
    with pytest.raises(ValueError):
        seg.segment_signal(np.zeros((48000, 2, 2), np.int16), sample_rate=48000)
    with pytest.raises(TypeError):
        seg.segment_signal(x.astype(np.float64), sample_rate=48000)
    with pytest.raises(TypeError):
        seg.segment_signals([x, torch.from_numpy(x.astype(np.int32)).cuda()], sample_rates=[48000, 48000])
    with pytest.raises(ValueError, match='2 signals but 1 sample rates'):
        seg.segment_signals([x, x], sample_rates=[48000])
    with pytest.raises(ValueError, match='<signal 1> holds 399 samples'):
        seg.segment_signals([x, x[:1197]], sample_rates=[48000, 48000])
    assert lib.iss_launch_count() == c0


# ------------------------------------------------------------------ VoiceFemininityScoring
def test_score_signal_and_signals_resampled(rt, synth_models):
    from inaspeechsegmenter_b200 import vbx_segmenter as vb
    from test_vfs_pack_gpu import vfs_models
    vfs = vb.VoiceFemininityScoring(ffmpeg=None, models=vfs_models(synth_models))
    x48 = _stereo(30, 48000, 70)
    q, tie, _, _ = reference(x48, 48000)
    assert not tie.any()

    def score(fn):
        try:
            return fn()
        except ZeroDivisionError as e:          # score_signal's own error when no window is kept
            return type(e)

    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        got = vfs.score_signal(x48, sample_rate=48000)
        assert got == vfs.score_signal(q) and got[2] > 0
        sigs, rates = _mixed_list()
        ref = [score(lambda: vfs.score_signal(s.cpu().numpy() if isinstance(s, torch.Tensor) and r == 16000 else s,
                                              'signal', r)) for s, r in zip(sigs, rates)]   # 16 kHz mono from the host
        err = next((r for r in ref if isinstance(r, type)), None)
        assert score(lambda: vfs.score_signals(sigs, sample_rates=rates)) == (ref if err is None else err)
        assert sum(isinstance(r, tuple) and r[2] > 0 for r in ref) >= 3, ref
