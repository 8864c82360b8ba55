"""Resampled live streams on the GPU (run with -m gpu on an H100): the 16 kHz samples a stream's calls produce against
resample.to16k on the whole stream, segments against segment_signal and the calibration-prefix reference, many mixed
streams against each stream alone, errors, the window checks of iss_resample_window_multi and launch counts."""
import os
import warnings

import numpy as np
import pytest

from conftest import synth_audio
from test_sample_rates_gpu import RATES, _recording
from test_stream_gpu import _prefix_reference

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')


@pytest.fixture(scope='module')
def rt():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from inaspeechsegmenter_b200 import _lib, engine, pack, resample, segmenter, stream
    return dict(lib=_lib, engine=engine, pack=pack, resample=resample, segmenter=segmenter, stream=stream)


def _segmenter(rt, synth_models, vad='smn', gender=True, fft='fp64'):
    return rt['segmenter'].Segmenter(vad_engine=vad, detect_gender=gender, ffmpeg=None, fft_precision=fft,
                                     models={'vad': synth_models[vad], 'gender': synth_models['gender']})


def _parts(n, how, rng, rate=16000):
    if how == 'one':
        return [(0, n)]
    if how == 'random':
        out, pos = [], 0
        while pos < n:
            m = max(1, int(rng.uniform(0.01, 3.0) * rate))
            out.append((pos, min(pos + m, n)))
            pos += m
        return out
    return [(a, min(a + how, n)) for a in range(0, n, how)]


def _on_device(c, misaligned):
    """A CUDA copy of c; misaligned: a view one frame into a larger buffer (not 16-byte aligned)."""
    if not misaligned:
        return torch.from_numpy(np.ascontiguousarray(c)).cuda()
    big = torch.from_numpy(np.concatenate([c[:1], c])).cuda()
    return big[1:]


def _backend_stream(be, sid, x, rate, parts, where):
    """The 16 kHz samples CudaBackend.resample hands on for one stream fed in `parts`, then flushed."""
    got = []
    for a, b in parts:
        c = x[a:b]
        if where != 'host':
            c = _on_device(c, where == 'view')
        got.append(be.resample({sid: c}, {sid: rate})[sid])
    got.append(be.resample({}, {sid: rate}, [sid])[sid])
    be.release(sid)
    return torch.cat(got)


# ---- the 16 kHz samples --------------------------------------------------------------------------------------
@pytest.mark.parametrize('rate', RATES)
@pytest.mark.parametrize('fmt', ['int16', 'float32'])
def test_streamed_samples_equal_whole_stream(rt, synth_models, rate, fmt):
    seg = _segmenter(rt, synth_models)
    resample = rt['resample']
    up, down = resample.factors(rate)
    rng = np.random.default_rng(rate)
    be = rt['stream'].CudaBackend(seg)
    for C in (1, 2, 6):
        if rate == 16000 and C == 1:
            continue                        # 16 kHz mono streams are never resampled
        x = _recording(rate, 2 * rate + 333, C, fmt, seed=rate + C)
        x = x[:, 0] if C == 1 else x
        for where in ('host', 'view'):
            for how in (1, max(down - 1, 1), down, down + 1, 997, 'random', 'one'):
                xs = x[:300 * how] if isinstance(how, int) and how < 100 else x      # at most 300 calls
                ref = resample.to16k(seg.ctx, xs, rate)
                got = _backend_stream(be, 0, xs, rate, _parts(len(xs), how, rng, rate), where)
                assert torch.equal(got, ref), (rate, fmt, C, where, how)


def test_mixed_streams_in_one_call_equal_streams_alone(rt, synth_models):
    seg = _segmenter(rt, synth_models)
    resample = rt['resample']
    spec = [(48000, 2, 'int16'), (44100, 1, 'float32'), (8000, 1, 'int16'), (48000, 2, 'int16'), (22050, 6, 'float32'),
            (16000, 2, 'int16'), (44100, 1, 'float32'), (192000, 1, 'int16'), (11025, 2, 'float32')] * 4
    xs = [_recording(r, int(r * 0.9) + 37 * i, C, f, seed=i) for i, (r, C, f) in enumerate(spec)]
    xs = [x[:, 0] if C == 1 else x for x, (_, C, _) in zip(xs, spec)]
    rates = {i: r for i, (r, _, _) in enumerate(spec)}
    chunk = {i: int(rates[i] * (0.05 + 0.01 * i)) for i in rates}
    be = rt['stream'].CudaBackend(seg)
    got = {i: [] for i in rates}
    pos = {i: 0 for i in rates}
    while any(pos[i] < len(xs[i]) for i in rates):
        feed = {}
        for i in rates:
            if pos[i] < len(xs[i]):
                c = xs[i][pos[i]:pos[i] + chunk[i]]
                feed[i] = _on_device(c, True) if i % 3 == 1 else c
                pos[i] += chunk[i]
        for i, v in be.resample(feed, {i: rates[i] for i in feed}).items():
            got[i].append(v)
    for i, v in be.resample({}, rates, list(rates)).items():
        got[i].append(v)
    alone = rt['stream'].CudaBackend(seg)
    for i in rates:
        whole = torch.cat(got[i])
        assert torch.equal(whole, resample.to16k(seg.ctx, xs[i], rates[i])), i
        assert torch.equal(whole, _backend_stream(alone, 0, xs[i], rates[i], _parts(len(xs[i]), chunk[i], None),
                                                  'host')), i


def test_feed_hands_the_pipeline_the_whole_stream_resampled(rt, synth_models):
    """What LiveStreams ingests for a resampled stream, over its feed and end calls, is to16k on the whole stream."""
    seg = _segmenter(rt, synth_models)
    x = np.stack([synth_audio(7, seed=3, sr=44100), synth_audio(7, seed=4, sr=44100)], axis=1)
    live = seg.stream(calibration_sec=2.0)
    seen = []
    ingest = live.backend.ingest

    def spy(chunks, keep):
        seen.extend(chunks.values())
        return ingest(chunks, keep)
    live.backend.ingest = spy
    for a in range(0, len(x), 30001):
        live.feed({'s': x[a:a + 30001]}, sample_rate=44100)
    live.end(['s'])
    assert torch.equal(torch.cat(seen), rt['resample'].to16k(seg.ctx, x, 44100))


# ---- end to end --------------------------------------------------------------------------------------------------
def _stream_alone(seg, x, rate, cal, how, seed=0, cuda=False):
    live = seg.stream(calibration_sec=cal)
    got = []
    for a, b in _parts(len(x), how, np.random.default_rng(seed), rate):
        c = torch.from_numpy(np.ascontiguousarray(x[a:b])).cuda() if cuda else x[a:b]
        got += live.feed({'k': c}, sample_rate=rate)['k']
    return got + live.end(['k'])['k']


def _media(media, name):
    from inaspeechsegmenter_b200.io import media2sig16kmono
    return media2sig16kmono(os.path.join(media, name), None, None, None, 'float32', return_int16=True)


def test_short_streams_equal_segment_signal(rt, synth_models, media):
    from scipy.signal import resample_poly
    seg = _segmenter(rt, synth_models)
    m = _media(media, 'musanmix.wav').astype(np.float64)
    up = resample_poly(m, 3, 1)
    musan48 = np.clip(np.round(np.stack([up, 0.5 * up], axis=1)), -32768, 32767).astype(np.int16)
    cases = [(musan48, 48000), (np.stack([synth_audio(9, seed=1, sr=44100)] * 2, axis=1), 44100),
             (synth_audio(4, seed=2, sr=8000), 8000), (_recording(22050, 30000, 6, 'float32', seed=3), 22050),
             (synth_audio(0.1, seed=5, sr=48000), 48000)]
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        for i, (x, rate) in enumerate(cases):
            ref = seg.segment_signal(x, sample_rate=rate)
            cal = len(x) / rate + 2
            for how in ('random', rate // 2 + 3) if i == 0 else ('one', 'random', 4001):
                assert _stream_alone(seg, x, rate, cal, how, seed=i, cuda=i == 1) == ref, (i, how)


@pytest.mark.parametrize('vad,gender,fft', [('smn', True, 'fp64'), ('sm', True, 'fp32'), ('smn', False, 'fp32'),
                                            ('sm', False, 'fp64')])
def test_long_streams_equal_prefix_threshold_reference(rt, synth_models, vad, gender, fft):
    seg = _segmenter(rt, synth_models, vad, gender, fft)
    for rate, seed in ((44100, 9), (48000, 10)):
        x = np.stack([synth_audio(180, seed=seed, sr=rate), synth_audio(180, seed=seed + 100, sr=rate) // 4], axis=1)
        y = rt['resample'].to16k(seg.ctx, x, rate).cpu().numpy()
        ref = _prefix_reference(rt, seg, y, 500)
        for how in (rate, 'random'):
            assert _stream_alone(seg, x, rate, 5.0, how, seed=3) == ref, (rate, how)


def test_many_mixed_streams_equal_streams_alone(rt, synth_models):
    seg = _segmenter(rt, synth_models)
    rng = np.random.default_rng(11)
    audio = {r: synth_audio(200, seed=21 + r // 1000, sr=r) for r in (16000, 48000, 44100, 8000)}
    N = 300
    sigs, rates, starts, chunk, cuda = [], [], [], [], []
    for i in range(N):
        kind = i % 5                        # 16 kHz int16, 16 kHz float, 48 kHz stereo, 44.1 kHz mono, 8 kHz
        rate = (16000, 16000, 48000, 44100, 8000)[kind]
        n = int(rng.uniform(0.3, 20.0) * rate)
        a = int(rng.integers(0, len(audio[rate]) - n))
        x = audio[rate][a:a + n]
        if kind == 1:
            x = x.astype(np.float32) / np.float32(32768)
        elif kind == 2:
            x = np.stack([x, audio[rate][a // 2:a // 2 + n]], axis=1)
        elif kind == 3 and i % 2:
            x = x.astype(np.float32) / np.float32(32768)
        sigs.append(x)
        rates.append(rate)
        starts.append(int(rng.integers(0, 8)))
        chunk.append(int(rng.choice([0.1, 0.5, 1.0, 1.4657]) * rate))
        cuda.append(i % 7 == 3)
    live = seg.stream(calibration_sec=3.0)
    got = {i: [] for i in range(N)}
    pos = [0] * N
    step = 0
    open_ = set()
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        while any(pos[i] < len(sigs[i]) for i in range(N)):
            feed = {}
            for i in range(N):
                if starts[i] <= step and pos[i] < len(sigs[i]):
                    c = sigs[i][pos[i]:pos[i] + chunk[i]]
                    feed[i] = torch.from_numpy(np.ascontiguousarray(c)).cuda() if cuda[i] else c
                    pos[i] += len(c)
            for k, v in live.feed(feed, sample_rate={i: rates[i] for i in feed}).items():
                got[k] += v
            open_ |= set(feed)
            done = [i for i in open_ if pos[i] >= len(sigs[i]) and i % 2 == 0 and rt['resample'].num_frames(
                len(sigs[i]), rates[i]) >= 400]
            for k, v in live.end(done).items():
                got[k] += v
            open_ -= set(done)
            step += 1
        for k, v in live.end(sorted(i for i in open_ if rt['resample'].num_frames(len(sigs[i]), rates[i]) >= 400)).items():
            got[k] += v
        # a key reused after end starts fresh, at another rate
        again = live.feed({0: sigs[2]}, sample_rate=rates[2])[0] + live.end([0])[0]
        assert again == _stream_alone(seg, sigs[2], rates[2], 3.0, 'one')
        for i in range(N):
            x = sigs[i]
            if rt['resample'].num_frames(len(x), rates[i]) < 400:
                continue
            assert got[i] == _stream_alone(seg, x, rates[i], 3.0, chunk[i], cuda=cuda[i]), i


def test_calibration_reached_only_at_the_flush(rt, synth_models):
    """The last 16 kHz samples of a 48 kHz stream, computed by end, complete its calibration: it is then decoded
    online and still gives segment_signal (a stream of exactly N_cal frames)."""
    seg = _segmenter(rt, synth_models)
    n16 = 299 * 160 + 400
    x = np.stack([synth_audio(n16 * 3 / 48000, seed=12, sr=48000)[:3 * n16]] * 2, axis=1)
    resample = rt['resample']
    assert resample.end_outputs(len(x), 48000) == n16 and rt['pack'].num_frames(resample.ready_outputs(len(x), 48000)) < 300
    live = seg.stream(calibration_sec=3.0)
    got = live.feed({'a': x}, sample_rate=48000)['a']
    assert not live.streams['a'].calibrated
    got += live.end(['a'])['a']
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        assert got == seg.segment_signal(x, sample_rate=48000)


def test_stream_short_after_resampling(rt, synth_models):
    seg = _segmenter(rt, synth_models)
    x = synth_audio(0.1, seed=3, sr=48000)[:1197]            # 399 samples at 16 kHz
    with pytest.raises(ValueError) as ref:
        seg.segment_signal(x, sample_rate=48000)
    live = seg.stream(calibration_sec=1.0)
    live.feed({'a': x[:600], 'b': synth_audio(1, seed=4, sr=48000)}, sample_rate=48000)
    live.feed({'a': x[600:]}, sample_rate=48000)
    with pytest.raises(ValueError) as got:
        live.end(['a'])
    assert str(got.value) == str(ref.value) and 'holds 399 samples' in str(got.value)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        assert live.end(['b'])['b'] == seg.segment_signal(synth_audio(1, seed=4, sr=48000), sample_rate=48000)


# ---- errors ------------------------------------------------------------------------------------------------------
def test_errors_change_nothing(rt, synth_models):
    seg = _segmenter(rt, synth_models)
    x = np.stack([synth_audio(6, seed=1, sr=48000)] * 2, axis=1)
    m = synth_audio(6, seed=2)

    def run(bad_calls):
        live = seg.stream(calibration_sec=2.0)
        out = {'s': [], 'm': []}
        for i in range(0, 6):
            for k, v in live.feed({'s': x[i * 48000:(i + 1) * 48000], 'm': m[i * 16000:(i + 1) * 16000]},
                                  sample_rate={'s': 48000, 'm': 16000}).items():
                out[k] += v
            if bad_calls and i == 2:
                for exc, chunks, rate in bad_calls:
                    with pytest.raises(exc):
                        live.feed(chunks, sample_rate=rate)
        for k, v in live.end(['s', 'm']).items():
            out[k] += v
        return out

    s1 = x[:4800]
    bad = [(ValueError, {'new': s1}, 7999), (ValueError, {'new': s1}, 192001), (ValueError, {'new': s1}, 44100.5),
           (ValueError, {'new': np.zeros((4800, 9), np.int16)}, 48000),
           (TypeError, {'new': s1.astype(np.float64)}, 48000),
           (ValueError, {'new': np.zeros((4800, 2, 2), np.int16)}, 48000),
           (ValueError, {'new': s1, 's': s1}, {'new': 48000}),
           (ValueError, {'s': s1}, 44100), (ValueError, {'s': s1[:, :1]}, 48000),
           (ValueError, {'s': s1.mean(axis=1).astype(np.int16)}, 48000),
           (TypeError, {'s': s1.astype(np.float32)}, 48000), (TypeError, {'s': torch.from_numpy(s1).cuda()}, 48000),
           (ValueError, {'m': m[:100]}, 8000), (ValueError, {'m': np.stack([m[:100]] * 2, axis=1)}, 16000),
           (ValueError, {'s': s1, 'm': m[:100]}, {'s': 48000, 'm': 44100})]
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        assert run(bad) == run([])


def test_window_entry_point_rejects_records_outside_their_window(rt, synth_models):
    """Host-side checks of iss_resample_window_multi; nothing is launched."""
    seg = _segmenter(rt, synth_models)
    lib, resample = rt['lib'], rt['resample']
    L = lib.load()
    resample._ensure_taps(seg.ctx, 48000)
    x = torch.zeros(600, dtype=torch.int16, device='cuda')
    out = torch.empty(400, dtype=torch.int16, device='cuda')
    s_min, e_max = resample.reach(48000)                       # -30, 31: output k reads frames 3k - 30 .. 3k + 30
    ptrs = (lib._c.c_void_p * 2)(x.data_ptr(), x.data_ptr())
    good = [0, 100, 0, resample.ready_outputs(100, 48000), 0, 0]

    def call(row, first=good):
        w = np.array([first, row], dtype=np.int64)
        c0 = L.iss_launch_count()
        rc = L.iss_resample_window_multi(seg.ctx.handle, 2, ptrs, lib.ptr(w), 1, 48000, lib.PCM_S16, lib.ptr(out), None)
        if rc != 0:
            assert L.iss_launch_count() == c0
        return rc, L.iss_last_error()

    assert call([200, 600, 77, 10, 100, 0])[0] == 0            # outputs 77..86 read frames 201 .. 288
    for row, what in (([202, 600, 77, 10, 100, 0], b'before the window'),          # output 77 reads frame 201
                      ([200, 600, 185, 10, 100, 0], b'has not ended'),               # output 194 reads frame 612
                      ([200, 600, 195, 10, 100, 1], b'past the'),                    # 200 outputs of 600 frames
                      ([-1, 600, 77, 10, 100, 0], b'bad field'), ([200, 100, 0, 0, 0, 0], b'bad field'),
                      ([200, 600, 77, 10, 100, 2], b'bad field')):
        rc, err = call(row)
        assert rc == -1, (row, rc)                             # ISS_ERR_INVALID
        assert b'record 1' in err and what in err, (row, err)
    assert call([200, 600, 190, 10, 100, 1])[0] == 0           # the stream's last outputs read its zero padding
    torch.cuda.synchronize()


def test_one_resampler_launch_per_group(rt, synth_models):
    seg = _segmenter(rt, synth_models)
    L = rt['lib'].load()
    x = np.stack([synth_audio(1, seed=7, sr=48000)] * 2, axis=1)
    for N in (1, 10, 300):
        be = rt['stream'].CudaBackend(seg)
        for step in range(3):
            feed = {i: x[step * 16000:(step + 1) * 16000] for i in range(N)}
            c0 = L.iss_launch_count()
            be.resample(feed, dict.fromkeys(feed, 48000))
            assert L.iss_launch_count() - c0 == 1, (N, step)
        c0 = L.iss_launch_count()
        be.resample({}, dict.fromkeys(range(N), 48000), list(range(N)))
        assert L.iss_launch_count() - c0 == 1, N
    # two groups, two launches
    be = rt['stream'].CudaBackend(seg)
    c0 = L.iss_launch_count()
    be.resample({0: x[:4800], 1: x[:4800, 0].copy()}, {0: 48000, 1: 48000})
    assert L.iss_launch_count() - c0 == 2
