"""Resampled live streams on the CPU: the readiness and retention rule of resample.py (ready_outputs, end_outputs,
first_kept) driving a windowed float64 evaluation (resample_window, a restatement of oracle/resample_ref.resample on
a window of the input), which must reproduce the whole-stream oracle exactly for every chunking; and stream.LiveStreams on a CPU oracle backend that resamples, against the oracle
segmentation of the whole stream's 16 kHz int16."""
import math

import numpy as np
import pytest

from conftest import synth_audio
from oracle import cnn_oracle
from oracle import resample_ref as rr
from oracle import sidekit_oracle as sk
from stream_oracle import OracleStreamBackend, segment_reference
from inaspeechsegmenter_b200 import models, resample
from inaspeechsegmenter_b200.stream import LiveStreams

RATES = [8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000, 96000, 192000]
RATIO = 0.03


def resample_window(xw, f_base, n_known, rate, k_first, n_out, end):
    """y[k_first .. k_first + n_out) of a stream as ``rr.resample`` evaluates them on the whole stream, from a window xw
    holding its frames [f_base, n_known) only: the same sum in the same order over the taps that hit the window, the
    others skipped or added as zeros, so the values are the same bits.  Frames past n_known are the stream's zero
    padding only once it has ended (end); ValueError if an output reads a frame in [0, f_base), or, before the end, a
    frame at or past n_known."""
    up, down = rr.factors(rate)
    xm = rr.downmix(xw) if len(xw) else np.zeros(0)
    if len(xm) != n_known - f_base:
        raise ValueError('the window holds %d frames, not [%d, %d)' % (len(xm), f_base, n_known))
    h = rr.taps(up, down)
    H = (len(h) - 1) // 2
    t = (k_first + np.arange(n_out, dtype=np.int64)) * down + H
    m_hi = t // up
    y = np.zeros(n_out)
    for j in range((2 * H) // up + 1):                      # rr.resample's loop, in its order
        m = m_hi - j
        hi = t - m * up
        need = (hi <= 2 * H) & (m >= 0)
        early = need & (m < f_base)
        if early.any():
            raise ValueError('output %d reads frame %d, before the window' % (k_first + np.argmax(early), m[early][0]))
        late = need & (m >= n_known)
        if not end and late.any():
            raise ValueError('output %d reads frame %d of %d before the end' % (k_first + np.argmax(late), m[late][0],
                                                                              n_known))
        ok = need & (m < n_known)
        if not ok.any():
            continue
        mm = np.where(ok, m - f_base, 0)
        hv = np.where(ok, h[np.minimum(hi, 2 * H)], 0.0)
        y += hv * xm[mm]
    return y


class StreamResampler:
    """One stream through the rule: its raw frames from first_kept on, outputs computed once ready_outputs says so and
    the rest at the end, each by the windowed evaluation (which raises if the window lacks a frame)."""

    def __init__(self, rate, C, dtype):
        self.rate, self.tail, self.f0, self.n, self.k = rate, np.zeros((0, C), dtype), 0, 0, 0
        self.tails = []                # retained frames after each call

    def push(self, x, end=False):
        if x is not None:
            self.tail = np.concatenate((self.tail, np.asarray(x).reshape(len(x), -1)))
            self.n += len(x)
        k_to = (resample.end_outputs if end else resample.ready_outputs)(self.n, self.rate)
        y = resample_window(self.tail, self.f0, self.n, self.rate, self.k, k_to - self.k, end)
        keep = min(resample.first_kept(k_to, self.rate), self.n)
        self.tail, self.f0, self.k = self.tail[keep - self.f0:], keep, k_to
        self.tails.append(len(self.tail))
        return y


def _signal(rate, n, C, fmt, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / rate
    x = np.clip(rng.standard_normal((n, C)) * 0.2 + 0.3 * np.sin(2 * np.pi * 440 * t[:, None]), -1, 1)
    if fmt == 'int16':
        return np.round(x * 32767).astype(np.int16)
    return x.astype(np.float32)


def _chunkings(rate, n, rng):
    up, down = rr.factors(rate)
    cuts = {1: None, 'down-1': max(down - 1, 1), 'down': down, 'down+1': down + 1, 997: 997}
    out = {}
    for name, c in cuts.items():
        size = 1 if c is None else c
        m = min(n, 400) if size == 1 else n
        out[name] = [(a, min(a + size, m)) for a in range(0, m, size)]
    bounds = np.unique(np.concatenate(([0, n], rng.integers(0, n, size=12))))
    out['random'] = list(zip(bounds[:-1].tolist(), bounds[1:].tolist()))
    out['one'] = [(0, n)]
    return out


def test_reach_matches_the_filter():
    """s_min / e_max from the phase algebra equal the frames each output reads by the filter's own index range:
    h[k down + H - m up] is a tap for 0 <= k down + H - m up <= 2H."""
    for rate in RATES + [12345, 191999]:
        up, down = rr.factors(rate)
        H = (len(rr.taps(up, down)) - 1) // 2
        k = np.arange(up, dtype=np.int64)
        a = k * down // up
        first = -((H - k * down) // up)                       # ceil((k down - H) / up)
        last = (k * down + H) // up
        assert resample.reach(rate) == (int((first - a).min()), int((last - a).max()) + 1), rate


def test_rule_restated():
    """ready_outputs, end_outputs and first_kept against a direct count of the rule they state."""
    for rate in RATES:
        up, down = rr.factors(rate)
        s_min, e_max = resample.reach(rate)
        for n in list(range(0, 3 * e_max + 2 * down + 3)) + [10 ** 6 + 7]:
            ks = np.arange(resample.num_frames(n, rate), dtype=np.int64)
            assert resample.ready_outputs(n, rate) == int((ks * down // up + e_max - 1 <= n - 1).sum()), (rate, n)
            assert resample.end_outputs(n, rate) == len(ks)
        for k in range(0, 4 * up + 5):
            assert resample.first_kept(k, rate) == max(0, k * down // up + s_min), (rate, k)


@pytest.mark.parametrize('rate', RATES)
@pytest.mark.parametrize('C', [1, 2, 6])
def test_windowed_stream_equals_whole_stream(rate, C):
    """Every chunking gives y bit for bit (so its int16 too), and the retained tail stays within one output's reach
    plus one step of the input."""
    up, down = rr.factors(rate)
    fmt = 'int16' if C != 2 else 'float32'
    n = max(2000, 6 * (20 * max(up, down) + 1) // up)
    x = _signal(rate, n, C, fmt, seed=rate + C)
    x = x[:, 0] if C == 1 else x
    rng = np.random.default_rng(rate * 7 + C)
    for name, parts in _chunkings(rate, n, rng).items():
        m = parts[-1][1]
        y_ref, _ = rr.resample(x[:m], rate)
        sr = StreamResampler(rate, C, x.dtype)
        ys = [sr.push(x[a:b]) for a, b in parts] + [sr.push(None, end=True)]
        y = np.concatenate(ys)
        assert np.array_equal(y, y_ref), (rate, C, name)
        assert np.array_equal(rr.quantise(y), rr.quantise(y_ref)), (rate, C, name)
        s_min, e_max = resample.reach(rate)
        assert max(sr.tails[:-1]) <= e_max - 1 - s_min + math.ceil(down / up), (rate, name)


def test_rule_off_by_one_fails(monkeypatch):
    """A readiness rule that releases one output early reads a frame not yet fed; a retention rule that drops one
    frame too many loses a frame a later output reads (48 kHz: one phase, so every output reads from a + s_min)."""
    x = _signal(48000, 4000, 2, 'int16', seed=1)
    ready, kept = resample.ready_outputs, resample.first_kept
    for name, fn in (('ready_outputs', lambda n, r: ready(n, r) + 1), ('first_kept', lambda k, r: kept(k, r) + 1)):
        with monkeypatch.context() as m:
            m.setattr(resample, name, fn)
            sr = StreamResampler(48000, 2, x.dtype)
            with pytest.raises(ValueError, match='reads frame'):
                for a in range(0, 4000, 250):
                    sr.push(x[a:a + 250])
                sr.push(None, end=True)


# ---- LiveStreams on a resampling oracle backend ------------------------------------------------------------------
class ResamplingOracleBackend(OracleStreamBackend):
    """OracleStreamBackend plus the resampler of CudaBackend, restated with StreamResampler: int16 numpy chunks of the
    16 kHz samples each call makes final."""

    def __init__(self, *a):
        super().__init__(*a)
        self.rs = {}

    def release(self, sid):
        super().release(sid)
        self.rs.pop(sid, None)

    def resample(self, chunks, rates, final=()):
        out = {}
        for sid in sorted(set(chunks) | set(final)):
            if sid not in self.rs:
                c = np.asarray(chunks[sid])
                self.rs[sid] = StreamResampler(rates[sid], 1 if c.ndim == 1 else c.shape[1], c.dtype)
            out[sid] = rr.quantise(self.rs[sid].push(chunks.get(sid), sid in final))
        return out


@pytest.fixture(scope='module')
def nets():
    vad = cnn_oracle.KerasLikeModel(*models.synthetic_keras_cnn(21, 3, seed=11, width=0.25), threads=2)
    gen = cnn_oracle.KerasLikeModel(*models.synthetic_keras_cnn(24, 2, seed=13, width=0.25), threads=2)
    return {'vad': (vad.predict, 21, ('speech', 'music', 'noise'), 80),
            'gender': (gen.predict, 24, ('female', 'male'), 80)}


def _live(nets, cal):
    from types import SimpleNamespace
    seg = SimpleNamespace(vad=SimpleNamespace(outlabels=nets['vad'][2]), gender=SimpleNamespace(outlabels=nets['gender'][2]),
                          detect_gender=True)
    return LiveStreams(seg, cal, backend=ResamplingOracleBackend(RATIO, nets))


def _expected(x, rate, n_cal, nets):
    q = rr.quantise(rr.resample(x, rate)[0])
    mspec, loge = sk.logmel_loge(q.astype(np.float32) / np.float32(32768))
    return segment_reference(mspec, loge, n_cal if len(loge) > n_cal else None, RATIO, nets)


def _feed_all(live, sigs, rates, sizes):
    """Every stream in the same calls, each cut in chunks of its own size, rates as a dict; segments per key."""
    got = {k: [] for k in sigs}
    pos = {k: 0 for k in sigs}
    while any(pos[k] < len(x) for k, x in sigs.items()):
        feed = {k: x[pos[k]:pos[k] + sizes[k]] for k, x in sigs.items() if pos[k] < len(x)}
        for k in feed:
            pos[k] += sizes[k]
        for k, v in live.feed(feed, sample_rate={k: rates[k] for k in feed}).items():
            got[k] += v
    for k, v in live.end(list(sigs)).items():
        got[k] += v
    return got


def test_resampled_streams_equal_oracle_segmentation(nets):
    a = synth_audio(14, seed=5, sr=48000)
    s48 = np.stack([a, (a // 3) + synth_audio(14, seed=6, sr=48000) // 8], axis=1)
    s8 = synth_audio(14, seed=8, sr=8000)
    sigs = {'48k long': s48, '8k long': s8, '48k short': s48[:48000 * 3 + 7], '8k short': s8[:8000 * 3 + 3]}
    rates = {'48k long': 48000, '8k long': 8000, '48k short': 48000, '8k short': 8000}
    sizes = {'48k long': 48000, '8k long': 3001, '48k short': 17777, '8k short': 8000}
    got = _feed_all(_live(nets, 5.0), sigs, rates, sizes)
    for k, x in sigs.items():
        ref = _expected(x, rates[k], 500, nets)
        assert got[k] == ref, k
    assert sum(len(_expected(x, rates[k], 500, nets)) for k, x in sigs.items()) >= 8


def test_calibration_reached_only_at_the_flush(nets):
    """A 48 kHz stream whose last 16 kHz samples, computed at the end, complete its 100-frame calibration."""
    n16 = 99 * 160 + 400
    x = synth_audio(3 * n16 / 48000, seed=12, sr=48000)[:3 * n16]
    assert resample.end_outputs(len(x), 48000) == n16 and resample.ready_outputs(len(x), 48000) < n16
    live = _live(nets, 1.0)
    got = live.feed({'a': x}, sample_rate=48000)['a']
    assert not live.streams['a'].calibrated
    got += live.end(['a'])['a']
    assert got == _expected(x, 48000, 100, nets)
