"""The resampler's whole domain on the CPU, at the rates of resample_fixtures.RATES (16000 phases, 3.8 million taps,
NTSC pull-down): oracle/resample_ref.py against scipy.signal.resample_poly, its tap-error bound against the kernel's
taps, the live-stream rule and windowed evaluation with 1 to 8 channels, and WAV files of every encoding with 3 to 8
channels read by io.wav_data against read_wav."""
import functools
import struct

import numpy as np
import pytest

from oracle import resample_ref as rr
from resample_fixtures import RATES, TILES, frames_for, reach, tap_err, tile_for
from test_stream_resample import StreamResampler, _chunkings, _signal
from wav_fixtures import CHANNEL_MASKS, DOMAIN_CHANNELS, DOMAIN_RATES, ENCODINGS, decode, domain_fixtures

from inaspeechsegmenter_b200 import io as iss_io
from inaspeechsegmenter_b200 import resample

signal = pytest.importorskip('scipy.signal')


@functools.lru_cache(maxsize=None)
def _firwin(rate):
    """resample_poly's default filter for `rate` (before its scaling by up), designed once."""
    up, down = rr.factors(rate)
    M = max(up, down)
    return signal.firwin(2 * 10 * M + 1, 1.0 / M, window=('kaiser', 5.0))


def _poly(x, rate):
    up, down = rr.factors(rate)
    return signal.resample_poly(x, up, down, window=_firwin(rate))


def _inputs(rate, n):
    rng = np.random.default_rng(rate + n)
    t = np.arange(n) / rate
    imp = np.zeros(n)
    imp[::max(n // 7, 1)] = 0.9
    return {'dc': np.full(n, 0.5), 'impulses': imp, 'square': np.where(np.sin(2 * np.pi * 997 * t) >= 0, 1.0, -1.0),
            'noise': np.clip(rng.standard_normal(n) * 0.3, -1, 1)}


@pytest.mark.parametrize('rate', RATES)
def test_oracle_equals_resample_poly(rate):
    up, down = rr.factors(rate)
    span = (20 * max(up, down) + 1) // up + 1
    worst = 0.0
    for n in sorted({1, 2, max(down - 1, 1), down, down + 1, span - 1, span, span + 1, frames_for(rate, 3001)}):
        for name, x in _inputs(rate, n).items():
            y, _ = rr.resample(x, rate)
            ref = _poly(x, rate)
            assert y.shape == ref.shape == (resample.num_frames(n, rate),), (rate, n, name)
            err = float(np.abs(y - ref).max())
            assert err <= 1e-12, (rate, n, name, err)
            worst = max(worst, err)
    print('%d Hz: worst |oracle - resample_poly| = %.2e' % (rate, worst))


def _with_kernel_taps(monkeypatch, x, rate):
    """y of rr.resample evaluated with the kernel's taps (resample.lowpass) in place of the oracle's."""
    with monkeypatch.context() as m:
        m.setattr(rr, 'taps', resample.lowpass)
        return rr.resample(x, rate)[0]


@pytest.mark.parametrize('rate', RATES)
def test_tap_error_bound_covers_the_kernel_taps(monkeypatch, rate):
    """The same sum over the kernel's taps lies within the bound that tap_err gives, for noise and for an input that
    puts +-1 on the taps of one output where the two designs differ most (the difference is then sum |dh| itself)."""
    up, down = rr.factors(rate)
    e = tap_err(rate)
    h = rr.taps(up, down)
    H = (len(h) - 1) // 2
    n = frames_for(rate, 600)
    noise = np.clip(np.random.default_rng(rate).standard_normal(n) * 0.3, -1, 1)
    k = 300                                        # y[k] = sum_m x[m] h[k down + H - m up]
    m = np.arange(n)
    i = k * down + H - m * up
    on = (i >= 0) & (i <= 2 * H)
    dh = resample.lowpass(up, down)[i[on]] - h[i[on]]
    adverse = np.zeros(n)
    adverse[m[on]] = np.where(e[i[on]] >= np.median(e[i[on]]), np.sign(dh), 0.0)
    for name, x in (('noise', noise), ('adverse', adverse)):
        y, bound = rr.resample(x, rate, e)
        y0, bound0 = rr.resample(x, rate)
        assert np.array_equal(y, y0) and np.all(bound >= bound0)
        diff = np.abs(_with_kernel_taps(monkeypatch, x, rate) - y)
        assert np.all(diff <= bound), (rate, name, float((diff / np.maximum(bound, 1e-300)).max()))
    assert abs(float(np.sum(dh * adverse[m[on]]))) <= bound[k]


def test_rule_restated_every_rate():
    """ready_outputs, end_outputs and first_kept against the rule they state, counted over a sorted table of
    floor(k down / up): at the first lengths, around the first multiples of down and at random lengths to 10^7."""
    rng = np.random.default_rng(3)
    for rate in RATES:
        up, down = rr.factors(rate)
        s_min, e_max = reach(rate)
        ns = set(range(0, 3 * e_max + 2 * (down // up) + 3))
        ns |= {j * down + c + d for j in range(1, 4) for c in (0, e_max) for d in range(-3, 4)}
        ns |= set(rng.integers(0, 10 ** 7, size=200).tolist())
        a = np.arange(resample.num_frames(max(ns), rate) + 1, dtype=np.int64) * down // up
        for n in sorted(ns):
            total = resample.num_frames(n, rate)
            assert resample.ready_outputs(n, rate) == min(total, int(np.searchsorted(a, n - e_max, 'right'))), (rate, n)
            assert resample.end_outputs(n, rate) == total
        k = np.arange(0, 4 * up + 5, dtype=np.int64)
        assert [resample.first_kept(int(j), rate) for j in k] == np.maximum(0, k * down // up + s_min).tolist(), rate


@pytest.mark.parametrize('rate', RATES)
def test_windowed_stream_equals_whole_stream_every_channel_count(rate):
    """The rule driving the windowed evaluation reproduces the whole-stream oracle bit for bit with 1 to 8 channels,
    each channel count with its own chunkings (one-frame chunks, down - 1 .. down + 1, random, whole)."""
    up, down = rr.factors(rate)
    s_min, e_max = reach(rate)
    n = max(2000, 3 * (20 * max(up, down) + 1) // up)
    names = list(_chunkings(rate, n, np.random.default_rng(0)))
    for C in range(1, 9):
        fmt = 'int16' if C % 2 else 'float32'
        x = _signal(rate, n, C, fmt, seed=rate + C)
        x = x[:, 0] if C == 1 else x
        rng = np.random.default_rng(rate * 7 + C)
        parts = _chunkings(rate, n, rng)
        for name in (names[C % len(names)], 'random', 'down+1'):
            p = parts[name]
            m = p[-1][1]
            y_ref, _ = rr.resample(x[:m], rate)
            sr = StreamResampler(rate, C, x.dtype)
            y = np.concatenate([sr.push(x[a:b]) for a, b in p] + [sr.push(None, end=True)])
            assert np.array_equal(y, y_ref), (rate, C, name)
            assert max(sr.tails[:-1]) <= e_max - 1 - s_min + -(-down // up), (rate, C, name)


def test_gpu_cases_cover_every_tile():
    """The in-memory and WAV cases of test_resample_domain_gpu.py run every tile from 64 to 1024 outputs per CTA."""
    import test_resample_domain_gpu as g
    seen = {tile_for(r, C, b) for r in RATES for C in range(1, 9) for b in (2, 4)}
    seen |= {tile_for(r, C, iss_io.BYTES[e]) for r in g.WAV_RATES for C in g.WAV_CHANNELS for e in g.WAV_ENCODINGS}
    assert seen == set(TILES), sorted(seen)
    assert all(tile_for(r, 8, 8) == 64 for r in (176400, 191999, 192000))


def test_domain_wavs_decode_equals_read_wav(tmp_path):
    """Every encoding with 3, 4, 5, 7 and 8 channels at 11.025 to 191.999 kHz, in WAVE_FORMAT_EXTENSIBLE headers with
    the channel mask of the layout: wav_data's byte range through wav_fixtures.decode is read_wav's signal exactly."""
    wavs = domain_fixtures(str(tmp_path))
    assert len(wavs) == len(ENCODINGS) * len(DOMAIN_CHANNELS) * len(DOMAIN_RATES)
    for name, (path, enc, C, rate) in wavs.items():
        with open(path, 'rb') as f:
            head = f.read(44)
        assert struct.unpack('<HH', head[20:24]) == (0xFFFE, C) and struct.unpack('<I', head[40:44])[0] == CHANNEL_MASKS[C]
        w = iss_io.wav_data(path)
        assert (w.encoding, w.channels, w.rate, w.frames) == (enc, C, rate, 2001), name
        with open(path, 'rb') as f:
            f.seek(w.start)
            raw = f.read(w.nbytes)
        ref, sr = iss_io.read_wav(path, 'float64')
        assert sr == rate and ref.shape == (2001, C), name
        assert np.array_equal(decode(raw, enc, C), ref), name
