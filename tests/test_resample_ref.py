"""The float64 resampling reference (oracle/resample_ref.py) against scipy.signal.resample_poly, the host taps of
inaspeechsegmenter_b200/resample.py against scipy.signal.firwin, and the pass plan over resampled lengths (CPU)."""
import numpy as np
import pytest

from oracle import resample_ref as rr

signal = pytest.importorskip('scipy.signal')

RATES = [8000, 11025, 22050, 24000, 32000, 44100, 48000, 96000, 192000]


def _lengths(rate):
    up, down = rr.factors(rate)
    span = (20 * max(up, down) + 1) // up + 1          # input frames under one output's taps
    return sorted({1, 2, max(down - 1, 1), down, down + 1, span - 1, span, span + 1, 10 * rate})


def _fixtures(rate, n):
    rng = np.random.default_rng(rate + n)
    t = np.arange(n) / rate
    imp = np.zeros(n)
    imp[::max(n // 7, 1)] = 0.9
    square = np.where(np.sin(2 * np.pi * 997 * t) >= 0, 1.0, -1.0)
    return {'dc': np.full(n, 0.5), 'impulses': imp, 'square': square,
            'noise': np.clip(rng.standard_normal(n) * 0.3, -1, 1)}


def _poly(x, rate):
    up, down = rr.factors(rate)
    return signal.resample_poly(x, up, down) if (up, down) != (1, 1) else np.array(x, dtype=np.float64)


@pytest.mark.parametrize('rate', RATES)
def test_oracle_equals_resample_poly(rate):
    worst = 0.0
    for n in _lengths(rate):
        for name, x in _fixtures(rate, n).items():
            y, bound = rr.resample(x, rate)
            ref = _poly(x, rate)
            assert y.shape == ref.shape == (-(-n * rr.factors(rate)[0] // rr.factors(rate)[1]),), (n, name)
            err = float(np.abs(y - ref).max())
            assert err <= 1e-12, (rate, n, name, err)
            worst = max(worst, err)
    print('rate %d: worst |oracle - resample_poly| = %.2e' % (rate, worst))


def test_full_scale_square_saturates():
    x = _fixtures(48000, 48000)['square']
    q, tie, y, _ = rr.reference(x, 48000)
    assert y.max() * 32768 > 32767.5 and y.min() * 32768 < -32768.5      # the overshoot of the filter
    assert q.max() == 32767 and q.min() == -32768
    assert np.array_equal(q, np.clip(np.rint(_poly(x, 48000) * 32768), -32768, 32767).astype(np.int16))


@pytest.mark.parametrize('C', [1, 2, 3, 6, 8])
@pytest.mark.parametrize('dtype', ['int16', 'float32'])
def test_downmix_is_the_channel_mean(C, dtype):
    rng = np.random.default_rng(C)
    if dtype == 'int16':
        x = rng.integers(-32768, 32768, size=(4000, C)).astype(np.int16)
        xf = x / 32768.0
    else:
        x = (rng.standard_normal((4000, C)) * 0.3).astype(np.float32)
        xf = x.astype(np.float64)
    assert np.abs(rr.downmix(x) - xf.mean(axis=1)).max() <= 4e-16
    y, bound = rr.resample(x, 44100)
    assert np.abs(y - _poly(xf.mean(axis=1), 44100)).max() <= 1e-12


def test_ties_at_16k_round_to_even():
    """Up == down == 1: the output is the downmix itself, so exact midpoints are no near ties and round to even."""
    x = np.array([[1, 2], [2, 3], [-1, -2], [-2, -3], [32767, 32767], [-32768, -32767]], dtype=np.int16)
    q, tie, _, _ = rr.reference(x, 16000)
    assert not tie.any()
    assert list(q) == [2, 2, -2, -2, 32767, -32768]
    x6 = np.array([[1, 1, 1, 0, 0, 0], [3, 3, 3, 3, 3, 6]], dtype=np.int16)          # 3 / 6 and 21 / 6
    q, tie, _, _ = rr.reference(x6, 16000)
    assert not tie.any() and list(q) == [0, 4]


@pytest.mark.parametrize('rate', RATES)
def test_host_taps_equal_firwin(rate):
    from inaspeechsegmenter_b200 import resample
    up, down = resample.factors(rate)
    assert (up, down) == rr.factors(rate)
    M = max(up, down)
    ref = signal.firwin(2 * 10 * M + 1, 1.0 / M, window=('kaiser', 5.0)) * up
    h = resample.lowpass(up, down)
    assert h.dtype == np.float64 and h.shape == ref.shape
    assert np.abs(h - ref).max() <= 1e-15 * np.abs(ref).max()
    assert np.abs(rr.taps(up, down) - ref).max() <= 1e-15 * np.abs(ref).max()


def test_taps_per_phase():
    """The sizes the kernel sees: 8 821 taps in 160 phases at 44.1 kHz (55 or 56 per output), 61 at 48 kHz."""
    from inaspeechsegmenter_b200 import resample
    assert resample.lowpass(160, 441).size == 8821
    assert resample.lowpass(1, 3).size == 61
    assert resample.lowpass(1, 1).tolist() == [1.0]


def test_num_frames_and_rates():
    from inaspeechsegmenter_b200 import resample
    for rate in RATES + [16000, 44101, 191999]:
        up, down = resample.factors(rate)
        for n in (0, 1, 2, down - 1, down, down + 1, 12345):
            assert resample.num_frames(n, rate) == len(_poly(np.zeros(n), rate)) if n else resample.num_frames(n, rate) == 0
    for bad in (7999, 192001, 44100.5, '48k', None, True):
        with pytest.raises(ValueError):
            resample.check_rate(bad)
    assert resample.check_rate(np.int64(48000)) == 48000 and resample.check_rate(48000.0) == 48000


def test_input_checks():
    from inaspeechsegmenter_b200 import resample
    assert resample.is_native(np.zeros(10, np.float64), 16000)
    assert resample.is_native(np.zeros((10, 1), np.int16), 16000)
    assert not resample.is_native(np.zeros((10, 2), np.int16), 16000)
    assert not resample.is_native(np.zeros(10, np.int16), 48000)
    with pytest.raises(TypeError):
        resample.as_input(np.zeros((10, 2), np.float64))
    with pytest.raises(ValueError):
        resample.as_input(np.zeros((10, 9), np.int16))
    with pytest.raises(ValueError):
        resample.as_input(np.zeros((10, 2, 2), np.int16))
    x = np.zeros((20, 2), np.int16)[::2]
    assert resample.as_input(x).flags.c_contiguous


def test_plan_groups_mixed_rates_and_routes_by_resampled_length():
    from inaspeechsegmenter_b200 import pack, resample
    long16 = (pack.LONG_FRAMES - 1) * 160 + 400                   # exactly LONG_FRAMES frames at 16 kHz
    sigs = [np.zeros(32000, np.float32),                           # 16 kHz mono float: its own kind
            np.zeros((96000, 2), np.int16),                        # 48 kHz stereo -> 32000 int16 samples
            np.zeros(long16 * 3, np.int16),                        # 48 kHz: LONG_FRAMES frames after resampling
            np.zeros(long16 * 3 - 3, np.float32),                  # one frame fewer: packed
            np.zeros(32000, np.int16),                             # 16 kHz mono int16 shares the resampled int16 pass
            np.zeros((44100, 6), np.float32)]
    rates = [16000, 48000, 48000, 48000, 16000, 44100]
    passes, long_ = resample.plan(sigs, rates)
    assert long_ == [2]
    assert sorted(map(sorted, passes)) == [[0], [1, 3, 4, 5]]
    with pytest.raises(ValueError, match='<signal 1> holds 399 samples'):
        resample.plan([np.zeros(400, np.int16), np.zeros(1197, np.int16)], [16000, 48000])
    resample.plan([np.zeros(1200, np.int16)], [48000])            # 400 samples at 16 kHz: one frame
