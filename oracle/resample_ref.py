"""float64 reference of the resampler (inaspeechsegmenter_b200/resample.py, resample.cu): downmix, then a direct
polyphase sum over the taps of resample_poly's default filter, with the float64 error bound of every output.  Written
without scipy, so that tests can hold it against ``scipy.signal.resample_poly`` and the kernel against it.

For a recording x of n frames, C channels at rate R (up = 16000 / g, down = R / g, g = gcd(16000, R)):
  x[m] = sum of the C channels of frame m in float64 (int16 s as s / 32768), over C,
  y[k] = sum over m of x[m] h[k down + H - m up], 0 <= k < ceil(n up / down), h the 2H + 1 taps (H = 10 max(up, down))
         of firwin(2H + 1, 1 / max(up, down), window=('kaiser', 5.0)) times up,
  out[k] = clip(round_half_even(y[k] 32768), -32768, 32767) as int16.
"""
import functools
import math

import numpy as np

U = 2.0 ** -53


def factors(rate):
    g = math.gcd(16000, rate)
    return 16000 // g, rate // g


@functools.lru_cache(maxsize=None)
def taps(up, down):
    """The 2H + 1 float64 taps of the filter, times up (kaiser(5.0) window, sinc, unit DC gain); read-only, computed
    once per (up, down) (3.8 million taps at 191999 Hz)."""
    if up == down == 1:
        h = np.ones(1)
    else:
        M = max(up, down)
        N = 20 * M + 1
        half = (N - 1) / 2
        t = np.arange(N) - half
        w = np.i0(5.0 * np.sqrt(1.0 - (t / half) ** 2)) / np.i0(5.0)
        h = np.sinc(t / M) / M * w
        h = h / h.sum() * up
    h.setflags(write=False)
    return h


def downmix(x):
    """float64 mean of the channels: their sum in channel order over C.  Additions and one division, each correctly
    rounded, so any IEEE evaluation in this order gives these bits: the definition holds them, not an error bound."""
    x = np.asarray(x)
    scale = 1.0 / 32768 if x.dtype == np.int16 else 1.0
    x2 = x.reshape(len(x), -1)
    s = np.zeros(len(x), dtype=np.float64)
    for c in range(x2.shape[1]):
        s = s + x2[:, c].astype(np.float64) * scale
    return s / x2.shape[1]


def resample(x, rate, tap_err=None):
    """(y float64, bound float64): y[k] as defined above, evaluated here in float64, and a bound on how far another float64
    evaluation of the same dot product (any order, FMA or not) can lie from it.  That evaluation may use other taps h':
    tap_err holds a bound on |h'[i] - h[i]| for each of the 2H + 1 taps, and each output's bound then grows by
    sum tap_err[i] |x[m]| over its taps.  Without tap_err the other evaluation uses these taps exactly.  With
    up == down == 1 the output is the downmix itself, and the bound is 0."""
    up, down = factors(rate)
    xm = downmix(x)
    n = len(xm)
    n_out = -(-n * up // down)
    h = taps(up, down)
    H = (len(h) - 1) // 2
    t = np.arange(n_out, dtype=np.int64) * down + H          # y[k] = sum_j h[t - m up] x[m], m = t // up - j
    m_hi = t // up
    if tap_err is not None:
        tap_err = np.asarray(tap_err, dtype=np.float64)
        assert tap_err.shape == h.shape, (tap_err.shape, h.shape)
    y = np.zeros(n_out)
    absum = np.zeros(n_out)
    errsum = np.zeros(n_out)
    ntap = 0
    for j in range((2 * H) // up + 1):
        m = m_hi - j
        hi = t - m * up
        ok = (hi <= 2 * H) & (m >= 0) & (m < n)
        if not ok.any():
            continue
        ntap += 1
        mm = np.where(ok, m, 0)
        hv = np.where(ok, h[np.minimum(hi, 2 * H)], 0.0)
        y += hv * xm[mm]
        absum += np.abs(hv * xm[mm])
        if tap_err is not None:
            errsum += np.where(ok, tap_err[np.minimum(hi, 2 * H)], 0.0) * np.abs(xm[mm])
    if up == down == 1:
        return y, np.zeros(n_out)
    # Both evaluations (this one with taps h, the other with h') lie within gamma_k times the sum of their absolute
    # products of their exact sums, gamma_k = k U / (1 - k U); the exact sums differ by at most errsum, and the other's
    # absolute products by at most absum + errsum.  The one-sided gamma_k on errsum also covers its own rounding here.
    k = ntap + 1
    g = k * U / (1 - k * U)
    return y, 2 * g * absum + (1 + 2 * g) * errsum


def quantise(y):
    """int16 clip(round_half_even(y * 32768), -32768, 32767)."""
    return np.clip(np.rint(y * 32768.0), -32768, 32767).astype(np.int16)


def near_tie(y, bound):
    """True where y * 32768 lies within its bound of a rounding midpoint m + 1/2: there, a correct float64 evaluation
    may round either way.  An output with bound 0 is the downmix itself, and an exact midpoint there rounds to even."""
    v = y * 32768.0
    return (bound > 0) & (np.abs(v - (np.floor(v) + 0.5)) <= bound * 32768.0)


def reference(x, rate, tap_err=None):
    """(int16 output, near-tie flags, y, bound) of a recording at `rate` Hz; tap_err as for resample."""
    y, bound = resample(x, rate, tap_err)
    return quantise(y), near_tie(y, bound), y, bound
