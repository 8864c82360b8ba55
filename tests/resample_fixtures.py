"""Cases for the resampler's domain tests (test_resample_domain.py on the CPU, test_resample_domain_gpu.py on an
H100): the rate set, the per-tap error of the kernel's taps against oracle/resample_ref.py, the rule that holds the
kernel's int16 output to the oracle at near ties, and a restatement of resample.cu's tile_for that picks lengths."""
import functools

import numpy as np

from oracle import resample_ref as rr

# 8001 / 15999 / 16001 and 191999 Hz: 16000 phases, up > down and up < down; 191999 Hz: 3.8 million taps, 240 per
# output, and k * down past 2^31 after 11185 outputs; 47952 Hz (NTSC pull-down): 1000 / 2997; 44056 Hz: 2000 / 5507
RATES = [8000, 8001, 11025, 12000, 15999, 16001, 22050, 32000, 37800, 44056, 44100, 47952, 48000, 64000, 88200, 96000,
         176400, 191999, 192000]
TILES = (64, 128, 256, 512, 1024)


@functools.lru_cache(maxsize=None)
def tap_err(rate):
    """|h' - h| tap by tap: h' the taps the kernel uses (resample.lowpass), h those of the oracle (rr.taps)."""
    from inaspeechsegmenter_b200 import resample
    up, down = rr.factors(rate)
    e = np.abs(resample.lowpass(up, down) - rr.taps(up, down))
    e.setflags(write=False)
    return e


def reference(x, rate):
    """rr.reference of a recording, its bound covering the kernel's taps."""
    return rr.reference(x, rate, tap_err(rate))


def check(got, x, rate, what):
    """The kernel's int16 output `got` equals the oracle's at every output not flagged as a near tie, and is one of
    the two integers around y * 32768 (clipped) at a flagged one.  Returns the number of flagged outputs."""
    q, tie, y, _ = reference(x, rate)
    got = np.asarray(got)
    assert got.shape == q.shape, (what, got.shape, q.shape)
    lo = np.clip(np.floor(y * 32768.0), -32768, 32767)
    ok = np.where(tie, (got == lo) | (got == np.clip(lo + 1, -32768, 32767)), got == q)
    bad = np.flatnonzero(~ok)
    assert not len(bad), (what, len(bad), bad[:5], got[bad][:5], q[bad][:5])
    return int(tie.sum())


@functools.lru_cache(maxsize=None)
def reach(rate):
    """(s_min, e_max) from the filter's index range (h[k down + H - m up] is a tap for 0 <= k down + H - m up <= 2H):
    output k reads frames floor(k down / up) + s_min .. + e_max - 1 at most."""
    up, down = rr.factors(rate)
    H = 0 if up == down == 1 else 10 * max(up, down)
    k = np.arange(up, dtype=np.int64)
    a = k * down // up
    return int((-((H - k * down) // up) - a).min()), int(((k * down + H) // up - a).max()) + 1


def tile_for(rate, channels, nbytes):
    """Outputs per CTA that resample.cu's tile_for picks for `channels` samples of `nbytes` bytes a frame: the largest
    power of two from 1024 down whose staged span (float64 frames, then the raw samples and one 16-byte vector of
    slack, each rounded up to 16 bytes) fits 96 KiB."""
    up, down = rr.factors(rate)
    s_min, e_max = reach(rate)
    to = 1024
    while True:
        span = ((to - 1) * down + up - 1) // up + 1 + (e_max - s_min)
        smem = (span * 8 + 15) // 16 * 16 + (span * channels * nbytes + 31) // 16 * 16
        if smem <= 96 * 1024 or to == 32:
            return to
        to //= 2


def frames_for(rate, n_out):
    """The fewest input frames that give n_out outputs or more (more only where up > down skips counts: every length
    gives an even count at 8 kHz)."""
    up, down = rr.factors(rate)
    return (n_out - 1) * down // up + 1


def lengths(rate, channels, nbytes):
    """Boundary lengths in input frames: 1, 2, down - 1 .. down + 1, one filter span - 1 .. + 1, and the length whose
    last tile holds one output (two at 8 kHz), some 3000 outputs in, or past 2^31 in k * down where that comes within
    30000 outputs (191999 Hz)."""
    up, down = rr.factors(rate)
    span = (20 * max(up, down) + 1) // up + 1            # input frames under one output's taps
    tile = tile_for(rate, channels, nbytes)
    target = 2 ** 31 // down + 1 if 2 ** 31 // down < 30000 else 3000
    n_out = tile * -(-target // tile) + 1
    return sorted({1, 2, max(down - 1, 1), down, down + 1, span - 1, span, span + 1, frames_for(rate, n_out)})
