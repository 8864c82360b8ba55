"""The rules live femininity scores decide by (vfs_stream), checked on the CPU: the dither as a restated MT19937 against
numpy's RandomState(3) draws, raw fbank rows against vbx_oracle on prefixes, the CMVN chunk replay of a window against
the replay of the whole recording, and window decidability against window_plan, over many chunkings."""
import numpy as np
import pytest

from oracle import vbx_oracle as vx
from inaspeechsegmenter_b200 import vfs_stream as vs
from vfs_stream_oracle import cmvn_rows as _replay

CHUNKINGS = (1, 159, 160, 161, 399, 400, 'random', 'one')


def _mt_twist(mt):
    """The MT19937 twist in its three dependent phases, as the kernel runs it."""
    mt = mt.copy()
    for lo, hi in ((0, 227), (227, 454), (454, 624)):
        i = np.arange(lo, hi)
        y = (mt[i] & 0x80000000) | (mt[(i + 1) % 624] & 0x7fffffff)
        mt[i] = mt[(i + 397) % 624] ^ (y >> 1) ^ np.where(y & 1, 0x9908b0df, 0).astype(np.uint32)
    return mt


def _mt_dither(state, n):
    """(next n dither values, state): tempering and res53 as numpy's legacy RandomState.rand."""
    mt, pos = state
    out = []
    while len(out) < n:
        if pos >= 624:
            mt, pos = _mt_twist(mt), 0
        m = min((624 - pos) // 2, n - len(out))
        y = mt[pos:pos + 2 * m].astype(np.uint64)
        y ^= y >> 11
        y ^= (y << 7) & 0x9d2c5680
        y ^= (y << 15) & 0xefc60000
        y ^= y >> 18
        a, b = (y[0::2] >> 5).astype(np.float64), (y[1::2] >> 6).astype(np.float64)
        out += list(8 * ((a * 67108864.0 + b) / 9007199254740992.0 * 2 - 1))
        pos += 2 * m
    return np.array(out), (mt, pos)


def _cuts(n, how, rng):
    if how == 'one':
        return [n]
    if how == 'random':
        return sorted(set(rng.integers(1, n, 25).tolist())) + [n]
    return list(range(how, n, how)) + [n]


def test_seed_row_is_randomstate_3():
    row = vs._mt_seed().view(np.uint32)
    _, key, pos = np.random.RandomState(3).get_state()[:3]
    assert np.array_equal(row[:624], key) and row[624] == pos == 624


@pytest.mark.parametrize('how', [1, 311, 312, 313, 623, 'random'])
def test_mt19937_restatement_equals_dither_stream(how):
    ref = vx.dither_stream(5000)
    row = vs._mt_seed().view(np.uint32)
    state = (row[:624].copy(), int(row[624]))
    got, pos, rng = [], 0, np.random.default_rng(2)
    for b in _cuts(5000, how, rng):
        d, state = _mt_dither(state, b - pos)
        got.append(d)
        pos = b
    assert np.array_equal(np.concatenate(got), ref)


def test_raw_rows_final_by_rule_and_not_before():
    """Row r of an open stream of n samples equals the whole stream's once 160 r + 280 <= n, and not one row later."""
    x = vx.quantise(np.random.default_rng(4).standard_normal(16000 * 2).astype(np.float32) * 0.1) / 32768.0
    whole = vx.raw_fbank(x)
    for n in (200, 279, 280, 281, 399, 400, 401, 439, 440, 441, 1000, 4321, 16000):
        pre = vx.raw_fbank(x[:n])
        R = vs.final_raw_rows(n)
        assert np.array_equal(pre[:R], whole[:R]), n
        if R < len(pre):
            assert not np.array_equal(pre[R], whole[R]), n
        assert len(pre) == vs.vbx_frames(n)


@pytest.mark.parametrize('M', [127, 128, 129, 143, 144, 145, 299, 300, 301, 450])
def test_cmvn_and_windows_by_rule(M):
    """Driven by the samples of every chunking, the retained raw rows and the final CMVN rows reproduce the replay on the
    whole recording (and, to rounding, get_features' cumulative-sum form), and the windows decided by the rule are
    window_plan(M)'s, each decided only once its rows are final."""
    rng = np.random.default_rng(M)
    raw = rng.standard_normal((M, 4)) * 3 + 10
    whole = _replay(raw, 0, M, 0, M)
    assert np.allclose(whole, vx.cmvn_floating(raw), rtol=0, atol=1e-9)
    n_total = 80 + 160 * (M - 1) + 37
    plan = vx.window_plan(M)
    for how in CHUNKINGS:
        R = T = w = 0
        keep = 0
        got, wins = [], []
        cuts = _cuts(n_total, how, rng)
        for i, n in enumerate(cuts):
            end = i == len(cuts) - 1
            R2 = vs.vbx_frames(n) if end else vs.final_raw_rows(n)
            T2 = R2 if end else vs.final_cmvn_rows(R2)
            assert vs.sample_keep(R2) <= max(0, 160 * R2 - 120)
            if T2 > T:
                got.append(_replay(raw[keep:R2], keep, R2, T, T2 - T))
                if not end:     # one row more with the same rows known is not the whole recording's
                    early = _replay(raw[keep:R2], keep, R2, T2, 1) if T2 < R2 else None
                    assert early is None or M <= T2 or not np.array_equal(early[0], whole[T2])
            keep = vs.raw_keep(T2, R2)
            R, T = R2, T2
            starts = vs.decided_windows(w, T, float('inf'), M if end else None)
            assert all(s + 144 <= T for s in starts)
            wins += [(s, 144, False) for s in starts]
            w += len(starts)
            if end:
                s = vs.tail_start(w, M)
                if s is not None:
                    wins.append((s, M - s, True))
        assert np.array_equal(np.concatenate(got), whole), how
        assert wins == plan, how
