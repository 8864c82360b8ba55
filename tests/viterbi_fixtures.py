"""Seeded Viterbi fixtures for the exact K3 comparisons: inputs at which an argmax decision depends on the last bit.

Every generator is deterministic and checked on the CPU (tests/test_viterbi_fixtures.py) before any GPU use:
the ties are exact ties as the C oracle sees them, the near-ties really flip under a reassociated step sum or a
one-ulp emission change, and no posterior has a log within a few float64 ulps of a float32 rounding midpoint (where
CUDA's double log and the host's could round to different float32 emissions).

``dp`` is a plain numpy restatement of the oracle's DP with switchable defects (last-max tie-break, reassociated
step sum); it is used only to show what a fixture is sensitive to -- the states every test compares with come from
the C oracle (``oracle/viterbi_oracle.c``).
"""
import numpy as np

from oracle import viterbi_oracle as vo

WARP_SEAMS = (31, 32, 33, 63, 64, 65)
CHUNK_SEAMS = (255, 256, 257, 511, 512, 513)
ECH = 16384                                 # chunk of the chunk-parallel energy decode (viterbi.cu)
ENERGY_SEAMS = (ECH - 1, ECH, ECH + 1, 2 * ECH, 3 * ECH, 4 * ECH - 1, 4 * ECH, 4 * ECH + 1, 5 * ECH)
MIDPOINT_MARGIN = 16                        # float64 ulps a fixture's log(p) keeps from a float32 rounding midpoint


def assert_clear_of_midpoints(p):
    m = vo.f32_midpoint_margin(np.asarray(p, dtype=np.float32).ravel())
    assert m.min() > MIDPOINT_MARGIN, 'a fixture posterior lies %.1f float64 ulps from a float32 midpoint' % m.min()


def _clear(p):
    """p (float32) with every value whose log is near a float32 rounding midpoint moved one float32 ulp down."""
    p = np.asarray(p, dtype=np.float32).copy()
    for _ in range(8):
        bad = vo.f32_midpoint_margin(p) <= MIDPOINT_MARGIN
        if not bad.any():
            return p
        p[bad] = np.nextafter(p[bad], np.float32(0))
    raise AssertionError('could not move the posteriors clear of float32 midpoints')


def dp(e, A, reassoc=False, last_max=False, vin=None):
    """The oracle's DP in numpy; returns (states, number of steps whose chosen candidate ties another, V[T-1]).
    reassoc: V[t, j] = (E[t, j] + V[t-1, k]) + A[k, j] instead of E[t, j] + (V[t-1, k] + A[k, j]);
    last_max: ties go to the last maximum instead of the first."""
    e = np.asarray(e, dtype=np.float64)
    T, K = e.shape
    bp = np.zeros((T, K), dtype=np.int64)
    ties = 0

    def pick(c):
        m = c.max()
        idx = np.flatnonzero(c == m)
        return (idx[-1] if last_max else idx[0]), len(idx) > 1

    if vin is None:
        V = e[0] + np.log(1.0 / K)
        bp[0] = np.arange(K)
        t0 = 1
    else:
        V = np.asarray(vin, dtype=np.float64).copy()
        t0 = 0
    for t in range(t0, T):
        Vn = np.empty(K)
        for j in range(K):
            c = V + A[:, j]
            a, tie = pick(c)
            ties += tie
            bp[t, j] = a
            Vn[j] = (e[t, j] + V[a]) + A[a, j] if reassoc else e[t, j] + c[a]
        V = Vn
    x, tie = pick(V)
    ties += tie
    X = np.empty(T, dtype=np.int64)
    X[T - 1] = x
    for t in range(T - 1, 0, -1):
        X[t - 1] = bp[t, X[t]]
    return X, ties, V


# ---- CNN posteriors --------------------------------------------------------------------------------------------

def tie_posteriors(K, T, seed):
    """[T, K] float32 posteriors whose decode is decided by first-max at exact ties: states 1 and 2 (and 3 for
    K = 4) carry bitwise-identical columns, so their V are equal at every step; runs of 0.5 override rows (every
    column equal, as segmenter.py sets non-finite patches); saturated rows with exact zeros (-inf emissions) in two
    states at once."""
    rng = np.random.default_rng(seed)
    p = rng.random((T, K)).astype(np.float32) ** 2 + np.float32(1e-4)
    dom = np.repeat(rng.integers(0, 2, T // 17 + 1), 17)[:T]          # spans where the tied twins win
    p[dom == 1, 1:] += np.float32(1.5)
    p[:, 2:] = p[:, 1:2]                                              # identical twins: states 1, 2 (, 3)
    p = (p / p.sum(1, keepdims=True)).astype(np.float32)
    p[:, 2:] = p[:, 1:2]
    for a in range(T // 7, T, max(T // 3, 1)):                        # runs of override rows
        p[a:a + 9] = 0.5
    sat = rng.integers(0, T, max(T // 50, 1))
    p[sat] = 0.0
    p[sat, 0] = 1.0                                                   # two (or more) states at -inf together
    p[T - min(T, 5):] = 0.5                                           # the final argmax is a tie among equal V
    return _clear(p)


def seam_flip_posteriors(K, T, flip_at, seed):
    """[T, K] posteriors whose decode switches state exactly at step ``flip_at`` (a warp-block or backtrack-chunk
    seam): one state dominates before, another after, and the transitions are cheap enough to switch."""
    rng = np.random.default_rng(seed)
    p = np.full((T, K), 0.02, dtype=np.float32) + rng.random((T, K)).astype(np.float32) * np.float32(0.01)
    a, b = 0, K - 1
    p[:flip_at, a] = 0.9
    p[flip_at:, b] = 0.9
    p = (p / p.sum(1, keepdims=True)).astype(np.float32)
    return _clear(p)


def _stay_scores(E, alpha, reassoc=False):
    """V[1] of a two-step chain that stays in one state, for every pair of emissions: [i * n + j] has e0 = E[i],
    e1 = E[j]."""
    v0 = E + np.log(0.5)
    if reassoc:
        return ((E[None, :] + v0[:, None]) + alpha).ravel()
    return (E[None, :] + (v0[:, None] + alpha)).ravel()


def near_tie_segments(seed, n_p=1500, want=300):
    """Two-step, two-state segments whose two non-switching paths tie or nearly tie at the final argmax.  Found by
    a meet-in-the-middle search: over all pairs (e0, e1) of emissions of posteriors just below 1 and in (0.05, 1),
    the stay-in-one-state score V[1] is computed once and sorted, and neighbours in that order become the two states'
    emission histories.  Returns (list of [2, 2] float32 posteriors, the 2x2 transition matrix, dict of boolean
    masks over the segments: 'tie' (exact tie in the oracle's order), 'reassoc' (the decode changes when the step sum
    is reassociated), 'np_log' (it changes with numpy's float32 log as the emission)).

    An exact tie resolves to state 0, so a one-ulp change of state 1's emission upwards or state 0's downwards flips
    the whole segment: the tie set is sensitive to the rounding of every emission it contains."""
    rng = np.random.default_rng(seed)
    A = vo.diag_trans_exp(80, 2)
    A[0, 0] = A[1, 1] = -0.1                # a non-zero diagonal, so that the step sum has three distinct terms
    near1 = (1 - rng.integers(1, 1 << 12, n_p // 2).astype(np.float64) * 2.0 ** -24).astype(np.float32)
    wide = rng.uniform(0.05, 1.0, n_p - len(near1)).astype(np.float32)
    pv = _clear(np.unique(np.concatenate((near1, wide))))
    n = len(pv)
    E = vo.emissions_kernel(pv)
    with np.errstate(divide='ignore'):
        E_np = np.log(pv).astype(np.float64)
    f = _stay_scores(E, A[0, 0])
    order = np.argsort(f, kind='stable')
    s0, s1 = order[:-1], order[1:]          # state 0 takes the lower-or-equal score: a tie or a one-ulp gap

    def decides_1(g):
        return g[s1] > g[s0]

    ref = decides_1(f)
    masks = {'tie': f[s1] == f[s0], 'reassoc': decides_1(_stay_scores(E, A[0, 0], True)) != ref,
             'np_log': decides_1(_stay_scores(E_np, A[0, 0])) != ref}
    distinct = (s0 // n) != (s1 // n)
    pick = []
    for m in (masks['reassoc'], masks['np_log'], masks['tie']):
        cand = np.flatnonzero(m & distinct)
        pick.extend(rng.permutation(cand)[:want // 3].tolist())
    pick = np.unique(pick)
    segs = [np.array([[pv[i0], pv[i1]], [pv[j0], pv[j1]]], dtype=np.float32)
            for (i0, j0), (i1, j1) in zip(zip(*divmod(s0[pick], n)), zip(*divmod(s1[pick], n)))]
    return segs, A, {k: v[pick] for k, v in masks.items()}


def pack(segs, K):
    """(concatenated float32 posteriors [n, K], int64 segment offsets)."""
    lens = [len(s) for s in segs]
    allp = np.concatenate([np.asarray(s, dtype=np.float32).reshape(-1, K) for s in segs]) if sum(lens) else \
        np.zeros((0, K), np.float32)
    return allp, np.concatenate(([0], np.cumsum(lens))).astype(np.int64)


def random_posteriors(K, T, seed):
    rng = np.random.default_rng(seed)
    p = rng.random((T, K)).astype(np.float32) ** 3 + np.float32(1e-7)
    dom = np.repeat(rng.integers(0, K, T // 40 + 1), 40)[:T]
    p[np.arange(T), dom] += rng.uniform(0.2, 2.0)
    return _clear((p / p.sum(1, keepdims=True)).astype(np.float32))


# ---- energy tracks ---------------------------------------------------------------------------------------------

def cpu_stats(lo):
    fin = np.isfinite(lo)
    return np.array([lo[fin].astype(np.float64).sum(), float(fin.sum())])


def energy_track(L, seed, ratio=0.03, n_near=2000, n_silent=500):
    """float32 loge of L frames: alternating quiet / active runs of 1 frame to 40 s, -inf (silent) frames, and
    ``n_near`` frames one float32 ulp above or below the kernel's threshold (placed after the threshold settles: a
    planted frame moves the mean itself)."""
    rng = np.random.default_rng(seed)
    lo = np.empty(L, dtype=np.float32)
    pos = 0
    while pos < L:
        n = int(min(L - pos, rng.choice([1, 2, 3, 7, 40, 300, 4000]) * (1 + rng.integers(0, 3))))
        lo[pos:pos + n] = rng.choice([-14.0, -9.0, -3.0, 1.5]) + rng.normal(0, 1.0, n)
        pos += n
    lo[rng.integers(0, L, n_silent)] = -np.inf
    near = rng.choice(L, size=min(n_near, L), replace=False)
    up = rng.random(len(near)) < 0.5
    for _ in range(6):
        below, above = threshold_neighbours(vo.energy_threshold_kernel(cpu_stats(lo), ratio))
        lo[near] = np.where(up, above, below)
    return lo


def threshold_neighbours(thr):
    """The float32 values just below (or at) and just above the float64 threshold ``thr``."""
    f = np.float32(thr)
    if float(f) > thr:
        return np.nextafter(f, np.float32(-np.inf)), f
    return f, np.nextafter(f, np.float32(np.inf))


def silent_track(L):
    return np.full(L, -np.inf, dtype=np.float32)
