"""CPU checks of the exact-Viterbi test infrastructure: the oracle's partial chains compose to the whole chain, the
kernel-definition helpers mean what they say, and every fixture generator really produces the ties, near-ties and
threshold-neighbour frames it claims, as the C oracle sees them.  No GPU."""
import numpy as np
import pytest

import viterbi_fixtures as vf
from oracle import viterbi_oracle as vo


def _chain_in_pieces(e, A, cuts, out_stride=1):
    """Decode e [T, K] as consecutive partial chains cut at `cuts`: forward pass piece by piece carrying V, then
    each piece backtracked from the state the next piece's back-map gives.  Returns (states, V[T-1])."""
    bounds = [0] + list(cuts) + [len(e)]
    pieces = list(zip(bounds[:-1], bounds[1:]))
    vin, fwd = None, []
    for a, b in pieces:
        _, vout, bmap = vo.viterbi_partial(e[a:b], A, vin=vin)
        fwd.append((vin, vout, bmap))
        vin = vout
    out, end = [], -1
    for (a, b), (vin_p, vout, bmap) in zip(reversed(pieces), reversed(fwd)):
        assert a % out_stride == 0
        st, _, _ = vo.viterbi_partial(e[a:b], A, vin=vin_p, end_state=end, out_stride=out_stride)
        out.append(st)
        end = int(bmap[end if end >= 0 else int(np.argmax(vout))])     # the previous piece's last state
    return np.concatenate(out[::-1]), vin


@pytest.mark.parametrize('K', [2, 3, 4])
def test_partial_chains_cut_anywhere_equal_the_whole_chain(K):
    rng = np.random.default_rng(K)
    for T, gen in ((700, 'tie'), (1500, 'random'), (300, 'seam')):
        p = {'tie': lambda: vf.tie_posteriors(K, T, 7), 'random': lambda: vf.random_posteriors(K, T, 8),
             'seam': lambda: vf.seam_flip_posteriors(K, T, 256, 9)}[gen]()
        e = vo.emissions_kernel(p)
        A = vo.diag_trans_exp(1 if gen != 'random' else 3, K)
        whole = vo.viterbi_c(e, A).astype(np.int32)
        _, v_whole, _ = vo.viterbi_partial(e, A)
        assert np.array_equal(vf.dp(e, A)[0], whole)
        cut_sets = [[1], [T - 1], [255, 256, 257], sorted(set(rng.integers(1, T, 12).tolist())), list(range(1, 40))]
        for cuts in cut_sets:
            got, vlast = _chain_in_pieces(e, A, cuts)
            assert np.array_equal(got, whole), (K, gen, cuts)
            assert np.array_equal(vlast, v_whole)
        even = sorted({c - c % 2 for c in cut_sets[3]} - {0})
        got2, _ = _chain_in_pieces(e, A, even, out_stride=2)
        assert np.array_equal(got2, whole[::2])


def test_partial_backmap_and_forced_end_state():
    e = vo.emissions_kernel(vf.random_posteriors(3, 400, 4))
    A = vo.diag_trans_exp(2, 3)
    S = 150
    _, v_head, _ = vo.viterbi_partial(e[:S], A)
    for end in (0, 1, 2):
        whole = vo.viterbi_partial(e, A, end_state=end)[0]
        assert whole[-1] == end
        st, _, bmap = vo.viterbi_partial(e[S:], A, vin=v_head, end_state=end)
        assert np.array_equal(st, whole[S:]) and bmap[end] == whole[S - 1]
        assert vo.viterbi_partial(e, A)[2][end] == vo.viterbi_partial(e, A, end_state=end)[0][0]
    # vin concentrated on one state (a max-plus basis vector): every end state traces back to it
    for i in range(3):
        basis = np.full(3, -np.inf)
        basis[i] = 0.0
        _, vout, bmap = vo.viterbi_partial(e, A, vin=basis)
        assert np.all(bmap == i) and np.all(np.isfinite(vout))


def test_emissions_kernel_is_correctly_rounded_and_numpy_log_is_not():
    rng = np.random.default_rng(0)
    p = rng.random(1_000_000, dtype=np.float32)
    p[p == 0] = 1
    ek = vo.emissions_kernel(p)
    assert np.array_equal(ek, np.log(p.astype(np.float64)).astype(np.float32).astype(np.float64))
    assert np.array_equal(vo.emissions_kernel(np.array([0.0, 1.0, 0.5], np.float32)), [-np.inf, 0.0, np.log(np.float32(0.5))])
    # the two definitions agree to a few float32 ulps, and the kernel's is never further from the float64 log
    d64 = np.log(p.astype(np.float64))
    npl = np.log(p).astype(np.float64)
    assert np.all(np.abs(ek - d64) <= np.abs(npl - d64))
    assert np.all(np.abs(npl - ek) <= 8 * np.spacing(np.abs(ek).astype(np.float32)).astype(np.float64))


def test_energy_activity_from_threshold_matches_segmenter_oracle():
    from oracle import segmenter_oracle as so
    lo = vf.energy_track(20001, 11)
    fin = np.isfinite(lo)
    thr = np.mean(lo[fin]) + np.log(0.03)                  # the reference's own threshold
    assert np.array_equal(vo.energy_activity_thr(lo, thr), so.energy_activity(lo, 0.03))
    assert not vo.energy_activity_thr(vf.silent_track(100), float('nan')).any()
    assert np.isnan(vo.energy_threshold_kernel([0.0, 0.0], 0.03))
    s = vf.cpu_stats(lo)
    assert vo.energy_threshold_kernel(s, 0.03) == float(np.float32(s[0] / s[1])) + np.log(0.03)


@pytest.mark.parametrize('K', [3, 4])
def test_tie_fixture_has_exact_ties_that_reach_the_output(K):
    for T in (40, 257, 700):
        p = vf.tie_posteriors(K, T, T)
        vf.assert_clear_of_midpoints(p)
        assert np.array_equal(p[:, 1], p[:, 2]) and (p == 0.5).all(1).any() and ((p == 0).sum(1) >= 2).any()
        e = vo.emissions_kernel(p)
        A = vo.diag_trans_exp(1, K)
        first, ties, V = vf.dp(e, A)
        assert np.array_equal(first, vo.viterbi_c(e, A))
        assert ties > T // 4 and V[1] == V[2]
        last = vf.dp(e, A, last_max=True)[0]
        assert (first != last).sum() > T // 10          # first-max decides a good share of the output
    all_half = np.full((9, K), 0.5, np.float32)
    assert not vo.viterbi_c(vo.emissions_kernel(all_half), vo.diag_trans_exp(1, K)).any()


def test_near_tie_fixture_flips_under_reassociation_and_numpy_log():
    segs, A, m = vf.near_tie_segments(5)
    assert m['tie'].sum() >= 60 and m['reassoc'].sum() >= 60 and m['np_log'].sum() >= 60
    for p, tie, re, nl in zip(segs, m['tie'], m['reassoc'], m['np_log']):
        vf.assert_clear_of_midpoints(p)
        e = vo.emissions_kernel(p)
        X, ties, _ = vf.dp(e, A)
        assert np.array_equal(X, vo.viterbi_c(e, A))
        assert (ties > 0) == tie
        assert (vf.dp(e, A, reassoc=True)[0][-1] != X[-1]) == re
        with np.errstate(divide='ignore'):
            assert (vf.dp(np.log(p).astype(np.float64), A)[0][-1] != X[-1]) == nl
        if tie:                                          # one float32 ulp in the losing direction flips the segment
            up = e.copy()
            up[1, 1] = np.float64(np.nextafter(np.float32(e[1, 1]), np.float32(np.inf)))
            assert vf.dp(up, A)[0][-1] != X[-1]


@pytest.mark.parametrize('K', [2, 3, 4])
def test_seam_fixture_switches_exactly_at_the_seam(K):
    for seam in vf.WARP_SEAMS + vf.CHUNK_SEAMS:
        p = vf.seam_flip_posteriors(K, seam + 40, seam, seam)
        st = vo.viterbi_c(vo.emissions_kernel(p), vo.diag_trans_exp(1, K))
        assert np.all(st[:seam] == 0) and np.all(st[seam:] == K - 1)


def test_energy_track_has_frames_one_ulp_around_the_kernel_threshold():
    lo = vf.energy_track(70001, 1)
    thr = vo.energy_threshold_kernel(vf.cpu_stats(lo), 0.03)
    below, above = vf.threshold_neighbours(thr)
    assert float(below) <= thr < float(above) and np.nextafter(below, above) == above
    assert (lo == below).sum() > 500 and (lo == above).sum() > 500 and np.isneginf(lo).sum() > 100
    raw = lo.astype(np.float64) > thr
    assert not raw[lo == below].any() and raw[lo == above].all()
    st = vo.energy_activity_thr(lo, thr)
    assert 0 < st.mean() < 1
