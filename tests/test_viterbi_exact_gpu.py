"""K3 (viterbi.cu) against the C oracle, state by state: every entry point, at exact ties, ulp-level near-ties, the
32-step warp blocks, the 256-step backtrack chunks, the 16384-frame chunks of the chunk-parallel energy decode and
the cuts of partial chains.  The kernels promise the reference's decisions bit for bit, so every comparison is
``np.array_equal``.  Emissions are the kernels' definition (``emissions_kernel``, a correctly rounded float32 log)
and energy thresholds are taken from the kernels' own ``loge_stats`` output, so what is checked is the Viterbi."""
import numpy as np
import pytest

import viterbi_fixtures as vf
from oracle import viterbi_oracle as vo

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')

RATIO = 0.03


@pytest.fixture(scope='module')
def rt():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from inaspeechsegmenter_b200 import _lib, engine
    return dict(ctx=engine.Context(0), engine=engine, lib=_lib.load())


def _oracle_segments(allp, off, A):
    out = np.zeros(len(allp), dtype=np.uint8)
    for a, b in zip(off[:-1], off[1:]):
        if b > a:
            out[a:b] = vo.viterbi_c(vo.emissions_kernel(allp[a:b]), A)
    return out


def _check_segments(rt, segs, K, A):
    allp, off = vf.pack(segs, K)
    vf.assert_clear_of_midpoints(allp)
    got = rt['engine'].viterbi_segments(rt['ctx'], torch.from_numpy(allp).cuda(), off, A).cpu().numpy()
    ref = _oracle_segments(allp, off, A)
    bad = [i for i, (a, b) in enumerate(zip(off[:-1], off[1:])) if not np.array_equal(got[a:b], ref[a:b])]
    assert not bad, 'K=%d: %d of %d segments differ, first %d (length %d)' % (K, len(bad), len(segs), bad[0],
                                                                               off[bad[0] + 1] - off[bad[0]])


# ---- iss_viterbi_segments --------------------------------------------------------------------------------------
@pytest.mark.parametrize('K', [2, 3, 4])
def test_segments_ties_seams_and_zero_length(rt, K):
    segs = [np.zeros((0, K), np.float32)]
    for T in (1, 2, 3) + vf.WARP_SEAMS + vf.CHUNK_SEAMS + (700, 1025):
        segs.append(vf.tie_posteriors(K, T, T) if K > 2 else vf.random_posteriors(K, T, T))
        segs.append(np.zeros((0, K), np.float32))                       # zero-length segments in the middle
    for s, seam in enumerate(vf.WARP_SEAMS + vf.CHUNK_SEAMS):           # a state switch exactly on the seam
        segs.append(vf.seam_flip_posteriors(K, seam + 1 + 97 * (s % 3), seam, seam))
        segs.append(vf.seam_flip_posteriors(K, 2 * seam + 3, seam, seam + 1))
    segs.append(np.full((300, K), 0.5, np.float32))                     # a whole segment of override rows
    segs.append(np.zeros((0, K), np.float32))
    _check_segments(rt, segs, K, vo.diag_trans_exp(1, K))
    _check_segments(rt, [vf.random_posteriors(K, T, 50 + T) for T in (1, 33, 256, 257, 5000, 20011)], K,
                    vo.diag_trans_exp(80, K))


def test_segments_near_ties(rt):
    segs, A, m = vf.near_tie_segments(5)
    assert m['tie'].sum() and m['reassoc'].sum() and m['np_log'].sum()
    _check_segments(rt, segs, 2, A)


def test_segments_one_hundred_thousand_short(rt):
    rng = np.random.default_rng(17)
    lens = rng.integers(0, 6, 100_000)
    lens[rng.integers(0, len(lens), 50)] = rng.integers(200, 700, 50)
    allp = vf.random_posteriors(3, int(lens.sum()), 18)
    off = np.concatenate(([0], np.cumsum(lens)))
    _check_segments(rt, [allp[a:b] for a, b in zip(off[:-1], off[1:])], 3, vo.diag_trans_exp(2, 3))


# ---- iss_energy_viterbi ----------------------------------------------------------------------------------------
def _energy_decode(rt, lo, stride, serial):
    eng, lib = rt['engine'], rt['lib']
    loge = torch.from_numpy(lo).cuda()
    stats = eng.loge_stats(rt['ctx'], loge)
    try:
        lib.iss_set_energy_viterbi_serial(1 if serial else 0)
        got = eng.energy_viterbi(rt['ctx'], loge, stats, RATIO, out_stride=stride).cpu().numpy()
    finally:
        lib.iss_set_energy_viterbi_serial(0)
    return got, vo.energy_threshold_kernel(stats.cpu().numpy(), RATIO)


@pytest.mark.parametrize('L', (1, 2, 31, 32, 33, 255, 256, 257, 513) + vf.ENERGY_SEAMS)
def test_energy_viterbi_serial_and_chunk_parallel(rt, L):
    lo = vf.energy_track(L, L, n_near=min(2000, L // 3), n_silent=min(500, L // 10))
    ref = None
    for serial in (True, False):
        for stride in (1, 2):
            got, thr = _energy_decode(rt, lo, stride, serial)
            if ref is None:
                ref = vo.energy_activity_thr(lo, thr).astype(np.uint8)
            assert np.array_equal(got, ref[::stride]), (L, serial, stride)


@pytest.mark.parametrize('L', [1000, 4 * vf.ECH + 5])
def test_energy_viterbi_all_silent(rt, L):
    lo = vf.silent_track(L)
    for serial in (True, False):
        got, thr = _energy_decode(rt, lo, 1, serial)
        assert np.isnan(thr) and not got.any()


def test_energy_viterbi_ten_hour_track(rt):
    lo = vf.energy_track(3_600_037, 4)
    for serial in (False, True):
        got, thr = _energy_decode(rt, lo, 2, serial)
        ref = vo.energy_activity_thr(lo, thr).astype(np.uint8)
        assert np.array_equal(got, ref[::2]), serial
        assert 0 < ref.mean() < 1


# ---- iss_energy_viterbi_multi ----------------------------------------------------------------------------------
@pytest.mark.parametrize('stride', [1, 2])
def test_energy_viterbi_multi(rt, stride):
    eng = rt['engine']
    lens = [0, 1, 31, 257, 0, 1001, 2, vf.ECH + 1, 3, 4 * vf.ECH - 1, 0, 700]
    tracks = [vf.energy_track(n, 100 + i, n_near=n // 4, n_silent=n // 20) if n else np.zeros(0, np.float32)
              for i, n in enumerate(lens)]
    tracks[6] = vf.silent_track(2)                                      # a recording with no finite frame
    lo = np.concatenate(tracks)
    loff = np.concatenate(([0], np.cumsum(lens))).astype(np.int64)
    nout = [(n + stride - 1) // stride for n in lens]
    ooff = np.concatenate(([0], np.cumsum([n + 3 for n in nout]))).astype(np.int64)   # gaps between outputs
    loge = torch.from_numpy(lo).cuda()
    nz = np.flatnonzero(np.diff(loff))                                 # loge_stats_multi takes non-empty ones
    stats = torch.zeros((len(lens), 2), dtype=torch.float64, device='cuda')
    stats[torch.from_numpy(nz).cuda()] = eng.loge_stats_multi(rt['ctx'], loge, loff[nz], np.diff(loff)[nz])
    got = eng.energy_viterbi_multi(rt['ctx'], loge, loff, stats, RATIO, ooff, out_stride=stride).cpu().numpy()
    st = stats.cpu().numpy()
    for r, n in enumerate(lens):
        if n == 0:
            continue
        ref = vo.energy_activity_thr(tracks[r], vo.energy_threshold_kernel(st[r], RATIO))[::stride]
        assert np.array_equal(got[ooff[r]:ooff[r] + nout[r]], ref.astype(np.uint8)), (r, n)


# ---- shard ABI: iss_energy_transfer / iss_energy_forward / iss_energy_emit -----------------------------------
def test_energy_shard_abi_at_arbitrary_cuts(rt):
    eng, ctx = rt['engine'], rt['ctx']
    L = 6000
    lo = vf.energy_track(L, 31, n_near=1500, n_silent=200)
    loge = torch.from_numpy(lo).cuda()
    stats = eng.loge_stats(ctx, loge)
    thr = vo.energy_threshold_kernel(stats.cpu().numpy(), RATIO)
    em = vo.pred2logemission(lo.astype(np.float64) > thr)
    A = vo.log_trans_exp(150, cost0=-5)
    whole = vo.energy_activity_thr(lo, thr).astype(np.uint8)
    cuts = [1, 2, 257, 513, 770, 1026, 1027, 2001, 4500, 4501]        # pieces of 1, 255, 256, 257 ... frames
    bounds = [0] + cuts + [L]
    # transfer matrices: the oracle's two basis-vector chains, bit for bit
    for a, b in zip(bounds[:-1], bounds[1:]):
        M = eng.energy_transfer(ctx, loge[a:b], stats, RATIO)
        for i in range(2):
            basis = np.full(2, -np.inf)
            basis[i] = 0.0
            _, vout, _ = vo.viterbi_partial(em[a:b], A, vin=basis)
            assert np.array_equal(M[:, i], vout), (a, b, i)
    # forward passes from the oracle's incoming scores, then emit from every end state
    vin, got = None, []
    for a, b in zip(bounds[:-1], bounds[1:]):
        vout, bmap = eng.energy_forward(ctx, loge[a:b], stats, RATIO, vin)
        _, r_vout, r_bmap = vo.viterbi_partial(em[a:b], A, vin=vin)
        assert np.array_equal(vout, r_vout) and np.array_equal(bmap, r_bmap.astype(np.uint8)), (a, b)
        for end in (-1, 0, 1):                                          # -1 (the forward's own argmax) first
            st = eng.energy_emit(ctx, loge[a:b], end, out_stride=1).cpu().numpy()
            ref = vo.viterbi_partial(em[a:b], A, vin=vin, end_state=end)[0]
            assert np.array_equal(st, ref.astype(np.uint8)), (a, b, end)
        vin = r_vout
    # stitched as shard.py does: each piece decoded from the end state its successor traces back to
    pieces = list(zip(bounds[:-1], bounds[1:]))
    fwd, vin = [], None
    for a, b in pieces:
        fwd.append((vin,) + eng.energy_forward(ctx, loge[a:b], stats, RATIO, vin))
        vin = fwd[-1][1]
    end, out = int(np.argmax(vin)), []
    for (a, b), (vin_p, vout, bmap) in zip(reversed(pieces), reversed(fwd)):
        eng.energy_forward(ctx, loge[a:b], stats, RATIO, vin_p)
        out.append(eng.energy_emit(ctx, loge[a:b], end, out_stride=1).cpu().numpy())
        end = int(bmap[end])
    assert np.array_equal(np.concatenate(out[::-1]), whole)


# ---- iss_viterbi_online ----------------------------------------------------------------------------------------
def _online(rt, kind, n_chain, seed):
    """n_chain chains in one launch per call, fed unequal pieces (a one-step start-and-end chain, end calls with
    no new steps, undecided spans far longer than 32 steps), slots in shuffled order.  After every call the decided
    prefix of each chain equals the oracle's offline decode; the end call completes it."""
    eng, ctx = rt['engine'], rt['ctx']
    rng = np.random.default_rng(seed)
    K = 2 if kind == 'energy' else int(kind)
    lens = [1] + [int(x) for x in rng.integers(200, 3000, n_chain - 1)]
    if kind == 'energy':
        data = [vf.energy_track(n, seed + i, n_near=n // 5, n_silent=n // 30) for i, n in enumerate(lens)]
        st = np.array([vf.cpu_stats(d) if np.isfinite(d).any() else [0.0, 0.0] for d in data])
        refs = [vo.energy_activity_thr(d, vo.energy_threshold_kernel(s, RATIO)).astype(np.uint8)
                for d, s in zip(data, st)]
        trans = None
    else:
        trans = vo.diag_trans_exp(3, K)
        data = [vf.tie_posteriors(K, n, seed + i) if K > 2 and i % 2 else vf.random_posteriors(K, n, seed + i)
                for i, n in enumerate(lens)]
        for d in data[2::3]:
            d[50:400] = 0.5                     # equal emissions: the K paths stay apart, nothing is decided
        refs = [vo.viterbi_c(vo.emissions_kernel(d), trans).astype(np.uint8) for d in data]
    slots = rng.permutation(n_chain)
    cap = max(lens) + 1
    scores = torch.zeros((n_chain, 4), dtype=torch.float64, device='cuda')
    hist = torch.zeros((n_chain, cap), dtype=torch.uint8, device='cuda')
    stats = None
    if kind == 'energy':
        stats = torch.from_numpy(np.ascontiguousarray(st[np.argsort(slots)])).cuda()   # row slots[i] = chain i
    pos, pend, done = [0] * n_chain, [0] * n_chain, [np.zeros(0, np.uint8) for _ in range(n_chain)]
    ended = [False] * n_chain
    max_pend = 0
    while not all(ended):
        rows, srcs, order = [], [], []
        src_off = out_off = 0
        for i in rng.permutation(n_chain):
            if ended[i]:
                continue
            left = lens[i] - pos[i]
            n = int(min(left, rng.choice([0, 1, 5, 31, 32, 33, 100, 400]))) if pos[i] else int(min(left, 1 + rng.integers(0, 64)))
            end = pos[i] + n == lens[i] and (n == 0 or rng.random() < 0.5 or lens[i] == 1)
            if n == 0 and not end and pos[i] == 0:
                continue
            fl = (eng.ONLINE_START if pos[i] == 0 else 0) | (eng.ONLINE_END if end else 0)
            rows.append([src_off, n, slots[i], pend[i], out_off, fl])
            srcs.append(data[i][pos[i]:pos[i] + n])
            order.append(i)
            src_off += n
            out_off += pend[i] + n
        if not rows:
            continue
        src = np.concatenate(srcs).astype(np.float32)
        if kind != 'energy':
            src = src.reshape(-1, K)
        if len(src) == 0:
            src = np.zeros((1,) if kind == 'energy' else (1, K), np.float32)
        buf = eng.viterbi_online(ctx, np.array(rows, np.int64), torch.from_numpy(np.ascontiguousarray(src)).cuda(),
                                 scores, hist, out_off, K=K, trans=trans, stats=stats,
                                 energy_ratio=RATIO if kind == 'energy' else None).cpu().numpy()
        nd, out = eng.split_online(buf, len(rows))
        for r, i in enumerate(order):
            n, o = rows[r][1], rows[r][4]
            done[i] = np.concatenate((done[i], out[o:o + nd[r]]))
            pos[i] += n
            pend[i] += n - int(nd[r])
            max_pend = max(max_pend, pend[i])
            assert np.array_equal(done[i], refs[i][:len(done[i])]), (kind, i, len(done[i]))
            if rows[r][5] & eng.ONLINE_END:
                ended[i] = True
                assert pend[i] == 0 and np.array_equal(done[i], refs[i]), (kind, i)
    return max_pend


@pytest.mark.parametrize('kind', ['energy', '2', '3', '4'])
def test_online_many_chains_equal_the_offline_decode(rt, kind):
    max_pend = _online(rt, kind, 40, {'energy': 1, '2': 2, '3': 3, '4': 4}[kind])
    if kind != 'energy':
        assert max_pend > 300                   # the history compaction ran over many 32-byte rounds
