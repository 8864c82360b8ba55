"""CPU model of the pipelined pooled gather convolution (csrc/conv_gemm_tc.cu, gather_pipe in conv_gemm_wg_kernel<1, BN, 2>).

* Protocol.  One CTA takes the tiles blockIdx.x, blockIdx.x + gridDim.x, ... in increasing order.  Producer warp 0 (one
  thread): per tile and tap, waits on wempty[s] (parity ph ^ 1), arms wfull[s] and issues one bulk copy into stage s.
  Producer warps 1..3: per tile, wait on hempty[b] (parity ph ^ 1), store their share of halo buffer b and arrive on
  hfull[b] (96 arrivals).  Consumers 0 and 1: per tile, wait on hfull[b]; per tap, gather the A operand from halo b
  into registers (ldmatrix: the read happens then), after the last tap's gather the four warps arrive on hempty[b];
  wait on wfull[s], issue the wgmmas, commit, wgmma.wait_group 0, and the four warps arrive on wempty[s].  Random
  interleavings must drain without a deadlock or a hazard, and each broken ordering must be caught.
* Addressing.  The halo planes (chunk q of pixel p at chunk q ^ (p & 7)) and the lanes' ldmatrix row addresses,
  assembled into the wgmma A fragments, give the im2col operand of the pooled input, and the three products per k16 step
  give the float64 convolution with pooling; on the VAD and gender shapes, odd un-pooled maps, stride 2, padding, and
  tiles spanning up to four images.
* Budget.  iss_gather_pipe_smem against the shared-memory arithmetic."""
import itertools
import random

import numpy as np
import pytest

from inaspeechsegmenter_b200 import _lib

TBM, C = 128, 64
FILL_WARPS, CONSUMER_WARPS = 3, 4
STAGES, HALOS = 3, 2
MAX_SMEM = 227 * 1024


# ============================ protocol ============================

class Bar:
    def __init__(self, count):
        self.count, self.pending, self.tx, self.phase = count, 0, 0, 0

    def _maybe_complete(self):
        while self.pending >= self.count and self.tx == 0:
            self.pending -= self.count
            self.phase += 1

    def arrive(self, n=1):
        self.pending += n
        self._maybe_complete()

    def arrive_expect_tx(self, nbytes):
        self.tx += nbytes
        self.arrive()

    def complete_tx(self, nbytes):
        self.tx -= nbytes
        self._maybe_complete()

    def done(self, parity):
        return (self.phase & 1) != parity


def run_cta(nkb, my_tiles, rng, bug=None):
    """One random interleaving of one CTA: the hazards seen (a deadlock ends the run) and the (tile, consumer) epilogues."""
    wfull = [Bar(1) for _ in range(STAGES)]
    wempty = [Bar(2 * CONSUMER_WARPS) for _ in range(STAGES)]
    hfull = [Bar(FILL_WARPS * 32) for _ in range(HALOS)]
    hempty = [Bar(2 * CONSUMER_WARPS) for _ in range(HALOS)]
    stage_data = [None] * STAGES                     # tap whose weights the stage holds (None while a copy writes it)
    copies = []
    halo_data = [[None] * FILL_WARPS for _ in range(HALOS)]
    inflight = [[], []]                              # per consumer, committed wgmma groups: the stage they read
    hazards, epilogues = [], []

    def weights():
        s, ph = 0, 0
        for _tile in my_tiles:
            for kb in range(nkb):
                if bug != 'weights_skip_empty_wait':
                    yield lambda s=s, ph=ph: wempty[s].done(ph ^ 1)
                wfull[s].arrive_expect_tx(1)
                if any(g == s for c in (0, 1) for g in inflight[c]):
                    hazards.append(('stage overwritten while read', s, kb))
                stage_data[s] = None
                copies.append((s, kb))
                yield None
                s += 1
                if s == STAGES:
                    s, ph = 0, ph ^ 1

    def fill(f):
        b, ph = 0, 0
        for tile in my_tiles:
            if bug != 'fill_skip_empty_wait':
                yield lambda b=b, ph=ph: hempty[b].done(ph ^ 1)
            halo_data[b][f] = None
            yield None                               # the stores take time; the other warpgroups run meanwhile
            halo_data[b][f] = tile
            hfull[b].arrive(32)
            yield None
            b += 1
            if b == HALOS:
                b, ph = 0, ph ^ 1

    def consumer(c):
        s, wph, b, hph = 0, 0, 0, 0
        for tile in my_tiles:
            if bug != 'consumer_skip_halo_wait':
                yield lambda b=b, hph=hph: hfull[b].done(hph)
            for kb in range(nkb):
                for w in range(CONSUMER_WARPS):      # each warp's ldmatrix gathers read the halo now
                    if halo_data[b] != [tile] * FILL_WARPS:
                        hazards.append(('gather read a halo that does not hold its tile', c, tile, kb))
                    if kb == nkb - 1 and bug != 'halo_release_early':
                        hempty[b].arrive()
                    if kb == 0 and bug == 'halo_release_early':
                        hempty[b].arrive()
                    yield None
                if bug != 'consumer_skip_full_wait':
                    yield lambda s=s, wph=wph: wfull[s].done(wph)
                if stage_data[s] != kb:
                    hazards.append(('tap read a stage that does not hold its weights', c, tile, kb))
                inflight[c].append(s)
                if bug == 'stage_release_before_wait':
                    wempty[s].arrive(CONSUMER_WARPS)
                    yield lambda: not inflight[c]
                else:
                    yield lambda: not inflight[c]    # wgmma.wait_group 0
                    wempty[s].arrive(CONSUMER_WARPS)
                s += 1
                if s == STAGES:
                    s, wph = 0, wph ^ 1
            b += 1
            if b == HALOS:
                b, hph = 0, hph ^ 1
            epilogues.append((tile, c))
            yield None

    actors = [weights()] + [fill(f) for f in range(FILL_WARPS)] + [consumer(c) for c in (0, 1)]
    waiting = [None] * len(actors)
    live = list(range(len(actors)))
    while live:
        events = [('land', i) for i in range(len(copies))] + [('retire', c) for c in (0, 1) if inflight[c]]
        runnable = [a for a in live if waiting[a] is None or waiting[a]()]
        if events and (not runnable or rng.random() < 0.4):
            kind, x = rng.choice(events)
            if kind == 'land':
                s, kb = copies.pop(x)
                stage_data[s] = kb
                wfull[s].complete_tx(1)
            else:
                inflight[x].pop(0)
            continue
        if not runnable:
            return hazards + [('deadlock',)], epilogues
        a = rng.choice(runnable)
        try:
            waiting[a] = next(actors[a])
        except StopIteration:
            live.remove(a)
    if copies or inflight[0] or inflight[1]:
        hazards.append(('copy or wgmma still in flight at exit',))
    return hazards, epilogues


def test_protocol_is_safe_and_never_deadlocks():
    rng = random.Random(20261017)
    for nkb, ntiles, _ in itertools.product((2, 3, 4, 9, 18), (1, 2, 3, 5), range(6)):
        tiles = list(range(3, 3 + 132 * ntiles, 132))
        hazards, epi = run_cta(nkb, tiles, rng)
        assert hazards == [], (nkb, ntiles, hazards[:3])
        assert sorted(epi) == sorted((t, c) for t in tiles for c in (0, 1))


@pytest.mark.parametrize('bug', ['weights_skip_empty_wait', 'fill_skip_empty_wait', 'consumer_skip_halo_wait',
                                 'consumer_skip_full_wait', 'stage_release_before_wait', 'halo_release_early'])
def test_model_catches_broken_orderings(bug):
    rng = random.Random(11)
    found = False
    for _ in range(300):
        hazards, _ = run_cta(9, [0, 4, 8, 12], rng, bug)
        if [h for h in hazards if h[0] != 'deadlock']:
            found = True
            break
    assert found, bug


# ============================ halo planes and ldmatrix addressing ============================

def halo_span(t, M, H, OH, OW, KH, SH, PT):
    ohw = OH * OW
    mf, ml = t * TBM, min(t * TBM + TBM, M) - 1
    img0, img1 = mf // ohw, ml // ohw
    oh0, oh1 = (mf - img0 * ohw) // OW, (ml - img1 * ohw) // OW
    g_lo = img0 * H + max(oh0 * SH - PT, 0)
    return g_lo, img1 * H + min(oh1 * SH - PT + KH - 1, H - 1) - g_lo + 1


def pool_floor(x):
    """2x2 / stride-2 max-pooling with floor of the [n, PH, PW, C] map."""
    n, ph, pw, c = x.shape
    h, w = ph // 2, pw // 2
    return x[:, :2 * h, :2 * w].reshape(n, h, 2, w, 2, c).max(axis=(2, 4))


def model_layer(x, wts, KH, KW, SH, SW, PT, PL, OH, OW, rows):
    """The pipelined path's operand gather: halo planes per tile (one value per channel; the hi and lo planes share
    their addressing), the ldmatrix lanes' row addresses and the fragment layout of wgmma's register A, and the products
    accumulated tap by tap.  Returns the [M, N] output."""
    pooled = pool_floor(x)
    n, H, W, _ = pooled.shape
    M = n * OH * OW
    zp = rows * W
    out = np.zeros((M, wts.shape[-1]))
    tall = pooled.reshape(n * H, W, C)
    for t in range((M + TBM - 1) // TBM):
        g_lo, hn = halo_span(t, M, H, OH, OW, KH, SH, PT)
        assert hn <= rows
        plane = np.full((zp + 1, 8, 8), np.nan)      # [pixel][physical chunk][channel in chunk]
        plane[zp] = 0.0
        for px in range(hn * W):
            g = g_lo * W + px
            for q in range(8):
                plane[px, q ^ (px & 7)] = tall[g // W, g % W, 8 * q:8 * q + 8]
        for c in (0, 1):
            for w in range(4):
                for kh, kw in itertools.product(range(KH), range(KW)):
                    kb = kh * KW + kw
                    addr = []                        # (pixel, physical chunk) per lane and k16 step
                    for lane in range(32):
                        r = 16 * w + (lane & 7) + 8 * ((lane >> 3) & 1)
                        m = t * TBM + 64 * c + r
                        ok = m < M
                        mm = m if ok else 0
                        img, rem = divmod(mm, OH * OW)
                        oh, ow = divmod(rem, OW)
                        ih, iw = oh * SH - PT + kh, ow * SW - PL + kw
                        p = (img * H - g_lo + ih) * W + iw if ok and 0 <= ih < H and 0 <= iw < W else zp
                        addr.append([(p, (2 * kk + (lane >> 4)) ^ (p & 7)) for kk in range(4)])
                    for kk in range(4):
                        # ldmatrix.x4: matrix i from the row addresses of lanes 8 i .. 8 i + 7; lane l receives row l / 4,
                        # elements 2 (l % 4), +1 of each.  Fragment of lane l: a[0] = (g, 2t..), a[1] = (g + 8, 2t..),
                        # a[2] = (g, 2t + 8..), a[3] = (g + 8, 2t + 8..).
                        mats = [np.stack([plane[addr[8 * i + j][kk]] for j in range(8)]) for i in range(4)]
                        A = np.zeros((16, 16))
                        for lane in range(32):
                            g, tq = lane // 4, lane % 4
                            for reg, (dr, dk) in enumerate(((0, 0), (8, 0), (0, 8), (8, 8))):
                                A[g + dr, 2 * tq + dk:2 * tq + dk + 2] = mats[reg][g, 2 * tq:2 * tq + 2]
                        m0 = t * TBM + 64 * c + 16 * w
                        valid = min(16, max(0, M - m0))
                        assert np.isfinite(A).all()   # every gathered row is a staged pixel or the zero pixel
                        out[m0:m0 + valid] += A[:valid] @ wts[kb, 16 * kk:16 * kk + 16]
    return out


def reference_layer(x, wts, KH, KW, SH, SW, PT, PL, OH, OW):
    pooled = pool_floor(x)
    n, H, W, _ = pooled.shape
    out = np.zeros((n, OH, OW, wts.shape[-1]))
    for kh, kw in itertools.product(range(KH), range(KW)):
        for oh in range(OH):
            ih = oh * SH - PT + kh
            if not 0 <= ih < H:
                continue
            for ow in range(OW):
                iw = ow * SW - PL + kw
                if 0 <= iw < W:
                    out[:, oh, ow] += pooled[:, ih, iw] @ wts[kh * KW + kw]
    return out.reshape(n * OH * OW, -1)


# (un-pooled map PH x PW, images, KH, KW, SH, SW, PT, PL): VAD / gender 3x3 pairs, odd maps, stride 2, padding
SHAPES = {
    'vad': ((61, 15), 3, 3, 3, 1, 1, 0, 0),
    'gender': ((61, 17), 3, 3, 3, 1, 1, 0, 0),
    'odd_padded': ((13, 11), 5, 3, 3, 1, 1, 1, 1),
    'stride2_four_images': ((19, 9), 9, 3, 3, 2, 2, 0, 0),
}


@pytest.mark.parametrize('name', sorted(SHAPES))
def test_halo_planes_and_ldmatrix_rows_give_the_pooled_convolution(name):
    (ph, pw), n, KH, KW, SH, SW, PT, PL = SHAPES[name]
    rng = np.random.default_rng(sorted(SHAPES).index(name))
    x = rng.standard_normal((n, ph, pw, C))
    H, W = ph // 2, pw // 2
    OH, OW = (H + 2 * PT - KH) // SH + 1, (W + 2 * PL - KW) // SW + 1
    rows = _lib.load(build_if_missing=False).iss_gather_halo_rows_bound(H, OH, OW, KH, SH, PT)
    wts = rng.standard_normal((KH * KW, C, 8))
    got = model_layer(x, wts, KH, KW, SH, SW, PT, PL, OH, OW, rows)
    ref = reference_layer(x, wts, KH, KW, SH, SW, PT, PL, OH, OW)
    assert np.allclose(got, ref, rtol=1e-12, atol=1e-12)


def test_planes_of_eight_consecutive_pixels_hit_every_bank():
    """A matrix of ldmatrix reads 8 rows of 16 bytes: for 8 consecutive pixels the swizzled chunks cover all 32 banks."""
    for p0, q in itertools.product(range(16), range(8)):
        banks = set()
        for p in range(p0, p0 + 8):
            off = p * 128 + ((q ^ (p & 7)) << 4)
            banks.update(((off >> 2) + i) % 32 for i in range(4))
        assert len(banks) == 32


# ============================ budget ============================

def pipe_smem(BN, rows, W):
    return STAGES * 2 * BN * 128 + HALOS * 2 * (rows * W + 1) * 128 + 1024


def test_pipe_smem_follows_the_budget_arithmetic():
    lib = _lib.load(build_if_missing=False)
    seen = {True: 0, False: 0}
    for H, W, KH, KW, SH, N in itertools.product((14, 30, 32, 33), (7, 8, 10, 11), (1, 2, 3, 5, 6, 7), (1, 3), (1, 2), (64, 128)):
        OH, OW = (H - KH) // SH + 1, (W - KW) // SH + 1
        if OH < 1 or OW < 1:
            continue
        rows = lib.iss_gather_halo_rows_bound(H, OH, OW, KH, SH, 0)
        for Cin in (64, 128):
            got = lib.iss_gather_pipe_smem(H, W, OH, OW, KH, KW, SH, 0, Cin, N)
            want = pipe_smem(N, rows, W)
            want = want if Cin == 64 and KH * KW > 1 and want <= MAX_SMEM else 0
            assert got == want, (H, W, KH, KW, SH, Cin, N)
            if Cin == 64 and KH * KW > 1:
                seen[got > 0] += 1
                # two halos fit only where one does
                assert got == 0 or lib.iss_gather_halo_smem(H, W, OH, OW, KH, KW, SH, 0, Cin, N) > 0
    assert seen[True] and seen[False]


def test_segmenter_layers_take_two_halos():
    lib = _lib.load(build_if_missing=False)
    for H, W, OH, OW in ((30, 7, 28, 5), (30, 8, 28, 6)):     # VAD (nmel 21) and gender (nmel 24) 64 -> 128 layers
        assert 0 < lib.iss_gather_pipe_smem(H, W, OH, OW, 3, 3, 1, 0, 64, 128) <= MAX_SMEM
