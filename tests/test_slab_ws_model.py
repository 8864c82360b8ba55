"""CPU model of the persistent, warp-specialized slab kernel's protocol (csrc/conv_gemm_tc.cu, conv_slab_kernel).

One CTA takes the tiles blockIdx.x, blockIdx.x + gridDim.x, ... in increasing order.  Its warpgroups:
  * producer warp 0 (one thread): per tile and tap, waits on wempty[s] (parity ph ^ 1), arms wfull[s] with the stage's
    bytes and issues one bulk copy into stage s, which lands later and completes the transaction on wfull[s];
  * producer warps 1..3: per tile, wait on sempty[b] (parity ph ^ 1), store their share of slab buffer b, fence and
    arrive on sfull[b] (96 arrivals complete it);
  * consumers 0 and 1: per tile, wait on sfull[b]; per tap, wait on wfull[s], issue the wgmmas of their 128 slots on
    stage s and slab b, commit, wgmma.wait_group 1, then the four warps arrive on wempty of the previous tap's stage; at
    the end of the tile wait_group 0 and arrive on wempty of the last stage and on sempty[b] (eight arrivals complete an
    empty barrier).
Stage and buffer indices wrap with a phase bit that flips at every wrap; ping-pong = two slab buffers and three stages,
the fallback for tall filters = one buffer and four stages.  mbarrier semantics: a wait on parity p returns once the
barrier's phase of parity p has completed (on a fresh barrier, parity 1 counts as completed).

The scheduler interleaves the warpgroups at random, lands copies and retires wgmma groups (in order, per consumer) at
random moments, and records a hazard whenever a buffer is written while an in-flight wgmma reads it, or a wgmma is
issued on a stage or slab that does not hold the data of its tap and tile.  The protocol must drain without deadlock
or hazard for every interleaving; each deliberately broken ordering must be caught."""
import itertools
import random

import pytest

TS, C, N = 256, 64, 64
FILL_WARPS, CONSUMER_WARPS = 3, 4


class Bar:
    def __init__(self, count):
        self.count, self.pending, self.tx, self.phase = count, 0, 0, 0

    def _maybe_complete(self):
        while self.pending >= self.count and self.tx == 0:   # surplus arrivals count toward the next phase
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


def cta_tiles(cta, grid, tiles):
    return list(range(cta, tiles, grid))


def run_cta(nkb, my_tiles, nbuf, stages, rng, bug=None):
    """One random interleaving of one CTA.  Returns the hazards seen (a deadlock ends the run as the last hazard) and the
    (tile, consumer, block) triples whose epilogue ran."""
    wfull = [Bar(1) for _ in range(stages)]
    wempty = [Bar(2 * CONSUMER_WARPS) for _ in range(stages)]
    sfull = [Bar(FILL_WARPS * 32) for _ in range(nbuf)]
    sempty = [Bar(2 * CONSUMER_WARPS) for _ in range(nbuf)]
    stage_data = [None] * stages                     # tap whose weights the stage holds (None while a copy writes it)
    copies = []                                      # in-flight bulk copies: (stage, tap)
    slab_data = [[None] * FILL_WARPS for _ in range(nbuf)]   # tile of each fill warp's share (None while written)
    inflight = [[], []]                              # per consumer, committed wgmma groups in order: (stage, buffer)
    hazards, epilogues = [], []

    def readers(kind, idx):
        return [g for c in (0, 1) for g in inflight[c] if (g[0] if kind == 'stage' else g[1]) == idx]

    def weights():
        s, ph = 0, 0
        for _tile in my_tiles:
            for kb in range(nkb):
                if bug != 'weights_skip_empty_wait':
                    yield lambda s=s, ph=ph: wempty[s].done(ph ^ 1)
                wfull[s].arrive_expect_tx(1)
                if readers('stage', s):
                    hazards.append(('stage overwritten while read', s, kb))
                stage_data[s] = None
                copies.append((s, kb))
                yield None
                s += 1
                if s == stages:
                    s, ph = 0, ph ^ 1

    def fill(f):
        b, ph = 0, 0
        for tile in my_tiles:
            if bug != 'fill_skip_empty_wait':
                yield lambda b=b, ph=ph: sempty[b].done(ph ^ 1)
            if readers('slab', b):
                hazards.append(('slab overwritten while read', b, tile))
            slab_data[b][f] = None
            yield None                               # the stores take time; other warpgroups run meanwhile
            if readers('slab', b):
                hazards.append(('slab overwritten while read', b, tile))
            slab_data[b][f] = tile
            sfull[b].arrive(32)                      # every thread of the warp: fence.proxy.async, then arrive
            yield None
            b += 1
            if b == nbuf:
                b, ph = 0, ph ^ 1

    def consumer(c):
        s, wph, b, sph = 0, 0, 0, 0
        for tile in my_tiles:
            yield lambda b=b, sph=sph: sfull[b].done(sph)
            prev = None
            for kb in range(nkb):
                if bug != 'consumer_skip_full_wait':
                    yield lambda s=s, wph=wph: wfull[s].done(wph)
                if stage_data[s] != kb:
                    hazards.append(('tap read a stage that does not hold its weights', c, tile, kb))
                if slab_data[b] != [tile] * FILL_WARPS:
                    hazards.append(('tap read a slab that does not hold its tile', c, tile, kb))
                inflight[c].append((s, b))
                if bug == 'consumer_release_before_wait':
                    wempty[s].arrive(CONSUMER_WARPS)
                    yield lambda: len(inflight[c]) <= 1
                else:
                    yield lambda: len(inflight[c]) <= 1      # wgmma.wait_group 1
                    if prev is not None:
                        wempty[prev].arrive(CONSUMER_WARPS)
                prev = s
                s += 1
                if s == stages:
                    s, wph = 0, wph ^ 1
            yield lambda: not inflight[c]                    # wgmma.wait_group 0
            if bug != 'consumer_release_before_wait':
                wempty[prev].arrive(CONSUMER_WARPS)
            sempty[b].arrive(CONSUMER_WARPS)
            b += 1
            if b == nbuf:
                b, sph = 0, sph ^ 1
            epilogues.extend((tile, c, k) for k in (0, 1))
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
                inflight[x].pop(0)                   # wgmma groups of one warpgroup retire in order
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


CONFIGS = [(2, 3), (1, 4)]                           # (slab buffers, weight stages): ping-pong, one-buffer fallback


@pytest.mark.parametrize('nbuf,stages', CONFIGS)
def test_protocol_is_safe_and_never_deadlocks(nbuf, stages):
    """Seeded random interleavings drain without deadlock and without a hazard, for tap counts around the ring size and
    for one to several tiles per CTA; every owned block of every tile runs its epilogue once."""
    rng = random.Random(20261015 + nbuf)
    for nkb, ntiles, _ in itertools.product((1, 2, 3, 4, 5, 20), (1, 2, 3, 5), range(6)):
        tiles = list(range(3, 3 + 7 * ntiles, 7))
        hazards, epi = run_cta(nkb, tiles, nbuf, stages, rng)
        assert hazards == [], (nkb, ntiles, hazards[:3])
        assert sorted(epi) == sorted((t, c, k) for t in tiles for c in (0, 1) for k in (0, 1))


@pytest.mark.parametrize('bug', ['weights_skip_empty_wait', 'fill_skip_empty_wait', 'consumer_skip_full_wait',
                                 'consumer_release_before_wait'])
@pytest.mark.parametrize('nbuf,stages', CONFIGS)
def test_model_catches_broken_orderings(bug, nbuf, stages):
    """A producer that does not wait on an empty barrier, a consumer that does not wait for its stage to land, or one
    that releases a stage before its wgmmas retired: some interleaving overwrites a buffer in use or reads stale data."""
    rng = random.Random(7)
    found = False
    for _ in range(300):
        hazards, _ = run_cta(5, [0, 4, 8, 12], nbuf, stages, rng, bug)
        if [h for h in hazards if h[0] != 'deadlock']:   # a broken ordering may also deadlock; that alone does not count
            found = True
            break
    assert found, bug


def test_persistent_tile_order():
    """grid = min(tiles, SMs); CTA i takes tiles i, i + grid, ... in increasing order; every tile exactly once, and at
    any round the CTAs work on consecutive tiles (shared first-layer map and input rows in L2)."""
    for tiles, sms in ((1, 132), (131, 132), (132, 132), (133, 132), (35456, 132), (1000, 7)):
        grid = min(tiles, sms)
        seen = []
        for cta in range(grid):
            mine = cta_tiles(cta, grid, tiles)
            assert mine == sorted(mine) and mine[0] == cta
            seen += mine
        assert sorted(seen) == list(range(tiles))
        for rnd in range(-(-tiles // grid)):
            cur = [cta_tiles(cta, grid, tiles)[rnd] for cta in range(grid) if rnd < len(cta_tiles(cta, grid, tiles))]
            assert cur == list(range(rnd * grid, rnd * grid + len(cur)))


def acc_rc(t, q):
    """Row and column of accumulator register q of thread t (m64nN, any N)."""
    return 16 * (t >> 5) + ((t & 31) >> 2) + 8 * ((q & 3) >> 1), 8 * (q >> 2) + 2 * (t & 3) + (q & 1)


@pytest.mark.parametrize('KH,KW,W', [(5, 4, 17), (5, 4, 20), (17, 9, 24), (1, 1, 3)])
def test_block_ownership_keeps_each_slots_wgmma_sequence(KH, KW, W):
    """Consumer c owns slots 128 c .. 128 c + 127 (blocks 2c and 2c + 1) as the N side of three m64n128k16 products per
    k16 step, hh = Bh^T.Ah, hl = Bl^T.Ah and lh = Bh^T.Al, with the 64 output channels as the M side.  Register
    q = 4 i + 2 h + e of thread t holds channel 16 (t / 32) + (t % 32) / 4 + 8 h of slot 128 c + 8 i + 2 (t % 4) + e:
    exactly what the wgmma accumulator layout gives that row and column.  Every (slot, channel) of the tile is held by
    exactly one (consumer, thread, register); each accumulator still sums the same products of one slot and channel,
    tap by tap and k16 step by k16 step; the 128-row window of every tap stays inside the slab."""
    rows = (TS + (KH - 1) * W + KW - 1 + 7) & ~7
    owner = {}
    for c in (0, 1):
        assert max(128 * c + kh * W + kw for kh in range(KH) for kw in range(KW)) + 128 <= rows
        for t, i, h, e in itertools.product(range(128), range(2 * N // 8), range(2), range(2)):
            ch = 16 * (t >> 5) + ((t & 31) >> 2) + 8 * h
            slot = 128 * c + 8 * i + 2 * (t & 3) + e
            assert acc_rc(t, 4 * i + 2 * h + e) == (ch, slot - 128 * c)
            assert (slot, ch) not in owner
            owner[(slot, ch)] = c
    assert len(owner) == TS * N
    assert all(c == (slot >= 128) for (slot, _), c in owner.items())


@pytest.mark.parametrize('H,W,OH,OW', [(65, 17, 61, 14), (65, 20, 61, 17), (9, 3, 5, 3), (4, 1, 2, 1), (24, 24, 8, 16)])
def test_epilogue_slot_walk(H, W, OH, OW):
    """The epilogue finds (img, oh, ow) of its slots 8 i + 2 (t % 4) + e by one division for i = 0 and then steps of 8
    (and + 1 for e = 1), wrapping ow at W and oh at H; that equals the division for every slot, for any W."""
    HW, n_img = H * W, 3
    for c, t4, tile in itertools.product((0, 1), range(4), (0, 1, 5, 11)):
        sl0 = tile * TS + 128 * c + 2 * t4
        img, rem = divmod(sl0, HW)
        oh, ow = divmod(rem, W)
        for i in range(2 * N // 8):
            for e in (0, 1):
                ie, he, we = img, oh, ow + e
                if we == W:
                    we, he = 0, he + 1
                    if he == H:
                        he, ie = 0, ie + 1
                sl = sl0 + 8 * i + e
                assert (ie, he, we) == (sl // HW, sl % HW // W, sl % W)
                live = ie < n_img and he < OH and we < OW
                assert live == (sl < n_img * HW and sl % HW // W < OH and sl % W < OW)
            ow += 8
            while ow >= W:
                ow -= W
                oh += 1
                if oh == H:
                    oh, img = 0, img + 1
