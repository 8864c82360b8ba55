"""CPU model of the shared-memory pipeline of the wgmma convolution kernel (csrc/conv_gemm_tc.cu, conv_gemm_wg_kernel).

Two warpgroups run the same k-block loop.  Per k-block kb each one
  fills its operand tile A[g][kb % 2]                    (st.shared; the tile was read by its own wgmmas of kb - 2),
  waits for the weight stage of kb                        (cp.async.wait_group 1: only the newest commit group may pend),
  meets the other warpgroup at __syncthreads,
  copies its share of the weights of kb + 2 into stage (kb + 2) % B_STAGES and commits a group (empty past the end),
  issues its wgmmas of kb on A[g][kb % 2] and stage kb % B_STAGES, then wgmma.wait_group 1 (its kb - 1 retires).
The weights of k-blocks 0 and 1 are copied before the loop.  A wgmma may retire at any moment after it is issued and
must have retired when wait_group says so.  Both sides must agree on the stage of every k-block, the commit groups must
make the weights of kb complete at its wait, and no tile or stage may be overwritten while a wgmma that reads it can
still be in flight -- for every interleaving of the two warpgroups."""
import itertools
import random

B_STAGES, A_STAGES, AHEAD = 4, 2, 2


def weight_schedule(nkb, stages=B_STAGES):
    """(k-block, stage) written by each commit group, in commit order; None = empty group."""
    groups = [(kb, kb % stages) if kb < nkb else None for kb in range(AHEAD)]
    for kb in range(nkb):
        nxt = kb + AHEAD
        groups.append((nxt, nxt % stages) if nxt < nkb else None)
    return groups


def test_producer_and_consumers_agree_on_every_box():
    for nkb in range(1, 40):
        groups = weight_schedule(nkb)
        written = {g[0]: g[1] for g in groups if g is not None}
        assert sorted(written) == list(range(nkb))
        for kb in range(nkb):
            assert written[kb] == kb % B_STAGES                       # the stage the wgmmas of kb read
            # at the wait of iteration kb the groups committed so far are the prologue's and those of iterations < kb;
            # wait_group 1 lets only the newest pend, so the group of kb must not be the newest
            committed = AHEAD + kb
            idx = next(i for i, g in enumerate(groups) if g is not None and g[0] == kb)
            assert idx < committed - 1, (nkb, kb)


def run(nkb, stages, rng):
    """One random interleaving of the two warpgroups; returns the hazards seen (empty when the pipeline is safe)."""
    steps = ['fill', 'wait', 'bar', 'copy', 'mma']
    pc = [[0, 0], [0, 0]]                                           # (k-block, step) per warpgroup
    inflight = [set(), set()]                                       # k-blocks whose wgmmas may still run
    at_bar = [False, False]
    hazards = []
    while any(p[0] < nkb for p in pc):
        for g in (0, 1):                                            # a wgmma may retire at any time
            for k in list(inflight[g]):
                if rng.random() < 0.3:
                    inflight[g].discard(k)
        movable = [g for g in (0, 1) if pc[g][0] < nkb and not at_bar[g]]
        if not movable:
            if all(at_bar[g] or pc[g][0] >= nkb for g in (0, 1)):
                for g in (0, 1):
                    if at_bar[g]:
                        at_bar[g] = False
                        pc[g][1] += 1
                continue
            raise AssertionError('deadlock')
        g = rng.choice(movable)
        kb, st = pc[g]
        step = steps[st]
        if step == 'fill':
            if any(k % A_STAGES == kb % A_STAGES for k in inflight[g]):
                hazards.append(('A', g, kb))
        elif step == 'bar':
            at_bar[g] = True
            if all(at_bar[h] or pc[h][0] >= nkb for h in (0, 1)):
                for h in (0, 1):
                    if at_bar[h]:
                        at_bar[h] = False
                        pc[h][1] += 1
            continue
        elif step == 'copy':
            nxt = kb + AHEAD
            if nxt < nkb and any(k % stages == nxt % stages for h in (0, 1) for k in inflight[h]):
                hazards.append(('B', g, nxt))
        elif step == 'mma':
            inflight[g].add(kb)
            inflight[g] = {k for k in inflight[g] if k >= kb}          # wait_group 1: only the group just committed may pend
        pc[g][1] += 1
        if pc[g][1] == len(steps):
            pc[g] = [kb + 1, 0]
    return hazards


def test_ring_never_deadlocks():
    """Random interleavings (seeded) of the two warpgroups drain without deadlock and without a hazard.  With three weight
    stages instead of four the copy of kb + 2 would land on the stage the other warpgroup may still be reading for
    kb - 1: the model finds that hazard, which is why the ring has four stages at this prefetch distance."""
    rng = random.Random(20261015)
    for nkb, _ in itertools.product((1, 2, 3, 5, 9, 20), range(60)):
        assert run(nkb, B_STAGES, rng) == [], nkb
    assert any(run(9, 3, rng) for _ in range(200))
