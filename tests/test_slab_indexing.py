"""CPU model of the slab kernel (csrc/conv_gemm_tc.cu, conv_slab_kernel) against a float64 convolution.

The kernel cannot run here; its numbering, fill, swizzled reads, accumulator mapping, epilogue and pipeline can.
  * The input of a batch is one tall image, pixel p = (img * H + ih) * W + iw; output slot s = (img * H + oh) * W + ow.
  * CTA b owns slots s0 = 256 b .. s0 + 255, warpgroup g the 64 from s0 + 64 g.  Its slab holds pixels s0 .. s0 + rows - 1
    (rows = 256 + (KH - 1) W + KW - 1 rounded up to 8), 16-byte chunk j of slab row r at chunk j ^ (r & 7) of a hi and a
    lo plane; pixels past the batch are zero.
  * The A operand of tap (kh, kw) for warpgroup g is the 64-row window from row 64 g + kh W + kw.  wgmma reads element
    k of window row i from chunk (k // 8) ^ ((start + i) & 7): the SWIZZLE_128B pattern follows the shared-memory address
    bits [7, 10), whatever the window's start row.
  * Ah.[Bh | Bl] is one m64n128 accumulator dm (columns 0..63 = Ah.Bh, 64..127 = Ah.Bl), Al.Bh one m64n64 accumulator dl;
    register q of thread t holds row 16 (t // 32) + (t % 32) // 4 + 8 ((q % 4) // 2), column 8 (q // 4) + 2 (t % 4) + q % 2,
    and the epilogue adds dm[q] + (dm[32 + q] + dl[q]) for its output column.
  * A slot is stored only when oh < OH, ow < OW and its image exists; every output position is stored exactly once.
The same file models the kernel's shared-memory pipeline (weight ring of cp.async groups, four warpgroups, one barrier
per k-block) over random interleavings."""
import itertools
import random

import numpy as np
import pytest

TS, C, N, G = 256, 64, 64, 4


def slab_rows(KH, KW, W):
    return (TS + (KH - 1) * W + KW - 1 + 7) & ~7


def n_tiles(n, H, W, OH, OW):
    slots = ((n - 1) * H + OH - 1) * W + OW                  # through the last output position
    return (slots + TS - 1) // TS


def split16(x):
    hi = x.astype(np.float16).astype(np.float64)
    return hi, (x - hi).astype(np.float16).astype(np.float64)


def fill_slab(X, s0, rows):
    """X [npix, C] (the tall image's pixels) -> swizzled slab [rows, 8 chunks, 8 values]."""
    p = s0 + np.arange(rows)
    vals = np.where((p < len(X))[:, None], X[np.minimum(p, len(X) - 1)], 0.0).reshape(rows, 8, 8)
    slab = np.full((rows, 8, 8), np.nan)
    r = np.arange(rows)[:, None]
    j = np.arange(8)[None, :]
    slab[r, j ^ (r & 7)] = vals
    return slab


def read_window(slab, start):
    """wgmma's view of the 64-row window from `start`: element k of row i at chunk (k // 8) ^ ((start + i) & 7)."""
    r = start + np.arange(64)[:, None]
    k = np.arange(C)[None, :]
    return slab[r, (k // 8) ^ (r & 7), k % 8]


def acc_rc(t, q):
    """Row and column of accumulator register q of thread t (m64nN, any N)."""
    return 16 * (t >> 5) + ((t & 31) >> 2) + 8 * ((q & 3) >> 1), 8 * (q >> 2) + 2 * (t & 3) + (q & 1)


def slab_conv(Xh, Xl, n, H, W, wh, wl, KH, KW):
    """The kernel's computation: Xh / Xl [npix, C] split planes, wh / wl [KH, KW, C, N] -> out [n * OH * OW, N]."""
    OH, OW = H - KH + 1, W - KW + 1
    rows = slab_rows(KH, KW, W)
    out = np.full((n * OH * OW, N), np.nan)
    stored = np.zeros(n * OH * OW, dtype=np.int64)
    t = np.arange(128)[:, None]
    for b in range(n_tiles(n, H, W, OH, OW)):
        s0 = b * TS
        sh, sl = fill_slab(Xh, s0, rows), fill_slab(Xl, s0, rows)
        for g in range(G):
            dm = np.zeros((64, 2 * N))
            dl = np.zeros((64, N))
            for kh, kw in itertools.product(range(KH), range(KW)):
                start = g * 64 + kh * W + kw
                assert start + 64 <= rows
                Ah, Al = read_window(sh, start), read_window(sl, start)
                dm += Ah @ np.concatenate([wh[kh, kw], wl[kh, kw]], axis=1)          # Ah.[Bh | Bl], one n128
                dl += Al @ wh[kh, kw]                                                 # Al.Bh, one n64
            # registers -> epilogue
            q = np.arange(N // 2)[None, :]
            r, c = acc_rc(t, q)
            r2, c2 = acc_rc(t, q + N // 2)
            assert np.array_equal(r2, r) and np.array_equal(c2, c + N)               # dm[32 + q]: the Ah.Bl of dm[q]'s column
            y = dm[r, c] + (dm[r2, c2] + dl[r, c])
            slot = s0 + g * 64 + r
            img, rem = slot // (H * W), slot % (H * W)
            oh, ow = rem // W, rem % W
            live = (img < n) & (oh < OH) & (ow < OW)
            m = (img * OH + oh) * OW + ow
            out[m[live], c[live]] = y[live]
            np.add.at(stored, np.unique(m[live]), 1)
    assert (stored == 1).all()                               # every output position exactly once, waste slots never
    return out


def reference_conv(x, w):
    n, H, W, _ = x.shape
    KH, KW = w.shape[:2]
    OH, OW = H - KH + 1, W - KW + 1
    y = np.zeros((n, OH, OW, w.shape[3]))
    for a, b in itertools.product(range(KH), range(KW)):
        y += np.einsum('nhwc,cd->nhwd', x[:, a:a + OH, b:b + OW], w[a, b])
    return y.reshape(-1, w.shape[3])


def three_products(xh, xl, wh, wl):
    return reference_conv(xh, wh) + reference_conv(xh, wl) + reference_conv(xl, wh)


SHAPES = [(65, 17, 5, 4), (65, 20, 5, 4)]


@pytest.mark.parametrize('H,W,KH,KW', SHAPES)
@pytest.mark.parametrize('n', [1, 2, 37])
def test_slab_packed_input_is_a_valid_convolution(n, H, W, KH, KW):
    """LD_PACKED / LD_F32: the tall image's pixel p is NHWC pixel p of the batch."""
    rng = np.random.default_rng(n * 100 + W)
    x = rng.standard_normal((n, H, W, C))
    w = rng.standard_normal((KH, KW, C, N))
    xh, xl = split16(x)
    wh, wl = split16(w)
    y = slab_conv(xh.reshape(-1, C), xl.reshape(-1, C), n, H, W, wh, wl, KH, KW)
    np.testing.assert_allclose(y, three_products(xh, xl, wh, wl), rtol=1e-12, atol=1e-9)
    np.testing.assert_allclose(y, reference_conv(x, w), rtol=0, atol=1e-4 * np.abs(y).max())


def first_layer_pixels(Yh, Yl, y_f0, row0, coef, post, n, H, W):
    """LD_FIRST fill, per slab pixel: the first layer from the map Y at the pixel's own patch rows and its coefficients."""
    p = np.arange(n * H * W)
    img, rem = p // (H * W), p % (H * W)
    ih, iw = rem // W, rem % W
    o = (row0[img] - y_f0 + ih) * W + iw
    al, bh, bl = coef[img, 0], coef[img, 1], coef[img, 2]
    v = (Yh.reshape(-1, C)[o] * al + bh) + (Yl.reshape(-1, C)[o] * al + bl)
    v = np.maximum(v, 0.0)
    return v * post[0] + post[1]


@pytest.mark.parametrize('H,W,KH,KW', SHAPES)
@pytest.mark.parametrize('n', [1, 2, 37])
def test_slab_fused_first_layer_uses_each_pixels_own_patch(n, H, W, KH, KW):
    """LD_FIRST: tiles straddle patches; each pixel takes its own patch's map rows (overlapping, hop 2) and coefficients."""
    rng = np.random.default_rng(7 * n + H)
    row0 = 40 + 2 * np.arange(n) + (rng.integers(0, 3, n) * 2 if n > 2 else 0)
    y_f0 = 30
    rows_y = int(row0.max()) - y_f0 + H
    Yh = rng.standard_normal((rows_y, W, C))
    Yl = rng.standard_normal((rows_y, W, C)) * 1e-7
    coef = np.stack([rng.uniform(0.5, 2.0, (n, C)), rng.standard_normal((n, C)), rng.standard_normal((n, C)) * 1e-7], axis=1)
    post = (rng.uniform(0.5, 1.5, C), rng.standard_normal(C))
    X = first_layer_pixels(Yh, Yl, y_f0, row0, coef, post, n, H, W)
    # reference: the patch of image i is rows row0[i] - y_f0 .. + H of the map, evaluated image by image
    x = np.stack([np.maximum((Yh[r - y_f0:r - y_f0 + H] * coef[i, 0] + coef[i, 1]) + (Yl[r - y_f0:r - y_f0 + H] * coef[i, 0] + coef[i, 2]), 0.0)
                  * post[0] + post[1] for i, r in enumerate(row0)])
    np.testing.assert_array_equal(X.reshape(x.shape), x)
    w = rng.standard_normal((KH, KW, C, N))
    xh, xl = split16(X)
    wh, wl = split16(w)
    y = slab_conv(xh, xl, n, H, W, wh, wl, KH, KW)
    np.testing.assert_allclose(y, three_products(xh.reshape(x.shape), xl.reshape(x.shape), wh, wl), rtol=1e-12, atol=1e-9)


def test_slab_rows_past_the_batch_are_zero():
    n, H, W = 1, 65, 17
    X = np.ones((n * H * W, C))
    rows = slab_rows(5, 4, W)
    last = n_tiles(n, H, W, 61, 14) - 1
    slab = fill_slab(X, last * TS, rows)
    p = last * TS + np.arange(rows)
    assert (slab[p >= n * H * W] == 0).all() and (slab[p < n * H * W] == 1).all()
    assert (p >= n * H * W).any()                            # the last tile does run past the batch


@pytest.mark.parametrize('start', range(16))
def test_window_read_at_every_residue(start):
    """A window may start at any row (residue start % 8): reading through the address-based swizzle returns the rows."""
    rng = np.random.default_rng(start)
    X = rng.standard_normal((200, C))
    slab = fill_slab(X, 0, 128)
    np.testing.assert_array_equal(read_window(slab, start), X[start:start + 64])


def test_tile_count_and_useful_fraction():
    """Slots with ow >= OW or oh >= OH are computed and dropped: the useful fraction is (OW / W) (OH / H); the last tile is
    partial.  VAD 5x4 layer: 0.77, gender: 0.80."""
    for (H, W, KH, KW), frac in zip(SHAPES, (0.77, 0.80)):
        OH, OW = H - KH + 1, W - KW + 1
        B = 8192
        tiles = n_tiles(B, H, W, OH, OW)
        assert tiles * TS >= ((B - 1) * H + OH - 1) * W + OW > (tiles - 1) * TS
        assert abs(B * OH * OW / (tiles * TS) - frac) < 0.01
        assert 2 * slab_rows(KH, KW, W) * 128 + 4 * 2 * N * 128 + 1024 <= 227 * 1024


# ------------------------------------------------------------------ the pipeline
AHEAD = 2


def run(nkb, stages, rng, groups=G):
    """One random interleaving of the warpgroups through the slab kernel's loop.  Before the loop every thread fills its
    part of the slab and the weights of k-blocks 0 and 1 are committed; per k-block kb each warpgroup waits for the group
    of kb (cp.async.wait_group 1), fences, meets the others at __syncthreads, commits the copy of kb + 2 into stage
    (kb + 2) % stages, issues its wgmmas of kb and waits until only those may pend (wgmma.wait_group 1).  Returns the
    hazards seen: a slab write or a weight copy that lands while a wgmma that reads the buffer may still run."""
    steps = ['wait', 'bar', 'copy', 'mma']
    pc = [[-1, 0] for _ in range(groups)]                        # k-block -1 = the slab fill
    inflight = [set() for _ in range(groups)]
    at_bar = [False] * groups
    hazards = []

    def release():
        if all(at_bar[h] or pc[h][0] >= nkb for h in range(groups)):
            for h in range(groups):
                if at_bar[h]:
                    at_bar[h] = False
                    pc[h][1] += 1
                    if pc[h][1] == len(steps):
                        pc[h] = [pc[h][0] + 1, 0]

    while any(p[0] < nkb for p in pc):
        for h in range(groups):
            for k in list(inflight[h]):
                if rng.random() < 0.3:
                    inflight[h].discard(k)
        movable = [h for h in range(groups) if pc[h][0] < nkb and not at_bar[h]]
        if not movable:
            if all(at_bar[h] or pc[h][0] >= nkb for h in range(groups)):
                release()
                continue
            raise AssertionError('deadlock')
        g = rng.choice(movable)
        kb, st = pc[g]
        if kb < 0:                                               # slab fill: st.shared into the slab
            if any(inflight[h] for h in range(groups)):
                hazards.append(('slab', g))
            pc[g] = [0, 0]
            continue
        step = steps[st]
        if step == 'bar':
            at_bar[g] = True
            release()
            continue
        if step == 'copy':
            nxt = kb + AHEAD
            if nxt < nkb and any(k % stages == nxt % stages for h in range(groups) for k in inflight[h]):
                hazards.append(('B', g, nxt))
        elif step == 'mma':
            inflight[g].add(kb)
            inflight[g] = {k for k in inflight[g] if k >= kb}
        pc[g][1] += 1
        if pc[g][1] == len(steps):
            pc[g] = [kb + 1, 0]
    return hazards


def test_slab_pipeline_is_safe_and_never_deadlocks():
    """Seeded random interleavings of the four warpgroups drain without deadlock, the slab is written only before any wgmma
    runs, and no weight stage is overwritten while a wgmma may read it.  With three stages instead of four the model finds
    the hazard (the copy of kb + 2 lands on the stage another warpgroup may still read for kb - 1)."""
    rng = random.Random(20261015)
    for nkb, _ in itertools.product((1, 2, 3, 9, 20), range(40)):
        assert run(nkb, 4, rng) == [], nkb
    assert any(run(9, 3, rng) for _ in range(200))
