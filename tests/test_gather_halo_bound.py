"""The gather convolution kernel stages the input rows a 128-row tile reads into a shared-memory halo, sized on the host
by iss_gather_halo_rows_bound.  The bound must cover every tile of every batch, or the staging would overrun the halo:
checked here against brute-force enumeration of the rows each tile's output rows and taps read, over every 3x3
convolution shape of the segmenter CNNs, of the layer probes and of ResNet101."""
import math

import numpy as np
import pytest

from inaspeechsegmenter_b200 import _lib
from oracle import resnet_ref

TBM = 128


def _out(x, k, s, p):
    return (x + 2 * p - k) // s + 1


def brute_rows(H, W, OH, OW, KH, SH, PT, n_img):
    """Largest (last - first + 1) over the tiles of an n_img batch, rows of the batch as one tall image."""
    M = n_img * OH * OW
    m = np.arange(M)
    img, rem = m // (OH * OW), m % (OH * OW)
    oh = rem // OW
    worst = 0
    for t0 in range(0, M, TBM):
        sl = slice(t0, min(t0 + TBM, M))
        ih = oh[sl, None] * SH - PT + np.arange(KH)[None, :]
        g = img[sl, None] * H + ih
        g = g[(ih >= 0) & (ih < H)]
        worst = max(worst, int(g.max() - g.min() + 1))
    return worst


def cnn_shapes():
    shapes = []
    for nmel in (21, 24):                        # VAD and gender: the two 3x3 layers behind the 2x2 pooling
        h, w = (68 - 3 - 4) // 2, (nmel - 4 - 3) // 2
        for _ in range(2):
            shapes.append((h, w, h - 2, w - 2, 3, 1, 0))
            h, w = h - 2, w - 2
    for H, W in ((65, 17), (65, 20), (63, 15), (30, 7), (13, 2)):        # probe maps
        for KH, S, same in ((3, 1, False), (3, 1, True), (3, 2, False), (3, 2, True), (4, 2, True), (7, 1, False), (17, 1, False)):
            if KH > H:
                continue
            P = (KH - 1) // 2 if same else 0
            OH = math.ceil(H / S) if same else _out(H, KH, S, 0)
            OW = math.ceil(W / (1 if W < 3 else S)) if same else max(_out(W, min(3, W), S, 0), 1)
            shapes.append((H, W, OH, OW, KH, S, P))
    return shapes


def resnet_shapes():
    arch = resnet_ref.plan(**resnet_ref.RELEASE)
    shapes = []
    for T in (144, 200):
        h, t = arch.feat_dim, T
        for blk in arch.blocks:
            c = blk['c2']
            oh, ot = _out(h, 3, c['stride'], 1), _out(t, 3, c['stride'], 1)
            shapes.append((h, t, oh, ot, 3, c['stride'], 1))            # either orientation of the map
            shapes.append((t, h, ot, oh, 3, c['stride'], 1))
            h, t = oh, ot
    return sorted(set(shapes))


@pytest.mark.parametrize('shape', cnn_shapes() + resnet_shapes())
def test_halo_rows_bound_is_exact_over_every_tile(shape):
    H, W, OH, OW, KH, SH, PT = shape
    lib = _lib.load()
    bound = lib.iss_gather_halo_rows_bound(H, OH, OW, KH, SH, PT)
    g = math.gcd(TBM, OH * OW)
    n_img = TBM // g + 3                         # every tile start residue of an image, and a partial last tile
    assert brute_rows(H, W, OH, OW, KH, SH, PT, n_img) == bound, shape
    for n in (1, 2, 5):                          # small batches never need more
        assert brute_rows(H, W, OH, OW, KH, SH, PT, n) <= bound, (shape, n)


def test_halo_budget_rule():
    """The first 3x3 layer of the segmenter CNNs (2x2 pooling folded in, 64 -> 128) takes the halo; more than 64
    channels, one-tap filters and halos past 227 KB keep the global fill."""
    lib = _lib.load()
    for H, W, OH, OW in ((30, 7, 28, 5), (30, 8, 28, 6)):
        smem = lib.iss_gather_halo_smem(H, W, OH, OW, 3, 3, 1, 0, 64, 128)
        assert 0 < smem <= 227 * 1024, (H, W, smem)
    assert lib.iss_gather_halo_smem(28, 5, 26, 3, 3, 3, 1, 0, 128, 128) == 0
    assert lib.iss_gather_halo_smem(30, 7, 30, 7, 1, 1, 1, 0, 64, 128) == 0
    # pooled 32 x 8 map, N = 128: a 6x3 filter fits (32 rows x 8 pixels x 256 B + 161 KB = 225 KB), a 7x3 filter
    # (34 rows, 229 KB) is just over
    assert lib.iss_gather_halo_smem(32, 8, 27, 6, 6, 3, 1, 0, 64, 128) == 230400
    assert lib.iss_gather_halo_smem(32, 8, 26, 6, 7, 3, 1, 0, 64, 128) == 0
