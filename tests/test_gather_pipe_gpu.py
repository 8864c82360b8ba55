"""The pipelined pooled gather convolution (conv_gemm_wg_kernel with the 2x2 pooling folded in, 64 input channels, two
halo buffers) against the float64 reference of the lowered network, on the GPU, with the probe machinery of
tests/test_layer_probes_gpu.py: the segmenter CNNs' 3x3 pair, grids with fewer tiles than SMs and tile counts that are
not a multiple of the grid, more than 8192 patches, shapes just inside and just outside the two-halo budget, non-finite
words inside a pooling window, and bit-identical results for a patch alone, inside a batch and across runs."""
import numpy as np
import pytest

import layer_probes as lp
import test_layer_probes_gpu as tp

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')


@pytest.fixture(scope='module')
def rt():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from inaspeechsegmenter_b200 import _lib, engine
    return dict(ctx=engine.Context(0), lib=_lib, engine=engine)


def _pooled(nmel=21):
    # 65 x W -> 5x4 -> 61 x (W - 3) -> pool -> 30 x 7 (nmel 21, odd) or 30 x 8 (nmel 24)
    return lp.ProbeNet(nmel).conv(64, (4, 5), pre=True, relu=True).conv(64, (5, 4), pre=True, relu=True).pool()


def _budget(nmel):
    # 68 x nmel -> 4x5 -> pool -> 32 x 8 (nmel 21) or 32 x 10 (nmel 24), then a 6x3 filter with 128 outputs
    return lp.ProbeNet(nmel).conv(64, (4, 5), pre=True, relu=True).pool().conv(128, (6, 3), pre=True, relu=True)


# (H, W, OH, OW, KH, KW, SH, PT, C, N) of the pooled layer and whether two halos fit
PIPE_SHAPES = {
    'pipe_pair_w21': ((30, 7, 28, 5, 3, 3, 1, 0, 64, 128), True),
    'pipe_pair_w24': ((30, 8, 28, 6, 3, 3, 1, 0, 64, 128), True),
    'pipe_inside_6x3_w21': ((32, 8, 27, 6, 6, 3, 1, 0, 64, 128), True),
    'pipe_outside_6x3_w24': ((32, 10, 27, 8, 6, 3, 1, 0, 64, 128), False),
}

CASES = {
    # 54 patches: 60 tiles of 128 rows, fewer than the SMs
    'pipe_pair_w21': lambda: dict(net=_pooled(21).conv(128, (3, 3), pre=True, relu=True).conv(128, (3, 3), pre=True, relu=True)),
    'pipe_pair_w24': lambda: dict(net=_pooled(24).conv(128, (3, 3), relu=True, post=True).conv(128, (3, 3), pre=True, relu=True)),
    # 700 patches of 140 output rows: 766 tiles, not a multiple of the grid
    'pipe_pair_w21_700': lambda: dict(net=_pooled(21).conv(128, (3, 3), pre=True, relu=True), ranges=[(0, 700)]),
    # N = 64: the 64-wide n-tile
    'pipe_w24_n64': lambda: dict(net=_pooled(24).conv(64, (3, 3), pre=True, relu=True)),
    # two halos just fit (nmel 21) / only one fits, the single-halo path (nmel 24)
    'pipe_inside_6x3_w21': lambda: dict(net=_budget(21), ranges=lp.SMALL),
    'pipe_outside_6x3_w24': lambda: dict(net=_budget(24), ranges=lp.SMALL),
}


def _case(name):
    spec = dict(mode=3, fuse=True, mspec='normal', ranges=lp.RANGES)
    spec.update(CASES[name]())
    return spec


@pytest.mark.parametrize('name', sorted(PIPE_SHAPES))
def test_pipe_rule_of_the_probe_shapes(rt, name):
    lib = rt['lib'].load()
    args, pipe = PIPE_SHAPES[name]
    assert (lib.iss_gather_pipe_smem(*args) > 0) == pipe, name
    assert lib.iss_gather_halo_smem(*args) > 0


@pytest.mark.parametrize('name', sorted(CASES))
def test_pipe_layer_vs_float64_reference(rt, name):
    """Random and one-hot heads: |got - ref| <= C_BOUND E on every patch."""
    from oracle import lowered_ref as lr
    spec = _case(name)
    net = spec['net']
    m = lp.make_mspec(spec['mspec'])
    z, finite = lr.patch_inputs(m, net.nmel, spec['ranges'])
    assert finite.all()
    heads = [lp.random_head(net.size, s) for s in tp.HEAD_SEEDS]
    heads.append(lp.selector_head(net.shape, lp.default_picks(net.shape)))
    body, worst = None, 0.0
    for head in heads:
        low, ref, E, body = tp._reference(net, head, z, finite, spec['mode'], body)
        got, _ = tp._forward(rt, low, torch.from_numpy(m).cuda(), spec['ranges'], spec['mode'], spec['fuse'])
        assert np.isfinite(got).all(), name
        worst = max(worst, float((np.abs(got - ref) / E).max()))
    assert worst <= tp.C_BOUND, (name, worst)


@pytest.mark.parametrize('name', ['pipe_pair_w21', 'pipe_pair_w24', 'pipe_inside_6x3_w21'])
def test_pipe_patch_alone_equals_patch_in_batch(rt, name):
    """A tile's halo and its CTA depend on where the tile lies in the batch: a patch alone and inside a 700-patch batch
    give the same bits, and a second run repeats them."""
    spec = _case(name)
    net = spec['net']
    low = net.lowered(lp.random_head(net.size, 7))
    dm = torch.from_numpy(lp.make_mspec('normal')).cuda()
    batch, _ = tp._forward(rt, low, dm, [(0, 700)], spec['mode'], spec['fuse'])
    again, _ = tp._forward(rt, low, dm, [(0, 700)], spec['mode'], spec['fuse'])
    assert np.array_equal(batch, again)
    for j in (0, 17, 18, 333, 699):
        alone, _ = tp._forward(rt, low, dm, [(j, j + 1)], spec['mode'], spec['fuse'])
        assert np.array_equal(alone[0], batch[j]), (name, j)


def test_pipe_more_than_8192_patches(rt):
    """8400 patches (more than one 8192-patch sweep): every patch has the bits it has in a short batch of its own."""
    net = _pooled(21).conv(128, (3, 3), pre=True, relu=True).conv(128, (3, 3), pre=True, relu=True)
    low = net.lowered(lp.random_head(net.size, 3))
    dm = torch.from_numpy(lp.make_mspec('normal', L=2 * 8400 + 80)).cuda()
    big, _ = tp._forward(rt, low, dm, [(0, 8400)], 3, True)
    assert big.shape[0] == 8400 and np.isfinite(big).all()
    for lo, hi in ((0, 40), (8150, 8240), (8360, 8400)):
        part, _ = tp._forward(rt, low, dm, [(lo, hi)], 3, True)
        assert np.array_equal(part, big[lo:hi]), (lo, hi)


def test_pipe_pooling_of_non_finite_words_is_never_silent(rt):
    """Split-half words whose value is NaN (first-layer activations past the fp16 range) win their pooling window in the
    pipelined fill too: the outputs that depend on them are not finite, every finite output is within the bound."""
    from oracle import lowered_ref as lr
    m = lp.make_mspec('normal')
    z, finite = lr.patch_inputs(m, 21, lp.RANGES)
    base = lp.ProbeNet(21, seed=5).conv(64, (4, 5), bias=False)
    low0 = base.lowered(lp.random_head(base.size, 0))
    peak = float(np.abs(lr.eval_layers(low0, z, stop=1)[0]).max())
    net = lp.ProbeNet(21, seed=5).conv(64, (4, 5), bias=False, gain=2e5 / peak).pool().conv(128, (3, 3), relu=True)
    lib = rt['lib'].load()
    assert lib.iss_gather_pipe_smem(32, 8, 30, 6, 3, 3, 1, 0, 64, 128) > 0
    head = lp.random_head(net.size, 0)
    low, ref, E, _ = tp._reference(net, head, z, finite, 3)
    got, _ = tp._forward(rt, low, torch.from_numpy(m).cuda(), lp.RANGES, 3, False)
    fin = np.isfinite(got).all(axis=1)
    assert not fin.all()
    wrong = fin & (np.abs(got - ref) > tp.C_BOUND * E).any(axis=1)
    assert not wrong.any(), int(wrong.sum())
