"""The gather kernel's shared-memory halo (conv_gemm_wg_kernel with the 2x2 pooling folded in, 64 input channels)
against the float64 reference of the lowered network, on the GPU: the probe networks of tests/layer_probes.py on shapes
the probe matrix lacks -- tiles spanning two to four images, a partial last tile, odd pooled maps, stride 2, shapes
just inside and just over the halo budget (the latter keeps the global fill), more than one 64-channel block (global
fill), and non-finite words inside a pooling window.  Which fill a layer takes is the host rule that
tests/test_gather_halo_bound.py checks; the kernel instances of these layer kinds are pinned by the probe matrix."""
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


CASES = {
    # the segmenter CNNs' 3x3 pair: 140 / 168 output rows per image (tiles across two images)
    'halo_pool_pair_w21': lambda: dict(net=_pooled(21).conv(128, (3, 3), pre=True, relu=True).conv(128, (3, 3), pre=True, relu=True)),
    'halo_pool_pair_w24': lambda: dict(net=_pooled(24).conv(128, (3, 3), relu=True, post=True).conv(128, (3, 3), pre=True, relu=True)),
    # stride 2: 14 x 3 = 42 output rows per image, a tile spans up to four images; N = 64
    'halo_pool_stride2': lambda: dict(net=_pooled(21).conv(64, (3, 3), (2, 2), pre=True, relu=True)),
    # C = 192 behind the pooling: three channel blocks keep the global fill
    'halo_c192_global': lambda: dict(net=_pooled(24).conv(192, (3, 3), relu=True).pool().conv(64, (3, 3), pre=True, relu=True)),
    # pooled 32 x 8 map, N = 128: a 6x3 filter's halo just fits, a 7x3 filter's does not (global fill); the rule is
    # checked in test_gather_halo_bound.py
    'halo_at_budget_6x3': lambda: dict(net=lp.ProbeNet(21).conv(64, (4, 5), pre=True, relu=True).pool().conv(128, (6, 3), pre=True, relu=True),
                                       ranges=lp.SMALL),
    'halo_over_budget_7x3': lambda: dict(net=lp.ProbeNet(21).conv(64, (4, 5), pre=True, relu=True).pool().conv(128, (7, 3), pre=True, relu=True),
                                         ranges=lp.SMALL),
}


def _case(name):
    spec = dict(mode=3, fuse=True, mspec='normal', ranges=lp.RANGES)
    spec.update(CASES[name]())
    return spec


@pytest.mark.parametrize('name', sorted(CASES))
def test_halo_layer_vs_float64_reference(rt, name):
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


@pytest.mark.parametrize('name', ['halo_pool_pair_w21', 'halo_pool_stride2', 'halo_at_budget_6x3'])
def test_halo_patch_alone_equals_patch_in_batch(rt, name):
    """A tile's halo starts wherever its first output row lies: a patch alone and inside a 700-patch batch give the same
    bits, and a second run repeats them."""
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


def test_halo_pooling_of_non_finite_words_is_never_silent(rt):
    """First-layer activations past the fp16 range give split-half words whose value is NaN (hi = inf, lo = -inf).  The
    halo's pooling keeps the word of a NaN in the window, so the outputs that depend on it are not finite; every finite
    output stays within the bound of the float64 reference."""
    from oracle import lowered_ref as lr
    m = lp.make_mspec('normal')
    z, finite = lr.patch_inputs(m, 21, lp.RANGES)
    base = lp.ProbeNet(21, seed=5).conv(64, (4, 5), bias=False)
    low0 = base.lowered(lp.random_head(base.size, 0))
    peak = float(np.abs(lr.eval_layers(low0, z, stop=1)[0]).max())
    net = lp.ProbeNet(21, seed=5).conv(64, (4, 5), bias=False, gain=2e5 / peak).pool().conv(128, (3, 3), relu=True)
    head = lp.random_head(net.size, 0)
    low, ref, E, _ = tp._reference(net, head, z, finite, 3)
    got, _ = tp._forward(rt, low, torch.from_numpy(m).cuda(), lp.RANGES, 3, False)
    fin = np.isfinite(got).all(axis=1)
    assert not fin.all()                         # the overflow reached the pooled words
    wrong = fin & (np.abs(got - ref) > tp.C_BOUND * E).any(axis=1)
    assert not wrong.any(), int(wrong.sum())
