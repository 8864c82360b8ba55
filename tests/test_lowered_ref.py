"""CPU: the float64 evaluator of lowered networks (oracle/lowered_ref.py) against the Keras-config interpreter
(oracle/cnn_oracle.py, fp32) on the stand-in networks, the second architecture of test_gpu_parity and every probe
network of tests/layer_probes.py: both must agree within the float32 round-off the evaluator bounds (u = 2^-24 per
GEMM term).  This pins the reference the GPU probes are checked against, without a GPU."""
import numpy as np
import pytest

import layer_probes as lp
from inaspeechsegmenter_b200 import models
from oracle import cnn_oracle, lowered_ref as lr
from test_gpu_parity import _alt_keras_cnn


def _oracle(cfg, w, z):
    return cnn_oracle.KerasLikeModel(cfg, w).predict(z.astype(np.float32)).astype(np.float64)


def test_patch_stats_follow_the_kernel():
    """float64 sums, float32 mean / std: the z-normalised patch has mean ~0 and std ~1; constant patches are flagged."""
    m = lp.make_mspec('const')
    z, finite = lr.patch_inputs(m, 21, [(0, 400), (590, 620)])
    assert finite.sum() < len(finite) and finite[:100].all()
    zf = z[finite].reshape(finite.sum(), -1)
    assert np.abs(zf.mean(axis=1)).max() < 1e-5 and np.abs(zf.std(axis=1) - 1).max() < 1e-5
    mu, sg, fin = lr.patch_stats(m[None, 420:488, :21])
    assert not fin[0] and sg[0] == 0
    lo = lp.mspec_low_variance()
    z, finite = lr.patch_inputs(lo, 24, [(100, 110)])
    assert finite.all() and np.abs(z.reshape(10, -1).std(axis=1) - 1).max() < 1e-3


@pytest.mark.parametrize('which', ['smn', 'gender', 'alt21', 'alt24'])
def test_reference_matches_keras_interpreter_on_stand_ins(synth_models, which):
    if which.startswith('alt'):
        nmel = int(which[3:])
        cfg, w = _alt_keras_cnn(nmel, 3, seed=nmel)
    else:
        cfg, w = synth_models[which]
        nmel = 21 if which == 'smn' else 24
    low = models.lower_keras_model(cfg, w, 68, nmel)
    m = lp.mspec_normal(600, seed=3)
    z, finite = lr.patch_inputs(m, nmel, [(0, 3), (100, 109)])
    y, E = lr.eval_layers(low, z, mode=0)
    ref = _oracle(cfg, w, z)
    assert y.shape == ref.shape
    # softmax heads: |d softmax| <= 2 max |d logit|
    assert (np.abs(y - ref) <= 2 * E.max(axis=1, keepdims=True) + 1e-7).all(), np.abs(y - ref).max()


@pytest.mark.parametrize('name', sorted(lp.CASES))
def test_reference_matches_keras_interpreter_on_probe(name):
    spec = lp.case(name)
    net = spec['net']
    head = lp.random_head(net.size, 0)
    low = net.lowered(head)
    m = lp.make_mspec(spec['mspec'], 700)
    z, finite = lr.patch_inputs(m, net.nmel, [(30, 33), (250, 253)])
    y, E = lr.eval_layers(low, z, mode=0)
    ref = _oracle(*net.with_head(head), z)
    ok = finite
    err = np.abs(y - ref)[ok]
    assert (err <= E[ok]).all(), (err / E[ok]).max()


# ------------------------------------------------------------------ softmax head
def _softmax_f32(l, max_sub=True, k0=0):
    """softmax_head_kernel in numpy float32: max subtraction, exp, the sum over k = k0 .. K-1, one division."""
    l = np.asarray(l, dtype=np.float32)
    z = l - l.max(axis=1, keepdims=True) if max_sub else l
    with np.errstate(over='ignore', invalid='ignore', divide='ignore'):
        e = np.exp(z)
        s = np.zeros(len(l), np.float32)
        for k in range(k0, l.shape[1]):
            s = s + e[:, k]
        return (e / s[:, None]).astype(np.float64)


def _logits(K, seed=0):
    """float32 logits: ordinary, past expf's range (|l| > 88.7), a few ulps apart, all far below zero."""
    r = np.random.default_rng(seed)
    rows = [r.standard_normal((200, K)) * 4, r.standard_normal((50, K)) * 300 + 150,
            np.float32(r.standard_normal((50, 1)) * 40) * (1 + np.arange(K)[None, :] * 2.0 ** -22),
            -1e4 + r.standard_normal((20, K)) * 60]
    return np.concatenate(rows).astype(np.float32)


@pytest.mark.parametrize('K', [1, 2, 3, 8])
def test_softmax_bound_holds_for_float32_softmax(K):
    """The float32 softmax of exact float32 logits (E = 0) lies inside the softmax bound, on ordinary and extreme logits;
    a softmax without the max subtraction or with a sum that skips k = 0 does not (K > 1)."""
    l = _logits(K)
    p, E = lr.softmax(l.astype(np.float64))
    got = _softmax_f32(l)
    assert (np.abs(got - p) <= E).all(), (np.abs(got - p) / E).max()
    if K > 1:
        for wrong in (_softmax_f32(l, max_sub=False), _softmax_f32(l, k0=1)):
            assert not (np.abs(wrong - p) <= 2 * E).all()


def test_softmax_bound_carries_the_logits_bound():
    """Logits perturbed within their bound E move the posteriors by at most the propagated bound (first order)."""
    r = np.random.default_rng(1)
    l = r.standard_normal((500, 3)) * 3
    El = np.abs(l) * 1e-5 + 1e-6
    p, E = lr.softmax(l, El)
    for s in range(4):
        q, _ = lr.softmax(l + El * r.choice([-1.0, 1.0], l.shape))
        assert (np.abs(q - p) <= E).all()


def test_override_rows_are_one_half_with_zero_bound(synth_models):
    cfg, w = synth_models['smn']
    low = models.lower_keras_model(cfg, w, 68, 21)
    m = lp.make_mspec('const', 700)
    y, E = lr.evaluate(low, m, [(190, 240)])
    _, finite = lr.patch_inputs(m, 21, [(190, 240)])
    assert (~finite).any() and finite.any()
    assert (y[~finite] == 0.5).all() and (E[~finite] == 0).all() and (E[finite] > 0).all()
    assert np.allclose(y[finite].sum(axis=1), 1.0)


# ------------------------------------------------------------------ MLP
@pytest.mark.parametrize('name', sorted(lp.MLP_CASES))
def test_mlp_bound_holds_for_float32_numpy(name):
    """numpy float32 evaluation of the MLP's Keras config (vfs_oracle: unfolded BatchNorm) lies inside the float64 bound
    of its lowered Dense stack, every layer at u = U32."""
    from oracle import vfs_oracle
    in_dim, layers = lp.MLP_CASES[name]
    cfg, w = lp.mlp_config(in_dim, layers, seed=4)
    low = models.lower_keras_model(cfg, w, 1, in_dim, allow_no_head=True)
    x = np.random.default_rng(2).standard_normal((300, in_dim)).astype(np.float32)
    y, E = lr.eval_layers(low, x, mode=0, first=False)
    got = vfs_oracle.mlp_numpy(cfg, w, x).astype(np.float64)
    assert y.shape == got.shape
    assert (np.abs(got - y) <= E).all(), (np.abs(got - y) / E).max()


# ------------------------------------------------------------------ dispatch mirror
@pytest.mark.parametrize('name', sorted(lp.CASES))
def test_mirror_predicts_the_probe_kernels(name):
    """In the probe's mode, the kernels the mirror of plan_forward / iss_conv_kernel predicts include every kernel the
    case lists by hand (the GPU probes check the mirror's whole list against a profiler trace)."""
    spec = lp.case(name)
    low = spec['net'].lowered(lp.random_head(spec['net'].size, 0))
    names = lr.kernel_names(low, spec['mode'], spec['fuse'])
    assert set(spec['kernels']) <= names, (sorted(set(spec['kernels']) - names), sorted(names))


GATHER_KERNELS = {   # the pooled 3x3 layers of test_gather_halo_gpu.py / test_gather_pipe_gpu.py
    'halo_pool_pair_w21': ['conv_gemm_wg_kernel<1,128,2>', 'conv_gemm_wg_kernel<1,128,1>', 'conv_slab_kernel<3>'],
    'halo_pool_stride2': ['conv_gemm_wg_kernel<1,64,2>'],
    'halo_c192_global': ['conv_slab_kernel<3>', 'conv_gemm_wg_kernel<1,64,2>', 'dense_small_n_kernel'],
    'halo_over_budget_7x3': ['conv_first_direct_kernel', 'conv_gemm_wg_kernel<1,128,2>'],
    'pipe_w24_n64': ['conv_gemm_wg_kernel<1,64,2>', 'conv_slab_kernel<3>'],
    'pipe_outside_6x3_w24': ['conv_gemm_wg_kernel<1,128,2>'],
}


@pytest.mark.parametrize('name', sorted(GATHER_KERNELS))
def test_mirror_predicts_the_gather_kernels(name):
    import test_gather_halo_gpu as th
    import test_gather_pipe_gpu as tq
    spec = (th._case if name.startswith('halo') else tq._case)(name)
    net = spec['net']
    names = lr.kernel_names(net.lowered(lp.random_head(net.size, 0)), spec['mode'], spec['fuse'])
    assert set(GATHER_KERNELS[name]) <= names, sorted(names)


def test_mirror_modes_and_switches():
    """Mode 0 runs every layer but the first and the small heads on conv_gemm_f32_kernel; mode 2 never takes an fp16
    kernel or split-half words; ISS_B200_FUSE_FIRST=0 / ISS_B200_FUSE_POOL=0 bring the stand-alone first layer and the
    pooling kernel back."""
    spec = lp.case('g3_pool_odd')
    low = spec['net'].lowered(lp.random_head(spec['net'].size, 0))
    assert lr.plan(low, 3) == [None, 'conv_slab_kernel<3>', None, 'conv_gemm_wg_kernel<1,128,2>',
                               'conv_gemm_f32_kernel<64,false>']
    assert lr.plan(low, 3, fuse_first=False, fuse_pool=False) == [
        'conv_first_direct_kernel', 'conv_slab_kernel<1>', 'maxpool_nhwc_kernel<uint4>', 'conv_gemm_wg_kernel<1,128,1>',
        'conv_gemm_f32_kernel<64,false>']
    assert lr.plan(low, 2) == ['conv_first_direct_kernel', 'conv_gemm_wg_kernel<0,64,0>', 'maxpool_nhwc_kernel<float4>',
                               'conv_gemm_wg_kernel<0,128,0>', 'conv_gemm_f32_kernel<64,false>']
    assert lr.plan(low, 0) == ['conv_first_direct_kernel', 'conv_gemm_f32_kernel<64,false>', 'maxpool_nhwc_kernel<float4>',
                               'conv_gemm_f32_kernel<128,false>', 'conv_gemm_f32_kernel<64,false>']
