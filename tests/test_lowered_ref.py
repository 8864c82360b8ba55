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
