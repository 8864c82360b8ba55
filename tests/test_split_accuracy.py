"""CPU: numerical design check of the operand-split schemes the tensor-core GEMM can use.

The tensor-core path evaluates fp32 layers as sums of low-precision products (DESIGN.md).  This
emulates the schemes on the stand-in VAD network in float64 (exact products, exact accumulation -- i.e.
the algorithmic error of the split alone, without the tensor core's truncating accumulate) and checks
them against the fp32 oracle with the north-star tolerance (1e-4 on the per-frame softmax):

  tf32x3  hi = x with the 13 low mantissa bits cleared, lo = (x - hi) truncated to TF32;  Ah.Bh + Ah.Bl + Al.Bh
          (the production engine)
  tf32x1  a single TF32 product (why one pass is not enough)
  fp16x2  hi = fp16(x), lo = fp16(x - hi), weights pre-scaled by a power of two per layer;  same three products at
          the kind::f16 rate (2x TF32) with half the operand bytes -- the round-2 candidate
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import synth_audio
from oracle import cnn_oracle, segmenter_oracle as so


def _tf32_trunc(x):
    return (x.view(torch.int32) & -8192).view(torch.float32)


def split_tf32x3(x):
    hi = _tf32_trunc(x)
    return hi, _tf32_trunc(x - hi)


def split_tf32x1(x):
    return _tf32_trunc(x), None


def split_fp16x2(x):
    hi = x.to(torch.float16).to(torch.float32)
    return hi, (x - hi).to(torch.float16).to(torch.float32)


def _gemm_like(op, a, b, split, scale_b):
    """op(a, b) evaluated as the sum of split products in float64, returned as float32."""
    s = 1.0
    if scale_b:                                        # exact power-of-two pre-scale of the weights
        s = float(2.0 ** np.floor(np.log2(1.0 / float(b.abs().max()))))
    ah, al = split(a)
    bh, bl = split(b * s)
    y = op(ah.double(), bh.double())
    if al is not None:
        y = y + op(ah.double(), bl.double()) + op(al.double(), bh.double())
    return (y / s).float()


def forward_split(config, weights, x, split, scale_b=False):
    layers = config['config']['layers']
    w = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in weights.items()}
    t = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).permute(0, 3, 1, 2).contiguous()
    first = True
    for l in layers:
        cls, c, n = l['class_name'], l['config'], l['config'].get('name')
        if cls == 'Conv2D':
            k = w[n + '/kernel'].permute(3, 2, 0, 1).contiguous()
            if first:                                   # Cin = 1: direct fp32 kernel in the product, not a GEMM
                t = F.conv2d(t, k)
                first = False
            else:
                t = _gemm_like(F.conv2d, t, k, split, scale_b)
            t = t + w[n + '/bias'].view(1, -1, 1, 1)
        elif cls == 'BatchNormalization':
            inv = torch.rsqrt(w[n + '/moving_variance'] + c.get('epsilon', 1e-3))
            scale = inv * w[n + '/gamma']
            shift = w[n + '/beta'] - w[n + '/moving_mean'] * scale
            shape = (1, -1, 1, 1) if t.dim() == 4 else (1, -1)
            t = t * scale.view(shape) + shift.view(shape)
        elif cls == 'Activation':
            t = F.relu(t) if c['activation'] == 'relu' else F.softmax(t, dim=-1)
        elif cls == 'MaxPooling2D':
            t = F.max_pool2d(t, tuple(c['pool_size']), stride=tuple(c['strides']))
        elif cls == 'Flatten':
            t = t.permute(0, 2, 3, 1).reshape(t.shape[0], -1)
        elif cls == 'Dense':
            if w[n + '/kernel'].shape[1] % 32 == 0:     # the 3-class head runs on the fp32 kernel
                t = _gemm_like(torch.matmul, t, w[n + '/kernel'], split, scale_b)
            else:
                t = t @ w[n + '/kernel']
            t = t + w[n + '/bias']
            if c.get('activation') == 'softmax':
                t = F.softmax(t, dim=-1)
        elif cls not in ('InputLayer', 'Dropout'):
            raise NotImplementedError(cls)
    return t.numpy()


@pytest.fixture(scope='module')
def patches_and_ref(synth_models):
    s16 = synth_audio(20, seed=7)
    mspec, loge, difflen = so.media2feats(s16.astype(np.float32) / np.float32(32768))
    patches, finite = so.get_patches(mspec[:, :21].copy(), 68, 2)
    x = patches[finite][::13][:48][:, :, :, None].astype(np.float32)
    cfg, w = synth_models['smn']
    ref = cnn_oracle.KerasLikeModel(cfg, w).predict(x)
    return cfg, w, x, ref


def test_split_schemes(patches_and_ref):
    cfg, w, x, ref = patches_and_ref
    err = {}
    for name, split, scale in (('tf32x3', split_tf32x3, False), ('tf32x1', split_tf32x1, False),
                               ('fp16x2', split_fp16x2, False), ('fp16x2_scaled', split_fp16x2, True)):
        with torch.no_grad():
            err[name] = float(np.abs(forward_split(cfg, w, x, split, scale) - ref).max())
    print('max |softmax - fp32 oracle|:', {k: '%.2e' % v for k, v in err.items()})
    assert err['tf32x3'] <= 5e-6                     # production scheme: algorithmic error far below the 1e-4 bar
    assert err['tf32x1'] > 10 * err['tf32x3']        # a single TF32 pass is an order of magnitude worse
    assert err['fp16x2_scaled'] <= 2e-5              # round-2 candidate stays inside the bar with margin
