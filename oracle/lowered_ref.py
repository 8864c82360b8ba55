"""Oracle (test infrastructure): float64 evaluation of a LOWERED CNN with a propagated error bound.

``cnn_oracle`` evaluates the Keras config; this module evaluates what the CUDA kernels are handed instead:
``LoweredModel.descs`` + ``blob`` (the ``iss_layer_desc`` semantics of csrc/cnn.cu), with the float32 parameters of
the blob -- so the folded BatchNorm is the one the kernels use:

  Conv2D     explicit pads / strides, then the epilogue bias -> pre-affine -> ReLU -> sigmoid -> post-affine
  Dense      the same epilogue on [n, cin] (the NHWC flatten order)
  MaxPool    -inf padding
  softmax    on the head only, then the non-finite override (rows of non-finite patches = 0.5)

The patch z-normalisation is the one ``patch_stats_kernel`` computes: float64 sums in its lane order, mean and
population std rounded to float32; the network input is (x - mu) / sigma of those float32 values, taken exactly.

Next to every value the evaluator carries a bound E on the error a kernel may make, propagated layer by layer:

  GEMM layer      E_out = |W| . E_in + u . |W| . |x|      (u: unit error of the layer's engine, fp32 accumulation included)
  epilogue        affines scale E by |s|, ReLU and max-pooling pass it on, sigmoid by 1/4; plus U32 |y| for the
                  float32 epilogue itself (and the split-half store of the result)

``u`` is 2^-22 for the tensor-core split engines (both split every operand into 11 + 11 significant bits), 2^-24
for layers on the fp32 CUDA cores and 2^-22 for the first layer (its input is rounded to fp32 first).  The split's
subnormal range adds an absolute term: fp16 lo parts are subnormal below 2^-14, so a split value carries up to 2^-25
absolute error there.  The bound is a scale, not a proof: tests compare |got - ref| <= c . E with a constant c
calibrated on the unmodified kernels.
"""
from fractions import Fraction

import numpy as np
import torch
import torch.nn.functional as F

PATCH_H, PATCH_HOP = 68, 2
PATCH_LFILL = PATCH_H // (2 * PATCH_HOP)

LAYER_CONV2D, LAYER_DENSE, LAYER_MAXPOOL = 1, 2, 3
F_BIAS, F_AFFINE_PRE, F_RELU, F_AFFINE_POST, F_SOFTMAX, F_SIGMOID = 1, 2, 4, 8, 16, 32

U_SPLIT = 2.0 ** -22       # engines 2 and 3: hi / lo split of both operands (the dropped lo . lo ~ 2^-22)
U32 = 2.0 ** -24           # fp32 CUDA cores
U_FIRST = 2.0 ** -22       # first layer: z rounded to fp32 before the products, taps accumulated in fp32 (a few U32)
ABS_SPLIT = 2.0 ** -25     # absolute error of an fp16 hi + lo pair whose lo part is subnormal


# ------------------------------------------------------------------ patches (patch_index_kernel + patch_stats_kernel)
def patch_rows(L, ranges, edge_left=True, edge_right=True):
    """First log-mel row of every requested padded patch index (patch_index_kernel)."""
    U = (L - PATCH_H) // PATCH_HOP + 1
    p = np.concatenate([np.arange(a, b) for a, b in ranges]).astype(np.int64)
    j = p - (PATCH_LFILL if edge_left else 0)
    j = np.maximum(j, 0)
    if edge_right:
        j = np.minimum(j, U - 1)
    return j * PATCH_HOP


def patch_stats(patches):
    """float32 (mu, sigma, finite) of [n, 68, w] float32 patches with the arithmetic of patch_stats_kernel: lane l of a
    warp sums the elements e = l, l + 32, ... (row-major) in float64, the lanes are combined by an xor tree, then
    mean = s1 / cnt, var = max(s2 / cnt - mean^2, 0) in float64 and both are rounded to float32."""
    n = patches.shape[0]
    v = patches.reshape(n, -1).astype(np.float64)
    cnt = v.shape[1]
    pad = (-cnt) % 32
    vp = np.concatenate((v, np.zeros((n, pad))), axis=1).reshape(n, -1, 32)
    s1 = np.zeros((n, 32))
    s2 = np.zeros((n, 32))
    for r in range(vp.shape[1]):                       # sequential per lane (padding adds exact zeros)
        s1 = s1 + vp[:, r]
        s2 = s2 + vp[:, r] * vp[:, r]                  # exact: a float32 squared fits in a float64
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        s1 = s1 + s1[:, lanes ^ o]
        s2 = s2 + s2[:, lanes ^ o]
    s1, s2 = s1[:, 0], s2[:, 0]
    m = s1 / cnt
    # the kernel's variance is one fused multiply-add, fma(-m, m, s2 / cnt): evaluated exactly, rounded once
    var = np.array([float(Fraction(q) - Fraction(a) * Fraction(a)) if np.isfinite(q) and np.isfinite(a) else q - a * a
                    for q, a in zip(s2 / cnt, m)])
    var = np.maximum(var, 0.0)
    with np.errstate(invalid='ignore', over='ignore'):
        mu, sg = m.astype(np.float32), np.sqrt(var).astype(np.float32)
    finite = np.isfinite(mu) & np.isfinite(sg) & (sg > 0)
    return mu, sg, finite


def patch_inputs(mspec, nmel, ranges, edge_left=True, edge_right=True):
    """Network input of the requested patches: z = (x - mu) / sigma in float64 of the float32 x, mu, sigma
    ([n, 68, nmel, 1]), and the finite mask (False: the row is overridden with 0.5)."""
    mspec = np.asarray(mspec, dtype=np.float32)
    rows = patch_rows(len(mspec), ranges, edge_left, edge_right)
    idx = rows[:, None] + np.arange(PATCH_H)[None, :]
    x = mspec[idx][:, :, :nmel]                        # [n, 68, nmel]
    mu, sg, finite = patch_stats(x)
    with np.errstate(invalid='ignore', divide='ignore'):
        z = (x.astype(np.float64) - mu.astype(np.float64)[:, None, None]) / sg.astype(np.float64)[:, None, None]
    z[~finite] = 0.0                                   # overridden rows: any finite stand-in
    return z[..., None], finite


# ------------------------------------------------------------------ layers
def _engine_u(d, li, in_shape, mode):
    """Unit error of the engine a layer runs on (the dispatch of cnn.cu / conv_gemm.cu, by shape)."""
    if li == 0:
        return U_FIRST
    if d['kind'] == LAYER_MAXPOOL or mode == 0 or d['flags'] & F_SIGMOID:
        return U32                                     # only the fp32 kernels evaluate a sigmoid
    cin = d['cin']
    K = cin if d['kind'] == LAYER_DENSE else d['kh'] * d['kw'] * cin
    N = d['cout']
    small_n = d['kind'] == LAYER_DENSE or (d['kh'] == 1 and d['kw'] == 1 and d['sh'] == 1 and d['sw'] == 1 and
                                           d['pad_top'] == 0 and d['pad_left'] == 0)
    if small_n and N <= 8 and K % 4 == 0 and K * N * 4 <= 48 * 1024:
        return U32                                     # dense_small_n_kernel
    if cin % 32 == 0 and K % 32 == 0 and N % 32 == 0:
        return U_SPLIT
    return U32


def _epilogue(d, blob, y, E):
    """bias -> pre-affine -> ReLU -> sigmoid -> post-affine on the last axis, with the bound."""
    f = d['flags']
    C = d['cout']

    def par(off):
        return blob[off:off + C].astype(np.float64)

    if f & F_BIAS:
        y = y + par(d['bias_off'])
    if f & F_AFFINE_PRE:
        s = par(d['pre_scale_off'])
        y = y * s + par(d['pre_shift_off'])
        E = E * np.abs(s)
    if f & F_RELU:
        y = np.where(np.isnan(y), y, np.maximum(y, 0.0))
    if f & F_SIGMOID:
        y = 1.0 / (1.0 + np.exp(-y))
        E = E * 0.25
    if f & F_AFFINE_POST:
        s = par(d['post_scale_off'])
        y = y * s + par(d['post_shift_off'])
        E = E * np.abs(s)
    return y, E + 4 * U32 * np.abs(y)


def _conv(x, w, d):
    """x [n, H, W, C] float64 (numpy) -> conv with the desc's pads / strides -> [n, OH, OW, N] (numpy)."""
    t = torch.from_numpy(np.ascontiguousarray(x)).permute(0, 3, 1, 2)
    t = F.pad(t, (d['pad_left'], d['pad_right'], d['pad_top'], d['pad_bottom']))
    k = torch.from_numpy(np.ascontiguousarray(w)).permute(3, 2, 0, 1)
    with torch.no_grad():
        y = F.conv2d(t, k, stride=(d['sh'], d['sw']))
    return y.permute(0, 2, 3, 1).contiguous().numpy()


def _maxpool(x, d):
    t = torch.from_numpy(np.ascontiguousarray(x)).permute(0, 3, 1, 2)
    t = F.pad(t, (d['pad_left'], d['pad_right'], d['pad_top'], d['pad_bottom']), value=float('-inf'))
    with torch.no_grad():
        y = F.max_pool2d(t, (d['kh'], d['kw']), stride=(d['sh'], d['sw']))
    return y.permute(0, 2, 3, 1).contiguous().numpy()


def eval_layers(lowered, x, E=None, mode=3, start=0, stop=None):
    """Layers [start, stop) of a LoweredModel on x (float64: [n, H, W, C], or [n, K] after a Dense) with bound E
    (zeros when None).  mode: the GEMM engine (0 = fp32 CUDA cores, 2 / 3 = the split engines).  Returns (y, E) as
    float64 numpy arrays, NHWC or [n, K]; the head's softmax, if any, is applied to y (E is left as the logits')."""
    descs, blob = lowered.descs, np.asarray(lowered.blob, dtype=np.float32)
    stop = len(descs) if stop is None else stop
    x = np.asarray(x, dtype=np.float64)
    E = np.zeros_like(x) if E is None else np.asarray(E, dtype=np.float64)
    for li in range(start, stop):
        d = descs[li]
        if d['kind'] == LAYER_MAXPOOL:
            x, E = _maxpool(x, d), _maxpool(E, d)      # max |a_i - b_i| bounds |max a - max b|
            continue
        u = _engine_u(d, li, x.shape, mode)
        K = d['cin'] if d['kind'] == LAYER_DENSE else d['kh'] * d['kw'] * d['cin']
        w = blob[d['w_off']:d['w_off'] + K * d['cout']].astype(np.float64)
        slack = E + u * np.abs(x) + (ABS_SPLIT if u == U_SPLIT else 0.0)
        if d['kind'] == LAYER_DENSE:
            x2, s2 = x.reshape(len(x), -1), slack.reshape(len(x), -1)
            w = w.reshape(d['cin'], d['cout'])
            y, E = x2 @ w, s2 @ np.abs(w)
        else:
            w = w.reshape(d['kh'], d['kw'], d['cin'], d['cout'])
            y, E = _conv(x, w, d), _conv(slack, np.abs(w), d)
        x, E = _epilogue(d, blob, y, E)
        if d['flags'] & F_SOFTMAX:
            z = x - x.max(axis=1, keepdims=True)
            x = np.exp(z) / np.exp(z).sum(axis=1, keepdims=True)
    return x, E


def evaluate(lowered, mspec, ranges, mode=3, edge_left=True, edge_right=True):
    """The network output of ``CnnModel.forward(mspec, ranges)`` in float64: (y [n, K], E [n, K]); rows of
    non-finite patches are 0.5 with E = 0."""
    z, finite = patch_inputs(mspec, lowered.in_w, ranges, edge_left, edge_right)
    y, E = eval_layers(lowered, z, mode=mode)
    y, E = y.reshape(len(y), -1), E.reshape(len(E), -1)
    y[~finite], E[~finite] = 0.5, 0.0
    return y, E
