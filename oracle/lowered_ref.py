"""Oracle (test infrastructure): float64 evaluation of a LOWERED CNN with a propagated error bound.

``cnn_oracle`` evaluates the Keras config; this module evaluates what the CUDA kernels are handed instead:
``LoweredModel.descs`` + ``blob`` (the ``iss_layer_desc`` semantics of csrc/cnn.cu), with the float32 parameters of
the blob -- so the folded BatchNorm is the one the kernels use:

  Conv2D     explicit pads / strides, then the epilogue bias -> pre-affine -> ReLU -> sigmoid -> post-affine
  Dense      the same epilogue on [n, cin] (the NHWC flatten order)
  MaxPool    -inf padding
  softmax    on the head only, then the non-finite override (rows of non-finite patches = 0.5, E = 0)

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

The head's softmax (softmax_head_kernel: max subtraction, expf, an fp32 sum over k = 0 .. K-1, one division) carries
the logits' bound to first order, p_k (E_k + sum_j p_j E_j), and adds its own rounding, relative to p_k: the rounded
z_k = l_k - max (U32 |z_k|, and the p-weighted mean of those in the sum), two expf of at most 2 ulp each (U_EXP), K - 1
fp32 additions and the division (U32 each), plus one subnormal ulp where an exponential underflows.

The MLP of VoiceFemininityScoring is the same Dense stack on the fp32 kernels: ``eval_layers(..., mode=0,
first=False)`` evaluates its lowered descs with u = U32 on every layer.

``kernel_names`` mirrors the dispatch (iss_conv_kernel, iss_prepare_weights, iss_slab_covers and plan_forward): the
CUDA kernels one forward of a lowered network launches in a GEMM mode.
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
U_EXP = 2.0 ** -22         # expf without fast-math: at most 2 ulp
ABS_EXP = 2.0 ** -149      # one subnormal ulp: an exponential (or a probability) that underflows


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
def _engine_u(d, li, in_shape, mode, first=True):
    """Unit error of the engine a layer runs on (the dispatch of cnn.cu / conv_gemm.cu, by shape).  first: layer 0
    is the CNN's first layer, which reads the z-normalised patch."""
    if li == 0 and first:
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


def softmax(logits, E=None):
    """Softmax over the last axis of float64 logits [n, K] with the bound of softmax_head_kernel: the logits' bound E
    (zeros when None) carried to first order plus the kernel's own rounding (module docstring).  Returns (p, E_p)."""
    lg = np.asarray(logits, dtype=np.float64)
    E = np.zeros_like(lg) if E is None else np.asarray(E, dtype=np.float64)
    z = lg - lg.max(axis=-1, keepdims=True)
    e = np.exp(z)
    p = e / e.sum(axis=-1, keepdims=True)
    K = lg.shape[-1]
    az = np.abs(z)
    rel = U32 * az + U32 * (p * az).sum(axis=-1, keepdims=True) + 2 * U_EXP + K * U32
    return p, p * (E + (p * E).sum(axis=-1, keepdims=True)) + p * rel + 2 * ABS_EXP


def eval_layers(lowered, x, E=None, mode=3, start=0, stop=None, first=True):
    """Layers [start, stop) of a LoweredModel on x (float64: [n, H, W, C], or [n, K] after a Dense) with bound E
    (zeros when None).  mode: the GEMM engine (0 = fp32 CUDA cores, 2 / 3 = the split engines).  first: layer 0 is the
    CNN's first layer (False for an MLP, whose layers all run on the fp32 kernels).  Returns (y, E) as float64 numpy
    arrays, NHWC or [n, K]; the head's softmax, if any, is applied to y and E."""
    descs, blob = lowered.descs, np.asarray(lowered.blob, dtype=np.float32)
    stop = len(descs) if stop is None else stop
    x = np.asarray(x, dtype=np.float64)
    E = np.zeros_like(x) if E is None else np.asarray(E, dtype=np.float64)
    for li in range(start, stop):
        d = descs[li]
        if d['kind'] == LAYER_MAXPOOL:
            x, E = _maxpool(x, d), _maxpool(E, d)      # max |a_i - b_i| bounds |max a - max b|
            continue
        u = _engine_u(d, li, x.shape, mode, first)
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
            x, E = softmax(x, E)
    return x, E


def evaluate(lowered, mspec, ranges, mode=3, edge_left=True, edge_right=True):
    """The network output of ``CnnModel.forward(mspec, ranges)`` in float64: (y [n, K], E [n, K]); rows of
    non-finite patches are 0.5 with E = 0."""
    z, finite = patch_inputs(mspec, lowered.in_w, ranges, edge_left, edge_right)
    y, E = eval_layers(lowered, z, mode=mode)
    y, E = y.reshape(len(y), -1), E.reshape(len(E), -1)
    y[~finite], E[~finite] = 0.5, 0.0
    return y, E


# ------------------------------------------------------------------ dispatch mirror (conv_gemm.cu, conv_gemm_tc.cu, cnn.cu)
K_F32, K_F32_FIRST, K_FIRST_DIRECT, K_SMALL_N, K_TF32, K_F16, K_SLAB = \
    'f32', 'f32_first', 'first_direct', 'small_n', 'tf32', 'f16', 'slab'
_SLAB_ROWS_MAX = (227 * 1024 - 1024 - 4 * 2 * 64 * 128) // 256      # one slab next to a four-stage weight ring


def _layer_args(lowered):
    """Per layer, the ConvArgs fields the dispatch reads (plan_forward's first loop), with the layer's shapes."""
    h, w, c = lowered.in_h, lowered.in_w, 1
    out = []
    for li, d in enumerate(lowered.descs):
        H, W, C = h, w, c
        if d['kind'] == LAYER_DENSE:
            h, w, c = 1, 1, d['cout']
            a = dict(K=d['cin'], C=d['cin'], H=1, W=1, OH=1, OW=1, KH=1, KW=1, SH=1, SW=1, PT=0, PL=0)
        else:
            h = (H + d['pad_top'] + d['pad_bottom'] - d['kh']) // d['sh'] + 1
            w = (W + d['pad_left'] + d['pad_right'] - d['kw']) // d['sw'] + 1
            c = d['cout'] if d['kind'] == LAYER_CONV2D else C
            a = dict(K=d['kh'] * d['kw'] * C, C=C, H=H, W=W, OH=h, OW=w, KH=d['kh'], KW=d['kw'], SH=d['sh'], SW=d['sw'],
                     PT=d['pad_top'], PL=d['pad_left'])
        # iss_prepare_weights: engine 2's image for C, K, N multiples of 32, engine 3's also with C, N multiples of 64
        tiled = li > 0 and d['kind'] != LAYER_MAXPOOL and a['C'] % 32 == 0 and a['K'] % 32 == 0 and d['cout'] % 32 == 0
        a.update(d=d, li=li, N=c, flags=d['flags'] & ~F_SOFTMAX, tiled=tiled,
                 f16=tiled and a['C'] % 64 == 0 and c % 64 == 0, in_packed=False, out_packed=False, pool_h=0, pool_w=0,
                 first=False)
        out.append(a)
    return out


def conv_kernel(a, mode):
    """iss_conv_kernel (conv_gemm.cu) for the fields of ``_layer_args``."""
    if a['li'] == 0:
        return K_FIRST_DIRECT if a['C'] == 1 and a['N'] in (16, 32, 64, 128) else K_F32_FIRST
    if (a['KH'] == 1 and a['KW'] == 1 and a['SH'] == 1 and a['SW'] == 1 and a['PT'] == 0 and a['PL'] == 0 and
            a['N'] <= 8 and a['K'] % 4 == 0 and a['K'] == a['C'] and a['K'] * a['N'] * 4 <= 48 * 1024 and
            not a['in_packed'] and not a['out_packed']):
        return K_SMALL_N
    if mode == 0 or not a['tiled'] or a['flags'] & F_SIGMOID:
        return K_F32
    if mode == 3 and a['f16']:
        slab = (a['C'] == 64 and a['N'] == 64 and a['K'] == a['KH'] * a['KW'] * a['C'] and a['pool_h'] == 0 and
                a['SH'] == 1 and a['SW'] == 1 and a['PT'] == 0 and a['PL'] == 0 and a['OH'] == a['H'] - a['KH'] + 1 and
                a['OW'] == a['W'] - a['KW'] + 1 and (256 + (a['KH'] - 1) * a['W'] + a['KW'] - 1 + 7) // 8 * 8 <= _SLAB_ROWS_MAX)
        pool_ok = a['pool_h'] == 0 or (not a['first'] and a['in_packed'] and a['pool_h'] // 2 == a['H'] and
                                       a['pool_w'] // 2 == a['W'])
        if pool_ok and (not a['first'] or slab):
            return K_SLAB if slab else K_F16
    return K_TF32


def _is_f16(k):
    return k in (K_F16, K_SLAB)


def _kernel_name(a, k):
    N = a['N']
    if k == K_FIRST_DIRECT:
        return 'conv_first_direct_kernel'
    if k in (K_F32, K_F32_FIRST):
        return 'conv_gemm_f32_kernel<%d,%s>' % (64 if N <= 64 else 128, 'true' if k == K_F32_FIRST else 'false')
    if k == K_SMALL_N:
        return 'dense_small_n_kernel'
    if k == K_SLAB:
        return 'conv_slab_kernel<%d>' % (3 if a['first'] else int(a['in_packed']))
    if k == K_F16:
        return 'conv_gemm_wg_kernel<1,%d,%d>' % (128 if N % 128 == 0 else 64, 2 if a['pool_h'] else int(a['in_packed']))
    return 'conv_gemm_wg_kernel<0,%d,0>' % (128 if N % 128 == 0 else 64 if N % 64 == 0 else 32)


def plan(lowered, mode, fuse_first=True, fuse_pool=True):
    """plan_forward (cnn.cu): per layer (kernel name, or None for a pooling folded into the next convolution or a
    first layer folded into the second), for a batch whose patches span few enough frames for the fused first layer's
    map (contiguous ascending ranges of up to 8192 patches).  fuse_first / fuse_pool: ISS_B200_FUSE_FIRST /
    ISS_B200_FUSE_POOL not '0'."""
    args = _layer_args(lowered)
    n = len(args)

    def reads_packed(j):
        return _is_f16(conv_kernel(dict(args[j], in_packed=True), mode))

    names = [None] * n
    packed, pool_h, pool_w, first_fused = False, 0, 0, False
    for li, a in enumerate(args):
        d = a['d']
        if d['kind'] == LAYER_MAXPOOL:
            nx = args[li + 1]['d'] if li + 1 < n else None
            if (packed and fuse_pool and nx is not None and (d['kh'], d['kw'], d['sh'], d['sw']) == (2, 2, 2, 2) and
                    d['pad_top'] == d['pad_left'] == d['pad_bottom'] == d['pad_right'] == 0 and
                    nx['kind'] == LAYER_CONV2D and nx['pad_bottom'] == 0 and nx['pad_right'] == 0 and
                    _is_f16(conv_kernel(dict(args[li + 1], in_packed=True, pool_h=a['H'], pool_w=a['W']), mode))):
                pool_h, pool_w = a['H'], a['W']
                continue
            names[li] = 'maxpool_nhwc_kernel<%s>' % ('uint4' if packed else 'float4' if a['C'] % 4 == 0 else 'float')
            continue
        a.update(in_packed=packed, pool_h=pool_h, pool_w=pool_w)
        pool_h = pool_w = 0
        j = li + 1
        while j < n and args[j]['d']['kind'] == LAYER_MAXPOOL:
            j += 1
        pools_vec4 = all(args[p]['C'] % 4 == 0 for p in range(li + 1, j))
        a['out_packed'] = j < n and pools_vec4 and reads_packed(j) and \
            (_is_f16(conv_kernel(a, mode)) or conv_kernel(a, mode) == K_FIRST_DIRECT)
        if li == 0:
            d1 = args[1]['d'] if n > 1 else None
            first_fused = (a['out_packed'] and fuse_first and d['sh'] == 1 and d['sw'] == 1 and
                           d['pad_top'] == d['pad_left'] == d['pad_bottom'] == d['pad_right'] == 0 and
                           not d['flags'] & F_SIGMOID and d1['kind'] == LAYER_CONV2D and d1['pad_bottom'] == 0 and
                           d1['pad_right'] == 0 and _is_f16(conv_kernel(dict(args[1], in_packed=True, first=True), mode)))
            if first_fused:
                continue
        if li == 1 and first_fused:
            a['first'] = True
        names[li] = _kernel_name(a, conv_kernel(a, mode))
        packed = a['out_packed']
    return names


def kernel_names(lowered, mode, fuse_first=True, fuse_pool=True):
    """Names (as the profiler shows them, white space removed) of the CUDA kernels one CnnModel.forward launches."""
    names = {'patch_index_kernel', 'patch_stats_kernel', 'softmax_head_kernel'}
    p = plan(lowered, mode, fuse_first, fuse_pool)
    if p[0] is None:
        names |= {'first_linear_kernel', 'first_coef_kernel'}
    return names | {k for k in p if k is not None}
