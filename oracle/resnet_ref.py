"""Oracle (test infrastructure): float64 evaluation of the ResNet x-vector extractor with a propagated error bound.

``vbx_oracle.ResNet101Oracle`` evaluates a state_dict in fp32; this module evaluates what ``iss_resnet_create`` is
handed instead: the blob in the layout of ``build_plan`` (csrc/resnet.cu), with its float32 folded BatchNorm scale and
shift as parameters, on windows gathered as ``window_gather_kernel`` does (x[f][t] = fea[start + t][f]):

  stem         3x3 conv, padding 1 -> scale / shift -> ReLU
  block        c1 (1x1) -> c2 (3x3, stride s, padding 1) -> c3 (1x1) + residual -> ReLU; the residual is the block
               input or the 1x1 stride-s shortcut convolution (scale / shift, no ReLU)
  stat pool    mean over time, sqrt(E[x^2] - E[x]^2 + 1e-10), flattened c * H + h (means, then stds)
  embedding    [2 C H] @ W + bias

Next to every value it carries a bound E on the error a kernel may make, with the rules of ``lowered_ref``:

  GEMM + epilogue   E_out = (sqrt(|W|^2 . E_in^2) + |W| . (u |x| + abs)) . |s| + 4 U32 |y|; a residual adds its E
                    and U_SPLIT |y| for every tensor resnet.cu stores as split-half words
  stat pool         the fp32 one-pass sums add ~ W U32 sum|v| and W U32 sum v^2; the std takes
                    min(E_var / (2 std), sqrt(E_var)), finite where the variance is ~0
  embedding         as a GEMM layer, plus U32 sqrt(n (p^2 . W^2)) for its fp32 accumulation over n non-zero weights

Over 104 layers the worst-case |W| . E of lowered_ref compounds to a useless bound (~1e110 on the release network), so
the error a layer receives is propagated as a root-sum-square (|W|^2 . E^2, and residual with branch) and ReLU drops
the bound where its input is certainly negative; the local rounding term |W| . u |x| stays worst-case.

``u`` (and ``abs``) belong to the kernel ``iss_conv_kernel`` picks for the layer in the GEMM mode (``conv_kernel``):
U32 for the fp32 and small-N kernels, U_SPLIT + ABS_SPLIT for engines 2 and 3.  The bound is a scale, not a proof: tests
compare |got - ref| <= c . E with a constant c calibrated on the unmodified kernels.

The arithmetic runs in torch float64 on any device (``device='cuda'`` for the full-size network)."""
from collections import namedtuple

import numpy as np
import torch
import torch.nn.functional as F

from .lowered_ref import ABS_SPLIT, U32, U_SPLIT

STRIDES = (1, 2, 2, 2)
RELEASE = dict(m=32, feat_dim=64, embed_dim=256, num_blocks=(3, 4, 23, 3))

# kernels of iss_conv_kernel (conv_gemm.cuh) a ResNet layer can run on
K_F32, K_SMALL_N, K_TF32, K_F16, K_SLAB = 'f32', 'small_n', 'tf32', 'f16', 'slab'

Arch = namedtuple('Arch', 'm feat_dim embed_dim num_blocks stem blocks emb blob_len')


def out_dim(x, k, s, p):
    return (x + 2 * p - k) // s + 1


def plan(m, feat_dim, embed_dim, num_blocks):
    """The architecture walk of build_plan (resnet.cu): every convolution with its blob offsets (weights
    [kh][kw][cin][cout], then scale[cout], shift[cout]); blocks in order c1, c2, c3, shortcut; then the embedding
    [2 C H][embed] and its bias."""
    off = 0

    def mk(k, stride, pad, cin, cout, images='f16'):
        nonlocal off
        c = dict(k=k, stride=stride, pad=pad, cin=cin, cout=cout, images=images, w_off=off)
        off += k * k * cin * cout
        c['scale_off'] = off
        off += cout
        c['shift_off'] = off
        off += cout
        return c

    stem = mk(3, 1, 1, 1, m, images=None)             # the stem gets no tensor-core images
    blocks, inp, h = [], m, feat_dim
    for li in range(4):
        planes = m << li
        for b in range(num_blocks[li]):
            s = STRIDES[li] if b == 0 else 1
            blk = dict(name='layer%d.%d' % (li + 1, b), c1=mk(1, 1, 0, inp, planes), c2=mk(3, s, 1, planes, planes),
                       c3=mk(1, 1, 0, planes, 4 * planes))
            blk['sc'] = mk(1, s, 0, inp, 4 * planes) if (s != 1 or inp != 4 * planes) else None
            blocks.append(blk)
            inp = 4 * planes
            h = out_dim(h, 3, s, 1)
    K = 2 * inp * h
    emb = dict(k=1, stride=1, pad=0, cin=K, cout=embed_dim, images='tiled', w_off=off, c_final=inp, h_final=h)
    off += K * embed_dim
    emb['b_off'] = off
    off += embed_dim
    return Arch(m, feat_dim, embed_dim, tuple(num_blocks), stem, blocks, emb, off)


def conv_kernel(c, mode, residual=False):
    """The kernel iss_conv_kernel picks for a ResNet convolution c (a ``plan`` entry) in GEMM mode 0 / 2 / 3.

      small-N   1x1 stride-1 unpadded, N <= 8, K % 4 == 0, K N 4 bytes <= 48 KiB, no residual (any mode)
      fp32      mode 0; the stem (no tensor-core images); C, K or N not a multiple of 32
      engine 3  mode 3 with an fp16 image: C and N multiples of 64 (the slab kernel for 1x1 64 -> 64)
      engine 2  every other layer: C, K and N multiples of 32 (the embedding in modes 2 and 3)"""
    k, cin, cout = c['k'], c['cin'], c['cout']
    K = k * k * cin
    unit = k == 1 and c['stride'] == 1 and c['pad'] == 0
    if unit and cout <= 8 and K % 4 == 0 and K * cout * 4 <= 48 * 1024 and not residual:
        return K_SMALL_N
    if mode == 0 or c['images'] is None or cin % 32 or K % 32 or cout % 32:
        return K_F32
    if mode == 3 and c['images'] == 'f16' and cin % 64 == 0 and cout % 64 == 0:
        return K_SLAB if unit and cin == 64 and cout == 64 else K_F16
    return K_TF32


def unit_error(kernel):
    return U_SPLIT if kernel in (K_TF32, K_F16, K_SLAB) else U32


def is_f16(c, mode):
    return conv_kernel(c, mode) in (K_F16, K_SLAB)


def packed_formats(arch, mode):
    """Per block: which tensors resnet.cu stores as split-half words (a: c1 -> c2, b: c2 -> c3, s: shortcut, y: the
    block output), as in iss_resnet_embed."""
    out = []
    for i, b in enumerate(arch.blocks):
        f = dict(a=is_f16(b['c1'], mode) and is_f16(b['c2'], mode), b=is_f16(b['c2'], mode) and is_f16(b['c3'], mode),
                 s=b['sc'] is not None and is_f16(b['sc'], mode) and is_f16(b['c3'], mode), y=False)
        if i + 1 < len(arch.blocks):
            nx = arch.blocks[i + 1]
            f['y'] = (is_f16(b['c3'], mode) and is_f16(nx['c1'], mode) and is_f16(nx['c3'], mode) and
                      (nx['sc'] is None or is_f16(nx['sc'], mode)))
        out.append(f)
    return out


def kernel_names(arch, mode):
    """Names (as the profiler shows them, white space removed) of the CUDA kernels one iss_resnet_embed launches."""
    names = {'window_gather_kernel', 'stat_pool_kernel'}

    def name(c, kern, in_packed):
        if kern == K_F32:
            return 'conv_gemm_f32_kernel<%d,false>' % (64 if c['cout'] <= 64 else 128)
        if kern == K_SMALL_N:
            return 'dense_small_n_kernel'
        if kern == K_SLAB:
            return 'conv_slab_kernel<%d>' % int(in_packed)
        if kern == K_F16:
            return 'conv_gemm_wg_kernel<1,%d,%d>' % (128 if c['cout'] % 128 == 0 else 64, int(in_packed))
        bn = 128 if c['cout'] % 128 == 0 else (64 if c['cout'] % 64 == 0 else 32)
        return 'conv_gemm_wg_kernel<0,%d,0>' % bn

    names.add(name(arch.stem, conv_kernel(arch.stem, mode), False))
    x_packed = False
    for b, f in zip(arch.blocks, packed_formats(arch, mode)):
        names.add(name(b['c1'], conv_kernel(b['c1'], mode), x_packed))
        names.add(name(b['c2'], conv_kernel(b['c2'], mode), f['a']))
        if b['sc'] is not None:
            names.add(name(b['sc'], conv_kernel(b['sc'], mode), x_packed))
        names.add(name(b['c3'], conv_kernel(b['c3'], mode, residual=True), f['b']))
        x_packed = f['y']
    names.add(name(arch.emb, conv_kernel(arch.emb, mode), False))
    return names


# ------------------------------------------------------------------ evaluation
def gather(fea, starts, win_len):
    """window_gather_kernel: [n, feat_dim, win_len] float64, x[w][f][t] = fea[starts[w] + t][f]."""
    fea = np.asarray(fea, dtype=np.float32)
    return np.stack([fea[s:s + win_len].T for s in starts]).astype(np.float64)


def _conv(arch_blob, x, E, c, mode, relu, out_packed, residual=None):
    kern = conv_kernel(c, mode, residual=residual is not None)
    u = unit_error(kern)
    k, cin, cout = c['k'], c['cin'], c['cout']
    w = arch_blob[c['w_off']:c['w_off'] + k * k * cin * cout].view(k, k, cin, cout).permute(3, 2, 0, 1)
    s = arch_blob[c['scale_off']:c['scale_off'] + cout].view(1, -1, 1, 1)
    t = arch_blob[c['shift_off']:c['shift_off'] + cout].view(1, -1, 1, 1)
    local = u * x.abs() + (ABS_SPLIT if u == U_SPLIT else 0.0)
    y = F.conv2d(x, w, stride=c['stride'], padding=c['pad']) * s + t
    E = (torch.sqrt(F.conv2d(E * E, w * w, stride=c['stride'], padding=c['pad'])) +
         F.conv2d(local, w.abs(), stride=c['stride'], padding=c['pad'])) * s.abs()
    if residual is not None:
        y, E = y + residual[0], torch.sqrt(E * E + residual[1] * residual[1])
    if relu:                                          # an input below -E gives exactly 0 on both sides
        E = (E - (-y).clamp_min(0.0)).clamp_min(0.0)
        y = torch.where(torch.isnan(y), y, y.clamp_min(0.0))
    E = E + 4 * U32 * y.abs()
    if out_packed:
        E = E + U_SPLIT * y.abs()
    return y, E


def stat_pool(x, E):
    """stat_pool_kernel on [n, C, H, W] with the bound of its fp32 one-pass sums: [n, 2 C H] (y, E)."""
    W = x.shape[-1]
    ax = x.abs()
    mean = x.mean(-1)
    msq = (x * x).mean(-1)
    E_mean = E.mean(-1) + W * U32 * ax.mean(-1) + U32 * mean.abs()
    var = (msq - mean * mean).clamp_min(0.0)
    # propagated: d var = 2 mean_t((x - mean) dx); rounded: the two sums, the division and msq - mean^2 in fp32
    E_var = (2 * (x - mean.unsqueeze(-1)).abs() * E + E * E).mean(-1) + (W + 2) * U32 * (msq + mean * mean)
    std = torch.sqrt(var + 1e-10)
    E_std = torch.minimum(E_var / (2 * std), torch.sqrt(E_var)) + U32 * std
    n = x.shape[0]
    return (torch.cat((mean.reshape(n, -1), std.reshape(n, -1)), 1),
            torch.cat((E_mean.reshape(n, -1), E_std.reshape(n, -1)), 1))


def forward(arch, blob, x, mode=3, device='cpu', pooled=False):
    """The network on x ([n, feat_dim, T], float64) in float64: (y [n, embed_dim], E [n, embed_dim]) as numpy; with
    pooled, also the stat-pooling output and its bound."""
    bl = torch.as_tensor(np.asarray(blob, dtype=np.float32), device=device).to(torch.float64)
    x = torch.as_tensor(np.asarray(x, dtype=np.float64), device=device).unsqueeze(1)
    E = torch.zeros_like(x)
    with torch.no_grad():
        x, E = _conv(bl, x, E, arch.stem, mode, relu=True, out_packed=False)
        for b, f in zip(arch.blocks, packed_formats(arch, mode)):
            a, Ea = _conv(bl, x, E, b['c1'], mode, relu=True, out_packed=f['a'])
            a, Ea = _conv(bl, a, Ea, b['c2'], mode, relu=True, out_packed=f['b'])
            res = (x, E) if b['sc'] is None else _conv(bl, x, E, b['sc'], mode, relu=False, out_packed=f['s'])
            x, E = _conv(bl, a, Ea, b['c3'], mode, relu=True, out_packed=f['y'], residual=res)
        p, Ep = stat_pool(x, E)
        e = arch.emb
        u = unit_error(conv_kernel(e, mode))
        w = bl[e['w_off']:e['w_off'] + e['cin'] * e['cout']].view(e['cin'], e['cout'])
        y = p @ w + bl[e['b_off']:e['b_off'] + e['cout']]
        # the embedding's fp32 accumulation runs over up to K = 2 C H = 16384 terms (10x the convolutions' K): n
        # roundings of partial sums that wander as sqrt(k) rms(p w), n counted per column over the non-zero weights
        n = (w != 0).sum(0).to(torch.float64)
        acc = U32 * torch.sqrt(n * ((p * p) @ (w * w)))
        Ey = (torch.sqrt((Ep * Ep) @ (w * w)) + (u * p.abs() + (ABS_SPLIT if u == U_SPLIT else 0.0)) @ w.abs() +
              acc + 4 * U32 * y.abs())
    out = (y.cpu().numpy(), Ey.cpu().numpy())
    return out + (p.cpu().numpy(), Ep.cpu().numpy()) if pooled else out


def evaluate(arch, blob, fea, starts, win_len, mode=3, device='cpu'):
    """iss_resnet_embed(fea, starts, win_len) in float64: (y, E) [n, embed_dim] numpy."""
    return forward(arch, blob, gather(fea, starts, win_len), mode, device)


# ------------------------------------------------------------------ seeded networks
def synthetic_blob(arch, seed=0, heads=None, bias=None):
    """A seeded blob for ``arch``: He-scaled weights, folded BatchNorm scale in [0.8, 1.2] (x 0.3 on every c3, as
    vbx_oracle.synthetic_resnet101_state keeps residual streams well scaled) and shift ~ N(0, 0.1).  ``heads``
    ([2 C H, embed_dim]) sets the embedding weight columns; ``bias`` its bias (zeros when None)."""
    rng = np.random.default_rng(seed)
    blob = np.zeros(arch.blob_len, dtype=np.float32)

    def fill(c, gain=1.0):
        k, cin, cout = c['k'], c['cin'], c['cout']
        n = k * k * cin * cout
        blob[c['w_off']:c['w_off'] + n] = rng.standard_normal(n) * np.sqrt(2.0 / (k * k * cin))
        blob[c['scale_off']:c['scale_off'] + cout] = rng.uniform(0.8, 1.2, cout) * gain
        blob[c['shift_off']:c['shift_off'] + cout] = rng.normal(0, 0.1, cout)

    fill(arch.stem)
    for b in arch.blocks:
        fill(b['c1'])
        fill(b['c2'])
        fill(b['c3'], 0.3)
        if b['sc'] is not None:
            fill(b['sc'])
    e = arch.emb
    if heads is None:
        heads = rng.standard_normal((e['cin'], e['cout'])) * np.sqrt(1.0 / e['cin'])
    assert heads.shape == (e['cin'], e['cout'])
    blob[e['w_off']:e['w_off'] + e['cin'] * e['cout']] = np.asarray(heads, dtype=np.float32).ravel()
    if bias is not None:
        blob[e['b_off']:e['b_off'] + e['cout']] = bias
    return blob


def layer(arch, name):
    """The ``plan`` entry of 'stem', 'emb' or '<block name>.c1|c2|c3|sc' (e.g. 'layer2.0.c3')."""
    if name in ('stem', 'emb'):
        return arch.stem if name == 'stem' else arch.emb
    blk, conv = name.rsplit('.', 1)
    return next(b for b in arch.blocks if b['name'] == blk)[conv]
