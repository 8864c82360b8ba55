"""Probe networks: one convolution path of the CNN operator at a time, in a short Keras-style Sequential that ends in
Flatten -> Dense(8, linear, no bias) with no softmax, so the operator returns 8 linear functionals of the probed
layer's whole output per patch (softmax_head_kernel copies a head without softmax verbatim).  A Dense head of 8 units
is not tensor-core eligible: it runs on the fp32 CUDA cores, and a one-hot ("selector") column reads one element of
the layer's output exactly.

Shared by tests/test_lowered_ref.py (the float64 reference against cnn_oracle on the CPU) and
tests/test_layer_probes_gpu.py (the kernels against the float64 reference)."""
import numpy as np

from inaspeechsegmenter_b200 import models


def _out(size, k, s, padding):
    return -(-size // s) if padding == 'same' else (size - k) // s + 1


class ProbeNet:
    """A Sequential under construction; ``shape`` is the current (H, W, C) or (K,) after a Dense."""

    def __init__(self, nmel, seed=0):
        self.nmel, self.rng = nmel, np.random.default_rng(seed)
        self.layers = [{'class_name': 'InputLayer', 'config': {'name': 'in', 'batch_input_shape': [None, 68, nmel, 1]}}]
        self.weights = {}
        self.shape = (68, nmel, 1)
        self.n = 0

    def _name(self, prefix):
        self.n += 1
        return '%s_%d' % (prefix, self.n)

    def bn(self, ch, spread=1.0):
        name = self._name('bn')
        r = self.rng
        self.weights[name + '/gamma'] = r.uniform(0.8, 1.2, ch).astype(np.float32) * np.float32(spread)
        self.weights[name + '/beta'] = r.normal(0, 0.1, ch).astype(np.float32)
        self.weights[name + '/moving_mean'] = r.normal(0, 0.2, ch).astype(np.float32)
        self.weights[name + '/moving_variance'] = r.uniform(0.5, 1.5, ch).astype(np.float32)
        self.layers.append({'class_name': 'BatchNormalization', 'config': {'name': name, 'axis': -1, 'epsilon': 1e-3}})

    def _epilogue(self, ch, pre, relu, post):
        if pre:
            self.bn(ch)
        if relu:
            self.layers.append({'class_name': 'Activation', 'config': {'name': self._name('act'), 'activation': 'relu'}})
        if post:
            self.bn(ch)

    def conv(self, cout, k=(3, 3), s=(1, 1), padding='valid', bias=True, pre=False, relu=False, post=False, gain=1.0,
             kernel=None, act='linear'):
        h, w, cin = self.shape
        name = self._name('conv')
        if kernel is None:
            kernel = self.rng.standard_normal((k[0], k[1], cin, cout)) * np.sqrt(2.0 / (k[0] * k[1] * cin)) * gain
        self.weights[name + '/kernel'] = np.asarray(kernel, dtype=np.float32)
        if bias:
            self.weights[name + '/bias'] = self.rng.normal(0, 0.05, cout).astype(np.float32)
        self.layers.append({'class_name': 'Conv2D', 'config': {
            'name': name, 'filters': cout, 'kernel_size': list(k), 'strides': list(s), 'padding': padding,
            'use_bias': bias, 'activation': act}})
        self._epilogue(cout, pre, relu, post)
        self.shape = (_out(h, k[0], s[0], padding), _out(w, k[1], s[1], padding), cout)
        return self

    def relay(self):
        """1x1 identity convolution without bias: on the fp16-split engine its weights scale to exactly 2^12 with a zero
        lo part, so its fp32 output is the split-half word it reads, decoded exactly."""
        c = self.shape[2]
        return self.conv(c, (1, 1), bias=False, kernel=np.eye(c, dtype=np.float32).reshape(1, 1, c, c))

    def widen(self, cout):
        """1x1 convolution without bias that repeats the C input channels up to cout (weights 0 / 1): a producer on the
        3xTF32 engine whose fp32 output carries almost no error of its own (2^-22 relative), so that an error of the
        layer behind it is not hidden under a loose input bound."""
        c = self.shape[2]
        return self.conv(cout, (1, 1), bias=False, kernel=(np.arange(cout)[None, :] % c == np.arange(c)[:, None])
                         .astype(np.float32).reshape(1, 1, c, cout))

    def pool(self, p=(2, 2), s=None, padding='valid'):
        s = s or p
        h, w, c = self.shape
        self.layers.append({'class_name': 'MaxPooling2D', 'config': {'name': self._name('pool'), 'pool_size': list(p),
                                                                     'strides': list(s), 'padding': padding}})
        self.shape = (_out(h, p[0], s[0], padding), _out(w, p[1], s[1], padding), c)
        return self

    def dense(self, units, pre=False, relu=False, post=False, act='linear'):
        if len(self.shape) == 3:
            self.layers.append({'class_name': 'Flatten', 'config': {'name': self._name('flat')}})
        cin = int(np.prod(self.shape))
        name = self._name('dense')
        self.weights[name + '/kernel'] = (self.rng.standard_normal((cin, units)) * np.sqrt(2.0 / cin)).astype(np.float32)
        self.weights[name + '/bias'] = self.rng.normal(0, 0.05, units).astype(np.float32)
        self.layers.append({'class_name': 'Dense', 'config': {'name': name, 'units': units, 'use_bias': True,
                                                              'activation': act}})
        self._epilogue(units, pre, relu, post)
        self.shape = (units,)
        return self

    @property
    def size(self):
        return int(np.prod(self.shape))

    def with_head(self, head):
        """(config, weights) of the body followed by Flatten -> Dense(8, linear, no bias) with kernel ``head`` [size, 8]."""
        layers = list(self.layers)
        if len(self.shape) == 3:
            layers.append({'class_name': 'Flatten', 'config': {'name': 'head_flat'}})
        layers.append({'class_name': 'Dense', 'config': {'name': 'head', 'units': 8, 'use_bias': False,
                                                         'activation': 'linear'}})
        weights = dict(self.weights)
        weights['head/kernel'] = np.asarray(head, dtype=np.float32)
        return {'class_name': 'Sequential', 'config': {'name': 'probe', 'layers': layers}}, weights

    def lowered(self, head):
        return models.lower_keras_model(*self.with_head(head), 68, self.nmel)


def random_head(size, seed):
    """Eight +-1 columns: every element of the layer's output enters every output."""
    return np.random.default_rng(seed).choice(np.float32([-1, 1]), (size, 8))


def selector_head(shape, picks):
    """One-hot columns on the elements ``picks`` ((oh, ow, c) of an (H, W, C) output, or (k,) of a flat one);
    negative coordinates count from the end."""
    head = np.zeros((int(np.prod(shape)), 8), np.float32)
    for j, p in enumerate(picks[:8]):
        coords = [int(v) % int(n) for v, n in zip(p, shape)]
        head[int(np.ravel_multi_index(coords, shape)), j] = 1.0
    return head


def default_picks(shape):
    """First and last output row / column / channel, the corners and the middle: with the batch offset of every
    patch these elements land on every slot position of a 256-slot tile and of a 128-row GEMM tile."""
    if len(shape) == 1:
        return [(0,), (-1,), (1,), (shape[0] // 2,), (-2,), (7,), (-8,), (shape[0] // 3,)]
    return [(0, 0, 0), (-1, -1, -1), (0, -1, -1), (-1, 0, 0), (shape[0] // 2, shape[1] // 2, -1),
            (-1, -1, 0), (1, 1, shape[2] // 2), (shape[0] // 3, -1, 7 % shape[2])]


def mspec_normal(L=1600, seed=0):
    return (np.random.default_rng(seed).standard_normal((L, 24)) * 3 - 5).astype(np.float32)


def mspec_low_variance(L=1600, seed=0):
    """Log-mel rows of mean -30 and std 1e-3: large |mean / std|, the first layer's bias and mean term cancel."""
    return (np.float32(-30) + np.random.default_rng(seed).standard_normal((L, 24)).astype(np.float32) * np.float32(1e-3))


# ------------------------------------------------------------------ the case matrix
# Each case: the network body, the GEMM engine, whether the first layer may be fused, the input, the patch ranges and
# the kernels one forward must launch (substrings of the demangled names).  Kernel template arguments:
# conv_slab_kernel<fill>, fill 0 = fp32 values split in the fill, 1 = split-half words, 3 = fused first layer;
# conv_gemm_wg_kernel<engine, BN, fill>, engine 0 = 3xTF32, 1 = fp16 split, fill 2 = words with the 2x2 pooling.
# 54 patches: many tiles and a partial last tile; the frames they span are few enough for the fused first layer's
# float64 map (a batch spread wider takes the stand-alone first layer)
RANGES = [(20, 60), (75, 89)]
SMALL = [(30, 46)]                              # 16 patches for the widest filters


def _first(nmel, k=(4, 5), seed=0, cout=64, **kw):
    return ProbeNet(nmel, seed).conv(cout, k, pre=True, relu=True, **kw)


EPILOGUES = [dict(pre=True, relu=True), dict(), dict(relu=True, post=True), dict(pre=True, relu=True, post=True),
             dict(bias=False, relu=True)]
SLAB_TAPS = [(1, 1), (2, 2), (3, 3), (5, 4), (4, 5), (7, 1), (1, 7)]
SLAB_FILL = {'first': 3, 'packed': 1, 'f32': 0}


def _slab_case(taps, fill, nmel, epi, relay=False, seed=0):
    if fill == 'f32':                            # producer on engine 2 (32 -> 64): the slab reads fp32 values
        net = _first(nmel, seed=seed, cout=32).widen(64)
    else:
        net = _first(nmel, seed=seed)
    net.conv(64, taps, **epi)
    if relay:
        net.relay()
    return dict(net=net, fuse=fill == 'first', kernels=['conv_slab_kernel<%d>' % SLAB_FILL[fill]])


def _cases():
    c = {}
    for i, taps in enumerate(SLAB_TAPS):
        for j, fill in enumerate(SLAB_FILL):
            nmel = (21, 24)[(i + j) % 2]
            c['slab_%s_%dx%d_w%d' % (fill, taps[0], taps[1], nmel)] = \
                lambda taps=taps, fill=fill, nmel=nmel, e=EPILOGUES[(i + j) % len(EPILOGUES)]: _slab_case(taps, fill, nmel, e)
    for fill in SLAB_FILL:
        c['slab_%s_5x4_relay' % fill] = lambda fill=fill: _slab_case((5, 4), fill, 21, EPILOGUES[3], relay=True)
    # OW = 1: a 2x17 filter on the 17-wide map of nmel 21
    c['slab_first_ow1'] = lambda: dict(net=_first(21).conv(64, (2, 17), pre=True, relu=True), fuse=True,
                                       kernels=['conv_slab_kernel<3>'])
    # the shared-memory boundary on a 24-wide map: 17x9 = 648 slab rows = 227 KB (slab), 17x10 = 656 rows (gather)
    c['slab_boundary_17x9'] = lambda: dict(net=_first(24, (3, 1)).conv(64, (17, 9), pre=True, relu=True), fuse=True,
                                           ranges=SMALL, kernels=['conv_slab_kernel<3>'])
    c['gather_boundary_17x10'] = lambda: dict(net=_first(24, (3, 1)).conv(64, (17, 10), pre=True, relu=True), fuse=True,
                                              ranges=SMALL, kernels=['conv_gemm_wg_kernel<1,64,1>'])
    # ---- gather kernel, engine 3
    c['g3_c64_n128'] = lambda: dict(net=_first(21).conv(128, (3, 3), pre=True, relu=True),
                                    kernels=['conv_gemm_wg_kernel<1,128,1>'])
    c['g3_c64_n256'] = lambda: dict(net=_first(24).conv(256, (3, 3), relu=True, post=True),
                                    kernels=['conv_gemm_wg_kernel<1,128,1>'])
    c['g3_c64_n64_same'] = lambda: dict(net=_first(21).conv(64, (3, 3), padding='same', pre=True, relu=True),
                                        kernels=['conv_gemm_wg_kernel<1,64,1>'])
    c['g3_c128_n192'] = lambda: dict(net=_first(21).conv(128, (3, 3), pre=True, relu=True).conv(192, (3, 3), pre=True, relu=True),
                                     kernels=['conv_gemm_wg_kernel<1,128,1>', 'conv_gemm_wg_kernel<1,64,1>'])
    c['g3_c192_n128_stride2_same'] = lambda: dict(
        net=_first(24).conv(192, (3, 3), relu=True).conv(128, (3, 3), (2, 2), 'same', pre=True, relu=True),
        kernels=['conv_gemm_wg_kernel<1,64,1>', 'conv_gemm_wg_kernel<1,128,1>'])
    c['g3_stride21_same_even'] = lambda: dict(net=_first(24, (3, 5)).conv(64, (4, 4), (2, 1), 'same', relu=True),
                                              kernels=['conv_gemm_wg_kernel<1,64,1>'])
    c['g3_pool_odd'] = lambda: dict(net=_first(21).conv(64, (3, 3), pre=True, relu=True).pool().conv(128, (3, 3), pre=True, relu=True),
                                    kernels=['conv_gemm_wg_kernel<1,128,2>'])
    c['g3_pool_even'] = lambda: dict(net=_first(24, (3, 5)).conv(64, (3, 3), pre=True, relu=True).pool().conv(64, (3, 3), relu=True),
                                     kernels=['conv_gemm_wg_kernel<1,64,2>'])
    c['g3_f32_input'] = lambda: dict(net=_first(21, cout=32).widen(64).conv(128, (3, 3), pre=True, relu=True),
                                     kernels=['conv_gemm_wg_kernel<0,64,0>', 'conv_gemm_wg_kernel<1,128,0>'])
    c['g3_dense_large_k'] = lambda: dict(net=_first(21).pool().dense(128, pre=True, relu=True),
                                         kernels=['conv_gemm_wg_kernel<1,128,1>'])
    c['g3_dense_chain'] = lambda: dict(net=_first(24, (3, 3)).conv(64, (3, 3), (2, 2), relu=True).dense(256, relu=True, post=True).dense(192),
                                       kernels=['conv_gemm_wg_kernel<1,128,1>', 'conv_gemm_wg_kernel<1,64,1>'])
    # ---- gather kernel, engine 2 (C % 64 != 0 or N % 64 != 0)
    c['g2_c32_n32'] = lambda: dict(net=_first(21, cout=32).conv(32, (3, 3), pre=True, relu=True),
                                   kernels=['conv_gemm_wg_kernel<0,32,0>'])
    c['g2_c32_n96_stride2_same'] = lambda: dict(net=_first(24, cout=32).conv(96, (3, 3), (2, 2), 'same', relu=True),
                                                kernels=['conv_gemm_wg_kernel<0,32,0>'])
    c['g2_c96_n160'] = lambda: dict(net=_first(21, cout=32).conv(96, (3, 3), relu=True).conv(160, (2, 3), (1, 2), 'same', pre=True, relu=True),
                                    kernels=['conv_gemm_wg_kernel<0,32,0>'])
    c['g2_mode2_c64_n128'] = lambda: dict(net=_first(21).conv(128, (3, 3), pre=True, relu=True), mode=2,
                                          kernels=['conv_gemm_wg_kernel<0,128,0>'])
    # ---- first layer
    for cout in (16, 32, 64, 128):
        c['first_direct_c%d_same_stride' % cout] = lambda cout=cout: dict(
            net=ProbeNet(21 if cout != 64 else 24).conv(cout, (3, 4), (2, 1) if cout % 32 else (1, 2), 'same', pre=True, relu=True),
            kernels=['conv_first_direct_kernel'])
    c['first_generic_c48'] = lambda: dict(net=ProbeNet(21).conv(48, (4, 5), relu=True, post=True),
                                          kernels=['conv_gemm_f32_kernel<64,true>'])
    for k in ((4, 5), (3, 3), (1, 1), (5, 1)):
        for name, epi in (('none', dict()), ('relu', dict(relu=True)), ('pre_relu', dict(pre=True, relu=True)),
                          ('pre_relu_post', dict(pre=True, relu=True, post=True))):
            c['first_fused_%dx%d_%s' % (k[0], k[1], name)] = lambda k=k, epi=epi: dict(
                net=ProbeNet(21).conv(64, k, **epi).conv(64, (3, 3), pre=True, relu=True), fuse=True,
                kernels=['conv_slab_kernel<3>'])
    for inp in ('lowvar', 'const'):
        c['first_fused_%s' % inp] = lambda inp=inp: dict(net=_first(21).conv(64, (5, 4), pre=True, relu=True), fuse=True,
                                                         mspec=inp, kernels=['conv_slab_kernel<3>'])
        c['first_direct_%s' % inp] = lambda inp=inp: dict(net=_first(21).conv(64, (5, 4), pre=True, relu=True), fuse=False,
                                                          mspec=inp, kernels=['conv_first_direct_kernel', 'conv_slab_kernel<1>'])
    # ---- max-pooling on split-half words, 'same' padding (-inf words at the border)
    c['pool_words_3x2_same'] = lambda: dict(
        net=_first(21).conv(64, (3, 3), pre=True, relu=True).pool((3, 2), (2, 2), 'same').conv(64, (3, 3), padding='same', pre=True, relu=True),
        kernels=['maxpool_nhwc_kernel<uint4>', 'conv_gemm_wg_kernel<1,64,1>'])
    # ---- max-pooling on fp32 values: four channels per thread ('same' padding, engine 2), and one (6 channels)
    c['pool_f32x4_3x2_same_mode2'] = lambda: dict(
        net=_first(21).conv(64, (3, 3), pre=True, relu=True).pool((3, 2), (2, 2), 'same').conv(64, (3, 3), padding='same', pre=True, relu=True),
        mode=2, kernels=['maxpool_nhwc_kernel<float4>', 'conv_gemm_wg_kernel<0,64,0>'])
    c['pool_f32_first_generic_c6'] = lambda: dict(net=ProbeNet(21).conv(6, (4, 5), relu=True).pool(),
                                                  kernels=['conv_gemm_f32_kernel<64,true>', 'maxpool_nhwc_kernel<float>'])
    # ---- sigmoid: layers whose shapes the tensor-core engines take still run on the fp32 kernels, which evaluate it
    c['sigmoid_conv_3x3_c64'] = lambda: dict(net=_first(21).conv(64, (3, 3), act='sigmoid'),
                                             kernels=['conv_first_direct_kernel', 'conv_gemm_f32_kernel<64,false>'])
    c['sigmoid_dense_128'] = lambda: dict(net=_first(21).pool().dense(128, act='sigmoid'),
                                          kernels=['conv_gemm_f32_kernel<128,false>'])
    return c


CASES = _cases()


def case(name):
    spec = dict(mode=3, fuse=True, mspec='normal', ranges=RANGES)
    spec.update(CASES[name]())
    return spec


def make_mspec(kind, L=1600, seed=0):
    if kind == 'lowvar':
        return mspec_low_variance(L, seed)
    m = mspec_normal(L, seed)
    if kind == 'const':                          # constant stretches: std 0 -> the 0.5 override; the rest normal
        m[400:560] = np.float32(-7.25)
        m[900:1000] = np.float32(0)
    return m


# ------------------------------------------------------------------ MLPs (the Dense stack of VoiceFemininityScoring)
def mlp_config(in_dim, layers, seed=0):
    """Keras-style Sequential (config, weights) of Dense layers; each entry of ``layers``: dict(units, bias=True,
    bn='none' | 'pre' (BatchNorm before the activation) | 'post' (after it), act='linear' | 'relu' | 'sigmoid')."""
    rng = np.random.default_rng(seed)
    L = [{'class_name': 'InputLayer', 'config': {'name': 'in', 'batch_input_shape': [None, in_dim]}}]
    W, cin = {}, in_dim
    for i, spec in enumerate(layers):
        units, bias, bn, act = spec['units'], spec.get('bias', True), spec.get('bn', 'none'), spec.get('act', 'linear')
        name = 'dense_%d' % i
        W[name + '/kernel'] = (rng.standard_normal((cin, units)) * np.sqrt(2.0 / cin)).astype(np.float32)
        if bias:
            W[name + '/bias'] = rng.normal(0, 0.1, units).astype(np.float32)
        L.append({'class_name': 'Dense', 'config': {'name': name, 'units': units, 'use_bias': bias,
                                                    'activation': 'linear' if bn == 'pre' else act}})
        if bn != 'none':
            b = 'bn_%d' % i
            W[b + '/gamma'] = rng.uniform(0.8, 1.2, units).astype(np.float32)
            W[b + '/beta'] = rng.normal(0, 0.1, units).astype(np.float32)
            W[b + '/moving_mean'] = rng.normal(0, 0.2, units).astype(np.float32)
            W[b + '/moving_variance'] = rng.uniform(0.5, 1.5, units).astype(np.float32)
            L.append({'class_name': 'BatchNormalization', 'config': {'name': b, 'axis': -1, 'epsilon': 1e-3}})
            if bn == 'pre' and act != 'linear':
                L.append({'class_name': 'Activation', 'config': {'name': 'act_%d' % i, 'activation': act}})
        cin = units
    return {'class_name': 'Sequential', 'config': {'name': 'mlp', 'layers': L}}, W


# 1 to 4 Dense layers over widths 256, 100, 37 and 1: bias and none, BatchNorm before and after the activation, linear /
# relu / sigmoid.  Which fp32 kernel a layer takes (conv_gemm.cu): dense_small_n_kernel for N <= 8 and K % 4 == 0, else
# conv_gemm_f32_kernel, with scalar A loads for K % 8 != 0 and scalar B loads / stores for N % 4 != 0.
MLP_CASES = {
    'd1_256_1_sigmoid': (256, [dict(units=1, act='sigmoid')]),
    'd2_256_100_1': (256, [dict(units=100, act='relu', bn='post'), dict(units=1, act='sigmoid')]),
    'd3_256_37_100_1': (256, [dict(units=37, bias=False, bn='pre', act='relu'), dict(units=100, act='relu', bn='post'),
                              dict(units=1, bias=False)]),
    'd4_256_100_37_8_1': (256, [dict(units=100, bn='pre', act='relu'), dict(units=37, act='sigmoid'),
                                dict(units=8, act='relu', bn='post'), dict(units=1, act='sigmoid')]),
    'd2_37_100_3': (37, [dict(units=100, act='relu'), dict(units=3, bias=False, bn='pre', act='sigmoid')]),
    'd2_100_37_1': (100, [dict(units=37, act='relu', bn='pre'), dict(units=1)]),
    'd3_256_256_128_1': (256, [dict(units=256, act='relu', bn='post'), dict(units=128, act='relu'),
                               dict(units=1, act='sigmoid')]),
}
