"""The fp32 CUDA-core kernels (conv_gemm_f32_kernel, dense_small_n_kernel), the softmax head (softmax_head_kernel) and
the femininity MLP (iss_mlp_forward) against the float64 reference of the lowered network (oracle/lowered_ref.py), on
the GPU, with the probe machinery of tests/test_layer_probes_gpu.py:

  mode matrix      every probe case of tests/layer_probes.py in GEMM mode 0 (fp32 CUDA cores everywhere) and mode 2
                   (3xTF32); mode 3 is the probe module's own
  fp32 edges       scalar A loads (C % 8 != 0), scalar B loads and stores (N % 4 != 0), two or more grid columns
                   (N > 128), a partial last k-tile (K % 16 != 0), 'same' padding with strides, filters with KH != KW,
                   M tails (M % 128 = 1, 127), the generic first layer, sigmoid layers the tensor-core engines would take
  heads            1, 2, 3 and 8 outputs with and without softmax, both sides of the small-N kernel's 48 KB weight limit
                   and of K % 4, logits past expf's range (the max subtraction matters), logits a few ulps apart, rows
                   of non-finite patches; the posteriors are compared against the softmax bound
  MLP              1 to 4 Dense layers through MlpModel and the C ABI, 1 to 40000 rows (past the small-N kernel's
                   grid-stride loop and past the tiles the GPU holds at once), a row alone against the same row in a
                   9000-row batch, an input view at an offset that is not a multiple of 16 bytes

Each output must satisfy |got - ref| <= C_BOUND . E (the constant of the probe module), and the kernels one forward
launches, read from a torch.profiler trace, must be exactly those the reference's mirror of the dispatch predicts
(lowered_ref.kernel_names).  With ISS_B200_REPORT_DIR set, the module writes fp32_paths_report.json there: the worst
err / E per case, mode and head, and the kernels seen."""
import ctypes
import json
import os

import numpy as np
import pytest

import layer_probes as lp
import test_layer_probes_gpu as tp

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')

REPORT = {}


@pytest.fixture(scope='module')
def rt():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from inaspeechsegmenter_b200 import _lib, engine
    return dict(ctx=engine.Context(0), lib=_lib, engine=engine)


@pytest.fixture(scope='module', autouse=True)
def _dump_report():
    yield
    out = os.environ.get('ISS_B200_REPORT_DIR')
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, 'fp32_paths_report.json'), 'w') as f:
            json.dump(REPORT, f, indent=1, sort_keys=True)


def _assert_kernels(rt, low, spec, dm, names):
    """The project kernels of the trace `names` are exactly the ones lowered_ref.kernel_names predicts (two more traced
    forwards when a record is missing: the activity trace may drop one).  Returns the predicted names."""
    from oracle import lowered_ref as lr
    want = sorted(lr.kernel_names(low, spec['mode'], spec['fuse']))
    if not isinstance(names, list):
        return want                                  # the profiler recorded no CUDA kernels
    seen = set(names)

    def missing():
        return [k for k in want if not any(k in n for n in seen)]
    for _ in range(2):
        if not missing():
            break
        seen |= set(tp._forward(rt, low, dm, spec['ranges'], spec['mode'], spec['fuse'], profile=True)[1] or [])
    extra = [n for n in seen if '_kernel' in n and not any(k in n for k in want)]
    assert not missing() and not extra, (missing(), extra)
    return want


# ------------------------------------------------------------------ mode matrix
@pytest.mark.parametrize('mode', [0, 2])
@pytest.mark.parametrize('name', sorted(lp.CASES))
def test_probe_in_mode(rt, name, mode):
    """Every probe case in GEMM modes 0 and 2 (the fused first layer is an engine-3 path: off), one random and the
    selector head."""
    from oracle import lowered_ref as lr
    spec = lp.case(name)
    spec.update(mode=mode, fuse=False)
    net = spec['net']
    m = lp.make_mspec(spec['mspec'])
    z, finite = lr.patch_inputs(m, net.nmel, spec['ranges'])
    sel = lp.selector_head(net.shape, lp.default_picks(net.shape))
    dm = torch.from_numpy(m).cuda()
    entry = tp._check_heads(rt, net, spec, dm, z, finite, [('rand0', lp.random_head(net.size, 0)), ('sel', sel)], name)
    REPORT['mode%d/%s' % (mode, name)] = entry
    assert entry['worst'] <= tp.C_BOUND, entry
    _assert_kernels(rt, net.lowered(sel), spec, dm, entry.get('kernels'))


# ------------------------------------------------------------------ conv_gemm_f32_kernel edges
def _first(nmel=21, cout=64):
    return lp.ProbeNet(nmel).conv(cout, (4, 5), pre=True, relu=True)


def _tail_ranges(pix, tail):
    """One range of n patches with n * pix % 128 == tail (pix: output positions per patch of the layer)."""
    n = tail * pow(pix % 128, -1, 128) % 128
    return [(17, 17 + n)]


EDGES = {
    # scalar A (C % 8 != 0); C = 6 under a 3x3 filter is K = 54, a partial last k-tile of 6
    'scalar_a_c6_k54': lambda: dict(net=lp.ProbeNet(21).conv(6, (4, 5), relu=True).conv(32, (3, 3), pre=True, relu=True)),
    'scalar_a_c12': lambda: dict(net=lp.ProbeNet(21).conv(12, (4, 5), relu=True).conv(48, (3, 3), relu=True, post=True)),
    'scalar_a_c20_k120': lambda: dict(net=lp.ProbeNet(24).conv(20, (3, 3), pre=True, relu=True).conv(40, (2, 3))),
    # KH != KW on the scalar path: a tap's row and column differ
    'scalar_a_c6_5x2': lambda: dict(net=lp.ProbeNet(21).conv(6, (3, 3), relu=True).conv(24, (5, 2), relu=True)),
    # scalar B loads and stores (N % 4 != 0); N = 70 on the 128-wide tile
    'scalar_b_n6': lambda: dict(net=_first(21).conv(6, (3, 3), relu=True)),
    'scalar_b_n10': lambda: dict(net=_first(24).conv(10, (3, 1), pre=True, relu=True)),
    'scalar_b_n70': lambda: dict(net=_first(21).conv(70, (3, 3), relu=True, post=True)),
    # two and more grid columns
    'n130': lambda: dict(net=_first(21, 32).conv(130, (3, 3), pre=True, relu=True)),
    'n256': lambda: dict(net=_first(21, 32).conv(256, (3, 3), relu=True)),          # engine 2 in mode 3
    # 'same' padding with strides
    'same_stride22': lambda: dict(net=_first(21, 32).conv(48, (3, 3), (2, 2), 'same', relu=True)),
    'same_stride21_c12': lambda: dict(net=lp.ProbeNet(21).conv(12, (4, 5), relu=True).conv(40, (4, 3), (2, 1), 'same', pre=True, relu=True)),
    # M tails: 63 x 15 output positions per patch
    'mtail_1': lambda: dict(net=lp.ProbeNet(21).conv(12, (4, 5), relu=True).conv(24, (3, 3), relu=True),
                            ranges=_tail_ranges(63 * 15, 1)),
    'mtail_127': lambda: dict(net=lp.ProbeNet(21).conv(12, (4, 5), relu=True).conv(24, (3, 3), relu=True),
                              ranges=_tail_ranges(63 * 15, 127)),
    # the generic first layer: one input channel, N outside {16, 32, 64, 128}
    'first_generic_n8': lambda: dict(net=lp.ProbeNet(21).conv(8, (4, 5), relu=True)),
    'first_generic_n24': lambda: dict(net=lp.ProbeNet(24).conv(24, (3, 3), pre=True, relu=True, post=True)),
    'first_generic_n40_same': lambda: dict(net=lp.ProbeNet(21).conv(40, (5, 4), (1, 2), 'same', relu=True)),
    # sigmoid: shapes the tensor-core engines take, still on the fp32 kernel
    'sigmoid_n70': lambda: dict(net=_first(21).conv(70, (3, 3), act='sigmoid')),
    'sigmoid_n128_stride21_same': lambda: dict(net=_first(21).conv(128, (3, 3), (2, 1), 'same', act='sigmoid')),
}


@pytest.mark.parametrize('mode', [0, 3])
@pytest.mark.parametrize('name', sorted(EDGES))
def test_fp32_kernel_edge(rt, name, mode):
    from oracle import lowered_ref as lr
    spec = dict(mode=mode, fuse=mode == 3, mspec='normal', ranges=lp.RANGES)
    spec.update(EDGES[name]())
    net = spec['net']
    m = lp.make_mspec(spec['mspec'])
    z, finite = lr.patch_inputs(m, net.nmel, spec['ranges'])
    sel = lp.selector_head(net.shape, lp.default_picks(net.shape))
    heads = [('rand0', lp.random_head(net.size, 0)), ('rand1', lp.random_head(net.size, 1)), ('sel', sel)]
    dm = torch.from_numpy(m).cuda()
    entry = tp._check_heads(rt, net, spec, dm, z, finite, heads, name)
    entry['patches'] = int(len(z))
    REPORT['edge/mode%d/%s' % (mode, name)] = entry
    assert entry['worst'] <= tp.C_BOUND, entry
    low = net.lowered(sel)
    _assert_kernels(rt, low, spec, dm, entry.get('kernels'))
    probed = lr.plan(low, mode, spec['fuse'])[-2]          # the layer in front of the head
    assert probed.startswith('conv_gemm_f32_kernel') or (mode == 3 and name == 'n256'), probed


# ------------------------------------------------------------------ small-N heads and the softmax
def _head_body(K, nmel=21):
    """68 x nmel -> 65 x (nmel - 4) x 16 -> 4x4 pooling -> Dense(K, relu): the head reads K values per patch."""
    return lp.ProbeNet(nmel).conv(16, (4, 5), pre=True, relu=True).pool((4, 4)).dense(K, relu=True)


def _with_head(body, N, softmax, scale=1.0, bias=True, kernel=None, seed=0):
    from inaspeechsegmenter_b200 import models
    cfg, w = body.with_head(np.zeros((body.size, 8), np.float32))
    cfg['config']['layers'][-1]['config'].update(units=N, use_bias=bias, activation='softmax' if softmax else 'linear')
    r = np.random.default_rng(seed)
    if kernel is None:
        kernel = r.standard_normal((body.size, N)) * np.sqrt(1.0 / body.size) * scale
    w['head/kernel'] = np.asarray(kernel, dtype=np.float32)
    if bias:
        w['head/bias'] = r.normal(0, 0.1, N).astype(np.float32)
    return models.lower_keras_model(cfg, w, 68, body.nmel)


def _ulps_apart(body):
    """Two columns whose weights differ by a relative 2^-21: logits a few ulps apart, posteriors near 1/2."""
    c = np.random.default_rng(3).standard_normal((body.size, 1)) * np.sqrt(1.0 / body.size) * 40
    return np.concatenate([c, c * (1 + 2.0 ** -21)], axis=1)


HEADS = {}
for _n in (1, 2, 3, 8):
    for _sm in (False, True):
        HEADS['k512_n%d%s' % (_n, '_softmax' if _sm else '')] = \
            lambda n=_n, sm=_sm: dict(K=512, N=n, softmax=sm, bias=n != 2, small_n=True)
HEADS.update({
    # K N 4 bytes against the 48 KB of the small-N kernel's shared memory: 1536 x 8 fits, 1540 x 8 does not
    'k1536_n8_softmax': lambda: dict(K=1536, N=8, softmax=True, small_n=True),
    'k1540_n8_softmax': lambda: dict(K=1540, N=8, softmax=True, small_n=False),
    'k514_n3_softmax': lambda: dict(K=514, N=3, softmax=True, small_n=False),           # K % 4 != 0
    # logits of a few hundred: expf(l) overflows without the max subtraction
    'k512_n3_softmax_large': lambda: dict(K=512, N=3, softmax=True, scale=300.0, small_n=True, large=True),
    'k512_n2_softmax_large': lambda: dict(K=512, N=2, softmax=True, scale=300.0, small_n=True, large=True),
    'k512_n2_softmax_ulps': lambda: dict(K=512, N=2, softmax=True, bias=False, kernel=_ulps_apart, small_n=True),
    # rows of non-finite patches (constant stretches of the log-mel): exactly 0.5
    'k512_n3_softmax_nonfinite': lambda: dict(K=512, N=3, softmax=True, small_n=True, mspec='const',
                                              ranges=[(150, 320), (420, 480)]),
    'k512_n1_nonfinite': lambda: dict(K=512, N=1, softmax=False, small_n=True, mspec='const', ranges=[(150, 320)]),
    # 700 patches: 88 CTAs of the small-N kernel
    'k512_n2_softmax_700': lambda: dict(K=512, N=2, softmax=True, small_n=True, ranges=[(0, 700)]),
})


@pytest.mark.parametrize('name', sorted(HEADS))
def test_head_vs_float64_reference(rt, name):
    from oracle import lowered_ref as lr
    h = HEADS[name]()
    spec = dict(mode=3, fuse=True, mspec=h.get('mspec', 'normal'), ranges=h.get('ranges', lp.RANGES))
    body = _head_body(h['K'])
    kernel = h['kernel'](body) if 'kernel' in h else None
    low = _with_head(body, h['N'], h['softmax'], h.get('scale', 1.0), h.get('bias', True), kernel)
    m = lp.make_mspec(spec['mspec'])
    dm = torch.from_numpy(m).cuda()
    ref, E = lr.evaluate(low, m, spec['ranges'], mode=3)
    _, finite = lr.patch_inputs(m, body.nmel, spec['ranges'])
    if h.get('large'):
        x, _ = lr.eval_layers(low, lr.patch_inputs(m, body.nmel, spec['ranges'])[0], mode=3, stop=len(low.descs) - 1)
        lg = x.reshape(len(x), -1) @ low.blob[low.descs[-1]['w_off']:][:h['K'] * h['N']].reshape(h['K'], h['N'])
        assert (np.abs(lg).max(axis=1)[finite] > 88.8).mean() > 0.9
    got, names = tp._forward(rt, low, dm, spec['ranges'], spec['mode'], spec['fuse'], profile=True)
    assert np.isfinite(got).all(), name
    assert (got[~finite] == 0.5).all(), name
    if h['softmax']:
        assert np.allclose(got[finite].sum(axis=1), 1.0, atol=1e-6)
    ratio = np.abs(got - ref)[finite] / E[finite]
    entry = dict(worst=float(ratio.max()), patches=int(len(got)), non_finite_rows=int((~finite).sum()),
                 kind='softmax' if h['softmax'] else 'linear', kernels=names)
    REPORT['head/%s' % name] = entry
    assert entry['worst'] <= tp.C_BOUND, entry
    want = _assert_kernels(rt, low, spec, dm, names)
    assert ('dense_small_n_kernel' in want) == h['small_n'], want


# ------------------------------------------------------------------ MLP
def _mlp(rt, name, seed=4):
    in_dim, layers = lp.MLP_CASES[name]
    return rt['engine'].MlpModel(rt['ctx'], *lp.mlp_config(in_dim, layers, seed=seed), in_dim)


def _mlp_kernels(low):
    """The kernel iss_mlp_forward launches for every Dense layer (iss_conv_kernel in mode 0)."""
    return {'dense_small_n_kernel' if d['cout'] <= 8 and d['cin'] % 4 == 0 and d['cin'] * d['cout'] * 4 <= 48 * 1024
            else 'conv_gemm_f32_kernel<%d,false>' % (64 if d['cout'] <= 64 else 128) for d in low.descs}


def _mlp_ratio(mlp, x, got):
    from oracle import lowered_ref as lr
    ref, E = lr.eval_layers(mlp.lowered, x, mode=0, first=False)
    return float((np.abs(got.astype(np.float64) - ref) / E).max())


@pytest.mark.parametrize('rows', [1, 127, 128, 129, 8449, 40000])
@pytest.mark.parametrize('name', sorted(lp.MLP_CASES))
def test_mlp_vs_float64_reference(rt, name, rows):
    """8449 rows: past dense_small_n_kernel's grid-stride loop (132 x 8 CTAs of 8 warps); 40000 rows: more 128-row
    tiles of conv_gemm_f32_kernel than the GPU holds at once, so a layer that overwrote its own input (the two hidden
    buffers aliased) would feed later tiles wrong rows."""
    mlp = _mlp(rt, name)
    x = (np.random.default_rng(rows).standard_normal((rows, mlp.in_dim)) * 2).astype(np.float32)
    entry = {}
    if rows == 129:
        xd = torch.from_numpy(x).cuda()
        got, seen = tp.traced(lambda: mlp.predict(xd))
        if seen:
            want = _mlp_kernels(mlp.lowered)
            entry['kernels'] = sorted(want)
            assert all(any(k in n for n in seen) for k in want), (sorted(want), sorted(seen))
    else:
        got = mlp.predict(torch.from_numpy(x).cuda())
    entry['worst'] = _mlp_ratio(mlp, x, got)
    REPORT['mlp/%s/rows%d' % (name, rows)] = entry
    mlp.close()
    assert got.shape == (rows, mlp.out_dim)
    assert entry['worst'] <= tp.C_BOUND, entry


@pytest.mark.parametrize('name', ['d4_256_100_37_8_1', 'd3_256_256_128_1', 'd1_256_1_sigmoid'])
def test_mlp_row_alone_equals_row_in_batch(rt, name):
    """A row's place in the batch (tile, warp, grid-stride step) does not change its bits; a second run repeats them."""
    mlp = _mlp(rt, name)
    x = torch.from_numpy(np.random.default_rng(9).standard_normal((9000, mlp.in_dim)).astype(np.float32)).cuda()
    batch = mlp.predict(x)
    assert np.array_equal(batch, mlp.predict(x))
    for j in (0, 1, 127, 128, 1055, 8447, 8448, 8449, 8999):
        assert np.array_equal(mlp.predict(x[j:j + 1]), batch[j:j + 1]), (name, j)
    mlp.close()


def test_mlp_c_abi_workspace_and_alignment(rt):
    """iss_mlp_forward with exactly iss_mlp_workspace_bytes of workspace matches the reference; a d_x that is not
    16-byte aligned, or a workspace one byte short, is refused with ISS_ERR_INVALID before anything runs."""
    from inaspeechsegmenter_b200 import _lib
    lib = rt['lib'].load()
    mlp = _mlp(rt, 'd2_256_100_1')
    ctx = rt['ctx']
    n = 300
    x = np.random.default_rng(1).standard_normal((n, 256)).astype(np.float32)
    buf = torch.zeros(n * 256 + 4, dtype=torch.float32, device='cuda')
    buf[:n * 256] = torch.from_numpy(x.ravel()).cuda()
    ws = lib.iss_mlp_workspace_bytes(mlp.handle, n)
    work = torch.empty(ws, dtype=torch.uint8, device='cuda')
    y = torch.empty((n, mlp.out_dim), dtype=torch.float32, device='cuda')
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.iss_mlp_forward(ctx.handle, mlp.handle, _lib.ptr(buf), n, _lib.ptr(y), _lib.ptr(work), ws, st), 'mlp')
    got = y.cpu().numpy()
    assert _mlp_ratio(mlp, x, got) <= tp.C_BOUND
    assert np.array_equal(got, mlp.predict(x))
    torch.cuda.synchronize()
    for off in (4, 8, 12):
        rc = lib.iss_mlp_forward(ctx.handle, mlp.handle, ctypes.c_void_p(buf.data_ptr() + off), n, _lib.ptr(y),
                                 _lib.ptr(work), ws, st)
        assert rc == -1 and b'16-byte' in lib.iss_last_error(), off
    assert lib.iss_mlp_forward(ctx.handle, mlp.handle, _lib.ptr(buf), n, _lib.ptr(y), _lib.ptr(work), ws - 1, st) == -1
    torch.cuda.synchronize()
    mlp.close()


@pytest.mark.parametrize('name', ['d2_256_100_1', 'd1_256_1_sigmoid', 'd2_100_37_1'])
def test_mlp_predict_misaligned_view(rt, name):
    """MlpModel.predict on a contiguous view 4 bytes past a 16-byte boundary (buf[1:1 + n * K].view(n, K)): the first
    layer's float4 loads need an aligned copy; the result equals the one of an aligned input, bit for bit."""
    mlp = _mlp(rt, name)
    n, K = 129, mlp.in_dim
    buf = torch.from_numpy(np.random.default_rng(5).standard_normal(1 + n * K).astype(np.float32)).cuda()
    view = buf[1:1 + n * K].view(n, K)
    assert view.is_contiguous() and view.data_ptr() % 16 == 4
    got = mlp.predict(view)
    assert np.array_equal(got, mlp.predict(view.clone()))
    assert _mlp_ratio(mlp, view.cpu().numpy(), got) <= tp.C_BOUND
    mlp.close()
