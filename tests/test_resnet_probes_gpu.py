"""The x-vector extractor (csrc/resnet.cu) on probe architectures against the float64 reference of its blob
(oracle/resnet_ref.py) -- on the GPU.

Each probe network is built through the C ABI (iss_resnet_create takes any m_channels / feat_dim / num_blocks; a stage
may have no blocks) with embed_dim = 32, whose weight columns are the heads:

  random heads     16 columns of +-1: widespread errors
  selector heads   16 one-hot columns on pooled features (mean and std of the first / last / middle channels and mel
                   rows): an error confined to one channel group, one row or one tile shows up at full size

Every output must satisfy |got - ref| <= C_BOUND . E in each GEMM mode (0, 2, 3), E the bound the reference propagates.
C_BOUND was calibrated once on the unmodified kernels.  Each case also checks, from a torch.profiler trace, that the
kernels which ran are the ones resnet_ref.conv_kernel predicts.  With ISS_B200_REPORT_DIR set, the module writes
resnet_probe_report.json there: the largest err / E per case, mode and head kind, and the kernels.

Also checked: tail-window lengths, batches across and beyond one 256-window sweep, a window alone and inside a batch give
the same bits, a constant channel pools to a finite std, and activations past the fp16 range are never silently wrong."""
import ctypes
import json
import os
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')

from oracle import resnet_ref as rr           # noqa: E402

REPORT = {}
C_BOUND = 2.0           # calibrated on H100 (as the CNN probes): the unmodified kernels reach 1.01 (m32_b1211, T = 17, engine 2)
# The release network with a residual stream of ~1e5 on engine 2 reaches 2.9 on H100: there the pooled means dwarf
# the stds, and the bound's model of the fp32 one-pass variance and of the embedding's accumulation is tighter than the
# kernels' rounding
C_RANGE = 4.0
EMBED = 32
MODES = (0, 2, 3)

# name -> (m, feat_dim, num_blocks)
CASES = {
    'm32_b1211': (32, 64, (1, 2, 1, 1)),     # stage 1 on engine 2 (fp32 residual), stage-2 entry LD_F32, words after
    'm64_b1100': (64, 64, (1, 1, 0, 0)),     # stage 1 on engine 3 reading the fp32 stem output (slab kernel for c1)
    'm16_b2110': (16, 64, (2, 1, 1, 0)),     # fp32 kernel with a residual, fp32 -> engine 2 -> engine 3
    'm8_b2100': (8, 64, (2, 1, 0, 0)),       # dense_small_n_kernel as a 1x1 convolution
    'm32_stem': (32, 64, (0, 0, 0, 0)),      # the stem alone + stat pool
    'm32_f40_b1111': (32, 40, (1, 1, 1, 1)),  # h_final = 5, embedding K = 10240
    'release': (32, 64, (3, 4, 23, 3)),
}
KERNEL_RE = re.compile(r'(conv_gemm_f32_kernel<[^>]*>|conv_gemm_wg_kernel<[^>]*>|conv_slab_kernel<[^>]*>|'
                       r'dense_small_n_kernel|window_gather_kernel|stat_pool_kernel)')


def _norm(name):
    return re.sub(r'\s|\(int\)|\(bool\)|\(anonymousnamespace\)::', '', name)


class Net:
    """An iss_resnet handle of any architecture, embedding through iss_resnet_embed."""

    def __init__(self, rt, arch, blob):
        self.rt, self.arch = rt, arch
        lib = rt['lib'].load()
        nb = (ctypes.c_int * 4)(*arch.num_blocks)
        self.blob = np.ascontiguousarray(blob, dtype=np.float32)
        h = ctypes.c_void_p()
        rt['lib'].check(lib.iss_resnet_create(rt['ctx'].handle, rt['lib'].ptr(self.blob), self.blob.size, arch.m,
                                              arch.feat_dim, arch.embed_dim, ctypes.cast(nb, ctypes.c_void_p),
                                              ctypes.byref(h)), 'iss_resnet_create')
        self.h = h

    def embed(self, fea, starts, T, mode, profile=False):
        lib, L = self.rt['lib'].load(), self.rt['lib']
        starts = np.ascontiguousarray(starts, dtype=np.int32)
        n = len(starts)
        emb = torch.empty((n, self.arch.embed_dim), dtype=torch.float32, device='cuda')
        work = torch.empty(lib.iss_resnet_workspace_bytes(self.h, n, T), dtype=torch.uint8, device='cuda')
        prev = lib.iss_get_gemm_mode()
        names = None
        try:
            L.check(lib.iss_set_gemm_mode(mode), 'set mode')

            def run():
                L.check(lib.iss_resnet_embed(self.rt['ctx'].handle, self.h, L.ptr(fea), fea.shape[0], L.ptr(starts), n, T,
                                             L.ptr(emb), L.ptr(work), work.numel(), None), 'iss_resnet_embed')
                torch.cuda.synchronize()
            if profile:
                from test_layer_probes_gpu import traced
                names = {m.group(1) for n in traced(run)[1] or [] for m in [KERNEL_RE.search(_norm(n))] if m}
            else:
                run()
        finally:
            lib.iss_set_gemm_mode(prev)
        out = emb.cpu().numpy().astype(np.float64)
        return (out, names) if profile else out

    def close(self):
        self.rt['lib'].load().iss_resnet_destroy(self.h)


@pytest.fixture(scope='module')
def rt():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from inaspeechsegmenter_b200 import _lib, engine
    return dict(ctx=engine.Context(0), lib=_lib)


@pytest.fixture(scope='module', autouse=True)
def _dump_report():
    yield
    out = os.environ.get('ISS_B200_REPORT_DIR')
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, 'resnet_probe_report.json'), 'w') as f:
            json.dump(REPORT, f, indent=1, sort_keys=True)


def selector_picks(arch):
    C, H = arch.emb['c_final'], arch.emb['h_final']
    ch = [(0, 0), (C - 1, H - 1), (0, H - 1), (C - 1, 0), (C // 2, H // 2), (1, H // 3), (C - 2, 1), (C // 3, H - 2)]
    return [c * H + h for c, h in ch] + [C * H + c * H + h for c, h in ch]


def heads(arch, seed=0):
    """[2 C H, 32]: 16 random +-1 columns, then 16 one-hot selectors (8 means, the same 8 stds)."""
    K = arch.emb['cin']
    W = np.zeros((K, EMBED), dtype=np.float32)
    W[:, :16] = np.random.default_rng(seed).choice([-1.0, 1.0], size=(K, 16))
    for j, k in enumerate(selector_picks(arch)):
        W[k, 16 + j] = 1.0
    return W


def probe(name, seed=1):
    m, feat, nb = CASES[name]
    arch = rr.plan(m, feat, EMBED, nb)
    return arch, rr.synthetic_blob(arch, seed=seed, heads=heads(arch))


def features(arch, rows, seed=3):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return torch.randn(rows, arch.feat_dim, generator=g).cuda()


def _ratio(got, ref, E):
    """|got - ref| / E elementwise; where E = 0 (a dead channel's exact zero) only an exact match passes."""
    d = np.abs(got - ref)
    return np.where(E > 0, d / np.where(E > 0, E, 1.0), np.where(d == 0, 0.0, np.inf))


def _ratios(got, ref, E):
    r = _ratio(got, ref, E)
    return float(r[:, :16].max()), float(r[:, 16:].max())


def _check(net, fea, starts, T, tag, modes=MODES, profile=False):
    """Every mode: finite outputs within C_BOUND . E; with profile, the kernels of the trace are the predicted ones."""
    arch = net.arch
    x = rr.gather(fea.cpu().numpy(), starts, T)
    entry = REPORT.setdefault(tag, {})
    for mode in modes:
        ref, E = rr.forward(arch, net.blob, x, mode, device='cuda')
        if profile:
            got, names = net.embed(fea, starts, T, mode, profile=True)
        else:
            got, names = net.embed(fea, starts, T, mode), None
        assert np.isfinite(got).all(), (tag, mode)
        rand, sel = _ratios(got, ref, E)
        e = entry.setdefault('mode%d' % mode, {})
        e.update(rand=max(rand, e.get('rand', 0.0)), sel=max(sel, e.get('sel', 0.0)))
        assert max(rand, sel) <= C_BOUND, (tag, mode, rand, sel)
        if profile:
            expected = rr.kernel_names(arch, mode)
            for _ in range(2):                       # the activity trace may drop a record: look at two more runs
                if names and expected <= names:
                    break
                names = (names or set()) | (net.embed(fea, starts, T, mode, profile=True)[1] or set())
            if not names:
                e['kernels'] = 'the profiler recorded no CUDA kernels: kernel assertion skipped'
                continue
            e['kernels'] = sorted(names)
            assert expected <= names and names <= expected, (tag, mode, sorted(expected - names), sorted(names - expected))


@pytest.mark.parametrize('name', sorted(CASES))
def test_probe_network_vs_float64_reference(rt, name):
    arch, blob = probe(name)
    net = Net(rt, arch, blob)
    try:
        n = 8 if name == 'release' else 5
        fea = features(arch, 24 * n + 144 + 7)
        starts = [24 * i + 3 * (i % 3) for i in range(n)][::-1]
        _check(net, fea, starts, 144, name, profile=True)
    finally:
        net.close()


@pytest.mark.parametrize('T', [10, 17, 131, 143])
def test_probe_tail_window_lengths(rt, T):
    """Odd widths into the stride-2 layers, down to a final width of 2 (T = 10 and 17)."""
    for name in ('m32_b1211', 'm16_b2110'):
        arch, blob = probe(name)
        net = Net(rt, arch, blob)
        try:
            fea = features(arch, 400, seed=T)
            _check(net, fea, [0, 399 - T, 123, 57], T, '%s_T%d' % (name, T))
        finally:
            net.close()


def _starts(n, rows, T, seed):
    """n unsorted, overlapping window starts in [0, rows - T], one of them ending at the last row."""
    s = np.random.default_rng(seed).integers(0, rows - T + 1, n)
    s[n // 2] = rows - T
    return s


@pytest.mark.parametrize('n', [1, 37, 256, 257, 700])
def test_probe_batches(rt, n):
    """Windows across one 256-window sweep, a sweep and one window, several sweeps."""
    arch, blob = probe('m32_b1211')
    net = Net(rt, arch, blob)
    try:
        rows = 24 * n + 144
        fea = features(arch, rows, seed=n)
        _check(net, fea, _starts(n, rows, 144, n), 144, 'm32_b1211_batch%d' % n)
    finally:
        net.close()


@pytest.mark.parametrize('name', ['m32_b1211', 'm16_b2110', 'release'])
def test_window_alone_equals_window_in_batch(rt, name):
    """The slot of a window in a 128-row tile, its sweep and its place in the grid must not change the arithmetic: a window
    embedded alone and inside a 700-window batch (three sweeps) give the same bits in every mode, as do two runs."""
    arch, blob = probe(name)
    net = Net(rt, arch, blob)
    try:
        rows = 24 * 700 + 144
        fea = features(arch, rows, seed=11)
        starts = _starts(700, rows, 144, 5)
        for mode in MODES:
            batch = net.embed(fea, starts, 144, mode)
            assert np.isfinite(batch).all()
            assert np.array_equal(batch, net.embed(fea, starts, 144, mode)), mode
            for j in (0, 127, 128, 255, 256, 350, 511, 699):
                alone = net.embed(fea, starts[j:j + 1], 144, mode)
                assert np.array_equal(alone[0], batch[j]), (name, mode, j)
    finally:
        net.close()


def test_constant_channel_std_is_finite(rt):
    """Zero stem weights and a positive shift: every channel of the stem output is constant over time, so every pooled
    std is sqrt(1e-10) = 1e-5 in float64.  The one-pass fp32 variance rounds to either side of 0; it must not be NaN."""
    arch, blob = probe('m32_stem')
    st = arch.stem
    blob[st['w_off']:st['w_off'] + 9 * arch.m] = 0.0
    blob[st['shift_off']:st['shift_off'] + arch.m] = np.random.default_rng(2).uniform(0.05, 4.0, arch.m)
    net = Net(rt, arch, blob)
    try:
        fea = features(arch, 600)
        for T in (144, 131, 17):
            x = rr.gather(fea.cpu().numpy(), [0, 5, 77], T)
            _, _, p, _ = rr.forward(arch, blob, x, 0, device='cuda', pooled=True)
            assert np.abs(p[:, p.shape[1] // 2:] - 1e-5).max() < 1e-12
            _check(net, fea, [0, 5, 77], T, 'constant_channel_T%d' % T)
    finally:
        net.close()


def _overflow_blob(shift):
    arch, blob = probe('m32_b1211')
    c3 = rr.layer(arch, 'layer2.0.c3')
    blob[c3['shift_off']:c3['shift_off'] + c3['cout']] = shift
    return arch, blob


def test_fp16_range_overflow_is_never_silent(rt):
    """A stage-2 BatchNorm shift of 1e5 pushes the residual stream past 65520: engine 3 carries it as split-half words
    (hi = inf, lo = -inf, a NaN).  It may return non-finite x-vectors, never finite wrong ones; engine 2 (fp32 range)
    must be right.  The extractor must refuse the non-finite x-vectors under engine 3 with an error naming the remedy."""
    from inaspeechsegmenter_b200 import _lib, vbx_segmenter as vb
    from oracle import vbx_oracle as vx
    arch, blob = _overflow_blob(1e5)
    net = Net(rt, arch, blob)
    entry = REPORT.setdefault('fp16_range_overflow', {})
    try:
        fea = features(arch, 400)
        starts = [0, 100, 256]
        x = rr.gather(fea.cpu().numpy(), starts, 144)
        for mode in (2, 3):
            ref, E = rr.forward(arch, blob, x, mode, device='cuda')
            got = net.embed(fea, starts, 144, mode)
            fin = np.isfinite(got).all(axis=1)
            wrong = fin & (_ratio(got, ref, E) > C_BOUND).any(axis=1)
            entry['mode%d' % mode] = dict(finite_rows=int(fin.sum()), rows=len(fin), finite_and_wrong_rows=int(wrong.sum()))
            assert not wrong.any(), entry
            if mode == 2:
                assert fin.all(), entry
    finally:
        net.close()

    sd = vx.synthetic_resnet101_state(seed=5)
    sd['layer2.0.bn3.bias'] = sd['layer2.0.bn3.bias'] + 1e5
    ext = vb.B200BackendExtractor(state_dict=sd, ctx=rt['ctx'])
    fea = features(rr.plan(**rr.RELEASE), 330, seed=7).cpu().numpy()
    lib = _lib.load()
    prev = lib.iss_get_gemm_mode()
    try:
        lib.iss_set_gemm_mode(3)
        with pytest.raises(_lib.IssError, match='ISS_B200_GEMM=tc_ts'):
            ext('clip', fea, 3.3)
        with pytest.raises(_lib.IssError, match='ISS_B200_GEMM=tc_ts'):
            ext.get_embedding(fea[:144])
        lib.iss_set_gemm_mode(2)
        out = ext('clip', fea, 3.3)
    finally:
        lib.iss_set_gemm_mode(prev)
    plan = vb.window_plan(len(fea))
    assert [k for k, _, _ in out] == ['clip_%08d-%08d' % (s, len(fea) if tail else s + n) for s, n, tail in plan]
    arch = rr.plan(**rr.RELEASE)
    blob = vb.resnet_blob_from_state(sd)
    worst = 0.0
    for (s, n, _), (_, _, got) in zip(plan, out):
        ref, E = rr.forward(arch, blob, rr.gather(fea, [s], n), 2, device='cuda')
        r = float(_ratio(got / 10, ref[0], E[0]).max())
        worst = max(worst, r)
        assert r <= C_RANGE, (s, n, r)
    entry['extractor_mode2_worst'] = worst
