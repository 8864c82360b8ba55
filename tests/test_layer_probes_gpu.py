"""Every convolution path of the CNN operator, one layer at a time, against the float64 reference of the lowered network
(oracle/lowered_ref.py) -- on the GPU.

The layer under test sits in a probe network (tests/layer_probes.py) that ends in Flatten -> Dense(8) without softmax,
so the operator returns 8 linear functionals of the layer's whole output per patch:

  random heads     +-1 columns, three seeds: widespread errors
  selector head    one-hot columns on chosen elements (first / last row, column and channel, corners, middle): with the
                   batch offset of each patch these land on every slot of a tile, so an error confined to one tap, one
                   warpgroup, one channel group or the last tile shows up at full size instead of averaged away

Each output must satisfy |got - ref| <= C_BOUND . E, E the error bound the reference propagates (2^-22 per term for
the split engines).  C_BOUND was calibrated once on the unmodified kernels.  With ISS_B200_REPORT_DIR set, the module
writes probe_report.json there: the largest err / E per case and head, and the kernels one forward launched
(torch.profiler trace).  A kernel that drops a whole correction product on a fraction of its outputs sits one to two
orders of magnitude above the bound.

Also checked: a patch alone and inside a multi-tile batch give the same bits; two runs give the same bits; a layer's
split-half words decode to exactly hi + lo of its fp32 output; the fp16 range of the split engine."""
import json
import os
import re
import time

import numpy as np
import pytest

import layer_probes as lp

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')

REPORT = {}
C_BOUND = 2.0           # calibrated on H100: the unmodified kernels reach 0.56 (17x10 taps, K = 9792), most cases < 0.3
HEAD_SEEDS = (0, 1, 2)


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
        with open(os.path.join(out, 'probe_report.json'), 'w') as f:
            json.dump(REPORT, f, indent=1, sort_keys=True)


def _norm(name):
    return re.sub(r'\s|\(int\)|\(bool\)|\(anonymousnamespace\)::', '', name)


def traced(run):
    """(run(), the names of the CUDA kernels it launched) from a torch.profiler trace; the names are None when the trace
    holds no kernels.  run() executes twice: in the profiler's warm-up step, whose records are discarded, and then,
    after a pause, recorded.  A trace that begins with the launches can lose the first kernels of a short run (a probe
    forward was seen three times running without its first three kernels), so the recorded run starts only once the
    activity tracing has been running for a while."""
    from torch.profiler import ProfilerActivity, profile, schedule
    with profile(activities=[ProfilerActivity.CUDA], schedule=schedule(wait=0, warmup=1, active=1, repeat=1)) as prof:
        run()
        torch.cuda.synchronize()
        prof.step()
        time.sleep(0.02)
        out = run()
        torch.cuda.synchronize()
        prof.step()
    names = sorted({_norm(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
    return out, names or None


def _forward(rt, low, dm, ranges, mode, fuse, profile=False):
    """Output of the operator ([n, 8] numpy) and, with profile, the names of the CUDA kernels it launched (None when
    the profiler records no kernels)."""
    lib = rt['lib'].load()
    prev_mode, prev_env = lib.iss_get_gemm_mode(), os.environ.get('ISS_B200_FUSE_FIRST')
    try:
        os.environ['ISS_B200_FUSE_FIRST'] = '1' if fuse else '0'
        rt['lib'].check(lib.iss_set_gemm_mode(mode), 'set mode')
        net = rt['engine'].CnnModel(rt['ctx'], low)
        names = None
        if profile:
            out, names = traced(lambda: net.forward(dm, ranges))
        else:
            out = net.forward(dm, ranges)
        out = out.cpu().numpy().astype(np.float64)
        net.close()
        return out, names
    finally:
        lib.iss_set_gemm_mode(prev_mode)
        if prev_env is None:
            os.environ.pop('ISS_B200_FUSE_FIRST', None)
        else:
            os.environ['ISS_B200_FUSE_FIRST'] = prev_env


def _reference(net, head, z, finite, mode, body=None):
    from oracle import lowered_ref as lr
    low = net.lowered(head)
    nl = len(low.descs)
    if body is None:
        body = lr.eval_layers(low, z, mode=mode, stop=nl - 1)
    y, E = lr.eval_layers(low, body[0], body[1], mode=mode, start=nl - 1)
    y[~finite], E[~finite] = 0.5, 0.0
    return low, y, E, body


def _check_heads(rt, net, spec, dm, z, finite, heads, tag):
    """Every head: |got - ref| <= C_BOUND E on finite patches, exactly 0.5 on the others.  Returns the report entry."""
    body, entry = None, {}
    for hname, head in heads:
        low, ref, E, body = _reference(net, head, z, finite, spec['mode'], body)
        got, names = _forward(rt, low, dm, spec['ranges'], spec['mode'], spec['fuse'], profile=hname == 'sel')
        assert np.isfinite(got).all(), (tag, hname)
        assert (got[~finite] == 0.5).all(), (tag, hname)
        ratio = np.abs(got - ref)[finite] / E[finite]
        entry[hname] = float(ratio.max())
        if names is not None:
            entry['kernels'] = names
        elif hname == 'sel':
            entry['kernels'] = 'the profiler recorded no CUDA kernels: kernel assertion skipped'
    entry['worst'] = max(v for k, v in entry.items() if k not in ('kernels',))
    return entry


@pytest.mark.parametrize('name', sorted(lp.CASES))
def test_probe_layer_vs_float64_reference(rt, name):
    from oracle import lowered_ref as lr
    spec = lp.case(name)
    net = spec['net']
    m = lp.make_mspec(spec['mspec'])
    z, finite = lr.patch_inputs(m, net.nmel, spec['ranges'])
    heads = [('rand%d' % s, lp.random_head(net.size, s)) for s in HEAD_SEEDS]
    heads.append(('sel', lp.selector_head(net.shape, lp.default_picks(net.shape))))
    entry = _check_heads(rt, net, spec, torch.from_numpy(m).cuda(), z, finite, heads, name)
    entry['patches'] = int(len(z))
    REPORT[name] = entry
    assert entry['worst'] <= C_BOUND, entry
    if isinstance(entry.get('kernels'), list):
        names = set(entry['kernels'])

        def missing():
            return [k for k in spec['kernels'] if not any(_norm(k) in n for n in names)]
        for _ in range(2):                           # the activity trace may drop a record: look at two more forwards
            if not missing():
                break
            names |= set(_forward(rt, net.lowered(heads[-1][1]), torch.from_numpy(m).cuda(), spec['ranges'],
                                  spec['mode'], spec['fuse'], profile=True)[1] or [])
        assert not missing(), (missing(), sorted(names))


BATCH_CASES = ['slab_first_5x4_w24', 'slab_packed_5x4_w21', 'slab_f32_3x3_w21', 'g3_c64_n128', 'g3_pool_odd',
               'g3_dense_large_k', 'g2_c96_n160', 'first_direct_c64_same_stride', 'pool_words_3x2_same']


@pytest.mark.parametrize('name', BATCH_CASES)
def test_probe_patch_alone_equals_patch_in_batch(rt, name):
    """The slot of a patch in a tile (and the tile's place in the grid) must not change the arithmetic: a patch evaluated
    alone and inside a 700-patch batch (several hundred tiles) give the same bits, and a second run repeats them."""
    spec = lp.case(name)
    net = spec['net']
    low = net.lowered(lp.random_head(net.size, 7))
    dm = torch.from_numpy(lp.make_mspec('normal')).cuda()
    batch, _ = _forward(rt, low, dm, [(0, 700)], spec['mode'], spec['fuse'])
    again, _ = _forward(rt, low, dm, [(0, 700)], spec['mode'], spec['fuse'])
    assert np.array_equal(batch, again)
    for j in (0, 17, 18, 333, 699):
        alone, _ = _forward(rt, low, dm, [(j, j + 1)], spec['mode'], spec['fuse'])
        assert np.array_equal(alone[0], batch[j]), (name, j)


def _split_words(y):
    """hi + lo of the split-half word of float32 y (hi = fp16(y), lo = fp16(y - hi)), in float32."""
    y = y.astype(np.float32)
    hi = y.astype(np.float16).astype(np.float32)
    lo = (y - hi).astype(np.float16).astype(np.float32)
    return hi + lo


@pytest.mark.parametrize('fill', sorted(lp.SLAB_FILL))
def test_packed_output_decodes_exactly(rt, fill):
    """A layer whose consumer is an fp16-split convolution stores split-half words.  Behind it, a 1x1 identity 'relay'
    (weights exactly 2^12 after scaling, lo = 0) returns the words decoded exactly; they must equal numpy's hi + lo of the
    same layer's fp32 output, read by one-hot heads from the network without the relay."""
    from oracle import lowered_ref as lr
    plain = lp._slab_case((5, 4), fill, 21, lp.EPILOGUES[3])
    relay = lp._slab_case((5, 4), fill, 21, lp.EPILOGUES[3], relay=True)
    dm = torch.from_numpy(lp.make_mspec('normal')).cuda()
    shape = plain['net'].shape
    picks = [(0, 0, 0), (-1, -1, -1), (3, 5, 17), (-2, 1, 40), (10, -1, 63), (20, 7, 1), (-1, 0, 32), (30, 3, 9)]
    head = lp.selector_head(shape, picks)
    ranges = lp.RANGES
    y, _ = _forward(rt, plain['net'].lowered(head), dm, ranges, 3, plain['fuse'])
    w, names = _forward(rt, relay['net'].lowered(head), dm, ranges, 3, relay['fuse'], profile=True)
    if names is not None:
        assert any('conv_slab_kernel<1>' in n for n in names)
    z, finite = lr.patch_inputs(lp.make_mspec('normal'), 21, ranges)
    assert finite.all()
    assert np.array_equal(w.astype(np.float32), _split_words(y)), np.abs(w - _split_words(y)).max()
    assert not np.array_equal(w.astype(np.float32), y.astype(np.float32))        # the words really are coarser


def _range_net(gain, bias=False):
    return lp.ProbeNet(21, seed=5).conv(64, (4, 5), bias=bias, gain=gain).conv(64, (3, 3), padding='same', relu=True)


def _first_layer_peak(z):
    from oracle import lowered_ref as lr
    net = _range_net(1.0)
    low = net.lowered(lp.random_head(net.size, 0))
    a, _ = lr.eval_layers(low, z, stop=1)
    return float(np.abs(a).max())


@pytest.mark.parametrize('peak', [65000.0, 0.0625])
def test_fp16_range_in_range(rt, peak):
    """First-layer activations up to +-65000 (just inside fp16) and below 2^-3 (the lo halves go subnormal; the bound
    has an absolute 2^-25 term per operand there) read as split-half words by an fp16-split convolution."""
    from oracle import lowered_ref as lr
    m = lp.make_mspec('normal')
    z, finite = lr.patch_inputs(m, 21, lp.RANGES)
    net = _range_net(peak / _first_layer_peak(z))
    spec = dict(mode=3, fuse=False, ranges=lp.RANGES)
    heads = [('rand0', lp.random_head(net.size, 0)), ('sel', lp.selector_head(net.shape, lp.default_picks(net.shape)))]
    entry = _check_heads(rt, net, spec, torch.from_numpy(m).cuda(), z, finite, heads, 'fp16_range_%g' % peak)
    REPORT['fp16_range_peak_%g' % peak] = entry
    assert entry['worst'] <= C_BOUND, entry


def test_fp16_range_overflow_is_never_silent(rt):
    """Activations past 65520 do not fit the split-half words of the fp16-split engine (hi = inf, lo = -inf, hi + lo =
    NaN).  The engine may fail -- non-finite outputs -- but it must never return finite values that differ from the
    float64 reference (and from the 3xTF32 engine, which carries fp32 values) beyond the bound; and the segmenter must
    refuse such posteriors with an error that names the remedy."""
    from oracle import lowered_ref as lr
    from inaspeechsegmenter_b200 import _lib, segmenter
    m = lp.make_mspec('normal')
    z, finite = lr.patch_inputs(m, 21, lp.RANGES)
    net = _range_net(2e5 / _first_layer_peak(z))
    head = lp.random_head(net.size, 0)
    dm = torch.from_numpy(m).cuda()
    entry = {}
    for mode in (2, 3):
        low, ref, E, _ = _reference(net, head, z, finite, mode)
        got, _ = _forward(rt, low, dm, lp.RANGES, mode, False)
        fin = np.isfinite(got).all(axis=1)
        wrong = fin & (np.abs(got - ref) > C_BOUND * E).any(axis=1)
        entry['mode%d' % mode] = dict(finite_rows=int(fin.sum()), rows=int(len(fin)), finite_and_wrong_rows=int(wrong.sum()),
                                      max_err_over_bound_finite=float((np.abs(got - ref)[fin] / E[fin]).max()) if fin.any() else None)
        if mode == 2:
            assert fin.all() and not wrong.any(), entry
    REPORT['fp16_range_overflow'] = entry
    assert entry['mode3']['finite_and_wrong_rows'] == 0, entry

    # the segmenter: a 2-class softmax head on the same body
    cfg, w = net.with_head(lp.random_head(net.size, 1))
    cfg['config']['layers'][-1]['config'].update(units=2, use_bias=False, activation='softmax')
    w['head/kernel'] = (w['head/kernel'][:, :2] * np.float32(1e-4)).copy()
    lib = rt['lib'].load()
    prev = lib.iss_get_gemm_mode()
    try:
        lib.iss_set_gemm_mode(3)
        seg = segmenter.SpeechMusic(32, ctx=rt['ctx'], model=(cfg, w))
        lseg = [('energy', 20, 63), ('noEnergy', 63, 400), ('energy', 400, 411)]
        with pytest.raises(_lib.IssError, match='ISS_B200_GEMM=tc_ts'):
            seg(dm, lseg)
        lib.iss_set_gemm_mode(2)
        out = seg(dm, lseg)
        assert out[0][1] == 20 and out[-1][2] == 411 and ('noEnergy', 63, 400) in out
    finally:
        lib.iss_set_gemm_mode(prev)
