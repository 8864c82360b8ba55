"""Live streams on the GPU (run with -m gpu on an H100): the online Viterbi kernel against the offline decoders, the
stream front end against K1 on the whole signal, and every stream's segments against the offline segmentation."""
import os
import warnings

import numpy as np
import pytest

from conftest import synth_audio

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')


@pytest.fixture(scope='module')
def rt():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from inaspeechsegmenter_b200 import _lib, engine, pack, segmenter, stream
    return dict(lib=_lib, engine=engine, pack=pack, segmenter=segmenter, stream=stream)


def _segmenter(rt, synth_models, vad='smn', gender=True, fft='fp64'):
    return rt['segmenter'].Segmenter(vad_engine=vad, detect_gender=gender, ffmpeg=None, fft_precision=fft,
                                     models={'vad': synth_models[vad], 'gender': synth_models['gender']})


def _chunks(x, rng, how):
    if how == 'one':
        return [x]
    if isinstance(how, int):
        return [x[i:i + how] for i in range(0, len(x), how)]
    out, pos = [], 0
    while pos < len(x):
        n = int(rng.uniform(0.01, 3.0) * 16000)
        out.append(x[pos:pos + n])
        pos += n
    return out


def _stream_alone(seg, x, cal, how, seed=0):
    live = seg.stream(calibration_sec=cal)
    got = []
    for c in _chunks(x, np.random.default_rng(seed), how):
        got += live.feed({'k': c})['k']
    got += live.end(['k'])['k']
    return got


def _prefix_reference(rt, seg, x, n_cal):
    """Offline segmentation with the energy threshold of the first n_cal loge values."""
    engine, sg = rt['engine'], rt['segmenter']
    mspec, loge, difflen = sg.feats_from_signal(x, 0, seg.fft_precision, 'main')
    stats = engine.loge_stats(seg.ctx, loge[:n_cal].contiguous())
    track = engine.energy_viterbi(seg.ctx, loge, stats, seg.energy_ratio, out_stride=2).cpu().numpy()
    lseg = [('noEnergy' if lab == 0 else 'energy', a, b) for lab, a, b in sg._rle(track)]
    lseg = seg.vad(mspec, lseg, difflen)
    if seg.detect_gender:
        lseg = seg.gender(mspec, lseg, difflen)
    return [(lab, 0 + a * .02, 0 + b * .02) for lab, a, b in lseg]


# ---- online Viterbi kernel -------------------------------------------------------------------------------------
def _online_run(rt, ctx, src, n, cuts, K, trans=None, stats=None, ratio=None):
    engine = rt['engine']
    scores = torch.zeros((1, 4), dtype=torch.float64, device='cuda')
    hist = torch.zeros((1, n + 1), dtype=torch.uint8, device='cuda')
    bounds = [0] + cuts + [n]
    got, pend = [], 0
    for i, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        end = i == len(bounds) - 2
        fl = (engine.ONLINE_START if a == 0 else 0) | (engine.ONLINE_END if end else 0)
        ch = np.array([[a, b - a, 0, pend, 0, fl]], dtype=np.int64)
        buf = engine.viterbi_online(ctx, ch, src, scores, hist, pend + b - a, K=K, trans=trans, stats=stats,
                                    energy_ratio=ratio)
        nd, st = engine.split_online(buf.cpu().numpy(), 1)
        got.append(st[:nd[0]].copy())
        pend += b - a - int(nd[0])
        yield np.concatenate(got), end


@pytest.mark.parametrize('K', [2, 3])
def test_online_kernel_equals_viterbi_segments(rt, synth_models, K):
    seg = _segmenter(rt, synth_models)
    engine = rt['engine']
    rng = np.random.default_rng(K)
    for T in (1, 37, 5000):
        p = torch.from_numpy(rng.dirichlet(np.ones(K) * 0.4, size=T).astype(np.float32)).cuda()
        trans = engine.diag_trans_exp(80, K)
        ref = engine.viterbi_segments(seg.ctx, p, [0, T], trans).cpu().numpy()
        for cuts in (sorted(set(rng.integers(1, T, size=20).tolist())) if T > 1 else [],
                     list(range(1, min(T, 300)))):
            for got, end in _online_run(rt, seg.ctx, p, T, cuts, K, trans=trans):
                assert np.array_equal(got, ref[:len(got)])
            assert end and np.array_equal(got, ref)


def test_online_kernel_equals_energy_viterbi_long(rt, synth_models):
    seg = _segmenter(rt, synth_models)
    engine = rt['engine']
    rng = np.random.default_rng(5)
    L = 70000                                               # decoded chunk-parallel by the offline path
    loge = torch.from_numpy(np.repeat(rng.normal(0, 3, size=L // 50), 50).astype(np.float32)[:L]).cuda()
    stats1 = engine.loge_stats(seg.ctx, loge[:1000].contiguous())
    ref = engine.energy_viterbi(seg.ctx, loge, stats1, seg.energy_ratio, out_stride=1).cpu().numpy()
    stats = stats1.view(1, 2)
    cuts = sorted(set(rng.integers(1, L, size=60).tolist()))
    for got, end in _online_run(rt, seg.ctx, loge, L, cuts, 2, stats=stats, ratio=seg.energy_ratio):
        assert np.array_equal(got, ref[:len(got)])
    assert np.array_equal(got, ref)


def test_loge_stats_multi_equals_single(rt, synth_models):
    seg = _segmenter(rt, synth_models)
    engine = rt['engine']
    x = torch.randn(20000, device='cuda')
    x[::97] = float('-inf')
    offs, lens = [0, 5, 1000, 19000], [1, 4999, 48 * 40 + 7, 1000]
    got = engine.loge_stats_multi(seg.ctx, x, offs, lens)
    for i, (o, n) in enumerate(zip(offs, lens)):
        assert torch.equal(got[i], engine.loge_stats(seg.ctx, x[o:o + n].contiguous())), i


# ---- front end -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('fmt', ['int16', 'float32'])
@pytest.mark.parametrize('where', ['host', 'cuda'])
def test_stream_front_end_equals_k1(rt, synth_models, fmt, where):
    seg = _segmenter(rt, synth_models)
    x = synth_audio(12, seed=3)
    if fmt == 'float32':
        x = x.astype(np.float32) / np.float32(32768)
    m1, l1, _ = rt['segmenter']._get_frontend('main', 0)(torch.from_numpy(x).cuda(), seg.fft_precision)
    rng = np.random.default_rng(1)
    for how in (1, 159, 160, 161, 399, 400, 'random', 'one'):
        xs = x[:3000] if how == 1 else x
        be = rt['stream'].CudaBackend(seg)
        pos = 0
        for c in _chunks(xs, rng, how):
            if where == 'cuda':                 # a misaligned view of a larger device buffer
                big = torch.from_numpy(np.concatenate((x[:3], c))).cuda()
                c = big[3:]
            be.ingest({0: c}, {0: 0})
            pos += len(c)
        F = be.frames[0]
        assert F == rt['pack'].num_frames(len(xs))
        assert torch.equal(be.mspec[:F], m1[:F]), how
        assert torch.equal(be.loge[:F], l1[:F]), how


# ---- end to end ------------------------------------------------------------------------------------------------
def _media(media, name):
    from inaspeechsegmenter_b200.io import media2sig16kmono
    return media2sig16kmono(os.path.join(media, name), None, None, None, 'float32', return_int16=True)


def test_short_streams_equal_segment_signal(rt, synth_models, media):
    seg = _segmenter(rt, synth_models)
    base = synth_audio(60, seed=7)
    sigs = [base[:400], base[1000:1559], base[3000:3560], base[5000:5719], base[9000:9720], base[20000:28000],
            base[40000:56000], base[60000:76160], np.zeros(32000, dtype=np.int16)]
    sigs += [_media(media, f) for f in ('musanmix.wav', 'silence2sec.wav', 'lamartine.wav')]
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        for i, x in enumerate(sigs):
            cal = max(1.0, (len(x) / 16000) + 1)
            ref = seg.segment_signal(x)
            for how in ('one', 'random', 4000):
                assert _stream_alone(seg, x, cal, how, seed=i) == ref, (i, how)
            # exactly N_cal frames: calibrated, decoded online
            n = rt['pack'].num_frames(len(x))
            if n >= 100:
                assert _stream_alone(seg, x, n / 100, 'random', seed=i) == ref, (i, 'n_cal == L')


@pytest.mark.parametrize('vad,gender,fft', [('smn', True, 'fp64'), ('sm', True, 'fp32'), ('smn', False, 'fp32'),
                                            ('sm', False, 'fp64')])
def test_long_streams_equal_prefix_threshold_reference(rt, synth_models, vad, gender, fft):
    seg = _segmenter(rt, synth_models, vad, gender, fft)
    x = synth_audio(180, seed=9)
    ref = _prefix_reference(rt, seg, x, 500)
    for how in (16000, 'random', 'one'):
        got = _stream_alone(seg, x, 5.0, how, seed=3)
        assert got == ref, how
    # segments are complete and never revised: the returned lists concatenate to the reference, in order
    live = seg.stream(calibration_sec=5.0)
    lags = []
    for i in range(0, len(x), 8000):
        live.feed({'a': x[i:i + 8000]})
        lags.append((i + 8000) / 16000 - live.decided_until('a'))
    assert min(lags) > 0
    live.end(['a'])


def test_many_streams_equal_streams_alone(rt, synth_models):
    seg = _segmenter(rt, synth_models)
    rng = np.random.default_rng(11)
    audio = synth_audio(600, seed=21)
    N = 300
    sigs, starts, chunk = [], [], []
    for i in range(N):
        n = int(rng.uniform(0.3, 25.0) * 16000)
        a = int(rng.integers(0, len(audio) - n))
        x = audio[a:a + n]
        if i % 3 == 1:
            x = x.astype(np.float32) / np.float32(32768)
        sigs.append(x)
        starts.append(int(rng.integers(0, 10)))
        chunk.append(int(rng.choice([1600, 8000, 16000, 23456])))
    live = seg.stream(calibration_sec=3.0)
    got = {i: [] for i in range(N)}
    pos = [0] * N
    step = 0
    open_ = set()
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        while any(pos[i] < len(sigs[i]) for i in range(N)):
            feed = {}
            for i in range(N):
                if starts[i] <= step and pos[i] < len(sigs[i]):
                    c = sigs[i][pos[i]:pos[i] + chunk[i]]
                    feed[i] = torch.from_numpy(c).cuda() if i % 5 == 2 else c
                    pos[i] += len(c)
            for k, v in live.feed(feed).items():
                got[k] += v
            open_ |= set(feed)
            done = [i for i in open_ if pos[i] >= len(sigs[i]) and i % 2 == 0]
            for k, v in live.end(done).items():
                got[k] += v
            open_ -= set(done)
            step += 1
        for k, v in live.end(sorted(open_)).items():
            got[k] += v
        # a key reused after end starts fresh
        again = live.feed({0: sigs[1]})[0] + live.end([0])[0]
        assert again == _stream_alone(seg, sigs[1], 3.0, 'one')
        for i in range(N):
            x = sigs[i]
            if len(x) < 400:
                continue
            assert got[i] == _stream_alone(seg, x, 3.0, chunk[i]), i


def test_launch_count_does_not_grow_with_streams(rt, synth_models):
    seg = _segmenter(rt, synth_models)
    lib = rt['lib'].load()
    audio = synth_audio(600, seed=12)
    counts = {}
    # 150 streams of 1 s are ~7500 patches per network: one CNN sweep (8192 patches) each, as for 10 streams; more
    # patches per call add sweeps, whatever the number of streams they come from
    for N, sec in ((10, 1), (150, 1), (75, 2)):
        live = seg.stream(calibration_sec=1.0)
        c = []
        n = 16000 * sec
        for s in range(4):
            feed = {i: audio[(i + s) * n % (len(audio) - n):][:n] for i in range(N)}
            c0 = lib.iss_launch_count()
            live.feed(feed)
            c.append(lib.iss_launch_count() - c0)
        live.end(list(range(N)))
        counts[N] = c
    # 75 streams of 2 s chunks decode as many patches per call as 150 streams of 1 s: the same launches once past
    # calibration, so launches follow the patches of a call, not its streams
    for a, b in zip(counts[150][2:], counts[75][2:]):
        assert abs(a - b) <= 4, counts
    # the first call only computes frames; the second decodes the calibration prefix too (twice the patches: a second
    # sweep for 150 streams); from the third on every call does the same work per stream
    assert counts[10][0] == counts[150][0], counts
    for a, b in zip(counts[10][2:], counts[150][2:]):
        assert abs(a - b) <= 4, counts          # up to the fused first layer of each network (two per network)


def test_errors(rt, synth_models):
    seg = _segmenter(rt, synth_models)
    with pytest.raises(ValueError, match='calibration_sec'):
        seg.stream(calibration_sec=0.5)
    live = seg.stream(calibration_sec=1.0)
    x = synth_audio(3, seed=1)
    live.feed({'a': x[:1000]})
    with pytest.raises(TypeError, match='opened with'):
        live.feed({'a': x[1000:2000].astype(np.float32)})
    with pytest.raises(TypeError, match='opened with'):
        live.feed({'a': torch.from_numpy(x[1000:2000]).cuda()})
    with pytest.raises(ValueError, match='16 kHz'):
        live.feed({'a': x[1000:2000]}, sample_rate=8000)
    with pytest.raises(TypeError):
        live.feed({'b': x.astype(np.float64)})
    with pytest.raises(KeyError):
        live.end(['nope'])
    live.feed({'c': x[:399]})
    with pytest.raises(ValueError, match='holds 399 samples'):
        live.end(['c'])
    assert live.end(['a'])['a'] == seg.segment_signal(x[:1000])


def test_cnn_on_retained_rows_equals_whole_recording(rt, synth_models, monkeypatch):
    """Patches of a stream read from a buffer that holds its rows from an even frame R0 on are padded patches p - R0/2
    of that buffer for iss_cnn_forward_multi (both edges replicated): at the stream start (R0 = 0, left replicas), in
    the middle (no replica) and at the end (right replicas)."""
    seg = _segmenter(rt, synth_models)
    stream = rt['stream']
    lib = rt['lib'].load()
    x = synth_audio(40, seed=4)
    m, _, _ = rt['segmenter'].feats_from_signal(x, 0, seg.fft_precision, 'main')
    L = m.shape[0]
    cases = [(0, 1000), (600, 2201), (1400, L)]            # (R0, frames so far): start, middle, end
    bufs, row_off, lens, rec, ranges, absolute = [], [], [], [], [], []
    pos = 0
    for i, (R0, F) in enumerate(cases):
        bufs.append(m[R0:F])
        row_off.append(pos)
        lens.append(F - R0)
        pos += F - R0
        a = R0 // 2 + (17 if R0 else 0)
        b = rt['pack'].num_patches(L) if F == L else stream.computable_patches(F)
        ranges.append((a - R0 // 2, b - R0 // 2))
        rec.append(i)
        absolute.append((a, b))
    packed = torch.cat(bufs).contiguous()
    mode0 = lib.iss_get_gemm_mode()
    try:
        for fuse in ('0', '1'):
            monkeypatch.setenv('ISS_B200_FUSE_FIRST', fuse)
            for mode in (3, 2, 0):
                lib.iss_set_gemm_mode(mode)
                for nn in (seg.vad.nn, seg.gender.nn):
                    got = nn.forward_multi(packed, row_off, lens, rec, ranges).cpu().numpy()
                    ref = nn.forward(m, absolute).cpu().numpy()
                    if fuse == '0':
                        assert np.array_equal(got, ref), (mode, nn.nmel)
                    else:
                        assert float(np.abs(got - ref).max()) <= 1e-6, (mode, nn.nmel)
    finally:
        lib.iss_set_gemm_mode(mode0)


def test_online_kernel_rejects_out_of_range_chains(rt, synth_models):
    seg = _segmenter(rt, synth_models)
    engine, lib = rt['engine'], rt['lib']
    probs = torch.full((10, 2), 0.5, dtype=torch.float32, device='cuda')
    scores = torch.zeros((2, 4), dtype=torch.float64, device='cuda')
    hist = torch.zeros((2, 64), dtype=torch.uint8, device='cuda')
    trans = engine.diag_trans_exp(80, 2)
    S = engine.ONLINE_START
    bad = {'negative field': [-1, 5, 0, 0, 0, S],
           'outside d_src ': [8, 5, 0, 0, 0, S],
           'slot': [0, 5, 2, 0, 0, S],
           'history capacity': [0, 5, 1, 60, 0, 0]}
    for what, row in bad.items():
        with pytest.raises(lib.IssError, match=what.strip()):
            engine.viterbi_online(seg.ctx, np.array([row]), probs, scores, hist, 70, K=2, trans=trans)
    with pytest.raises(lib.IssError, match='outside d_out'):
        engine.viterbi_online(seg.ctx, np.array([[0, 5, 0, 0, 0, S]]), probs, scores, hist, 4, K=2, trans=trans)
    buf = engine.viterbi_online(seg.ctx, np.array([[0, 5, 0, 0, 0, S | engine.ONLINE_END]]), probs, scores, hist, 5,
                                K=2, trans=trans)
    nd, st = engine.split_online(buf.cpu().numpy(), 1)
    assert nd[0] == 5 and not st[:5].any()
