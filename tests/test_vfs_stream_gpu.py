"""Live femininity scores on the GPU (run with -m gpu on an H100): the dither generator against numpy's RandomState(3),
the windowed VBx front end against iss_vbx_features on the whole stream, and every stream's final score against the
offline score on its live VAD segments."""
import ctypes
import os

import numpy as np
import pytest

from conftest import synth_audio
from test_vfs_pack_gpu import samples_for, vfs_models

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')


@pytest.fixture(scope='module')
def rt():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from inaspeechsegmenter_b200 import _lib, engine, vbx_segmenter as vb, vfs_stream as vs
    ctx = engine.Context(0)
    return dict(lib=_lib, vb=vb, vs=vs, ctx=ctx, fe=vb.VbxFrontEnd(ctx))


@pytest.fixture(scope='module')
def vfs(rt, synth_models):
    return rt['vb'].VoiceFemininityScoring(ffmpeg=None, models=vfs_models(synth_models))


def _dither_ref(n):
    return 8 * (np.random.RandomState(3).rand(n) * 2 - 1)


def _draw(rt, table, recs):
    lib = rt['lib']
    r = np.ascontiguousarray(recs, dtype=np.int64).reshape(-1, 3)
    out = torch.full((int(r[:, 1].sum()) + 1,), np.nan, dtype=torch.float64, device='cuda')
    rc = lib.load().iss_dither_mt19937_multi(rt['ctx'].handle, len(r), lib.ptr(r), lib.ptr(table), table.shape[0],
                                             lib.ptr(out), None)
    return rc, out.cpu().numpy()


def test_dither_generator_equals_randomstate(rt):
    """Many streams in one launch, each drawn in its own chunking, across 312-double twist boundaries."""
    seed = torch.from_numpy(rt['vs']._mt_seed()).cuda()
    cuts = [[1, 311, 1, 312, 5000], [312] * 4 + [7], [623, 1, 2, 3000], [16000, 16000], [0, 313, 0, 311]]
    table = seed.repeat(len(cuts), 1).contiguous()
    ref = _dither_ref(40000)
    pos = [0] * len(cuts)
    for step in range(max(len(c) for c in cuts)):
        recs, off = [], 0
        for s, c in enumerate(cuts):
            if step < len(c):
                recs.append((s, c[step], off))
                off += c[step]
        rc, got = _draw(rt, table, recs)
        assert rc == 0
        for s, n, o in recs:
            assert np.array_equal(got[o:o + n], ref[pos[s]:pos[s] + n]), (s, step)
            pos[s] += n


def test_dither_generator_rejects_bad_records(rt):
    table = torch.from_numpy(rt['vs']._mt_seed()).cuda().repeat(2, 1).contiguous()
    before = table.clone()
    lib = rt['lib'].load()
    c0 = lib.iss_launch_count()
    for recs in ([(2, 10, 0)], [(-1, 10, 0)], [(0, 10, 0), (0, 5, 10)], [(0, -1, 0)]):
        rc, _ = _draw(rt, table, recs)
        assert rc != 0
    r = np.array([[0, 10, 0]], dtype=np.int64)
    assert lib.iss_dither_mt19937_multi(rt['ctx'].handle, 1, rt['lib'].ptr(r), rt['lib'].ptr(table), 1 << 31,
                                        rt['lib'].ptr(table), None) != 0
    assert lib.iss_launch_count() == c0
    assert torch.equal(table, before)
    # a position the table cannot hold (odd, or past 624) is read as 624: the draw twists first and goes on
    for bad in (3, 625, -1):
        table[0] = torch.from_numpy(rt['vs']._mt_seed()).cuda()
        table[0, 624] = bad
        rc, got = _draw(rt, table, [(0, 700, 0)])
        assert rc == 0 and np.array_equal(got[:700], _dither_ref(700)), bad


def _stream_rows(rt, sig, cuts, where='host'):
    """The windowed K4 driven as LiveScores drives it, over one stream cut at `cuts`: the rows of every call."""
    vs = rt['vs']
    be = vs.CudaBackend.__new__(vs.CudaBackend)
    be.ctx, be.dev = rt['ctx'], rt['ctx'].device
    from inaspeechsegmenter_b200.segmenter import _stage_pass
    be._stage_pass = _stage_pass
    be.seed = torch.from_numpy(vs._mt_seed()).to(be.dev)
    be.mt = torch.zeros((0, 625), dtype=torch.int32, device=be.dev)
    be.tails, be.dtype, be.raw_at, be.fea_at = {}, {}, {}, {}
    be.raw = torch.empty((0, 64), dtype=torch.float64, device=be.dev)
    be.fea = torch.empty((0, 64), dtype=torch.float32, device=be.dev)
    be.open(0)
    n = R = T = 0
    keep = (0, 0, 0)
    got = []
    bounds = list(cuts) + [len(sig)]
    a = 0
    whole = torch.from_numpy(np.ascontiguousarray(sig)).cuda() if where == 'cuda' else sig
    for i, b in enumerate(bounds):
        c = whole[a:b]                  # CUDA chunks are views at any offset
        a = b
        end = i == len(bounds) - 1
        n += len(c)
        R2 = vs.vbx_frames(n) if end else vs.final_raw_rows(n)
        T2 = R2 if end else vs.final_cmvn_rows(R2)
        be.features({0: (c, n, (R, R2 - R), (T, T2 - T), end, (vs.sample_keep(R2), vs.raw_keep(T2, R2), None))},
                    {0: keep})
        f0, nf, off = be.fea_at[0]
        assert f0 <= T and f0 + nf == T2
        got.append(be.fea[off + T - f0:off + nf].cpu())
        keep = (vs.sample_keep(R2), vs.raw_keep(T2, R2), T2)      # features kept only from the rows still to come
        R, T = R2, T2
    return torch.cat(got)


@pytest.mark.parametrize('fmt', ['int16', 'float32'])
@pytest.mark.parametrize('where', ['host', 'cuda'])
def test_windowed_k4_equals_whole_stream(rt, fmt, where):
    x = synth_audio(30, seed=31)
    sig = x if fmt == 'int16' else x.astype(np.float32) / np.float32(32768)
    rng = np.random.default_rng(5)
    ref = rt['fe'](torch.from_numpy(np.ascontiguousarray(sig)).cuda()).cpu()
    for how in (1999, 160, 16001, 'random', 'one'):
        if how == 'one':
            cuts = []
        elif how == 'random':
            cuts = sorted(set(rng.integers(1, len(sig), 40).tolist()))
        else:
            cuts = list(range(how, len(sig), how))
        assert torch.equal(_stream_rows(rt, sig, cuts, where), ref), how


@pytest.mark.parametrize('M', [127, 128, 129, 143, 144, 145, 299, 300, 301, 450])
def test_windowed_k4_boundary_lengths(rt, M):
    """Streams that end with M < 300, at the 128-row chunk and window boundaries, fed in small chunks."""
    x = synth_audio(6, seed=M)[:samples_for(M, 37)]
    ref = rt['fe'](torch.from_numpy(x).cuda()).cpu()
    for how in (159, 160, 161, 399, 400):
        assert torch.equal(_stream_rows(rt, x, list(range(how, len(x), how))), ref), how


def test_windowed_k4_rejects_out_of_window_records(rt):
    lib, ctx = rt['lib'], rt['ctx']
    L = lib.load()
    pcm = torch.zeros(4000, dtype=torch.int16, device='cuda')
    raw = torch.zeros((64, 64), dtype=torch.float64, device='cuda')
    fea = torch.zeros((64, 64), dtype=torch.float32, device='cuda')
    P = (ctypes.c_void_p * 1)(pcm.data_ptr())
    D = (ctypes.c_void_p * 1)(None)
    c0 = L.iss_launch_count()
    # 4000 samples: M = 25 rows once the stream has ended
    for w in ([200, 4000, 1, 1, 0, 0],          # row 1 reads sample 40, before the window
              [0, 4000, 23, 2, 0, 0],           # row 24 reads sample 4119 and the stream is open
              [0, 4000, 24, 1, 0, 1],           # the last row once the stream has ended: accepted
              [0, 4000, 25, 1, 0, 1]):          # past the last row
        w = np.array(w, dtype=np.int64)
        rc = L.iss_vbx_fbank_window_multi(ctx.handle, 1, P, D, lib.ptr(w), lib.PCM_S16, lib.ptr(raw), None)
        assert (rc != 0) == (w[2] != 24), w
    c1 = L.iss_launch_count()
    assert c1 - c0 == 1
    for w in ([0, 299, 0, 10, 0, 0, 0],         # open stream under 300 rows
              [0, 400, 200, 52, 0, 0, 0],       # row 251 is not final with 400 rows (251 + 150 > 400)
              [60, 400, 200, 10, 0, 0, 0],      # the chunk of row 200 starts at row 128, whose window starts at row 0
              [0, 400, 400, 1, 0, 0, 1]):       # row 400 of 400 rows
        w = np.array(w, dtype=np.int64)
        rc = L.iss_vbx_cmvn_window_multi(ctx.handle, 1, lib.ptr(w), lib.ptr(raw), lib.ptr(fea), None)
        assert rc != 0, w
    assert L.iss_launch_count() == c1


# ------------------------------------------------------------------ the scorer
def _media(media, name):
    from inaspeechsegmenter_b200.io import media2sig16kmono
    return media2sig16kmono(os.path.join(media, name), None, None, None, 'float32', return_int16=True)


def _feed_all(live, sigs, how, rate=16000, seed=0):
    """Feed every stream of `sigs` in the same calls, cut `how` (in frames of the stream's rate: `rate`, or a dict
    {key: rate}); returns (windows per key, end results)."""
    rng = np.random.default_rng(seed)
    parts = {}
    for k, x in sigs.items():
        r = rate[k] if isinstance(rate, dict) else rate
        if how == 'one':
            parts[k] = [x]
        elif how == 'random':
            out, pos = [], 0
            while pos < len(x):
                n = int(rng.uniform(0.05, 3.0) * r)
                out.append(x[pos:pos + n])
                pos += n
            parts[k] = out
        else:
            parts[k] = [x[i:i + how] for i in range(0, len(x), how)]
    wins = {k: [] for k in sigs}
    for step in range(max(len(p) for p in parts.values())):
        feed = {k: p[step] for k, p in parts.items() if step < len(p)}
        got = live.feed(feed, sample_rate={k: rate[k] for k in feed} if isinstance(rate, dict) else rate)
        for k, v in got.items():
            wins[k] += v
    return wins, live.end(list(sigs))


def _same(a, b):
    if isinstance(a, Exception) or isinstance(b, Exception):
        return type(a) is type(b)
    return a == b


def test_short_streams_equal_score_signal(rt, vfs, media):
    """Streams of at most N_cal frames: the golden media, boundary lengths, and musanmix at 48 kHz stereo."""
    sigs = {f: _media(media, f) for f in ('musanmix.wav', 'silence2sec.wav', 'lamartine.wav')}
    base = synth_audio(40, seed=9)
    for M in (143, 144, 145, 300, 301):
        sigs['M%d' % M] = base[:samples_for(M)]
    for how in ('one', 16000, 'random'):
        _, got = _feed_all(vfs.stream(calibration_sec=75.0), sigs, how)
        for k, x in sigs.items():
            try:
                ref = vfs.score_signal(x)
            except ZeroDivisionError as e:
                ref = e
            assert _same(got[k], ref), (k, how, got[k], ref)
    m = sigs['musanmix.wav']
    x48 = np.stack([np.repeat(m, 3), np.repeat(m // 2, 3)], axis=1)
    _, got = _feed_all(vfs.stream(calibration_sec=75.0), {'s': x48}, 24000, rate=48000)
    assert got['s'] == vfs.score_signal(x48, sample_rate=48000)


def _prefix_reference(vfs, x, segs, vad_thresh):
    """The offline score on the live VAD segments: score_signal's x-vectors, selection rule and MLP."""
    vb = __import__('inaspeechsegmenter_b200.vbx_segmenter', fromlist=['x'])
    speech = [(b, e) for lab, b, e in segs if lab == 'speech']
    dur = sum(e - b for b, e in speech)
    if not dur:
        return None, dur, 0
    pcm = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    xv = vfs.xvector_model('s', vfs.frontend(pcm), len(x) / 16000)
    kept = vfs.apply_vad(xv, speech)
    p = vfs.gender_detection_mlp_model.predict(np.asarray([v for _, _, v in kept]))
    try:
        score, nb = vb.score_kept([seg for _, seg, _ in kept], p)
    except ZeroDivisionError as e:
        return e
    return score, dur, nb


def test_long_stream_equals_prefix_vad_reference(rt, vfs, media):
    """A 3-minute stream with a 5 s calibration, in several chunkings: the offline score on its live VAD segments."""
    x = np.tile(_media(media, 'musanmix.wav'), 3)[:180 * 16000]
    segs = vfs.vad.stream(calibration_sec=5.0)
    got_segs = []
    for i in range(0, len(x), 16000):
        got_segs += segs.feed({'s': x[i:i + 16000]})['s']
    got_segs += segs.end(['s'])['s']
    ref = _prefix_reference(vfs, x, got_segs, vfs.vad_thresh)
    assert not isinstance(ref, Exception) and ref[2] > 10
    for how in (16000, 'random', 4321):
        wins, got = _feed_all(vfs.stream(calibration_sec=5.0), {'s': x}, how)
        assert got['s'] == ref, how
        assert all(a < b for a, b in zip(wins['s'], wins['s'][1:]))


def test_many_streams_equal_streams_alone(rt, vfs, media):
    """300 streams of mixed formats and lengths in one object: int16 and float32 host arrays, int16 and float32 CUDA
    views at unaligned offsets, 48 kHz stereo and 44.1 kHz mono streams (resampled by the VAD's live streams, whose
    16 kHz chunks the scorer continues from).  Each gets what it gets alone."""
    rng = np.random.default_rng(3)
    m = _media(media, 'musanmix.wav')
    base = np.tile(m, 3)
    dev = torch.from_numpy(base).cuda()
    devf = torch.from_numpy(base.astype(np.float32) / np.float32(32768)).cuda()
    b48 = np.stack([np.repeat(m, 3), np.repeat(m // 2, 3)], axis=1)
    b44 = synth_audio(40, seed=45, sr=44100).astype(np.float32) / np.float32(32768)
    sigs, rates = {}, {}
    for i in range(300):
        sec = float(rng.uniform(0.3, 14.0))
        kind = i % 6
        rate = {4: 48000, 5: 44100}.get(kind, 16000)
        n = int(sec * rate)
        src = {0: base, 1: base, 2: dev, 3: devf, 4: b48, 5: b44}[kind]
        a = int(rng.integers(0, len(src) - n)) | 1                      # odd offsets: unaligned CUDA views
        x = src[a:a + n]
        sigs[i] = x.astype(np.float32) / np.float32(32768) if kind == 0 else x
        rates[i] = rate
    _, together = _feed_all(vfs.stream(calibration_sec=3.0), sigs, 'random', rate=rates, seed=1)
    scored = 0
    for i in list(range(6)) + list(range(6, 300, 10)):
        _, alone = _feed_all(vfs.stream(calibration_sec=3.0), {i: sigs[i]}, 8000, rate=rates)
        assert _same(together[i], alone[i]), i
        scored += isinstance(alone[i], tuple) and alone[i][0] is not None
    assert scored >= 10


def test_launch_count_does_not_grow_with_streams(rt, vfs):
    lib = rt['lib'].load()
    x = synth_audio(60, seed=47)
    counts = []
    for N, C in ((40, 32000), (80, 16000)):
        live = vfs.stream(calibration_sec=2.0)
        off = [(i * 7919) % (len(x) - 40 * C) for i in range(N)]
        for step in range(8):
            live.feed({i: x[off[i] + step * C:off[i] + (step + 1) * C] for i in range(N)})
        c0 = lib.iss_launch_count()
        live.feed({i: x[off[i] + 8 * C:off[i] + 9 * C] for i in range(N)})
        counts.append(lib.iss_launch_count() - c0)
    assert counts[0] == counts[1], counts


def test_errors_leave_state_unchanged(rt, vfs):
    live = vfs.stream(calibration_sec=2.0)
    x = synth_audio(8, seed=53)
    live.feed({'a': x[:48000]})

    def state():
        st, be, ls = live.streams['a'], live.backend, live.live.streams['a']
        return ((st.n, st.R, st.T, st.w, st.keep, list(st.speech), len(st.wins)), be.mt[st.sid].clone(),
                tuple(t.data_ptr() for t in be.tails[st.sid][:2]), be.tails[st.sid][2], dict(be.raw_at),
                dict(be.fea_at), be.raw.data_ptr(), be.fea.data_ptr(), (ls.samples, ls.F, ls.fin, ls.open),
                set(live.streams), set(live.live.streams))

    before = state()
    with pytest.raises(TypeError):
        live.feed({'a': x[48000:64000].astype(np.float32)})
    with pytest.raises(TypeError):
        live.feed({'a': x[48000:64000], 'b': x[:100].astype(np.float64)})
    with pytest.raises(ValueError):
        live.feed({'a': x[48000:64000]}, sample_rate=44100)
    after = state()
    assert after[0] == before[0] and torch.equal(after[1], before[1]) and after[2:] == before[2:]
    with pytest.raises(KeyError):
        live.end(['zz'])
    live.feed({'a': x[48000:]})
    got = live.end(['a'])['a']
    ref = vfs.stream(calibration_sec=2.0)
    ref.feed({'a': x})
    assert got == ref.end(['a'])['a']
    with pytest.raises(ValueError):
        live2 = vfs.stream(calibration_sec=2.0)
        live2.feed({'s': x[:300]})
        live2.end(['s'])
    assert 's' not in live2.streams
