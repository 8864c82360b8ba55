"""VoiceFemininityScoring.score_signals and the multi-recording VBx path on the GPU: every recording of a packed pass
gets exactly what the single-recording calls give it (run with -m gpu on an H100)."""
import os
import warnings

import numpy as np
import pytest

from conftest import synth_audio

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')

LONG_SAMPLES = (65536 - 1) * 160 + 400 + 1234          # 65536 sidekit frames: routed to score_signal


def samples_for(M, extra=0):
    """Sample counts with exactly M VBx frames."""
    return 80 + 160 * (M - 1) + extra


def _as(sig, fmt):
    if fmt == 'float32':
        return sig if sig.dtype == np.float32 else sig.astype(np.float32) / np.float32(32768)
    if fmt == 'float64':
        return _as(sig, 'float32').astype(np.float64)
    return sig if sig.dtype == np.int16 else np.clip(np.round(sig * 32768), -32768, 32767).astype(np.int16)


def _media(media, name):
    from inaspeechsegmenter_b200.io import media2sig16kmono
    return media2sig16kmono(os.path.join(media, name), None, None, None, 'float32', return_int16=True)


def _synthetic_mlp(seed=3):
    """A 256-128-64-1 sigmoid MLP in the Keras layout of the reference's gender models."""
    rng = np.random.default_rng(seed)
    L, W = [{'class_name': 'InputLayer', 'config': {'name': 'in', 'batch_input_shape': [None, 256]}}], {}
    dims = [256, 128, 64, 1]
    for i in range(3):
        n = 'dense_%d' % i
        W[n + '/kernel'] = (rng.standard_normal((dims[i], dims[i + 1])) * np.sqrt(1.0 / dims[i])).astype(np.float32)
        W[n + '/bias'] = rng.normal(0, 0.1, dims[i + 1]).astype(np.float32)
        L.append({'class_name': 'Dense', 'config': {'name': n, 'units': dims[i + 1], 'use_bias': True,
                                                    'activation': 'sigmoid' if i == 2 else 'relu'}})
    return {'class_name': 'Sequential', 'config': {'name': 'mlp', 'layers': L}}, W


@pytest.fixture(scope='module')
def rt():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from inaspeechsegmenter_b200 import _lib, engine, pack, vbx_segmenter as vb
    from oracle import vbx_oracle as vx
    ctx = engine.Context(0)
    return dict(lib=_lib, pack=pack, vb=vb, ctx=ctx, fe=vb.VbxFrontEnd(ctx),
                ext=vb.B200BackendExtractor(state_dict=vx.synthetic_resnet101_state(seed=5), ctx=ctx))


@pytest.fixture(scope='module')
def recordings(media):
    """The K4 boundary lengths (200 / 201 / 399 / 400 samples; M = 33-35, 143-170, 300 / 301; 16-frame tiles and 128-frame
    CMVN chunks), a 150-sample recording without frames in the middle, a 2 s clip (under 300 frames) next to a 60 s one,
    and the three golden media files."""
    base = synth_audio(120, seed=7)
    Ms = [33, 34, 35, 143, 144, 145, 150, 167, 168, 169, 170, 300, 301, 16, 17, 127, 128, 129, 257]
    lens = [200, 201, 399, 400] + [samples_for(M) for M in Ms] + [samples_for(300, 159)]
    sigs, pos = [], 0
    for k, n in enumerate(lens):
        sigs.append(base[pos:pos + n])
        pos += n
        if k == 6:
            sigs.append(base[pos:pos + 150])
    sigs += [base[200000:232000], synth_audio(60, seed=8)]
    sigs += [_media(media, f) for f in ('musanmix.wav', 'silence2sec.wav', 'lamartine.wav')]
    return sigs


# ------------------------------------------------------------------ K4
@pytest.mark.parametrize('dither', [True, False])
@pytest.mark.parametrize('fmt', ['int16', 'float32'])
def test_k4_multi_equals_single(rt, recordings, fmt, dither):
    lib, pack = rt['lib'].load(), rt['pack']
    pcms = [torch.from_numpy(_as(s, fmt)).cuda() for s in recordings]
    fea, off = rt['fe'].multi(pcms, dither=dither)
    assert [int(off[i + 1] - off[i]) for i in range(len(pcms))] == [lib.iss_vbx_num_frames(p.numel()) for p in pcms]
    assert list(off) == list(pack.VbxPlan([p.numel() for p in pcms]).fea_off)
    assert 0 in np.diff(off)                                        # the frameless recording
    for i, p in enumerate(pcms):
        assert torch.equal(fea[off[i]:off[i + 1]], rt['fe'](p, dither=dither)), (i, p.numel())


def test_k4_multi_one_recording_and_reordered(rt, recordings):
    """The n = 1 case and a reversed list give the same rows: nothing depends on the neighbours."""
    pcms = [torch.from_numpy(s).cuda() for s in recordings[:12]]
    fea, off = rt['fe'].multi(pcms)
    rev, roff = rt['fe'].multi(pcms[::-1])
    n = len(pcms)
    for i in range(n):
        j = n - 1 - i
        assert torch.equal(fea[off[i]:off[i + 1]], rev[roff[j]:roff[j + 1]]), i
    one, ooff = rt['fe'].multi(pcms[-1:])
    assert torch.equal(one, fea[off[-2]:off[-1]])


# ------------------------------------------------------------------ packed K5
def _tail_case(rt):
    """Features of clips whose tails have many lengths, clips with only a tail window, and longer clips."""
    audio = synth_audio(200, seed=21)
    Ms = [34, 35, 50, 80, 100, 143, 144, 145, 150, 160, 167, 168, 169, 170, 171, 200, 250, 300, 301, 500, 777]
    lens = [samples_for(M) for M in Ms] + [32000, 80000, 160000]
    pos, pcms = 0, []
    for n in lens:
        pcms.append(torch.from_numpy(audio[pos:pos + n]).cuda())
        pos += n
    fea, off = rt['fe'].multi(pcms)
    return pcms, fea, off


def test_packed_k5_equals_call(rt):
    pack, vb, ext = rt['pack'], rt['vb'], rt['ext']
    lib = rt['lib'].load()
    pcms, fea, off = _tail_case(rt)
    plan = pack.VbxPlan([p.numel() for p in pcms])
    assert len(plan.tails) >= 15
    names = ['clip%d' % i for i in range(len(pcms))]
    durs = [p.numel() / 16000 for p in pcms]
    mode0 = lib.iss_get_gemm_mode()
    try:
        for mode in (3, 2, 0):
            lib.iss_set_gemm_mode(mode)
            got = ext.call_packed(fea, plan, names, durs)
            for i in range(len(pcms)):
                ref = ext(names[i], fea[off[i]:off[i + 1]].contiguous(), durs[i])
                assert [(k, s) for k, s, _ in got[i]] == [(k, s) for k, s, _ in ref], (mode, i)
                assert all(np.array_equal(a, b) for (_, _, a), (_, _, b) in zip(got[i], ref)), (mode, i)
    finally:
        lib.iss_set_gemm_mode(mode0)


def test_packed_k5_tail_offsets_are_each_recordings(rt):
    """Each tail group's x-vector of recording i is the embedding of that recording's own last rows."""
    pack, ext = rt['pack'], rt['ext']
    pcms, fea, off = _tail_case(rt)
    plan = pack.VbxPlan([p.numel() for p in pcms])
    reg, tails = ext.embed_packed(fea, plan)
    for n, (recs, starts) in plan.tails.items():
        for pos, i in enumerate(recs):
            alone = ext.embed_windows(fea[off[i + 1] - n:off[i + 1]].contiguous(), [0], n).cpu().numpy()[0]
            assert np.array_equal(tails[n][pos], alone), (n, i)


# ------------------------------------------------------------------ score_signals
def _speech_vad(synth_models, boost=1.5):
    """The smn stand-in with its 'speech' logit raised: the seeded network alone labels almost nothing speech, and the
    x-vector path only runs on recordings with speech."""
    cfg, w = synth_models['smn']
    w = dict(w)
    last = max((k for k in w if k.startswith('dense_') and k.endswith('/bias')), key=lambda k: int(k[6:-5]))
    w[last] = w[last] + np.array([boost, 0, 0], dtype=np.float32)
    return cfg, w


def vfs_models(synth_models):
    """The VAD, MLP and ResNet101 weights of these tests and of tools/vfs_pack_times.py: the speech-biased smn stand-in,
    the synthetic MLP and the seeded synthetic ResNet101 of bench.py."""
    from oracle import vbx_oracle as vx
    return {'vad': _speech_vad(synth_models), 'mlp': _synthetic_mlp(), 'resnet': vx.synthetic_resnet101_state(seed=5)}


def _vfs(rt, synth_models, criteria='bgc'):
    return rt['vb'].VoiceFemininityScoring(criteria, ffmpeg=None, models=vfs_models(synth_models))


def _score_each(vfs, sigs):
    out = []
    for s in sigs:
        try:
            out.append(vfs.score_signal(s.cpu().numpy() if isinstance(s, torch.Tensor) else s))
        except ZeroDivisionError as e:
            out.append(type(e))
    return out


def _check(vfs, sigs):
    """score_signals(sigs) against score_signal on each: the same list, or the exception of the first signal that raises."""
    ref = _score_each(vfs, sigs)
    err = next((r for r in ref if isinstance(r, type)), None)
    try:
        got = vfs.score_signals(sigs)
    except ZeroDivisionError as e:
        got = type(e)
    assert got == (ref if err is None else err)
    return ref


@pytest.fixture(scope='module')
def clips():
    """2-12 s clips, a 0.7 s one, two all-zero clips (no speech) and the golden media."""
    audio = synth_audio(200, seed=31)
    rng = np.random.default_rng(4)
    out, pos = [], 0
    for _ in range(10):
        n = int(rng.integers(32000, 192000))
        out.append(audio[pos:pos + n])
        pos += n
    out.insert(3, np.zeros(48000, dtype=np.int16))
    out.insert(7, audio[pos:pos + 11200])
    out.append(np.zeros(20000, dtype=np.int16))
    return out


@pytest.mark.parametrize('criteria,inp', [('bgc', 'int16'), ('vfp', 'mixed'), ('bgc', 'cuda'), ('vfp', 'float64')])
def test_score_signals_equals_score_signal(rt, synth_models, clips, media, long_recording, criteria, inp):
    vfs = _vfs(rt, synth_models, criteria)
    sigs = list(clips) + [_media(media, f) for f in ('musanmix.wav', 'lamartine.wav')]
    sigs.insert(5, long_recording)
    fmts = ('int16', 'float32', 'float64')
    if inp == 'mixed':
        sigs = [_as(s, fmts[i % 3]) for i, s in enumerate(sigs)]
        sigs[2] = torch.from_numpy(_as(sigs[2], 'int16')).cuda()
    elif inp == 'float64':
        sigs = [_as(s, 'float64') for s in sigs]
    elif inp == 'cuda':
        sigs = [torch.from_numpy(s).cuda() for s in sigs]
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        ref = _check(vfs, sigs)
    print(criteria, inp, ref)
    assert any(r[0] is None for r in ref) and sum(isinstance(r, tuple) and r[0] is not None for r in ref) >= 3, ref


@pytest.fixture(scope='module')
def long_recording():
    return synth_audio(LONG_SAMPLES / 16000, seed=10)


def test_300_clips_in_one_pass(rt, synth_models):
    vfs = _vfs(rt, synth_models)
    rng = np.random.default_rng(6)
    audio = synth_audio(1500, seed=32)
    sigs, pos = [], 0
    for _ in range(320):
        n = int(rng.integers(16000, 64000))
        sigs.append(audio[pos:pos + n])
        pos += n
    passes, long_ = rt['pack'].plan_passes([len(s) for s in sigs], ['int16'] * len(sigs))
    assert len(passes) == 1 and not long_
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        ref = _check(vfs, sigs)
    scored = sum(isinstance(r, tuple) and r[0] is not None for r in ref)
    print('scored clips:', scored, 'of', len(ref))
    assert scored >= 30, scored


def test_empty_list_and_short_input(rt, synth_models, clips):
    vfs = _vfs(rt, synth_models)
    assert vfs.score_signals([]) == []
    with pytest.raises(ValueError, match='<signal 1> holds 399 samples'):
        vfs.score_signals([clips[0], clips[0][:399]])
    with pytest.raises(ValueError):
        vfs.score_signal(clips[0][:399])


def _all_speech(vfs, monkeypatch):
    """Make the VAD call every sample speech, so that windows decide alone what is retained."""
    full = lambda s: [('speech', 0.0, len(s) / 16000)]                       # noqa: E731
    monkeypatch.setattr(vfs.vad, 'segment_signal', full)
    monkeypatch.setattr(vfs.vad, 'segment_signals', lambda sigs: [full(s) for s in sigs])


def test_zero_division_matches_score_signal(rt, synth_models, clips, monkeypatch):
    """A recording with speech but no window (400 samples: 3 VBx frames) raises ZeroDivisionError, as in the reference."""
    vfs = _vfs(rt, synth_models)
    _all_speech(vfs, monkeypatch)
    tiny = clips[0][:400]
    with pytest.raises(ZeroDivisionError):
        vfs.score_signal(tiny)
    with pytest.raises(ZeroDivisionError):
        vfs.score_signals([clips[0], tiny, clips[1]])
    assert vfs.score_signals([clips[0], clips[1]]) == [vfs.score_signal(clips[0]), vfs.score_signal(clips[1])]


SENTINEL = 12345.0


def _poison(vfs, monkeypatch, n_bad):
    """Non-finite x-vectors for the recordings of n_bad samples: their features are tagged in column 0 and the ResNet's
    output rows of windows starting on a tagged row are replaced by NaN, in the single and the packed path alike."""
    fe, ext = vfs.frontend, vfs.xvector_model
    call, multi, embed = type(fe).__call__, type(fe).multi, type(ext).embed_windows

    def call_(self, pcm, dither=True, stream=None):
        fea = call(self, pcm, dither, stream)
        if self is fe and pcm.numel() == n_bad:
            fea[:, 0] = SENTINEL
        return fea

    def multi_(pcms, dither=True, stream=None):
        fea, off = multi(fe, pcms, dither, stream)
        for i, p in enumerate(pcms):
            if p.numel() == n_bad:
                fea[off[i]:off[i + 1], 0] = SENTINEL
        return fea, off

    def embed_(fea, starts, win_len, stream=None):
        emb = embed(ext, fea, starts, win_len, stream)
        bad = fea[torch.as_tensor(np.asarray(starts, dtype=np.int64), device=fea.device), 0] == SENTINEL
        emb[bad] = float('nan')
        return emb

    monkeypatch.setattr(type(fe), '__call__', call_)
    monkeypatch.setattr(fe, 'multi', multi_)
    monkeypatch.setattr(ext, 'embed_windows', embed_)


def test_engine3_error_names_the_signal(rt, synth_models, clips, monkeypatch):
    vfs = _vfs(rt, synth_models)
    lib = rt['lib'].load()
    _all_speech(vfs, monkeypatch)
    sigs = [clips[0], np.zeros(32000, dtype=np.int16), _as(clips[2], 'float32'), synth_audio(4, seed=77)[:54321], clips[5]]
    _poison(vfs, monkeypatch, 54321)
    mode0 = lib.iss_get_gemm_mode()
    try:
        lib.iss_set_gemm_mode(3)
        with pytest.raises(rt['lib'].IssError, match='non-finite'):
            vfs.score_signal(sigs[3])
        with pytest.raises(rt['lib'].IssError, match=r'\(signal 3\)'):
            vfs.score_signals(sigs)
        assert vfs.score_signals(sigs[:3]) == [vfs.score_signal(s) for s in sigs[:3]]
        # the fp32-range engines drop the windows with a warning: no window is left, as score_signal finds
        lib.iss_set_gemm_mode(0)
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            with pytest.raises(ZeroDivisionError):
                vfs.score_signal(sigs[3])
            with pytest.raises(ZeroDivisionError):
                vfs.score_signals(sigs)
    finally:
        lib.iss_set_gemm_mode(mode0)


def test_launch_count_does_not_grow_with_clips(rt, synth_models):
    vfs = _vfs(rt, synth_models)
    lib = rt['lib'].load()
    audio = synth_audio(1400, seed=12)
    speech, silent = [], []
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        for i in range(700):                          # 2 s clips for which score_signal does not raise, half with speech
            c = audio[i * 32000:(i + 1) * 32000]
            try:
                r = vfs.score_signal(c)
            except ZeroDivisionError:
                continue
            (speech if r[1] else silent).append(c)
            if len(speech) >= 50 and len(silent) >= 50:
                break
        assert len(speech) >= 50 and len(silent) >= 50, (len(speech), len(silent))
        clips = [c for pair in zip(speech[:50], silent[:50]) for c in pair]
        vfs.score_signals(clips[:10])
        counts, live = {}, {}
        for k in (10, 100):
            c0 = lib.iss_launch_count()
            res = vfs.score_signals(clips[:k])
            counts[k] = lib.iss_launch_count() - c0
            live[k] = sum(r[1] > 0 for r in res)
        # the ResNet sweeps 256 windows at a time: the regular windows (3 per 2 s clip) of 100 clips take more sweeps than
        # those of 10, which is work, not per-recording overhead
        fea = torch.zeros((200, 64), dtype=torch.float32, device='cuda')
        sweeps = {}
        for k in (10, 100):
            c0 = lib.iss_launch_count()
            vfs.xvector_model.embed_windows(fea, [0] * (3 * live[k]), 144)
            sweeps[k] = lib.iss_launch_count() - c0
        c0 = lib.iss_launch_count()
        vfs.score_signal(clips[0])
        single = lib.iss_launch_count() - c0
    assert live == {10: 5, 100: 50}, live
    assert abs((counts[100] - sweeps[100]) - (counts[10] - sweeps[10])) <= 2, (counts, sweeps)
    assert counts[100] <= 3 * single, (counts, single)
