"""Segmenter.segment_signals and the multi-recording entry points on the GPU: every recording of a packed pass gives
exactly what the single-recording calls give it (run with -m gpu on an H100)."""
import os
import warnings

import numpy as np
import pytest

from conftest import synth_audio

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')

LONG_SAMPLES = (65536 - 1) * 160 + 400 + 1234          # 65536 frames: routed to segment_signal


def _as(sig, fmt):
    """A recording as int16 or float32 samples (lamartine.wav is stored as float32)."""
    if fmt == 'float32':
        return sig if sig.dtype == np.float32 else sig.astype(np.float32) / np.float32(32768)
    return sig if sig.dtype == np.int16 else np.clip(np.round(sig * 32768), -32768, 32767).astype(np.int16)


def _media(media, name):
    from inaspeechsegmenter_b200.io import media2sig16kmono
    return media2sig16kmono(os.path.join(media, name), None, None, None, 'float32', return_int16=True)


@pytest.fixture(scope='module')
def rt():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from inaspeechsegmenter_b200 import _lib, engine, pack, segmenter
    return dict(lib=_lib, engine=engine, pack=pack, segmenter=segmenter)


@pytest.fixture(scope='module')
def recordings(media):
    """Sample counts at the frame boundaries, a 0.5 s clip (48 frames < 68), odd and even L, silence, 2 s / 10 s /
    3 min (more than one 8192-patch sweep) and the three golden media files; int16 but lamartine.wav (float32), none
    routed."""
    base = synth_audio(200, seed=7)
    sigs = [base[:400], base[1000:1559], base[3000:3560], base[5000:5719], base[9000:9720],
            base[20000:28000],                     # 0.5 s
            base[40000:56000],                     # 2 s, L = 98 (even)
            base[60000:76160],                     # L = 99 (odd)
            np.zeros(32000, dtype=np.int16),       # all-zero: NaN threshold, no energy segment
            synth_audio(10, seed=8), synth_audio(180, seed=9)]
    sigs += [_media(media, f) for f in ('musanmix.wav', 'silence2sec.wav', 'lamartine.wav')]
    return sigs


@pytest.fixture(scope='module')
def long_recording():
    return synth_audio(LONG_SAMPLES / 16000, seed=10)


def _segmenter(rt, synth_models, vad='smn', gender=True, fft='fp64'):
    return rt['segmenter'].Segmenter(vad_engine=vad, detect_gender=gender, ffmpeg=None, fft_precision=fft,
                                     models={'vad': synth_models[vad], 'gender': synth_models['gender']})


@pytest.mark.parametrize('fft', ['fp64', 'fp32'])
@pytest.mark.parametrize('fmt', ['int16', 'float32'])
def test_features_stats_and_energy_bit_identical(rt, synth_models, recordings, fft, fmt):
    seg = _segmenter(rt, synth_models, fft=fft)
    pack, engine = rt['pack'], rt['engine']
    sigs = [_as(s, fmt) for s in recordings]
    pcms = [torch.from_numpy(s).cuda() for s in sigs]
    lay = pack.PassLayout([len(s) for s in sigs], pcms[0].element_size())
    fe = rt['segmenter']._get_frontend('main', 0)
    mspec, loge, stats = fe.multi(pcms, lay, seg.fft_precision)
    track = engine.energy_viterbi_multi(seg.ctx, loge, lay.loge_off, stats, seg.energy_ratio, lay.out_off)
    for i, pcm in enumerate(pcms):
        m1, l1, s1 = fe(pcm, seg.fft_precision)
        L = int(lay.frames[i])
        a = int(lay.row_off[i])
        assert torch.equal(mspec[a:a + L], m1), i
        assert torch.equal(loge[lay.loge_off[i]:lay.loge_off[i + 1]], l1), i
        assert torch.equal(stats[i], s1), i
        t1 = engine.energy_viterbi(seg.ctx, l1, s1, seg.energy_ratio, out_stride=2)
        assert torch.equal(track[lay.out_off[i]:lay.out_off[i + 1]], t1), i


def test_energy_multi_refuses_long_recordings(rt, synth_models):
    seg = _segmenter(rt, synth_models)
    loge = torch.zeros(65536 + 10, dtype=torch.float32, device='cuda')
    stats = torch.tensor([[1.0, 1.0], [1.0, 1.0]], dtype=torch.float64, device='cuda')
    with pytest.raises(rt['lib'].IssError, match='65536'):
        rt['engine'].energy_viterbi_multi(seg.ctx, loge, [0, 10, 65546], stats, 0.03, [0, 5, 32773])


def _packed_cnn_case(rt, seg, sigs):
    """Single-recording padded features, their packed copy and the energy ranges of every recording."""
    feats = [rt['segmenter'].feats_from_signal(s, 0, seg.fft_precision, 'main') for s in sigs]
    lay = rt['pack'].PassLayout([len(s) for s in sigs])
    mspec = torch.cat([m for m, _, _ in feats]).contiguous()
    assert mspec.shape[0] == lay.total_rows
    ranges, rec, per = [], [], []
    for i, (m, loge, difflen) in enumerate(feats):
        r = [(a, b) for lab, a, b in seg.energy_segments(loge) if lab == 'energy']
        if i % 3 == 0:                     # also whole recordings, replicated ends included
            r = r + [(0, rt['pack'].num_patches(m.shape[0]) - int(difflen / 2))]
        ranges += r
        rec += [i] * len(r)
        per.append((m, r))
    return lay, mspec, ranges, rec, per


def test_cnn_multi_equals_single(rt, synth_models, recordings, monkeypatch):
    seg = _segmenter(rt, synth_models)
    lib = rt['lib'].load()
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        lay, mspec, ranges, rec, per = _packed_cnn_case(rt, seg, recordings)
    mode0 = lib.iss_get_gemm_mode()
    worst = {}
    try:
        for fuse in ('0', '1'):
            monkeypatch.setenv('ISS_B200_FUSE_FIRST', fuse)
            for mode in (3, 2, 0):
                lib.iss_set_gemm_mode(mode)
                for nn in (seg.vad.nn, seg.gender.nn):
                    got = nn.forward_multi(mspec, lay.row_off, lay.rows, rec, ranges).cpu().numpy()
                    ref = np.concatenate([nn.forward(m, r).cpu().numpy() for m, r in per if r])
                    assert got.shape == ref.shape
                    if fuse == '0':
                        assert np.array_equal(got, ref), (mode, nn.nmel)
                    else:
                        err = float(np.abs(got - ref).max())
                        worst[(mode, nn.nmel)] = err
                        assert err <= 1e-6, (mode, nn.nmel, err)
    finally:
        lib.iss_set_gemm_mode(mode0)
    print('fused first layer, packed vs single, max |diff| per (mode, nmel):', worst)


@pytest.mark.parametrize('vad,gender,fft,inp', [
    ('smn', True, 'fp64', 'int16'),
    ('sm', True, 'fp64', 'float32'),
    ('smn', False, 'fp32', 'int16'),
    ('sm', False, 'fp32', 'cuda'),
    ('smn', True, 'fp32', 'cuda'),
])
def test_segment_signals_equals_segment_signal(rt, synth_models, recordings, long_recording, vad, gender, fft, inp):
    seg = _segmenter(rt, synth_models, vad, gender, fft)
    sigs = list(recordings)
    sigs.insert(5, long_recording)
    if inp == 'float32':
        sigs = [_as(s, 'float32') for s in sigs]
    elif inp == 'cuda':
        sigs = [torch.from_numpy(s).cuda() for s in sigs]
    starts = [0.5 * i for i in range(len(sigs))]
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        got = seg.segment_signals(sigs, starts)
        ref = [seg.segment_signal(s, t) for s, t in zip(sigs, starts)]
        assert got == ref
        assert seg.segment_signals(sigs[6:9]) == [seg.segment_signal(s) for s in sigs[6:9]]


def test_mixed_formats_come_back_in_order(rt, synth_models, recordings):
    seg = _segmenter(rt, synth_models)
    sigs = [_as(s, 'float32' if i % 2 else 'int16') for i, s in enumerate(recordings)]
    sigs[3] = torch.from_numpy(recordings[3]).cuda()
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        assert seg.segment_signals(sigs) == [seg.segment_signal(s) for s in sigs]


def test_500_clips_in_one_pass(rt, synth_models):
    seg = _segmenter(rt, synth_models)
    rng = np.random.default_rng(5)
    audio = synth_audio(1500, seed=11)
    clips, pos = [], 0
    for _ in range(500):
        n = int(rng.integers(16000, 48000))
        clips.append(audio[pos:pos + n])
        pos += n
    passes, long_ = rt['pack'].plan_passes([len(c) for c in clips], ['int16'] * 500)
    assert len(passes) == 1 and not long_
    assert seg.segment_signals(clips) == [seg.segment_signal(c) for c in clips]


def test_launch_count_does_not_grow_with_clips(rt, synth_models):
    seg = _segmenter(rt, synth_models)
    lib = rt['lib'].load()
    audio = synth_audio(400, seed=12)
    clips = [audio[i * 32000:(i + 1) * 32000] for i in range(100)]
    seg.segment_signals(clips[:10])
    counts = {}
    for k in (10, 100):
        c0 = lib.iss_launch_count()
        seg.segment_signals(clips[:k])
        counts[k] = lib.iss_launch_count() - c0
    # 100 clips of 2 s are ~5000 patches per network: one CNN sweep each, the same launches as 10 clips up to the
    # fused first layer (two launches instead of one), which each network's sweep may or may not take
    assert abs(counts[100] - counts[10]) <= 2, counts
    c0 = lib.iss_launch_count()
    seg.segment_signal(clips[0])
    assert counts[100] <= 2 * (lib.iss_launch_count() - c0), counts


def test_errors_and_empty_list(rt, synth_models, recordings):
    seg = _segmenter(rt, synth_models)
    assert seg.segment_signals([]) == []
    with pytest.raises(ValueError, match='<signal 1> holds 399 samples'):
        seg.segment_signals([recordings[0], recordings[0][:399]])
