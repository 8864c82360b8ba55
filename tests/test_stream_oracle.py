"""The live-stream state machine (stream.LiveStreams: chain planning, row retention, label tracks, segment emission)
driven by a CPU oracle backend, against oracle/segmenter_oracle.py: with the calibration-prefix energy threshold for
streams longer than the calibration, and exactly the reference segmentation for shorter ones."""
import warnings
from types import SimpleNamespace

import numpy as np
import pytest

from conftest import synth_audio
from oracle import cnn_oracle
from oracle import segmenter_oracle as so
from oracle import sidekit_oracle as sk
from stream_oracle import OracleStreamBackend, segment_reference
from inaspeechsegmenter_b200 import models
from inaspeechsegmenter_b200.stream import LiveStreams

RATIO = 0.03


@pytest.fixture(scope='module')
def nets():
    vad = cnn_oracle.KerasLikeModel(*models.synthetic_keras_cnn(21, 3, seed=11, width=0.25), threads=2)
    gen = cnn_oracle.KerasLikeModel(*models.synthetic_keras_cnn(24, 2, seed=13, width=0.25), threads=2)
    return {'vad': (vad.predict, 21, ('speech', 'music', 'noise'), 80),
            'gender': (gen.predict, 24, ('female', 'male'), 80)}


def _live(nets, cal, gender=True):
    use = dict(nets) if gender else {'vad': nets['vad']}
    seg = SimpleNamespace(vad=SimpleNamespace(outlabels=nets['vad'][2]), gender=SimpleNamespace(outlabels=nets['gender'][2]),
                          detect_gender=gender)
    return LiveStreams(seg, cal, backend=OracleStreamBackend(RATIO, use)), use


def _cut(x, how, rng):
    if how == 'random':
        out, pos = [], 0
        while pos < len(x):
            n = int(rng.uniform(0.01, 3.0) * 16000)
            out.append(x[pos:pos + n])
            pos += n
        return out
    return [x] if how == 'one' else [x[i:i + how] for i in range(0, len(x), how)]


def _run_together(live, sigs, hows, seed=0):
    """Feed several streams in the same calls, each cut its own way; returns every stream's segments in order."""
    rng = np.random.default_rng(seed)
    parts = {k: _cut(x, h, rng) for (k, x), h in zip(sigs.items(), hows)}
    got = {k: [] for k in sigs}
    step = 0
    while any(step < len(p) for p in parts.values()):
        feed = {k: p[step] for k, p in parts.items() if step < len(p)}
        for k, v in live.feed(feed).items():
            got[k] += v
        step += 1
    for k, v in live.end(list(sigs)).items():
        got[k] += v
    return got


@pytest.mark.parametrize('gender', [True, False])
def test_streams_equal_prefix_threshold_oracle(nets, gender):
    x = synth_audio(150, seed=9)
    mspec, loge = sk.logmel_loge(x.astype(np.float32) / np.float32(32768))
    live, use = _live(nets, 5.0, gender)
    ref = segment_reference(mspec, loge, 500, RATIO, use)
    assert any(lab == 'noEnergy' for lab, _, _ in ref) and len(ref) > 10
    got = _run_together(live, {'1s': x, 'random': x, 'quarter': x, 'one': x}, [16000, 'random', 4000, 'one'])
    for k, segs in got.items():
        assert segs == ref, k


def test_streams_shorter_than_calibration_equal_reference(nets):
    base = synth_audio(30, seed=7)
    sigs = {i: s for i, s in enumerate([base[:400], base[1000:1559], base[5000:5719], base[20000:28000],
                                        base[40000:56000], base[60000:76160], np.zeros(32000, dtype=np.int16),
                                        base[100000:420000]])}
    live, use = _live(nets, 25.0)
    vad = so.DnnSegmenterOracle(use['vad'][0], **so.VAD_SMN)
    gen = so.DnnSegmenterOracle(use['gender'][0], **so.GENDER)
    got = _run_together(live, sigs, [3000] * len(sigs), seed=1)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        for k, x in sigs.items():
            ref = so.segment_feats(*so.media2feats(x.astype(np.float32) / np.float32(32768)), 0, vad, gen, RATIO)
            assert got[k] == ref, k
    # a stream exactly N_cal frames long is calibrated and decoded online, and still gives the reference
    x = base[:(1000 - 1) * 160 + 400]
    live, _ = _live(nets, 10.0)
    ref = so.segment_feats(*so.media2feats(x.astype(np.float32) / np.float32(32768)), 0, vad, gen, RATIO)
    assert _run_together(live, {'x': x}, [7000])['x'] == ref


def test_failed_call_leaves_the_object_unusable(nets):
    live, _ = _live(nets, 1.0)
    x = synth_audio(4, seed=2)
    live.feed({'a': x[:16000]})

    def boom(*a):
        raise RuntimeError('device failure')
    live.backend.energy = boom
    with pytest.raises(RuntimeError, match='device failure'):
        live.feed({'a': x[16000:32000]})
    with pytest.raises(RuntimeError, match='stopped in a failed call'):
        live.feed({'a': x[32000:]})
    with pytest.raises(RuntimeError, match='stopped in a failed call'):
        live.end(['a'])
    # a chunk rejected before any work does not break the object
    live2, _ = _live(nets, 1.0)
    live2.feed({'a': x[:16000]})
    with pytest.raises(TypeError):
        live2.feed({'a': x[16000:32000].astype(np.float32)})
    live2.feed({'a': x[16000:]})
