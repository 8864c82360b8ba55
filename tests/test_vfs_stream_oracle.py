"""The live femininity-score state machine (vfs_stream.LiveScores: row finality, retention, window decisions against
the VAD's decided time, overlap ratios, speech duration, the tail window at the end) driven by CPU oracle backends, the
VAD by stream.LiveStreams on tests/stream_oracle.py's backend, against oracle/vfs_oracle.py's femininity on the whole
stream with that stream's VAD segments."""
import numpy as np
import pytest

from conftest import synth_audio
from oracle import cnn_oracle
from oracle import vbx_oracle as vx
from oracle import vfs_oracle
from stream_oracle import OracleStreamBackend
from test_vfs_pack_gpu import _synthetic_mlp
from vfs_stream_oracle import OracleVfsBackend, StandinNet, whole_features
from inaspeechsegmenter_b200 import models
from inaspeechsegmenter_b200.stream import LiveStreams
from inaspeechsegmenter_b200.vfs_stream import LiveScores

RATIO, THRESH = 0.03, 0.7


@pytest.fixture(scope='module')
def vad():
    cfg, w = models.synthetic_keras_cnn(21, 3, seed=11, width=0.25)
    w = dict(w)
    last = max((k for k in w if k.startswith('dense_') and k.endswith('/bias')), key=lambda k: int(k[6:-5]))
    w[last] = w[last] + np.array([1.5, 0, 0], dtype=np.float32)          # speech-biased, as the GPU tests' VAD
    net = cnn_oracle.KerasLikeModel(cfg, w, threads=2)
    return {'vad': (net.predict, 21, ('speech', 'music', 'noise'), 80)}


def _live(vad, cal):
    from types import SimpleNamespace
    seg = SimpleNamespace(vad=SimpleNamespace(outlabels=vad['vad'][2]), gender=None, detect_gender=False)
    return LiveStreams(seg, cal, backend=OracleStreamBackend(RATIO, vad))


def _cut(x, how, rng):
    if how == 'one':
        return [x]
    if how == 'random':
        out, pos = [], 0
        while pos < len(x):
            n = int(rng.uniform(0.01, 2.5) * 16000)
            out.append(x[pos:pos + n])
            pos += n
        return out
    return [x[i:i + how] for i in range(0, len(x), how)]


def _feed(live, sigs, hows, seed=0, after=None):
    """Feed every stream in the same calls, each cut its own way: (what feed returned per key, what end returned).
    after(got) is called after each feed call."""
    rng = np.random.default_rng(seed)
    parts = {k: _cut(x, h, rng) for (k, x), h in zip(sigs.items(), hows)}
    got = {k: [] for k in sigs}
    for step in range(max(len(p) for p in parts.values())):
        now = live.feed({k: p[step] for k, p in parts.items() if step < len(p)})
        for k, v in now.items():
            got[k] += v
        if after is not None:
            after(now)
    return got, live.end(list(sigs))


def _oracle_windows(x, segs, mlp):
    """(start, stop, overlap ratio, MLP row) of every x-vector window whose midpoint lies in speech, computed from the
    whole stream and its final VAD segments as oracle/vfs_oracle.py computes them."""
    fea = whole_features(x.astype(np.float32) / np.float32(32768))
    speech = [(b, e) for lab, b, e in segs if lab == 'speech']
    out = []
    for _, (a, b), v in vx.extract_xvectors(fea, StandinNet(), 's', len(x) / 16000):
        if any(s < (a + b) / 2 < e for s, e in speech):
            inter = 0.0
            for s, e in speech:
                lo, hi = max(a, s), min(b, e)
                if hi > lo:
                    inter += hi - lo
            out.append((a, b, inter / (b - a), vfs_oracle.mlp_numpy(*mlp, v[None])[0]))
    return out


def _reference(x, segs, mlp):
    """vfs_oracle.femininity on the whole stream: its features (checked against get_features), the stand-in x-vectors
    of vbx_oracle.extract_xvectors, the stream's VAD segments."""
    sig = x.astype(np.float32) / np.float32(32768)
    fea = whole_features(sig)
    assert np.allclose(fea, vx.get_features(sig), rtol=0, atol=1e-4)
    xv = vx.extract_xvectors(fea, StandinNet(), 's', len(x) / 16000)
    try:
        return vfs_oracle.femininity(segs, xv, lambda v: vfs_oracle.mlp_numpy(*mlp, v), THRESH)
    except ZeroDivisionError as e:
        return e


def _same(a, b):
    if isinstance(a, Exception) or isinstance(b, Exception):
        return type(a) is type(b)
    return a == b


def test_live_scores_equal_femininity_oracle(vad):
    """Streams longer than the calibration (one of them float32), one shorter, and one without speech, fed together in
    different chunkings: each stream's end equals the oracle score on its own VAD segments, and the windows returned
    along the way are the ones the score is made of."""
    mlp = _synthetic_mlp()
    base = synth_audio(60, seed=61)
    sigs = {'a': base[:16000 * 14], 'b': base[16000 * 20:16000 * 31], 'short': base[16000 * 40:16000 * 42],
            'silent': np.zeros(16000 * 6, dtype=np.int16), 'f32': base[16000 * 44:16000 * 56]}
    hows = [16000, 'random', 7000, 3999, 'one']
    fed, last = _feed(_live(vad, 3.0), sigs, hows)        # the VAD segments, from a LiveStreams of their own
    segs = {k: fed[k] + last[k] for k in sigs}
    live = LiveScores(None, backend=OracleVfsBackend(mlp), live=_live(vad, 3.0), vad_thresh=THRESH)
    feed_sigs = dict(sigs)
    feed_sigs['f32'] = sigs['f32'].astype(np.float32) / np.float32(32768)
    held = {}

    def after(now):
        # a window is returned only once the VAD is final up to its stop time; the stream objects keep every window
        for k, v in now.items():
            assert all(w[1] <= live.live.decided_until(k) for w in v), k
        held.update(live.streams)
    wins, got = _feed(live, feed_sigs, hows, after=after)
    assert not live.streams
    # the rows computed window by window are those of the whole stream (every stream opens in the first call, in order)
    for sid, (k, x) in enumerate(sigs.items()):
        rows = np.concatenate(live.backend.computed[sid])
        assert np.array_equal(rows, whole_features(x.astype(np.float32) / np.float32(32768))), k
    speech = 0
    for k, x in sigs.items():
        ref = _reference(x, segs[k], mlp)
        assert _same(got[k], ref), (k, got[k], ref)
        speech += bool(any(lab == 'speech' for lab, _, _ in segs[k]))
        # every window that can enter the score, with its ratio and MLP row, the tail window included
        ref_w = _oracle_windows(x, segs[k], mlp)
        assert [w[:3] for w in held[k].wins] == [w[:3] for w in ref_w], k
        # (numpy's product of one row and of a batch may round apart: the MLP rows agree to float32 precision)
        assert all(np.allclose(a[3], b[3], rtol=1e-5, atol=1e-6) for a, b in zip(held[k].wins, ref_w)), k
        assert [w[:3] for w in wins[k]] == [w[:3] for w in held[k].wins[:len(wins[k])]], k
    assert got['silent'] == (None, 0, 0)
    assert speech >= 3 and all(got[k][2] > 0 for k in ('a', 'b', 'f32'))


def test_score_and_decided_until_follow_the_stream(vad):
    mlp = _synthetic_mlp()
    x = synth_audio(16, seed=62)
    live = LiveScores(None, backend=OracleVfsBackend(mlp), live=_live(vad, 2.0), vad_thresh=THRESH)
    assert live.feed({'s': x[:16000]}) == {'s': []}       # nothing is decided before the calibration
    assert live.decided_until('s') == 0 and live.score('s') == (None, 0, 0)
    last = 0
    for i in range(1, 16):
        live.feed({'s': x[16000 * i:16000 * (i + 1)]})
        assert live.decided_until('s') >= last
        last = live.decided_until('s')
    assert last > 5
    score, dur, nb = live.score('s')
    assert dur > 0 and nb > 0
    fed, last = _feed(_live(vad, 2.0), {'s': x}, [16000])
    segs = fed['s'] + last['s']
    assert live.end(['s'])['s'] == _reference(x, segs, mlp)
