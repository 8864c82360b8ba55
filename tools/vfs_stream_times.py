"""Live femininity-score throughput on one GPU: ``VoiceFemininityScoring.stream().feed`` over N streams with chunks of
C seconds, stand-in networks (the speech-biased smn VAD, the synthetic MLP and the seeded synthetic ResNet101 of the
tests; the release weights are not used).

    python tools/vfs_stream_times.py [--streams 100,1000] [--chunks 1,2] [--calls 8] [--rounds 2] [--out FILE]

Each stream reads the golden musanmix.wav (speech, music and noise) tiled to --audio-sec, from its own offset.  Per
configuration: feed until calibration is over plus two warm-up calls, then time `--calls` calls with a host clock
(every call ends in the copy that returns the decided windows, which synchronises) and split each call's time between
the backends (device work, launches, copies) and the host state machines.  Reports the feed median and slowest call,
the host share, the x-vector windows embedded per second, the decision lag (fed time - decided_until) of every stream
after every timed call, and the peak device memory per stream.  The configurations run --rounds times, alternated.
Prints one JSON line per configuration and round, after the card name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


def run(vfs, audio, N, C, calls, cal):
    n = int(C * 16000)
    off = [(i * len(audio)) // N for i in range(N)]
    pos = [0] * N

    def chunk(i):
        a = (off[i] + pos[i]) % (len(audio) - n)
        pos[i] += n
        return audio[a:a + n]

    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    m0 = torch.cuda.memory_allocated()
    live = vfs.stream(calibration_sec=cal)
    for _ in range(int(np.ceil(cal / C)) + 2):
        live.feed({i: chunk(i) for i in range(N)})
    spent = [0.0]
    for obj, names in ((live.backend, ('features', 'embed')),
                       (live.live.backend, ('resample', 'ingest', 'calibrate', 'energy', 'decode'))):
        for name in names:
            fn = getattr(obj, name)

            def timed(*args, _fn=fn):
                t = time.perf_counter()
                try:
                    return _fn(*args)
                finally:
                    spent[0] += time.perf_counter() - t
            setattr(obj, name, timed)
    ts, tb, lags, nwin = [], [], [], 0
    for _ in range(calls):
        feed = {i: chunk(i) for i in range(N)}
        spent[0] = 0.0
        t0 = time.perf_counter()
        got = live.feed(feed)
        ts.append(time.perf_counter() - t0)
        tb.append(spent[0])
        nwin += sum(len(v) for v in got.values())
        fed = pos[0] / 16000
        lags += [fed - live.decided_until(i) for i in range(N)]
    lags = np.array(lags)
    peak = (torch.cuda.max_memory_allocated() - m0) / N
    live.end(list(range(N)))
    t = float(np.median(ts))
    host = float(np.median(np.array(ts) - np.array(tb)))
    return dict(streams=N, chunk_s=C, feed_s_median=round(t, 4), feed_s_max=round(max(ts), 4),
                host_state_machine_s_median=round(host, 4), host_share=round(host / t, 3),
                real_time_every_call=max(ts) < C, windows_embedded_per_s=round(nwin / sum(ts), 1),
                peak_device_bytes_per_stream=int(peak),
                lag_s_p50=round(float(np.percentile(lags, 50)), 2), lag_s_max=round(float(lags.max()), 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', default='100,1000')
    ap.add_argument('--chunks', default='1,2')
    ap.add_argument('--calls', type=int, default=8)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--calibration', type=float, default=5.0)
    ap.add_argument('--audio-sec', type=float, default=600)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'vfs_stream_times measures on a GPU'
    from test_vfs_pack_gpu import _media, vfs_models
    from inaspeechsegmenter_b200 import models
    from inaspeechsegmenter_b200.vbx_segmenter import VoiceFemininityScoring
    vad = {'smn': models.synthetic_keras_cnn(21, 3, seed=11)}                    # tests/conftest.py synth_models
    vfs = VoiceFemininityScoring(ffmpeg=None, models=vfs_models(vad))
    m = _media(os.path.join(ROOT, 'tests', 'golden', 'media'), 'musanmix.wav')
    audio = np.tile(m, int(np.ceil(a.audio_sec * 16000 / len(m))))[:int(a.audio_sec * 16000)]
    lines = [json.dumps({'card': card()})]
    print(lines[0], flush=True)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        for rnd in range(1, a.rounds + 1):
            for N in [int(x) for x in a.streams.split(',')]:
                for C in [float(x) for x in a.chunks.split(',')]:
                    lines.append(json.dumps(dict(round=rnd, **run(vfs, audio, N, C, a.calls, a.calibration))))
                    print(lines[-1], flush=True)
    if a.out:
        with open(a.out, 'w') as f:
            f.write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
