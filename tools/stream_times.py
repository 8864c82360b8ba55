"""Live-stream throughput on one GPU: ``Segmenter.stream().feed`` over N streams with chunks of C seconds, stand-in
networks (the release weights are not used), against ``segment_signals`` on the same audio cut into clips of C seconds.

    python tools/stream_times.py [--streams 100,1000,4000] [--chunks 0.5,1,2] [--calls 10] [--out FILE]

Each stream reads one hour of synthetic audio from its own offset.  Per configuration: feed until calibration is over
plus two warm-up calls, then time `--calls` calls with a host clock (every call ends in the copy that returns the
decided states, which synchronises), and split each call's time between the backend (device work, launches, copies)
and the host state machine.  The decision lag of every stream is sampled after every timed call.  The configurations
run twice, alternated.  Prints one JSON line per
configuration and round, and the card name and power limit."""
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


def run(seg, audio, N, C, calls, cal):
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
    live = seg.stream(calibration_sec=cal)
    warm = int(np.ceil(cal / C)) + 2
    for _ in range(warm):
        live.feed({i: chunk(i) for i in range(N)})
    # time spent inside the backend (device work, launches and the synchronising copies) vs the host state machine
    spent = [0.0]
    for name in ('ingest', 'calibrate', 'energy', 'decode'):
        fn = getattr(live.backend, name)

        def timed(*args, _fn=fn):
            t = time.perf_counter()
            try:
                return _fn(*args)
            finally:
                spent[0] += time.perf_counter() - t
        setattr(live.backend, name, timed)
    ts, tb, lags = [], [], []
    for _ in range(calls):
        feed = {i: chunk(i) for i in range(N)}
        spent[0] = 0.0
        t0 = time.perf_counter()
        live.feed(feed)
        ts.append(time.perf_counter() - t0)
        tb.append(spent[0])
        fed = pos[0] / 16000
        lags += [fed - live.decided_until(i) for i in range(N)]       # every stream after every timed call
    lags = np.array(lags)
    peak = (torch.cuda.max_memory_allocated() - m0) / N
    live.end(list(range(N)))
    t = float(np.median(ts))
    clips = [chunk(i) for i in range(N)]
    seg.segment_signals(clips)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    seg.segment_signals(clips)
    torch.cuda.synchronize()
    t_off = time.perf_counter() - t0
    host = float(np.median(np.array(ts) - np.array(tb)))
    return dict(streams=N, chunk_s=C, feed_s_median=round(t, 4), feed_s_max=round(max(ts), 4),
                host_state_machine_s_median=round(host, 4), real_time_every_call=max(ts) < C,
                audio_hours_per_s=round(N * C / 3600 / t, 3), real_time=t < C,
                offline_clips_s=round(t_off, 4), offline_audio_hours_per_s=round(N * C / 3600 / t_off, 3),
                peak_device_bytes_per_stream=int(peak),
                lag_s_p50=round(float(np.percentile(lags, 50)), 2), lag_s_p99=round(float(np.percentile(lags, 99)), 2),
                lag_s_max=round(float(lags.max()), 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', default='100,1000,4000')
    ap.add_argument('--chunks', default='0.5,1,2')
    ap.add_argument('--calls', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--calibration', type=float, default=5.0)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'stream_times measures on a GPU'
    from conftest import synth_audio
    from inaspeechsegmenter_b200 import Segmenter, models
    mods = {'vad': models.synthetic_keras_cnn(21, 3, seed=11), 'gender': models.synthetic_keras_cnn(24, 2, seed=13)}
    seg = Segmenter(vad_engine='smn', detect_gender=True, ffmpeg=None, models=mods)
    audio = synth_audio(3600, seed=2026)
    lines = [json.dumps({'card': card()})]
    print(lines[0], flush=True)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        for rnd in range(1, a.rounds + 1):
            for N in [int(x) for x in a.streams.split(',')]:
                for C in [float(x) for x in a.chunks.split(',')]:
                    r = dict(round=rnd, **run(seg, audio, N, C, a.calls, a.calibration))
                    lines.append(json.dumps(r))
                    print(lines[-1], flush=True)
    if a.out:
        with open(a.out, 'w') as f:
            f.write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
