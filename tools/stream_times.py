"""Live-stream throughput on one GPU: ``Segmenter.stream().feed`` over N streams with chunks of C seconds, stand-in
networks (the release weights are not used), against ``segment_signals`` on the same audio cut into clips of C seconds.

    python tools/stream_times.py [--streams 100,1000,4000] [--chunks 0.5,1,2] [--calls 10] [--out FILE]
                                 [--rate 16000[,48000,...]] [--channels 1[,2,...]] [--dtype int16[,float32,...]]
                                 [--profile-resampler]

--rate, --channels and --dtype list the stream formats, zipped: every configuration runs in each format, alternated
within a round (defaults: 16 kHz mono int16, fed to the 16 kHz path as it is).  Other formats are resampled by the
live streams on the device; --profile-resampler then also runs 3 more calls under torch.profiler, after the timed
calls, and reports the resampler kernel's device time per call.

Each stream reads one hour (--audio-sec) of synthetic audio from its own offset.  Per configuration: feed until calibration is over
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


def run(seg, audio, rate, N, C, calls, cal, profile):
    n = int(C * rate)
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
        live.feed({i: chunk(i) for i in range(N)}, sample_rate=rate)
    # time spent inside the backend (device work, launches and the synchronising copies) vs the host state machine
    spent = [0.0]
    for name in ('resample', 'ingest', 'calibrate', 'energy', 'decode'):
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
        live.feed(feed, sample_rate=rate)
        ts.append(time.perf_counter() - t0)
        tb.append(spent[0])
        fed = pos[0] / rate
        lags += [fed - live.decided_until(i) for i in range(N)]       # every stream after every timed call
    lags = np.array(lags)
    peak = (torch.cuda.max_memory_allocated() - m0) / N
    kernel = None
    if profile:
        from torch.profiler import ProfilerActivity, profile as prof
        with prof(activities=[ProfilerActivity.CUDA]) as p:
            for _ in range(3):
                live.feed({i: chunk(i) for i in range(N)}, sample_rate=rate)
            torch.cuda.synchronize()
        us = sum(e.device_time_total for e in p.key_averages() if 'resample_kernel' in e.key)
        kernel = round(us / 3 / 1000, 4)
    live.end(list(range(N)))
    t = float(np.median(ts))
    clips = [chunk(i) for i in range(N)]
    seg.segment_signals(clips, sample_rates=[rate] * N)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    seg.segment_signals(clips, sample_rates=[rate] * N)
    torch.cuda.synchronize()
    t_off = time.perf_counter() - t0
    host = float(np.median(np.array(ts) - np.array(tb)))
    return dict(rate=rate, channels=1 if audio.ndim == 1 else audio.shape[1], dtype=str(audio.dtype), streams=N, chunk_s=C, feed_s_median=round(t, 4), feed_s_max=round(max(ts), 4),
                host_state_machine_s_median=round(host, 4), real_time_every_call=max(ts) < C,
                audio_hours_per_s=round(N * C / 3600 / t, 3), real_time=t < C,
                offline_clips_s=round(t_off, 4), offline_audio_hours_per_s=round(N * C / 3600 / t_off, 3),
                peak_device_bytes_per_stream=int(peak),
                lag_s_p50=round(float(np.percentile(lags, 50)), 2), lag_s_p99=round(float(np.percentile(lags, 99)), 2),
                lag_s_max=round(float(lags.max()), 2), resample_kernel_ms_per_call=kernel)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', default='100,1000,4000')
    ap.add_argument('--chunks', default='0.5,1,2')
    ap.add_argument('--calls', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--calibration', type=float, default=5.0)
    ap.add_argument('--rate', default='16000')
    ap.add_argument('--channels', default='1')
    ap.add_argument('--dtype', default='int16')
    ap.add_argument('--audio-sec', type=float, default=3600)
    ap.add_argument('--profile-resampler', action='store_true')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'stream_times measures on a GPU'
    from conftest import synth_audio
    from inaspeechsegmenter_b200 import Segmenter, models
    mods = {'vad': models.synthetic_keras_cnn(21, 3, seed=11), 'gender': models.synthetic_keras_cnn(24, 2, seed=13)}
    seg = Segmenter(vad_engine='smn', detect_gender=True, ffmpeg=None, models=mods)
    fmts = list(zip([int(x) for x in a.rate.split(',')], [int(x) for x in a.channels.split(',')], a.dtype.split(',')))
    audios = []
    for rate, ch, dt in fmts:
        x = synth_audio(a.audio_sec, seed=2026, sr=rate)
        if ch > 1:                          # the other channels: the same audio, shifted by 1.7 s per channel
            x = np.stack([np.roll(x, int(1.7 * rate * c)) for c in range(ch)], axis=1)
        audios.append((rate, x.astype(np.float32) / np.float32(32768) if dt == 'float32' else x))
    lines = [json.dumps({'card': card()})]
    print(lines[0], flush=True)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        for rnd in range(1, a.rounds + 1):
            for N in [int(x) for x in a.streams.split(',')]:
                for C in [float(x) for x in a.chunks.split(',')]:
                    for rate, audio in audios:
                        r = dict(round=rnd, **run(seg, audio, rate, N, C, a.calls, a.calibration,
                                                  a.profile_resampler and rnd == a.rounds))
                        lines.append(json.dumps(r))
                        print(lines[-1], flush=True)
    if a.out:
        with open(a.out, 'w') as f:
            f.write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
