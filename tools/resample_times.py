"""Device resampler timings (resample.cu) and segment_signals on native-rate clips.

1. Device time per audio-hour of one iss_resample_to16k_multi launch over one hour of seeded audio already on the
   device: 48 kHz stereo int16 and 44.1 kHz mono int16 (CUDA events around ITERS launches, after a warm-up launch).
2. ``segment_signals`` on one hour of 48 kHz stereo int16 clips in host memory (10 s each), two ways, alternated REPS
   rounds: in place (``sample_rates=[48000] * n``: one upload of the native-rate audio, then device resampling), and
   host ``scipy.signal.resample_poly`` of each clip (downmix, resample, int16 as the resampler defines it) followed
   by the 16 kHz call.  The host time of the resample_poly step is also reported on its own.  Also the time of the
   pinned upload of the native-rate hour, to see whether the upload dominates.

Reports the card's name and power limit read in the same process.

    python tools/resample_times.py [--reps 2] [--out RESULT.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from conftest import synth_audio  # noqa: E402
from inaspeechsegmenter_b200 import engine, models, resample  # noqa: E402
from inaspeechsegmenter_b200.segmenter import Segmenter  # noqa: E402

ITERS = 20


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        out = 'nvidia-smi unavailable: %s' % e
    return {'query': q, 'value': out, 'torch_name': torch.cuda.get_device_name(0)}


def kernel_time(ctx, x, rate):
    """ms per launch over one recording on the device, and audio-hours of that recording."""
    n16 = resample.num_frames(x.shape[0], rate)
    out = torch.empty(n16, dtype=torch.int16, device='cuda')
    resample.to16k_multi(ctx, [x], rate, out, [0])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(ITERS):
        resample.to16k_multi(ctx, [x], rate, out, [0])
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / ITERS, x.shape[0] / rate / 3600


def host_resample(clips, rate):
    from scipy.signal import resample_poly
    up, down = resample.factors(rate)
    out = []
    for c in clips:
        y = resample_poly(c.astype(np.float64).mean(axis=1) / 32768, up, down)
        out.append(np.clip(np.rint(y * 32768), -32768, 32767).astype(np.int16))
    return out


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--seconds', type=float, default=3600.0, help='audio per workload')
    ap.add_argument('--clip', type=float, default=10.0, help='clip length in seconds for segment_signals')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('resample_times.py measures the GPU: no CUDA device')
    ctx = engine.Context(0)
    result = {'card': card(), 'kernel': {}}

    rate = 48000
    n = int(args.seconds * rate)
    stereo = np.stack([synth_audio(args.seconds, seed=1, sr=rate), synth_audio(args.seconds, seed=2, sr=rate)], axis=1)
    mono44 = synth_audio(args.seconds, seed=3, sr=44100)
    for name, x, r in (('48k_stereo_int16', stereo, 48000), ('44.1k_mono_int16', mono44, 44100)):
        ms, hours = kernel_time(ctx, torch.from_numpy(x).cuda(), r)
        result['kernel'][name] = {'ms_per_launch': ms, 'audio_hours': hours, 'ms_per_audio_hour': ms / hours,
                                  'input_GB': x.nbytes / 1e9, 'input_GB_per_s': x.nbytes / 1e9 / (ms / 1e3)}
        print(json.dumps({name: result['kernel'][name]}), flush=True)

    host = torch.from_numpy(stereo).pin_memory()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(3):
        host.to('cuda', non_blocking=True)
    torch.cuda.synchronize()
    result['upload_48k_stereo_hour_ms'] = (time.perf_counter() - t0) / 3 * 1e3

    mods = {'vad': models.synthetic_keras_cnn(21, 3, seed=11), 'gender': models.synthetic_keras_cnn(24, 2, seed=13)}
    seg = Segmenter(vad_engine='smn', detect_gender=True, ffmpeg=None, models=mods)
    c = int(args.clip * rate)
    clips = [stereo[i:i + c] for i in range(0, n - c + 1, c)]
    hours = len(clips) * c / rate / 3600
    methods = {'device': lambda: seg.segment_signals(clips, sample_rates=[rate] * len(clips)),
               'host_resample_poly': lambda: seg.segment_signals(host_resample(clips, rate))}
    same = methods['device']() == methods['host_resample_poly']()
    rows = []
    for rep in range(args.reps):
        for name in (('device', 'host_resample_poly') if rep % 2 == 0 else ('host_resample_poly', 'device')):
            _, dt = timed(methods[name])
            rows.append({'rep': rep, 'method': name, 'sec': dt, 'audio_hours_per_s': hours / dt})
            print(json.dumps(rows[-1]), flush=True)
        _, dt = timed(lambda: host_resample(clips, rate))
        rows.append({'rep': rep, 'method': 'resample_poly_only', 'sec': dt, 'audio_hours_per_s': hours / dt})
        print(json.dumps(rows[-1]), flush=True)
    result.update({'clips': len(clips), 'clip_s': args.clip, 'audio_hours': hours, 'segments_equal': same, 'rows': rows})
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)
    print(json.dumps({k: v for k, v in result.items() if k != 'rows'}, indent=1))


if __name__ == '__main__':
    main()
