"""Short-clip throughput: ``[segment_signal(s) for s in clips]`` against ``segment_signals(clips)``.

One hour of seeded int16 audio (tests/conftest.py synth_audio) is cut into 2 s, 10 s and 60 s clips (1800 / 360 / 60
recordings) and segmented with the synthetic stand-in networks (smn VAD + gender).  Inputs are host numpy arrays (the
corpus case) or device-resident tensors; every (workload, input, method) shape is warmed up first and the cases are
then alternated in one process, REPS rounds.  Also sweeps the pass budget (pack.PASS_FRAMES) on the 2 s clips.
Reports audio-hours/s, recordings/s, library launches per recording, whether the segment lists are equal, and the
card's name, power limit and SM clock read in the same process.

    python tools/pack_times.py [--reps 3] [--out RESULT.json]
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

import torch  # noqa: E402

from conftest import synth_audio  # noqa: E402
from inaspeechsegmenter_b200 import _lib, models, pack  # noqa: E402
from inaspeechsegmenter_b200.segmenter import Segmenter  # noqa: E402

CLIP_SECONDS = (2, 10, 60)
BUDGETS = (1 << 16, 1 << 17, 1 << 18, 1 << 19, 1 << 20, 1 << 22)


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        out = 'nvidia-smi unavailable: %s' % e
    return {'query': q, 'value': out, 'torch_name': torch.cuda.get_device_name(0)}


def timed(fn):
    lib = _lib.load()
    torch.cuda.synchronize()
    c0 = lib.iss_launch_count()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0, lib.iss_launch_count() - c0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--seconds', type=float, default=3600.0, help='audio per workload')
    ap.add_argument('--out', default=None, help='also write every timed row and the summary as JSON to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('pack_times.py measures the GPU: no CUDA device')

    mods = {'vad': models.synthetic_keras_cnn(21, 3, seed=11), 'gender': models.synthetic_keras_cnn(24, 2, seed=13)}
    seg = Segmenter(vad_engine='smn', detect_gender=True, ffmpeg=None, models=mods)
    audio = synth_audio(args.seconds, seed=20261016)
    hours = len(audio) / 16000 / 3600
    work = {}
    for s in CLIP_SECONDS:
        n = int(s * 16000)
        host = [audio[i:i + n] for i in range(0, len(audio) - n + 1, n)]
        work[s] = {'host': host, 'device': [torch.from_numpy(c).cuda() for c in host]}
    methods = {'single': lambda clips: [seg.segment_signal(c) for c in clips],
               'packed': lambda clips: seg.segment_signals(clips)}

    # warm every shape, and check the results once per workload and input
    equal = {}
    for s, w in work.items():
        for inp, clips in w.items():
            ref = methods['single'](clips)
            equal['%ds/%s' % (s, inp)] = methods['packed'](clips) == ref
    rows = []
    for rep in range(args.reps):
        for s, w in work.items():
            for inp, clips in w.items():
                for name in (('single', 'packed') if rep % 2 == 0 else ('packed', 'single')):
                    _, dt, launches = timed(lambda: methods[name](clips))
                    rows.append({'rep': rep, 'clip_s': s, 'input': inp, 'method': name, 'n': len(clips), 'sec': dt,
                                 'audio_hours_per_s': hours / dt, 'recordings_per_s': len(clips) / dt,
                                 'launches_per_recording': launches / len(clips)})
                    print(json.dumps(rows[-1]), flush=True)
    sweep = []
    default = pack.PASS_FRAMES
    clips = work[2]['host']
    try:
        for b in BUDGETS:
            pack.PASS_FRAMES = b
            methods['packed'](clips)
        for rep in range(args.reps):
            for b in BUDGETS:
                pack.PASS_FRAMES = b
                _, dt, launches = timed(lambda: methods['packed'](clips))
                sweep.append({'rep': rep, 'budget_frames': b, 'sec': dt, 'audio_hours_per_s': hours / dt,
                              'launches_per_recording': launches / len(clips)})
                print(json.dumps(sweep[-1]), flush=True)
    finally:
        pack.PASS_FRAMES = default

    summary = {}
    for r in rows:
        k = '%ds/%s/%s' % (r['clip_s'], r['input'], r['method'])
        summary.setdefault(k, []).append(round(r['audio_hours_per_s'], 3))
    for r in sweep:
        summary.setdefault('sweep/2s/host/%d' % r['budget_frames'], []).append(round(r['audio_hours_per_s'], 3))
    result = {'card': card(), 'audio_hours': hours, 'default_budget_frames': default, 'equal': equal,
              'summary_audio_hours_per_s': summary, 'rows': rows, 'sweep': sweep}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)
    print(json.dumps({'card': result['card'], 'equal': equal, 'summary': summary}, indent=1))


if __name__ == '__main__':
    main()
