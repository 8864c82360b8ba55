"""Short-clip throughput of VoiceFemininityScoring: ``[score_signal(c) for c in clips]`` against ``score_signals(clips)``.

One hour of seeded int16 audio (tests/conftest.py synth_audio) is cut into 2 s, 5 s and 10 s clips (1800 / 720 / 360
recordings) and scored with the models of tests/test_vfs_pack_gpu.py (vfs_models): the seeded synthetic ResNet101 of
bench.py, the smn stand-in VAD with its speech logit raised and a synthetic 256-128-64-1 MLP.  Inputs are host numpy
arrays (the corpus case) or device-resident tensors.  The two result lists are checked for equality on every workload and input before anything is timed, which also
warms every shape; the cases are then alternated in one process, REPS rounds.  Reports audio-hours/s, recordings/s,
x-vector windows/s, library launches per recording, the share of the packed time spent in the ResNet calls of the
tail-length groups (CUDA events, a separate round), and the card's name, power limit and SM clock read in the same
process.

    python tools/vfs_pack_times.py [--reps 2] [--out RESULT.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import torch  # noqa: E402

from conftest import synth_audio  # noqa: E402
from test_vfs_pack_gpu import vfs_models  # noqa: E402
from inaspeechsegmenter_b200 import _lib, models, pack  # noqa: E402
from inaspeechsegmenter_b200.vbx_segmenter import VoiceFemininityScoring  # noqa: E402

CLIP_SECONDS = (2, 5, 10)


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        out = 'nvidia-smi unavailable: %s' % e
    return {'query': q, 'value': out, 'torch_name': torch.cuda.get_device_name(0)}


def guarded(fn):
    """fn() or the type of the exception it raised (a clip with speech but no retained window raises, as in the
    reference)."""
    try:
        return fn()
    except ZeroDivisionError as e:
        return type(e)


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
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--seconds', type=float, default=3600.0, help='audio per workload')
    ap.add_argument('--out', default=None, help='also write every timed row and the summary as JSON to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('vfs_pack_times.py measures the GPU: no CUDA device')
    warnings.simplefilter('ignore')

    vad = {'smn': models.synthetic_keras_cnn(21, 3, seed=11)}                    # tests/conftest.py synth_models
    vfs = VoiceFemininityScoring('bgc', ffmpeg=None, models=vfs_models(vad))
    audio = synth_audio(args.seconds, seed=20261016)
    hours = len(audio) / 16000 / 3600
    work = {}
    for s in CLIP_SECONDS:
        n = int(s * 16000)
        host = [audio[i:i + n] for i in range(0, len(audio) - n + 1, n)]
        work[s] = {'host': host, 'device': [torch.from_numpy(c).cuda() for c in host]}
    single = lambda clips: [guarded(lambda: vfs.score_signal(c.cpu().numpy() if isinstance(c, torch.Tensor) else c))   # noqa: E731
                            for c in clips]
    methods = {'single': single, 'packed': lambda clips: vfs.score_signals(clips)}

    # check (and warm) every workload and input; the packed call may only raise where a single call does
    equal, windows, scored = {}, {}, {}
    for s, w in work.items():
        for inp, clips in w.items():
            ref = single(clips)
            err = next((r for r in ref if isinstance(r, type)), None)
            if err is not None:                 # such clips would abort the packed call: time the others
                keep = [i for i, r in enumerate(ref) if not isinstance(r, type)]
                w[inp] = clips = [clips[i] for i in keep]
                ref = [ref[i] for i in keep]
            equal['%ds/%s' % (s, inp)] = methods['packed'](clips) == ref
            assert equal['%ds/%s' % (s, inp)], (s, inp)
            live = [c for c, r in zip(clips, ref) if r[1]]
            windows[s] = int(sum(len(pack.window_plan(pack.vbx_num_frames(c.shape[0]))) for c in live))
            scored[s] = len(live)
    rows = []
    for rep in range(args.reps):
        for s, w in work.items():
            for inp, clips in w.items():
                for name in (('single', 'packed') if rep % 2 == 0 else ('packed', 'single')):
                    _, dt, launches = timed(lambda: methods[name](clips))
                    h = sum(c.shape[0] for c in clips) / 16000 / 3600
                    rows.append({'rep': rep, 'clip_s': s, 'input': inp, 'method': name, 'n': len(clips), 'sec': dt,
                                 'audio_hours_per_s': h / dt, 'recordings_per_s': len(clips) / dt,
                                 'windows_per_s': windows[s] / dt, 'launches_per_recording': launches / len(clips)})
                    print(json.dumps(rows[-1]), flush=True)

    # share of the packed time in the ResNet calls of the tail-length groups (CUDA events around each embed_windows call
    # whose window length is not 144, a separate round from host memory)
    ext = vfs.xvector_model
    embed = ext.embed_windows
    tail_share = {}
    for s, w in work.items():
        ev = []

        def probe(fea, starts, win_len, stream=None):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = embed(fea, starts, win_len, stream)
            b.record()
            ev.append((win_len, a, b))
            return out

        ext.embed_windows = probe
        try:
            _, dt, _ = timed(lambda: vfs.score_signals(w['host']))
        finally:
            ext.embed_windows = embed
        tails = sum(a.elapsed_time(b) for n, a, b in ev if n != 144) * 1e-3
        regs = sum(a.elapsed_time(b) for n, a, b in ev if n == 144) * 1e-3
        tail_share[s] = {'tail_groups': sum(n != 144 for n, _, _ in ev), 'tail_sec': tails, 'regular_sec': regs,
                         'total_sec': dt, 'tail_share': tails / dt}
        print(json.dumps({'clip_s': s, **tail_share[s]}), flush=True)

    summary = {}
    for r in rows:
        k = '%ds/%s/%s' % (r['clip_s'], r['input'], r['method'])
        summary.setdefault(k, {'audio_hours_per_s': [], 'recordings_per_s': [], 'windows_per_s': [],
                               'launches_per_recording': []})
        for f in summary[k]:
            summary[k][f].append(round(r[f], 3))
    result = {'card': card(), 'audio_hours': hours, 'equal': equal, 'clips_with_speech': scored, 'windows': windows,
              'summary': summary, 'tail_share': tail_share, 'rows': rows}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)
    print(json.dumps({k: result[k] for k in ('card', 'equal', 'clips_with_speech', 'summary', 'tail_share')}, indent=1))


if __name__ == '__main__':
    main()
