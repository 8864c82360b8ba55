"""WAV input without ffmpeg: the device route (the data chunk read into pinned memory, uploaded as stored, decoded and
resampled by the resampler kernel) against the host route (``read_wav(path, 'float32')``, then ``segment_signal(x,
sample_rate=rate)``).

1. One seeded hour as a 48 kHz stereo 24-bit WAV (1.04 GB): ``Segmenter(ffmpeg=None)(path)`` against the host route.
2. 360 files of 10 s at 44.1 kHz stereo 16-bit: ``batch_process`` (CSV output) against the host route per file, with
   the same CSV written.
The two routes alternate over --reps rounds, after one untimed run of each that also warms the page cache; the host
``read_wav`` time is reported on its own.  Both routes must give equal segments.  Reports the card's name and power
limit read in the same process.  The WAV files go to a temporary directory, removed at the end.

    python tools/wav_times.py [--reps 2] [--out RESULT.json]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from conftest import synth_audio  # noqa: E402
from resample_times import card  # noqa: E402
from wav_fixtures import encode, write_wav  # noqa: E402
from inaspeechsegmenter_b200 import models  # noqa: E402
from inaspeechsegmenter_b200.export_funcs import seg2csv  # noqa: E402
from inaspeechsegmenter_b200.io import read_wav  # noqa: E402
from inaspeechsegmenter_b200.segmenter import Segmenter  # noqa: E402


def hour_wav(path, seconds, rate=48000, block=60):
    """A seeded stereo 24-bit WAV of `seconds` seconds, written block by block (each block its own seeds)."""
    parts = []
    for k in range(int(seconds // block)):
        x = np.stack([synth_audio(block, seed=1000 + 2 * k, sr=rate), synth_audio(block, seed=1001 + 2 * k, sr=rate)],
                     axis=1) / 32768.0
        parts.append(encode(x * 0.9, 's24'))
    return write_wav(path, b''.join(parts), 's24', 2, rate)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def warm(paths):
    for p in paths:
        with open(p, 'rb') as f:
            while f.read(1 << 24):
                pass


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--seconds', type=float, default=3600.0, help='length of the long file')
    ap.add_argument('--files', type=int, default=360, help='number of 10 s files')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('wav_times.py measures the GPU: no CUDA device')
    result = {'card': card(), 'rows': []}
    mods = {'vad': models.synthetic_keras_cnn(21, 3, seed=11), 'gender': models.synthetic_keras_cnn(24, 2, seed=13)}
    seg = Segmenter(vad_engine='smn', detect_gender=True, ffmpeg=None, models=mods)
    tmp = tempfile.mkdtemp(prefix='wav_times_')
    try:
        long_path = hour_wav(os.path.join(tmp, 'hour_48k_s24_stereo.wav'), args.seconds)
        hours = args.seconds / 3600
        result['long_file_GB'] = os.path.getsize(long_path) / 1e9

        def host_long():
            x, sr = read_wav(long_path, 'float32')
            return seg.segment_signal(x, sample_rate=sr)

        small = []
        os.makedirs(os.path.join(tmp, 'in'))
        for i in range(args.files):
            x = np.stack([synth_audio(10, seed=5000 + 2 * i, sr=44100), synth_audio(10, seed=5001 + 2 * i, sr=44100)],
                         axis=1) / 32768.0
            small.append(write_wav(os.path.join(tmp, 'in', 'f%03d.wav' % i), encode(x, 's16'), 's16', 2, 44100))
        outs = {m: [os.path.join(tmp, m, os.path.basename(p)[:-4] + '.csv') for p in small] for m in ('device', 'host')}
        os.makedirs(os.path.join(tmp, 'host'))
        small_hours = args.files * 10 / 3600

        def host_small():
            for p, o in zip(small, outs['host']):
                x, sr = read_wav(p, 'float32')
                seg2csv(seg.segment_signal(x, sample_rate=sr), o)

        def device_small():
            _, n_ok, _, _ = seg.batch_process(small, outs['device'])
            assert n_ok == len(small)

        warm([long_path] + small)
        result['long_equal'] = seg(long_path) == host_long()
        device_small()
        host_small()
        result['small_equal'] = all(open(a, 'rb').read() == open(b, 'rb').read()
                                    for a, b in zip(outs['device'], outs['host']))
        print(json.dumps({k: result[k] for k in ('card', 'long_equal', 'small_equal')}), flush=True)
        work = {('long', 'device'): lambda: seg(long_path), ('long', 'host'): host_long,
                ('small', 'device'): device_small, ('small', 'host'): host_small,
                ('long', 'read_wav_only'): lambda: read_wav(long_path, 'float32'),
                ('small', 'read_wav_only'): lambda: [read_wav(p, 'float32') for p in small]}
        for rep in range(args.reps):
            order = ('device', 'host') if rep % 2 == 0 else ('host', 'device')
            for what, h in (('long', hours), ('small', small_hours)):
                for method in order + ('read_wav_only',):
                    _, dt = timed(work[(what, method)])
                    result['rows'].append({'rep': rep, 'workload': what, 'method': method, 'sec': dt,
                                           'audio_hours_per_s': h / dt})
                    print(json.dumps(result['rows'][-1]), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
