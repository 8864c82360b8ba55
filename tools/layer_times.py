"""Per-layer times of the two segmenter CNNs on the GPU.

Builds the synthetic-weight stand-ins of the VAD (smn) and gender networks that bench.py runs
(models.synthetic_keras_cnn(21, 3, seed=11) and (24, 2, seed=13)), feeds each about 30 minutes of synthetic log-mel
(8192-patch batches) and times every convolution / dense layer with iss_cnn_profile / iss_cnn_profile_read, which
brackets one layer per forward pass with CUDA events.  Pooling layers are not profiled: profiling a 2x2 pooling layer
would keep it from being folded into the next convolution and so change what runs.

    python tools/layer_times.py [--minutes 30] [--json OUT]

Prints the card, its power limit, and per layer: ms per forward, useful TFLOP/s (fp32-equivalent FLOPs of the layer)
and share of the forward's time.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

KIND = {1: 'Conv2D', 2: 'Dense', 3: 'MaxPool'}


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = [s.strip() for s in q.split(',')]
        return {'name': name, 'power_limit': power, 'max_sm_clock': clk}
    except Exception as e:                                   # the GPU's name still identifies the card
        import torch
        return {'name': torch.cuda.get_device_name(0), 'power_limit': 'unknown (%r)' % e}


def time_network(torch, _lib, lib, engine, ctx, cfg, w, nmel, frames, seed):
    rng = np.random.default_rng(seed)
    mspec = torch.from_numpy((rng.standard_normal((frames, nmel)) * 3 - 5).astype(np.float32)).cuda()
    net = engine.CnnModel.from_keras(ctx, cfg, w, nmel)
    P = (frames + 1) // 2
    ranges = [(0, P)]
    net.forward(mspec, ranges)                               # warm-up: module load, workspace
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    net.forward(mspec, ranges)
    e1.record()
    e1.synchronize()
    total_ms = e0.elapsed_time(e1)
    rows = []
    for li, d in enumerate(net.lowered.descs):
        name = '%s %dx%d %d->%d' % (KIND[d['kind']], d['kh'], d['kw'], d['cin'], d['cout'])
        if d['kind'] == 3:
            rows.append({'layer': li, 'name': name, 'ms': None})
            continue
        _lib.check(lib.iss_cnn_profile(net.handle, li), 'iss_cnn_profile')
        net.forward(mspec, ranges)
        tms, nl, fl = ctypes.c_double(), ctypes.c_int64(), ctypes.c_double()
        _lib.check(lib.iss_cnn_profile_read(net.handle, ctypes.byref(tms), ctypes.byref(nl), ctypes.byref(fl)), 'profile_read')
        _lib.check(lib.iss_cnn_profile(net.handle, -1), 'iss_cnn_profile')
        rows.append({'layer': li, 'name': name, 'ms': tms.value, 'launches': int(nl.value), 'flops': fl.value,
                     'tflops': fl.value / (tms.value * 1e-3) / 1e12 if tms.value > 0 else 0.0, 'share': tms.value / total_ms})
    del net
    return {'patches': P, 'forward_ms': total_ms, 'layers': rows}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--minutes', type=float, default=30.0, help='synthetic log-mel per network (100 frames/s)')
    ap.add_argument('--json', default=None, help='also write the result to this file')
    args = ap.parse_args()
    import torch
    from inaspeechsegmenter_b200 import _lib, engine, models
    assert torch.cuda.is_available(), 'layer_times.py needs a CUDA device'
    lib = _lib.load()
    ctx = engine.Context(0)
    frames = int(args.minutes * 60 * 100)
    out = {'card': card(), 'minutes': args.minutes, 'networks': {}}
    for key, nmel, nc, seed in (('vad', 21, 3, 11), ('gender', 24, 2, 13)):
        cfg, w = models.synthetic_keras_cnn(nmel, nc, seed=seed)
        out['networks'][key] = time_network(torch, _lib, lib, engine, ctx, cfg, w, nmel, frames, seed)
    c = out['card']
    print('%s, power limit %s, max SM clock %s' % (c['name'], c['power_limit'], c.get('max_sm_clock', '?')))
    for key, r in out['networks'].items():
        print('\n%s network: %d patches, %.2f ms per forward' % (key, r['patches'], r['forward_ms']))
        print('  %-5s %-22s %10s %10s %7s' % ('layer', 'kind', 'ms', 'TFLOP/s', 'share'))
        for row in r['layers']:
            if row['ms'] is None:
                print('  %-5d %-22s %10s %10s %7s' % (row['layer'], row['name'], '(not timed)', '', ''))
            else:
                print('  %-5d %-22s %10.3f %10.1f %6.1f%%' % (row['layer'], row['name'], row['ms'], row['tflops'], 100 * row['share']))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
