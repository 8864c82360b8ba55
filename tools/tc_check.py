#!/usr/bin/env python
"""Bring-up check of the GEMM engines: run the VAD stand-in CNN on synthetic
log-mel with one GEMM mode, compare with the fp32 CUDA-core result saved by mode 0,
and time a larger batch.  Each mode runs in its own process (a hung kernel must not
take the others down):  python tools/tc_check.py <mode 0|2|3> [minutes]
(3 = the default fp16-split engine; run mode 0 first so the reference file exists)."""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from conftest import synth_audio                       # noqa: E402
from inaspeechsegmenter_b200 import _lib, engine, models   # noqa: E402
from inaspeechsegmenter_b200.sidekit_mfcc import SidekitFrontEnd   # noqa: E402

mode = int(sys.argv[1])
minutes = float(sys.argv[2]) if len(sys.argv) > 2 else 20.0
lib = _lib.load()
_lib.check(lib.iss_set_gemm_mode(mode), 'set mode')
ctx = engine.Context(0)
fe = SidekitFrontEnd(ctx)
pcm = torch.from_numpy(synth_audio(60 * minutes, seed=4)).cuda()
mspec, loge, stats = fe(pcm, _lib.FFT_FP64)
L = mspec.shape[0]
P = (L + 1) // 2
out = os.path.join(ROOT, 'gpurun_out')
os.makedirs(out, exist_ok=True)
for name, nmel, K, seed in (('vad', 21, 3, 11), ('gender', 24, 2, 13)):
    cfg, w = models.synthetic_keras_cnn(nmel, K, seed=seed)
    net = engine.CnnModel.from_keras(ctx, cfg, w, nmel)
    small = net.forward(mspec, [(0, 3000)]).cpu().numpy()
    torch.cuda.synchronize()
    ref_path = os.path.join(out, 'tc_ref_%s.npy' % name)
    if mode == 0:
        np.save(ref_path, small)
        err = 0.0
    else:
        if os.path.exists(ref_path):
            ref = np.load(ref_path)
            fin = np.isfinite(ref).all(1)
            err = float(np.abs(small - ref)[fin].max())
        else:
            err = float('nan')
    # timing
    net.forward(mspec, [(0, P)])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    probs = net.forward(mspec, [(0, P)])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    tf = net.flops_per_patch * P / (ms * 1e-3) / 1e12
    print('mode %d %-6s  max|softmax - fp32| = %.3e   %d patches in %.1f ms = %.1f TFLOP/s (fp32-equivalent)  nan=%d'
          % (mode, name, err, P, ms, tf, int(np.isnan(probs.cpu().numpy()).sum())), flush=True)
