import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, 'tests', 'golden')
MEDIA = os.path.join(GOLDEN_DIR, 'media')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run on an H100 with -m gpu)')


@pytest.fixture(scope='session')
def golden():
    return np.load(os.path.join(GOLDEN_DIR, 'reference_golden.npz'), allow_pickle=False)


@pytest.fixture(scope='session')
def media():
    return MEDIA


def synth_audio(seconds, seed=20260922, sr=16000):
    """Deterministic int16 test signal: spans of exact silence, white noise,
    a harmonic 'speech-like' source with 4 Hz AM and multi-tone 'music'
    (the generator SURVEY 8(d) describes), some spans shorter than 0.68 s."""
    rng = np.random.default_rng(seed)
    n = int(seconds * sr)
    out = np.zeros(n, dtype=np.float64)
    pos = 0
    kinds = ['silence', 'noise', 'speech', 'music']
    first = True
    while pos < n:
        dur = int(rng.uniform(0.3, 6.0) * sr) if not first else int(1.5 * sr)
        kind = kinds[rng.integers(0, 4)] if not first else 'noise'
        first = False
        end = min(n, pos + dur)
        t = np.arange(end - pos) / sr
        if kind == 'noise':
            out[pos:end] = rng.standard_normal(end - pos) * rng.uniform(1e-3, 0.3)
        elif kind == 'speech':
            f0 = rng.uniform(100, 250)
            sig = sum(np.sin(2 * np.pi * f0 * h * t + rng.uniform(0, 6.28)) / h for h in range(1, 12))
            out[pos:end] = 0.08 * sig * (0.6 + 0.4 * np.sin(2 * np.pi * 4 * t)) + rng.standard_normal(end - pos) * 2e-3
        elif kind == 'music':
            fs_ = rng.uniform(200, 3000, size=5)
            out[pos:end] = 0.05 * sum(np.sin(2 * np.pi * f * t) for f in fs_) + rng.standard_normal(end - pos) * 1e-3
        pos = end
    return np.clip(np.round(out * 32768), -32768, 32767).astype(np.int16)


@pytest.fixture(scope='session')
def synth_models():
    from inaspeechsegmenter_b200 import models
    return {
        'smn': models.synthetic_keras_cnn(21, 3, seed=11),
        'sm': models.synthetic_keras_cnn(21, 2, seed=12),
        'gender': models.synthetic_keras_cnn(24, 2, seed=13),
    }
