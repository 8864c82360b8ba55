"""Oracle (test infrastructure): Viterbi smoothing as the reference calls it.

Restates reference ``inaSpeechSegmenter/pyannote_viterbi.py:118-224`` (plain
max-sum DP, uniform prior, first-max tie-break) and the transition / emission
helpers of ``inaSpeechSegmenter/viterbi_utils.py:29-49``.

Two implementations of the same order of floating-point operations:
``viterbi_numpy`` (pure numpy/Python loop, small cases) and ``viterbi_c``
(``viterbi_oracle.c`` through ctypes, long sequences).  Both are pinned
against the real ``viterbi_decoding`` by ``tests/golden/make_golden.py``.
``viterbi_partial`` runs a cut of a longer chain (incoming scores, outgoing
scores, back-map, forced end state, output stride) in the same order of
operations; ``emissions_kernel`` and ``energy_threshold_kernel`` are the CUDA
kernels' own emission and threshold, for the exact GPU comparisons.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build():
    subprocess.run(['make', '-s', '-C', _HERE], check=True)


def _lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, '_build', 'liboracle.so')
        if not os.path.exists(path):
            build()
        lib = ctypes.CDLL(path)
        for name, etype in (('oracle_viterbi', ctypes.c_double), ('oracle_viterbi_f32', ctypes.c_float)):
            fn = getattr(lib, name)
            fn.restype = ctypes.c_int
            fn.argtypes = [ctypes.POINTER(etype), ctypes.POINTER(ctypes.c_double),
                           ctypes.c_int64, ctypes.c_int, ctypes.POINTER(ctypes.c_int32)]
        lib.oracle_viterbi_partial.restype = ctypes.c_int
        lib.oracle_viterbi_partial.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int,
                                               ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                               ctypes.c_int, ctypes.c_void_p]
        _LIB = lib
    return _LIB


# ---- viterbi_utils.py restated -------------------------------------------

def pred2logemission(pred, eps=1e-10):
    """viterbi_utils.py:29-34 -- 2-state log emissions from a boolean track."""
    pred = np.asarray(pred)
    em = np.full((len(pred), 2), eps)
    em[pred == 0, 0] = 1 - eps
    em[pred == 1, 1] = 1 - eps
    return np.log(em)


def log_trans_exp(exp, cost0=0, cost1=0):
    """viterbi_utils.py:36-42."""
    c = -exp * np.log(10)
    return np.array([[cost0, c], [c, cost1]], dtype=np.float64)


def diag_trans_exp(exp, dim):
    """viterbi_utils.py:44-49."""
    a = np.full((dim, dim), -exp * np.log(10))
    a[np.arange(dim), np.arange(dim)] = 0
    return a


# ---- the DP -----------------------------------------------------------------

def viterbi_numpy(emission, transition):
    """Straight numpy restatement; returns float array like the reference
    (``_update_states`` builds ``np.empty(states.shape)``, :106)."""
    emission = np.asarray(emission)
    T, K = emission.shape
    V = emission[0] + np.log(np.ones(K) / K)
    P = np.zeros((T, K), dtype=np.int64)
    cols = np.arange(K)
    for t in range(1, T):
        cand = V[:, None] + transition           # cand[k, j] = V[k] + A[k, j]
        P[t] = np.argmax(cand, axis=0)
        V = emission[t] + cand[P[t], cols]
    X = np.empty(T, dtype=np.int64)
    X[-1] = np.argmax(V)
    for t in range(T - 1, 0, -1):
        X[t - 1] = P[t, X[t]]
    return X.astype(np.float64)


def viterbi_c(emission, transition):
    emission = np.asarray(emission)
    T, K = emission.shape
    trans = np.ascontiguousarray(transition, dtype=np.float64)
    out = np.empty(T, dtype=np.int32)
    if T == 0:
        return out.astype(np.float64)
    lib = _lib()
    if emission.dtype == np.float32:
        em = np.ascontiguousarray(emission)
        rc = lib.oracle_viterbi_f32(em.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                                    trans.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                    T, K, out.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)))
    else:
        em = np.ascontiguousarray(emission, dtype=np.float64)
        rc = lib.oracle_viterbi(em.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                trans.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                T, K, out.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)))
    if rc != 0:
        raise RuntimeError('oracle_viterbi failed rc=%d' % rc)
    return out.astype(np.float64)


def viterbi_partial(emission, transition, vin=None, end_state=-1, out_stride=1):
    """Steps [0, T) of a longer chain (``oracle_viterbi_partial``): with ``vin`` (V of the step before) the first
    step is an ordinary transition, without it the prior log(1/K) applies.  Returns (states int32 [ceil(T /
    out_stride)], vout float64 [K] = V[T-1], backmap int32 [K]: for each end state, the state before the first step
    (with vin) or at the first step (without)).  ``end_state`` -1 backtracks from the first argmax of V[T-1]."""
    em = np.ascontiguousarray(emission, dtype=np.float64)
    T, K = em.shape
    trans = np.ascontiguousarray(transition, dtype=np.float64)
    states = np.empty((T + out_stride - 1) // out_stride, dtype=np.int32)
    vout = np.empty(K, dtype=np.float64)
    bmap = np.empty(K, dtype=np.int32)
    vin_arr = None if vin is None else np.ascontiguousarray(vin, dtype=np.float64)
    rc = _lib().oracle_viterbi_partial(em.ctypes.data, trans.ctypes.data, T, K,
                                       None if vin_arr is None else vin_arr.ctypes.data, vout.ctypes.data,
                                       bmap.ctypes.data, int(end_state), int(out_stride), states.ctypes.data)
    if rc != 0:
        raise RuntimeError('oracle_viterbi_partial failed rc=%d' % rc)
    return states, vout, bmap


# ---- emissions and thresholds as the CUDA kernels define them ---------------------------------

def emissions_kernel(p):
    """The K3 kernels' emission: float32(log(float64(p))), a correctly rounded float32 log, widened to double.
    numpy's float32 ``np.log`` (what the reference applies, segmenter.py:176) is not correctly rounded; this is the
    definition the GPU comparisons use, so they do not depend on the host's SIMD log."""
    with np.errstate(divide='ignore'):
        return np.log(np.asarray(p, dtype=np.float32).astype(np.float64)).astype(np.float32).astype(np.float64)


def f32_midpoint_margin(p):
    """Distance of log(float64(p)) from the nearest float32 rounding midpoint, in float64 ulps of the log (inf for
    p = 0 or 1).  A value within a few ulps could round to a different float32 in another double log (CUDA's or the
    host's), so fixtures assert a margin."""
    with np.errstate(divide='ignore'):
        d = np.log(np.asarray(p, dtype=np.float32).astype(np.float64))
    f = d.astype(np.float32).astype(np.float64)
    up = np.nextafter(d.astype(np.float32), np.float32(np.inf)).astype(np.float64)
    dn = np.nextafter(d.astype(np.float32), np.float32(-np.inf)).astype(np.float64)
    other = np.where(f <= d, up, dn)
    mid = 0.5 * (f + other)                          # exact: float32 neighbours need 25 bits
    with np.errstate(invalid='ignore'):
        m = np.abs(d - mid) / np.spacing(np.abs(d))
    return np.where(np.isfinite(d) & (d != 0), m, np.inf)


def energy_threshold_kernel(stats, ratio):
    """The K3 kernels' energy threshold from the ``loge_stats`` pair {sum, count}: float32(sum / count) + log(ratio)
    (NaN for an all-silent track)."""
    s, c = float(stats[0]), float(stats[1])
    with np.errstate(invalid='ignore', divide='ignore'):
        mean = np.float32(np.float64(s) / np.float64(c))
    return float(np.float64(mean) + np.log(ratio))


def energy_activity_thr(loge, thr):
    """segmenter.py:69-73 from a given threshold: ``loge > thr`` (float64 compare; a NaN threshold marks nothing
    active), then the 2-state Viterbi with the energy transitions.  int32 states."""
    raw = np.asarray(loge, dtype=np.float32).astype(np.float64) > thr
    return viterbi_partial(pred2logemission(raw), log_trans_exp(150, cost0=-5))[0]


def viterbi_decoding(emission, transition):
    """Drop-in for the reference call signature used on the hot path."""
    return viterbi_c(emission, transition)
