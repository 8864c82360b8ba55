"""CPU: the float64 front-end reference (oracle/frontend_ref.py) against the computations whose error it bounds, on the
fixtures of the GPU probes (test_frontend_probes_gpu.py) -- so the bound model is pinned without a GPU.

  sidekit_oracle.logmel_loge (bit-pinned to the real sidekit_mfcc.py)   inside the reference-recipe bound
  a numpy complex64 emulation of the FFT_FP32 recipe                    inside the FFT_FP32 bound
  vbx_oracle.get_features (bit-pinned to the real features_vbx.py)      faithfully rounded within the K4 float64 term

Each test prints how tight the bound is: the median of bound / error over the values with an error, and the worst
error / bound."""
import numpy as np
import pytest

from conftest import synth_audio
from oracle import frontend_ref as fr
from oracle import sidekit_oracle as sk
from oracle import vbx_oracle as vx
from test_frontend_probes_gpu import K1_FIX, K4_FIX

K1_CPU = dict({k: v.astype(np.float32) / np.float32(32768) for k, v in K1_FIX.items()},
              synth20=synth_audio(20).astype(np.float32) / np.float32(32768))


def emulate_fp32(sig):
    """K1's FFT_FP32 recipe with numpy float32 arithmetic: float32 window table, complex64 rfft, float32 power, the
    kernel's mel tasks (two chains, then the filter's partials) and float32 log; loge from a double sum, as the kernel."""
    y = fr.preemphasised_frames(sig)
    v = y * sk.hann_window().astype(np.float32)
    X = np.fft.rfft(v, sk.NFFT, axis=-1)
    assert X.dtype == np.complex64
    P = X.real * X.real + X.imag * X.imag
    bank = sk.mel_filterbank()[0]
    lo, _, tasks = fr.mel_tasks(bank)
    B = np.zeros((len(y), sk.NMEL), dtype=np.float32)
    for m in range(sk.NMEL):
        k0, acc = lo[m], np.zeros(len(y), dtype=np.float32)
        for n in tasks[m]:
            a0, a1 = np.zeros(len(y), np.float32), np.zeros(len(y), np.float32)
            for b in range(0, n - 1, 2):
                a0 = a0 + P[:, k0 + b] * bank[m, k0 + b]
                a1 = a1 + P[:, k0 + b + 1] * bank[m, k0 + b + 1]
            if n % 2:
                a0 = a0 + P[:, k0 + n - 1] * bank[m, k0 + n - 1]
            acc = acc + (a0 + a1)
            k0 += n
        B[:, m] = acc
    with np.errstate(divide='ignore'):
        mspec = np.log(B)
        loge = np.log((y.astype(np.float64) ** 2).sum(axis=1).astype(np.float32))
    return mspec, loge


def _report(tag, got, ref, E):
    med, worst = fr.tightness(got, ref, E)
    print('%-28s median bound/err %10.3g   worst err/bound %.3g' % (tag, med, worst))
    return worst


@pytest.mark.parametrize('name', sorted(K1_CPU))
def test_reference_recipe_within_bound(name):
    sig = K1_CPU[name]
    ref = fr.K1Ref(sig)
    mspec, loge = sk.logmel_loge(sig)
    Em, El = ref.bound('ref')
    assert _report('ref mspec ' + name, mspec, ref.mspec, Em) <= 1.0
    assert _report('ref loge ' + name, loge, ref.loge, El) <= 1.0


@pytest.mark.parametrize('name', sorted(K1_CPU))
def test_fp32_emulation_within_bound(name):
    sig = K1_CPU[name]
    ref = fr.K1Ref(sig)
    mspec, loge = emulate_fp32(sig)
    Em, El = ref.bound('fp32')
    assert _report('fp32 mspec ' + name, mspec, ref.mspec, Em) <= 1.0
    assert _report('fp32 loge ' + name, loge, ref.loge, El) <= 1.0


def test_fp64_bound_is_a_few_float32_ulps():
    """In FFT_FP64 the float32 power rounding dominates: on speech-like audio the bound is a few float32 ulps of the
    log-mel value plus the power's relative rounding, not a blanket tolerance."""
    ref = fr.K1Ref(K1_CPU['synth20'])
    Em, El = ref.bound('fp64')
    fin = np.isfinite(ref.mspec) & (ref.B > 1e-6 * ref.B.max(axis=1, keepdims=True))
    assert np.isfinite(Em[fin]).all()
    assert (Em[fin] <= 8 * fr.U32 * (1 + np.abs(ref.mspec[fin]))).all()
    finl = np.isfinite(ref.loge)
    assert (El[finl] <= 4 * fr.U32 * (1 + np.abs(ref.loge[finl]))).all()


@pytest.mark.parametrize('name', ['silence_runs', 'impulse_last', 'impulse_first', 'dc_half', 'len400'])
def test_inf_exactly_where_the_exact_value_is_zero(name):
    """mspec is -inf exactly where the windowed frame is all zero (the Hann window is 0 at both ends: an impulse on a
    frame's last sample leaves its loge finite and its mspec -inf), loge exactly where y is all zero; the reference
    follows the same pattern."""
    sig = K1_CPU[name]
    ref = fr.K1Ref(sig)
    y = ref.y32
    assert np.array_equal(np.isneginf(ref.loge), ~y.any(axis=1))
    assert np.array_equal(np.isneginf(ref.mspec), np.repeat(~y[:, 1:-1].any(axis=1)[:, None], sk.NMEL, axis=1))
    mspec, loge = sk.logmel_loge(sig)
    assert np.array_equal(np.isneginf(mspec), np.isneginf(ref.mspec))
    assert np.array_equal(np.isneginf(loge), np.isneginf(ref.loge))
    if name == 'impulse_last':
        only_edge = y[:, 1:-1].any(axis=1) == 0
        assert (only_edge & y.any(axis=1)).any()                  # the case is really there
    # a finite value where the exact one is 0 fails the check, and so does -inf where it is not
    Em, El = ref.bound('ref')
    if np.isneginf(ref.mspec).any():
        bad = np.where(np.isneginf(ref.mspec), 0.0, ref.mspec)
        assert np.isinf(fr.ratio(bad, ref.mspec, Em)).any()
    fin = np.isfinite(ref.mspec) & np.isfinite(Em)
    if fin.any():
        bad = np.where(fin, -np.inf, ref.mspec)
        assert np.isinf(fr.ratio(bad, ref.mspec, Em)).any()


def test_mel_tasks_follow_the_upload_rule():
    """32 tasks at most, at most 24 bins each, up to 3 per filter, covering each filter's support exactly once."""
    bank = sk.mel_filterbank()[0]
    lo, cnt, tasks = fr.mel_tasks(bank)
    assert sum(len(t) for t in tasks) <= 32
    assert max(max(t) for t in tasks) <= 24 and max(len(t) for t in tasks) <= 3
    assert [sum(t) for t in tasks] == cnt
    for m in range(sk.NMEL):
        assert np.count_nonzero(bank[m, lo[m]:lo[m] + cnt[m]]) == np.count_nonzero(bank[m])


@pytest.mark.parametrize('name', sorted(k for k in K4_FIX if K4_FIX[k][2]))
def test_vbx_reference_faithfully_rounded(name):
    sig = K4_FIX[name][0]
    ref = fr.K4Ref(sig, dither=True)
    got = vx.get_features(sig)
    ok, r = ref.check(got)
    print('%-28s worst err/(E + ulp) %.3g   median E/ulp %.3g' % (
        'k4 ' + name, r.max(), np.median(ref.E / np.spacing(np.abs(ref.fea).astype(np.float32)))))
    assert ok.all(), (name, np.argwhere(~ok)[:4])


def test_vbx_clamp_rule():
    """Silence without dither: every band sum is 0, the clamp gives raw = 0 and the features are exactly 0; a sum within
    its bound of 1 accepts both sides of the clamp."""
    ref = fr.K4Ref(np.zeros(16000), dither=False)
    assert (ref.acc == 0).all() and (ref.fea == 0).all()
    ok, _ = ref.check(np.zeros_like(ref.fea))
    assert ok.all()
    ok, _ = ref.check(np.full_like(ref.fea, 1e-3))
    assert not ok.any()
