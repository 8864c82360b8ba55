"""Oracle (test infrastructure): the two feature front ends in float64, with an error bound next to every value.

K1 (``feat_sidekit.cu``, log-mel + log-energy).  The exact input is the float32 pre-emphasised frame
``y = fl32(x - fl32(0.97f * x_prev))`` (a frame's first sample is its own predecessor): the kernel (``__fsub_rn`` /
``__fmul_rn``) and the reference (``sidekit_oracle.pre_emphasise``, numpy float32) compute it identically, so ``y`` is
shared and not a source of error.  From ``y``, in float64: ``v = y * hanning``, the 512-point DFT ``X``, ``P = |X|^2``,
``B = P @ bank.T`` with the float32 bank, ``mspec = log B``; ``loge = log(sum y^2)``.  Next to each value sits a bound
for three recipes:

  fp64  K1 in FFT_FP64: window, FFT and power in float64, power stored as float32, mel sums in float64, log in float64
  fp32  K1 in FFT_FP32: float32 window table, FFT, power, mel sums and logf
  ref   the reference's own recipe (sidekit_mfcc.py): float64 FFT, power stored as float32, float32 dot, float32 log

Terms, per frame and bin, for unit round-off u_T of the recipe:
  window   (u_T + u_w) sqrt(512) ||v||_2 with u_w = 2^-24 for the float32 window table of fp32 mode
  FFT      D = C_FFT log2(512) u_T sqrt(512) ||v||_2 (Parseval: a norm bound on the error vector, applied to every bin;
           it covers the rounded twiddles, the 1/sqrt2 products and FMA contraction)
  power    2 |X_k| D + D^2, the recipe's power arithmetic, and the rounding of the power to float32
  mel      the kernel's accumulation: at most ceil(bins / 2) + 1 steps per task (two chains) and the filter's tasks
           (``iss_sidekit_upload_tables``' rule, mirrored by ``mel_tasks``); the reference's float32 dot gets one step
           per non-zero weight (adding exact zeros is exact, so BLAS' order does not matter).  Then the rounding to float32.
  log      dB / (B - dB) (unbounded when dB >= B), the log's own error and the output ulp
The float64 evaluation here adds its own FFT and window term to D.  loge: the kernel's double sum makes its bound about
one float32 ulp; the reference's float32 pairwise sum (numpy: 400 -> 200 -> 96 | 104, eight running sums of <= 13
terms, then three combining levels) gets 18 u32 with the squares.

C_FFT is not the worst-case constant of the classic analysis (about 7 per level): the levels' rounding errors add as a
random walk (about sqrt(9) levels' worth on the error norm), so C_FFT = 2 still leaves a factor of about 6 over that
norm, which itself bounds every bin.  The worst-case constant would hide an error of a few hundred ulps in one window
sample, which is what a wrongly computed window table makes at the window's edges.

K4 (``feat_vbx.cu``, VBx fbank + floating CMVN) restates ``vbx_oracle.raw_fbank`` and ``cmvn_floating`` (pinned bit
for bit to the reference).  The kernel is all float64, so the bound is a float64 term (the same FFT model with
u_T = 2^-53, plus the frame-mean and pre-emphasis roundings, for the kernel and for this evaluation, carried through
``log(max(1, acc))`` and the CMVN mean), and the check is faithful rounding of the float32 output: ``got`` is a float32
neighbour of a value within the float64 term of the exact one.  The clamp: ``[log max(1, acc - dacc),
log max(1, acc + dacc)]`` is accepted, so within the bound of ``acc = 1`` either side is.
"""
import numpy as np

from . import sidekit_oracle as sk
from . import vbx_oracle as vx

U32, U64 = 2.0 ** -24, 2.0 ** -53
ETA32 = 2.0 ** -150                 # half the smallest float32 subnormal: absolute rounding error of a result near 0
C_FFT = 2.0
LOG2N = 9                           # log2(512)
SQRTN = np.sqrt(512.0)
RECIPES = ('fp64', 'fp32', 'ref')
# the log's error with the output rounding, in float32 ulps of the result (ulp(r) <= 2^-23 |r|): double log then
# rounded; CUDA logf (1 ulp, CUDA C Programming Guide); numpy's float32 log (3.3 ulps measured on 2.5e7 values)
LOG_ULPS = {'fp64': 0.5 + 1e-6, 'fp32': 1.0, 'ref': 4.0}
LOGE_REF_STEPS = 18                 # the square + numpy's pairwise float32 sum of 400 terms (see above)
LOGE_KERNEL_STEPS = 18              # the kernel's double sum: 13 terms per lane + 5 shuffle levels


def _gamma(n, u):
    n = np.asarray(n, dtype=np.float64)
    return n * u / (1.0 - n * u)


def mel_tasks(bank):
    """The kernel's balanced mel tasks (iss_sidekit_upload_tables): the smallest cap of bins per task for which all
    filters fit 32 tasks, a filter's bins dealt to its tasks as evenly as possible.  Returns (lo, cnt) per filter and
    the list of task lengths per filter."""
    nz = [np.flatnonzero(r) for r in bank]
    lo = [int(z[0]) if len(z) else 0 for z in nz]
    cnt = [int(z[-1] - z[0] + 1) if len(z) else 0 for z in nz]
    cap = 1
    while sum((c + cap - 1) // cap for c in cnt) > 32:
        cap += 1
    tasks = []
    for c in cnt:
        parts = (c + cap - 1) // cap
        lens, done = [], 0
        for q in range(parts):
            n = (c - done + (parts - q) - 1) // (parts - q)
            lens.append(n)
            done += n
        tasks.append(lens)
    return lo, cnt, tasks


def _k1_mel_steps(bank):
    """Rounding steps a term of filter m goes through: the recipe of feat_sidekit.cu (fp32 / fp64) or a dot (ref)."""
    _, cnt, tasks = mel_tasks(bank)
    kernel = np.array([(max(t) + 1) // 2 + 1 + 1 + len(t) if t else 0 for t in tasks], dtype=np.float64)
    ref = np.array(cnt, dtype=np.float64)
    return kernel, ref


def _log_error(val, dval):
    """Bound on |log(val_hat) - log(val)| for |val_hat - val| <= dval: -log1p(-dval / val), inf when dval >= val."""
    with np.errstate(divide='ignore', invalid='ignore'):
        q = dval / val
        return np.where(q < 1.0, -np.log1p(-np.where(q < 1.0, q, 0.0)), np.inf)


def preemphasised_frames(sig):
    """[L, 400] float32 y of a float32 signal, exactly as K1 and the reference compute it."""
    return sk.pre_emphasise(sk.frame_signal(np.asarray(sig, dtype=np.float32)))


class K1Ref:
    """Float64 values of K1's outputs for one float32 signal (int16 PCM is its samples / 32768) and their bounds.

    mspec [L, 24], loge [L] (float64, -inf where the exact value is 0); B, E the exact mel sums and energies;
    bound(recipe) -> (E_mspec, E_loge) with inf where the bound is unbounded."""

    def __init__(self, sig):
        y32 = preemphasised_frames(sig)
        self.y32 = y32
        y = y32.astype(np.float64)
        self.win = sk.hann_window()
        self.bank32 = sk.mel_filterbank()[0]
        bank = self.bank32.astype(np.float64)
        self.bank = bank
        v = y * self.win
        X = np.fft.rfft(v, sk.NFFT, axis=-1)
        self.A = np.abs(X)
        self.P = self.A ** 2
        self.B = self.P @ bank.T
        self.E = (y * y).sum(axis=1)
        self.nv = np.sqrt((v * v).sum(axis=1))[:, None]
        with np.errstate(divide='ignore'):
            self.mspec = np.log(self.B)
            self.loge = np.log(self.E)
        self.kernel_steps, self.ref_steps = _k1_mel_steps(self.bank32)

    def mel_sum_error(self, recipe):
        """dB: the bound on |B_hat - B| before the log, [L, 24]."""
        uT = U32 if recipe == 'fp32' else U64
        uw = U32 if recipe == 'fp32' else 0.0
        # the recipe's window + FFT, and this evaluation's own (float64 rfft of a float64 product)
        D = ((C_FFT * LOG2N * uT + uT + uw) + (C_FFT * LOG2N + 2.0) * U64) * SQRTN * self.nv
        Ph = (self.A + D) ** 2
        dP = 2.0 * self.A * D + D * D + 2.0 * uT * Ph
        if recipe == 'fp32':
            dP += 2.0 * ETA32                                   # float32 squares near the underflow
        else:
            dP += U32 * (self.P + dP) + ETA32                   # power stored as float32
        dB = dP @ self.bank.T
        Bh = self.B + dB
        if recipe == 'fp32':
            dB = dB + _gamma(self.kernel_steps, U32) * Bh + self.kernel_steps * ETA32
        elif recipe == 'fp64':
            dB = dB + _gamma(self.kernel_steps, U64) * Bh
            dB = dB + U32 * (self.B + dB) + ETA32                # (float) acc
        else:
            dB = dB + _gamma(self.ref_steps, U32) * Bh + self.ref_steps * ETA32
        return dB

    def energy_error(self, recipe):
        if recipe == 'ref':
            dE = _gamma(LOGE_REF_STEPS, U32) * self.E + 400 * ETA32
        else:
            dE = _gamma(LOGE_KERNEL_STEPS, U64) * self.E
            dE = dE + U32 * (self.E + dE) + ETA32                # (float) e
        return dE + _gamma(LOGE_KERNEL_STEPS, U64) * self.E     # this evaluation's pairwise double sum

    def bound(self, recipe):
        ulps = LOG_ULPS[recipe]
        Em = _log_error(self.B, self.mel_sum_error(recipe))
        El = _log_error(self.E, self.energy_error(recipe))
        with np.errstate(invalid='ignore'):
            Em = Em + ulps * 2 * U32 * (np.abs(self.mspec) + Em) + ETA32
            El = El + ulps * 2 * U32 * (np.abs(self.loge) + El) + ETA32
        Em[self.B == 0] = 0.0
        El[self.E == 0] = 0.0
        return Em, El


def ratio(got, ref, E):
    """|got - ref| / E elementwise.  Where the exact value is 0 (ref = -inf) only -inf passes; where the bound is
    unbounded (E = inf) anything but NaN / +inf passes, -inf included (the float32 sums may underflow)."""
    got = np.asarray(got, dtype=np.float64)
    zero = np.isneginf(ref)
    with np.errstate(invalid='ignore'):
        d = np.abs(got - ref)
        r = np.where(np.isfinite(E) & (E > 0), d / np.where(np.isfinite(E) & (E > 0), E, 1.0), np.where(d == 0, 0.0, np.inf))
    r = np.where(zero, np.where(np.isneginf(got), 0.0, np.inf), r)
    r = np.where(~zero & ~np.isfinite(E), np.where(np.isnan(got) | np.isposinf(got), np.inf, 0.0), r)
    return np.where(np.isnan(r), np.inf, r)


def tightness(got, ref, E):
    """(median of E / err over values with a finite bound and a non-zero error, worst err / E): how far the bound sits
    above the error actually made."""
    got = np.asarray(got, dtype=np.float64)
    ok = np.isfinite(ref) & np.isfinite(E) & np.isfinite(got)
    err = np.abs(got[ok] - ref[ok])
    nz = err > 0
    med = float(np.median(E[ok][nz] / err[nz])) if nz.any() else float('inf')
    r = ratio(got, ref, E)
    return med, float(r.max()) if r.size else 0.0


# ------------------------------------------------------------------ K4
def _down32(a):
    f = a.astype(np.float32)
    return np.where(f.astype(np.float64) > a, np.nextafter(f, np.float32(-np.inf)), f).astype(np.float64)


def _up32(a):
    f = a.astype(np.float32)
    return np.where(f.astype(np.float64) < a, np.nextafter(f, np.float32(np.inf)), f).astype(np.float64)


class K4Ref:
    """Float64 features of K4 for one signal and their float64 error term.

    signal: the samples as float64 (int16 PCM is its samples / 32768; float input its float32 values); dither: whether
    the kernel adds the reference's dither stream.  fea [M, 64], E [M, 64]; check(got, c) -> (ok mask, ratio)."""

    def __init__(self, signal, dither=True):
        x = vx.quantise(signal).astype(np.float64)
        if dither:
            x = x + vx.dither_stream(len(signal))
        seg = np.r_[x[vx.NOVERLAP // 2 - 1::-1], x, x[-1:-vx.FRAME // 2 - 1:-1]]
        M = (len(seg) - vx.FRAME) // (vx.FRAME - vx.NOVERLAP) + 1
        fr = np.lib.stride_tricks.sliding_window_view(seg, vx.FRAME)[::vx.FRAME - vx.NOVERLAP][:M]
        xmax = np.abs(fr).max(axis=1, keepdims=True)
        xc = fr - fr.mean(axis=1, keepdims=True)
        xp = np.c_[xc[:, :1], xc[:, :-1]]
        win = vx.povey_window()
        v = (xc - xp * 0.97) * win
        X = np.fft.rfft(v, vx.NFFT, axis=-1)
        A = np.abs(X)
        P = A ** 2
        mfb = vx.mel_bank()
        acc = P @ mfb
        # float64 term, kernel and this evaluation alike: the frame mean (<= 18 steps over |x| <= xmax) shifts every
        # sample, the pre-emphasis and the window round, and the FFT adds C_FFT log2(512) u64 of the norm
        dmean = _gamma(LOGE_KERNEL_STEPS, U64) * xmax
        dv = win * (2.0 * dmean + 3.0 * U64 * (np.abs(xc) + np.abs(xp)))
        nv = np.sqrt((v * v).sum(axis=1, keepdims=True))
        D = 2.0 * (dv.sum(axis=1, keepdims=True) + (C_FFT * LOG2N + 1.0) * U64 * SQRTN * nv)
        dP = 2.0 * A * D + D * D + 2.0 * U64 * (A + D) ** 2
        cnt = np.count_nonzero(mfb, axis=0).astype(np.float64)
        dacc = dP @ mfb
        dacc = dacc + 2.0 * _gamma(cnt, U64) * (acc + dacc)
        raw = np.log(np.maximum(1.0, acc))
        hi = np.log(np.maximum(1.0, acc + dacc))
        lo = np.log(np.maximum(1.0, acc - dacc))
        Eraw = np.maximum(hi - raw, raw - lo) + 4.0 * U64 * np.abs(raw)
        # floating CMVN (cmvn_floating_kaldi, LC = 150, RC = 149): the window shifts at the edges, it does not shrink
        N = M
        wl = min(N, 300)
        ws = np.maximum(np.minimum(np.arange(-150, N - 150), N - wl), 0)
        sums = np.lib.stride_tricks.sliding_window_view(raw, wl, axis=0).sum(axis=-1)     # [N - wl + 1, 64]
        esums = np.lib.stride_tricks.sliding_window_view(Eraw, wl, axis=0).sum(axis=-1)
        mean = sums[ws] / wl
        absmax = np.abs(raw).max(axis=0, keepdims=True)
        # kernel: a direct sum of wl rows, then <= 127 one-row slides of two roundings each; this evaluation: one sum
        dsum = U64 * (2 * wl + 2 * 128 + 4) * wl * absmax
        self.M = M
        self.acc, self.dacc, self.raw, self.Eraw = acc, dacc, raw, Eraw
        self.fea = raw - mean
        self.E = Eraw + esums[ws] / wl + dsum / wl + 4.0 * U64 * (np.abs(raw) + np.abs(mean))

    def check(self, got, c=1.0):
        """(ok, ratio): ok where got is a float32 neighbour of a value within c . E of the exact one; ratio is
        |got - fea| / (c . E + ulp32(fea)), below 1 for a faithfully rounded result with no float64 error."""
        got = np.asarray(got, dtype=np.float64)
        lo, hi = _down32(self.fea - c * self.E), _up32(self.fea + c * self.E)
        ok = (got >= lo) & (got <= hi)
        ulp = np.spacing(np.abs(self.fea).astype(np.float32)).astype(np.float64)
        return ok, np.abs(got - self.fea) / (c * self.E + ulp)
