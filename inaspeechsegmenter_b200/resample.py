"""Audio at any integer sample rate from 8 to 192 kHz with 1 to 8 channels, turned into the 16 kHz mono int16 PCM the
front ends take, on the device (resample.cu, DESIGN.md "Resampling").

For a recording x of n frames, C channels at rate R: the float64 mean of the channels of each frame (int16 s as
s / 32768), then ``scipy.signal.resample_poly(x, up, down)`` with up = 16000 / g, down = R / g, g = gcd(16000, R) and
scipy's default filter, then ``clip(rint(y * 32768), -32768, 32767)`` as int16: what a pcm_s16le decode delivers.  This
is not ffmpeg's resampler.  16 kHz mono input never comes here: it keeps the float path of the front ends.

Only the filter taps are computed on the host (float64, a numpy restatement of scipy's design, as ``trfbank_htk24``
restates sidekit's filterbank); they are uploaded once per context and rate.
"""
import functools
import math
import weakref

import numpy as np
import torch

from . import _lib, pack

TARGET_RATE = 16000
MIN_RATE, MAX_RATE = 8000, 192000
MAX_CHANNELS = 8
KAISER_BETA = 5.0
# pcm_format of each WAV encoding (io.wav_data); the device reads u8 / s24 / s32 / f64 only through WAV files
PCM_FORMATS = {'u8': _lib.PCM_U8, 's16': _lib.PCM_S16, 's24': _lib.PCM_S24, 's32': _lib.PCM_S32, 'f32': _lib.PCM_F32,
               'f64': _lib.PCM_F64}


def check_rate(rate):
    """The rate as an int; ValueError unless it is an integer in [8000, 192000]."""
    try:
        r = int(rate)
    except (TypeError, ValueError, OverflowError):
        raise ValueError('sample rate %r is not an integer' % (rate,)) from None
    if isinstance(rate, bool) or r != rate:
        raise ValueError('sample rate %r is not an integer' % (rate,))
    if not MIN_RATE <= r <= MAX_RATE:
        raise ValueError('sample rate %d Hz is outside [%d, %d]' % (r, MIN_RATE, MAX_RATE))
    return r


def factors(rate):
    """(up, down) of resample_poly for a rate of `rate` Hz to 16 kHz."""
    g = math.gcd(TARGET_RATE, rate)
    return TARGET_RATE // g, rate // g


def num_frames(n, rate):
    """16 kHz samples of a recording of n frames at `rate` Hz: ceil(n * up / down) (iss_resample_num_frames)."""
    up, down = factors(rate)
    return -(-n * up // down)


@functools.lru_cache(maxsize=None)
def reach(rate):
    """(s_min, e_max) of `rate`: output k, with k * down = a * up + q, reads the frames a + s_q .. a + s_q + n_q - 1; s_min
    is the least s_q and e_max the largest s_q + n_q over the phases (the phase table of iss_resample_upload_taps)."""
    up, down = factors(rate)
    half = 0 if up == down == 1 else 10 * max(up, down)
    b, r = divmod(half, up)
    q = np.arange(up)
    carry = (q + r >= up).astype(np.int64)
    nq = (2 * half - (q + r - carry * up)) // up + 1
    s = b + carry - (nq - 1)
    return int(s.min()), int((s + nq).max())


# Live streams (stream.py) resample chunk by chunk: a stream's outputs are computed once the frames they read have
# arrived, from a window of its input that starts at its first frame still needed, and are the outputs of the whole
# stream bit for bit (iss_resample_window_multi).  These three functions are the whole rule.
def ready_outputs(n, rate):
    """Outputs final once n frames have arrived: every k with floor(k * down / up) + e_max - 1 <= n - 1."""
    return min(num_frames(max(n - reach(rate)[1] + 1, 0), rate), num_frames(n, rate))


def end_outputs(n, rate):
    """Outputs of a stream that ended after n frames (the last ones read the zeros past its end)."""
    return num_frames(n, rate)


def first_kept(k_next, rate):
    """First input frame any output from k_next on reads (0 while that is before the stream): the start of a
    stream's retained tail once its outputs below k_next are computed."""
    up, down = factors(rate)
    return max(k_next * down // up + reach(rate)[0], 0)


@functools.lru_cache(maxsize=None)
def lowpass(up, down):
    """float64 taps of resample_poly's default filter, ``firwin(2 * 10 * M + 1, 1 / M, window=('kaiser', 5.0)) * up``
    with M = max(up, down); the single tap 1 when up == down == 1 (resample_poly then returns its input)."""
    if up == down == 1:
        return np.ones(1)
    M = max(up, down)
    N = 2 * 10 * M + 1
    cutoff = 1.0 / M
    alpha = 0.5 * (N - 1)
    m = np.arange(N, dtype=np.float64) - alpha
    h = cutoff * np.sinc(cutoff * m)
    h *= np.i0(KAISER_BETA * np.sqrt(1 - (m / alpha) ** 2.0)) / np.i0(KAISER_BETA)
    h /= np.sum(h)
    h *= up
    h.setflags(write=False)
    return h


def shape(sig):
    return tuple(sig.shape) if hasattr(sig, 'shape') else np.shape(sig)


def channels(sig):
    s = shape(sig)
    return 1 if len(s) == 1 else int(s[1])


def is_native(sig, rate):
    """True for 16 kHz mono (1-D, or one column), which takes the front ends' own path.  Checks the rate."""
    return check_rate(rate) == TARGET_RATE and len(shape(sig)) in (1, 2) and channels(sig) == 1


def as_input(sig):
    """A recording to resample as a C-contiguous [frames] or [frames, channels] int16 / float32 numpy array or CUDA
    tensor.  TypeError for another sample type, ValueError for another shape or channel count."""
    if isinstance(sig, torch.Tensor) and not sig.is_cuda:
        sig = sig.numpy()
    if isinstance(sig, torch.Tensor):
        if sig.dtype not in (torch.int16, torch.float32):
            raise TypeError('resampled pcm must be int16 or float32, got %s' % sig.dtype)
    else:
        sig = np.asarray(sig)
        if sig.dtype not in (np.int16, np.float32):
            raise TypeError('resampled pcm must be int16 or float32, got %s' % sig.dtype)
    if sig.ndim not in (1, 2):
        raise ValueError('pcm must be [frames] or [frames, channels], got shape %r' % (tuple(sig.shape),))
    if not 1 <= channels(sig) <= MAX_CHANNELS:
        raise ValueError('%d channels: 1 to %d are supported' % (channels(sig), MAX_CHANNELS))
    if isinstance(sig, torch.Tensor):
        return sig.contiguous()
    return np.ascontiguousarray(sig)


def _dtype_name(sig):
    return str(sig.dtype).split('.')[-1]


def plan(sigs, rates):
    """pack.plan_passes over the 16 kHz lengths: signals as _pass_input returns them, each with its checked rate.
    Resampled recordings count as int16 (what the front ends read), native ones by their dtype.  Raises the
    ValueError of pack.check_lengths for a recording too short after resampling.  Returns (passes, long)."""
    n16 = [s.shape[0] if r == TARGET_RATE and s.ndim == 1 else num_frames(int(s.shape[0]), r)
           for s, r in zip(sigs, rates)]
    kinds = [_dtype_name(s) if r == TARGET_RATE and s.ndim == 1 else 'int16' for s, r in zip(sigs, rates)]
    pack.check_lengths(n16)
    return pack.plan_passes(n16, kinds)


def check_rates(sample_rates, n):
    rates = [TARGET_RATE] * n if sample_rates is None else [check_rate(r) for r in sample_rates]
    if len(rates) != n:
        raise ValueError('%d signals but %d sample rates' % (n, len(rates)))
    return rates


_uploaded = weakref.WeakKeyDictionary()        # engine.Context -> rates whose taps it holds


def _ensure_taps(ctx, rate):
    done = _uploaded.setdefault(ctx, set())
    if rate not in done:
        h = np.ascontiguousarray(lowpass(*factors(rate)))
        _lib.check(_lib.load().iss_resample_upload_taps(ctx.handle, rate, _lib.ptr(h), h.size), 'iss_resample_upload_taps')
        done.add(rate)


def to16k_multi(ctx, pcms, rate, out, out_off, stream=None, encoding=None):
    """Resamples CUDA tensors of one rate, channel count and dtype ([frames] or [frames, channels], contiguous) in one
    launch; recording i's num_frames(len, rate) samples go to the int16 CUDA tensor `out` from out_off[i].  With an
    `encoding` (a key of PCM_FORMATS), the tensors are uint8 [frames, channels, bytes per sample]: samples as a WAV
    stores them (io.WavData.shape)."""
    x0 = pcms[0]
    if encoding is None:
        fmt = {torch.int16: _lib.PCM_S16, torch.float32: _lib.PCM_F32}[x0.dtype]
    else:
        fmt = PCM_FORMATS[encoding]
        assert x0.dtype == torch.uint8 and x0.dim() == 3
    C = channels(x0)
    assert all(p.is_cuda and p.is_contiguous() and p.dtype == x0.dtype and channels(p) == C for p in pcms)
    _ensure_taps(ctx, rate)
    n = len(pcms)
    ptrs = (_lib._c.c_void_p * n)(*[p.data_ptr() for p in pcms])
    frames = np.ascontiguousarray([p.shape[0] for p in pcms], dtype=np.int64)
    off = np.ascontiguousarray(out_off[:n], dtype=np.int64)
    st = stream if stream is not None else torch.cuda.current_stream(x0.device)
    _lib.check(_lib.load().iss_resample_to16k_multi(
        ctx.handle, n, ptrs, _lib.ptr(frames), C, rate, fmt, _lib.ptr(out), _lib.ptr(off), _lib._c.c_void_p(st.cuda_stream)),
        'iss_resample_to16k_multi')


def window_multi(ctx, pcms, win, rate, out, stream=None):
    """Windows of streams of one rate, channel count and dtype in one launch (iss_resample_window_multi): pcms[i] is a
    contiguous CUDA tensor holding frames [f_base, n_known) of stream i, win an int64 array of rows (f_base, n_known,
    k_first, n_out, out_off, flags); the outputs go to the int16 CUDA tensor `out`."""
    x0 = pcms[0]
    fmt = {torch.int16: _lib.PCM_S16, torch.float32: _lib.PCM_F32}[x0.dtype]
    C = channels(x0)
    assert all(p.is_cuda and p.is_contiguous() and p.dtype == x0.dtype and channels(p) == C for p in pcms)
    _ensure_taps(ctx, rate)
    n = len(pcms)
    ptrs = (_lib._c.c_void_p * n)(*[p.data_ptr() for p in pcms])
    win = np.ascontiguousarray(win, dtype=np.int64).reshape(n, 6)
    st = stream if stream is not None else torch.cuda.current_stream(x0.device)
    _lib.check(_lib.load().iss_resample_window_multi(
        ctx.handle, n, ptrs, _lib.ptr(win), C, rate, fmt, _lib.ptr(out), _lib._c.c_void_p(st.cuda_stream)),
        'iss_resample_window_multi')


def resample_pass(ctx, pcms, rates, encodings=None):
    """16 kHz mono device views of the device recordings of one pass (what _stage_pass returns), one launch per
    (rate, channels, dtype, encoding) group.  encodings[i] is None, or the encoding of a WAV's stored bytes (see
    to16k_multi).  16 kHz mono recordings are returned as they are; the others land in one int16 buffer, each 16-byte
    aligned."""
    encodings = encodings or [None] * len(pcms)
    todo = [i for i, (p, r) in enumerate(zip(pcms, rates)) if not (r == TARGET_RATE and p.dim() == 1)]
    if not todo:
        return list(pcms)
    n16 = [num_frames(int(pcms[i].shape[0]), rates[i]) for i in todo]
    off = pack.PassLayout(n16, 2).stage_off
    out = torch.empty(int(off[-1]), dtype=torch.int16, device=pcms[todo[0]].device)
    groups = {}
    for j, i in enumerate(todo):
        groups.setdefault((rates[i], channels(pcms[i]), pcms[i].dtype, encodings[i]), []).append(j)
    for (rate, _, _, enc), js in groups.items():
        to16k_multi(ctx, [pcms[todo[j]] for j in js], rate, out, [off[j] for j in js], encoding=enc)
    res = list(pcms)
    for j, i in enumerate(todo):
        res[i] = out[off[j]:off[j] + n16[j]]
    return res


def to16k(ctx, sig, rate):
    """One recording (numpy array or tensor, [frames] or [frames, channels]) at `rate` Hz as a 16 kHz int16 CUDA
    tensor, through the same launch as a pass of one."""
    from .segmenter import _stage_pass
    return resample_pass(ctx, _stage_pass([as_input(sig)], ctx.device), [check_rate(rate)])[0]
