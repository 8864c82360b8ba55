"""Host mirror of the reference feature operator ``mfcc(sig, get_mspec=True)``
(inaSpeechSegmenter/sidekit_mfcc.py:278-352), computed by the K1 CUDA kernel.

Only the host-side constant tables are computed here (once, in float64, with
the reference's formulas -- they are inputs of the kernel, exactly as the
reference recomputes ``trfbank`` on every call, sidekit_mfcc.py:332); all
per-sample work happens on the GPU.
"""
import numpy as np
import torch

from . import _lib

WIN, HOP, NFFT, NMEL = 400, 160, 512, 24


def trfbank_htk24(fs=16000, nfft=NFFT, lowfreq=100, maxfreq=8000, nfilt=NMEL):
    """The 24 area-normalised HTK-mel triangles ``trfbank(16000, 512, 100,
    8000, 0, 24)[0]`` builds (sidekit_mfcc.py:118-197, nlinfilt == 0 branch
    :146-154): float32 [24, 257]."""
    mel = lambda f: 2595 * np.log10(1 + f / 700.)           # noqa: E731  (hz2mel, :54-63)
    imel = lambda z: 700. * (10 ** (z / 2595.) - 1)          # noqa: E731  (mel2hz, :86-95)
    lo, hi = mel(lowfreq), mel(maxfreq)
    pts = np.zeros(nfilt + 2)
    pts[:] = lo + np.arange(nfilt + 2) * ((hi - lo) / (nfilt + 1))
    f = imel(pts)
    height = 2. / (f[2:] - f[:-2])
    table = np.zeros((nfilt, nfft // 2 + 1), dtype=np.float32)
    hz = np.arange(nfft) / (1. * nfft) * fs
    for i in range(nfilt):
        b_lo = np.floor(f[i] * nfft / fs) + 1
        b_mid = np.floor(f[i + 1] * nfft / fs) + 1
        b_hi = min(np.floor(f[i + 2] * nfft / fs) + 1, nfft)
        rise = np.arange(b_lo, b_mid, dtype=np.int32)
        fall = np.arange(b_mid, b_hi, dtype=np.int32)[:-1]     # the right slope drops its last bin (:195)
        table[i][rise] = (height[i] / (f[i + 1] - f[i])) * (hz[rise] - f[i])
        table[i][fall] = (height[i] / (f[i + 2] - f[i + 1])) * (f[i + 2] - hz[fall])
    return table


def num_frames(n_samples):
    return int(_lib.load().iss_sidekit_num_frames(int(n_samples)))


def _pcm_format(dtype):
    if dtype == torch.int16:
        return _lib.PCM_S16
    if dtype == torch.float32:
        return _lib.PCM_F32
    raise TypeError('pcm must be int16 or float32, got %s' % dtype)


class SidekitFrontEnd:
    """Owns one library context with the front-end tables uploaded."""

    def __init__(self, ctx):
        self.ctx = ctx
        self._fbank = np.ascontiguousarray(trfbank_htk24())
        self._window = np.ascontiguousarray(np.hanning(WIN), dtype=np.float64)      # sidekit_mfcc.py:223
        lib = _lib.load()
        _lib.check(lib.iss_sidekit_upload_tables(ctx.handle, _lib.ptr(self._fbank), _lib.ptr(self._window)),
                   'iss_sidekit_upload_tables')

    def multi(self, pcms, layout, fft_precision=_lib.FFT_FP64, stream=None):
        """pcms: 1-D contiguous CUDA tensors of one dtype (int16 or float32); layout: pack.PassLayout of their sample
        counts.  Returns (mspec[layout.total_rows, 24] f32 with recording i at rows layout.row_off[i] ..,
        loge f32 packed at layout.loge_off, stats[n, 2] f64), all on device; each recording's values are those of
        __call__ on it.  Rows reserved past a recording's frames are left unwritten."""
        fmt = _pcm_format(pcms[0].dtype)
        assert all(p.is_cuda and p.dim() == 1 and p.is_contiguous() and p.dtype == pcms[0].dtype for p in pcms)
        n = len(pcms)
        dev = pcms[0].device
        mspec = torch.empty((layout.total_rows, NMEL), dtype=torch.float32, device=dev)
        loge = torch.empty((int(layout.loge_off[-1]),), dtype=torch.float32, device=dev)
        stats = torch.empty((n, 2), dtype=torch.float64, device=dev)
        ptrs = (_lib._c.c_void_p * n)(*[p.data_ptr() for p in pcms])
        n_samples = np.ascontiguousarray([p.numel() for p in pcms], dtype=np.int64)
        row_off = np.ascontiguousarray(layout.row_off, dtype=np.int64)
        loge_off = np.ascontiguousarray(layout.loge_off[:-1], dtype=np.int64)
        st = stream if stream is not None else torch.cuda.current_stream(dev)
        _lib.check(_lib.load().iss_sidekit_features_multi(
            self.ctx.handle, n, ptrs, _lib.ptr(n_samples), fmt, int(fft_precision), _lib.ptr(mspec), _lib.ptr(row_off),
            _lib.ptr(loge), _lib.ptr(loge_off), _lib.ptr(stats), _lib._c.c_void_p(st.cuda_stream)),
            'iss_sidekit_features_multi')
        return mspec, loge, stats

    def __call__(self, pcm, fft_precision=_lib.FFT_FP64, stream=None):
        """pcm: CUDA tensor, int16 or float32, 1-D.  Returns (mspec[L,24] f32,
        loge[L] f32, stats[2] f64 = (sum, count) of finite loge), all on device."""
        assert pcm.is_cuda and pcm.dim() == 1 and pcm.is_contiguous()
        fmt = _pcm_format(pcm.dtype)
        n = pcm.numel()
        L = num_frames(n)
        dev = pcm.device
        mspec = torch.empty((L, NMEL), dtype=torch.float32, device=dev)
        loge = torch.empty((L,), dtype=torch.float32, device=dev)
        stats = torch.empty((2,), dtype=torch.float64, device=dev)
        st = stream if stream is not None else torch.cuda.current_stream(dev)
        _lib.check(_lib.load().iss_sidekit_features(
            self.ctx.handle, _lib.ptr(pcm), fmt, n, int(fft_precision), _lib.ptr(mspec), _lib.ptr(loge),
            _lib.ptr(stats), _lib._c.c_void_p(st.cuda_stream)), 'iss_sidekit_features')
        return mspec, loge, stats
