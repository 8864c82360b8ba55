"""VBx x-vector path on the GPU: host mirror of the numeric part of the reference's
``vbx_segmenter.py`` (constants :21-25, ``get_features`` :72-89, the
``VBxExtractor`` plugin ABC :205-246 and a backend :249-266).

``B200BackendExtractor`` is a drop-in for ``OnnxBackendExtractor``: same
``get_embedding(fea[T,64]) -> [256]`` and ``__call__(basename, fea, duration)``
contract, but ``__call__`` embeds all windows in batches on the GPU instead of
one ONNX call per 0.24 s of audio.  ``VoiceFemininityScoring`` (:92-202, SURVEY
N3) is mirrored at the end of the file: the MLP runs on device (``iss_mlp_*``),
the pyannote interval bookkeeping is restated in plain Python.
"""
import ctypes
import logging
import os
from abc import ABC, abstractmethod

import numpy as np
import torch

from . import _lib, pack
from .engine import Context, _stream_ptr
from .pack import window_plan  # noqa: F401  (kept importable from this module)

logger = logging.getLogger(__name__)

STEP = 24
WINLEN = 144
FEAT_DIM = 64
EMBED_DIM = 256
SR = 16000
NUM_BLOCKS = (3, 4, 23, 3)          # resnet.py:133-135 (ResNet101)
M_CHANNELS = 32                     # resnet.py:79


# ------------------------------------------------------------------ host tables (features_vbx.py)
def povey_window(winlen=400):
    """features_vbx.py:123-124."""
    return np.power(0.5 - 0.5 * np.cos(np.linspace(0, 2 * np.pi, winlen)), 0.85)


def mel_fbank_htk64(nfft=512, fs=SR, nchan=FEAT_DIM, lofreq=20.0, hifreq=7600.0):
    """mel_fbank_mx(400, 16000, NUMCHANS=64, LOFREQ=20, HIFREQ=7600, htk_bug=False)
    (features_vbx.py:31-59): float64 [257, 64]."""
    warp = lambda x: 1127. * np.log(1. + x / 700.)         # noqa: E731
    unwarp = lambda x: (np.exp(x / 1127.) - 1.) * 700.     # noqa: E731
    bins = warp(np.arange(nfft / 2 + 1, dtype=float) * fs / nfft)
    cent = np.linspace(warp(lofreq), warp(hifreq), nchan + 2)
    idx = np.floor(unwarp(cent) / fs * nfft).astype(int) + 1
    mx = np.zeros((len(bins), nchan))
    for i in range(nchan):
        mx[idx[i]:idx[i + 1], i] = (cent[i] - bins[idx[i]:idx[i + 1]]) / (cent[i] - cent[i + 1])
        mx[idx[i + 1]:idx[i + 2], i] = (cent[i + 2] - bins[idx[i + 1]:idx[i + 2]]) / (cent[i + 2] - cent[i + 1])
    return mx


class DitherCache:
    """Device-resident prefix of the dither the reference draws with
    ``np.random.seed(3); 8 * (np.random.rand(n) * 2 - 1)`` (vbx_segmenter.py:84-85,
    features_vbx.py:127-128).  The stream does not depend on the signal, so it is
    generated once (legacy MT19937 via RandomState(3): same doubles, no global
    RNG side effect) and kept in HBM; longer requests regenerate a longer prefix."""

    def __init__(self, device, level=8):
        self.device, self.level, self.buf = device, level, None

    def get(self, n):
        if self.buf is None or self.buf.numel() < n:
            cap = max(n, 16000 * 60)
            host = self.level * (np.random.RandomState(3).rand(cap) * 2 - 1)
            self.buf = torch.from_numpy(host).to(self.device)
        return self.buf


class VbxFrontEnd:
    def __init__(self, ctx):
        self.ctx = ctx
        self._fbank = np.ascontiguousarray(mel_fbank_htk64(), dtype=np.float64)
        self._window = np.ascontiguousarray(povey_window(400), dtype=np.float64)
        _lib.check(_lib.load().iss_vbx_upload_tables(ctx.handle, _lib.ptr(self._fbank), _lib.ptr(self._window)),
                   'iss_vbx_upload_tables')
        self.dither = DitherCache(ctx.device)

    def __call__(self, pcm, dither=True, stream=None):
        """pcm: CUDA int16 or float32 [n] -> CUDA float32 [M, 64] (CMVN'd log-mel)."""
        assert pcm.is_cuda and pcm.dim() == 1 and pcm.is_contiguous()
        fmt = {torch.int16: _lib.PCM_S16, torch.float32: _lib.PCM_F32}[pcm.dtype]
        lib = _lib.load()
        n = pcm.numel()
        M = lib.iss_vbx_num_frames(n)
        fea = torch.empty((M, FEAT_DIM), dtype=torch.float32, device=pcm.device)
        if M == 0:
            return fea
        work = self.ctx.workspace('vbx', lib.iss_vbx_work_bytes(n))
        d = self.dither.get(n) if dither else None
        _lib.check(lib.iss_vbx_features(self.ctx.handle, _lib.ptr(pcm), fmt, n, _lib.ptr(d), _lib.ptr(fea),
                                        _lib.ptr(work), _stream_ptr(pcm.device, stream)), 'iss_vbx_features')
        return fea

    def multi(self, pcms, dither=True, stream=None):
        """pcms: 1-D contiguous CUDA tensors of one dtype (int16 or float32) -> (CUDA float32 [sum M_i, 64], int64 numpy
        row offsets [n + 1]): recording i's features are rows off[i] .. off[i + 1], equal to __call__ on it."""
        assert len(pcms) and all(p.is_cuda and p.dim() == 1 and p.is_contiguous() and p.dtype == pcms[0].dtype for p in pcms)
        fmt = {torch.int16: _lib.PCM_S16, torch.float32: _lib.PCM_F32}[pcms[0].dtype]
        lib = _lib.load()
        n = len(pcms)
        n_samples = np.ascontiguousarray([p.numel() for p in pcms], dtype=np.int64)
        off = pack._starts([pack.vbx_num_frames(int(k)) for k in n_samples], total=True)
        dev = pcms[0].device
        fea = torch.empty((int(off[-1]), FEAT_DIM), dtype=torch.float32, device=dev)
        if off[-1] == 0:
            return fea, off
        work = self.ctx.workspace('vbx', FEAT_DIM * 8 * int(off[-1]) + 256)      # float64 log-fbank rows + 256
        d = self.dither.get(int(n_samples.max())) if dither else None
        ptrs = (ctypes.c_void_p * n)(*[p.data_ptr() for p in pcms])
        fea_off = np.ascontiguousarray(off[:-1])
        _lib.check(lib.iss_vbx_features_multi(self.ctx.handle, n, ptrs, _lib.ptr(n_samples), fmt, _lib.ptr(d), _lib.ptr(fea),
                                              _lib.ptr(fea_off), _lib.ptr(work), _stream_ptr(dev, stream)),
                   'iss_vbx_features_multi')
        return fea, off


_frontends = {}


def get_features(signal, LC=150, RC=149, device=0):
    """Same contract as the reference (vbx_segmenter.py:72-89): float64 (or
    float32 / int16) signal in [-1, 1) -> float32 [M, 64] numpy array."""
    assert (LC, RC) == (150, 149), 'only the reference window (150, 149) is built into the kernel'
    if device not in _frontends:
        _frontends[device] = VbxFrontEnd(Context(device))
    fe = _frontends[device]
    sig = np.asarray(signal)
    if sig.dtype == np.int16:
        pcm = torch.from_numpy(np.ascontiguousarray(sig))
    else:
        f32 = sig.astype(np.float32)
        if not np.array_equal(f32.astype(np.float64), sig.astype(np.float64)):
            raise ValueError('signal is not exactly representable in float32 (the decoder yields PCM16/float32 data)')
        pcm = torch.from_numpy(np.ascontiguousarray(f32))
    return fe(pcm.to(fe.ctx.device)).cpu().numpy()


# ------------------------------------------------------------------ ResNet101 weights -> blob
def resnet_blob_from_state(sd, m=M_CHANNELS, num_blocks=NUM_BLOCKS, eps=1e-5):
    """PyTorch state_dict of resnet.ResNet101 (``raw_81.pth`` layout, resnet.py:78-113)
    -> the float32 blob iss_resnet_create expects (BatchNorm folded to scale/shift)."""
    g = lambda k: np.asarray(sd[k].detach().cpu().numpy() if hasattr(sd[k], 'detach') else sd[k], dtype=np.float32)   # noqa: E731
    parts = []

    def conv_bn(conv, bn):
        w = g(conv + '.weight')                                   # [cout, cin, kh, kw]
        parts.append(np.ascontiguousarray(w.transpose(2, 3, 1, 0)).ravel())       # [kh][kw][cin][cout]
        scale = g(bn + '.weight') / np.sqrt(g(bn + '.running_var') + np.float32(eps))
        shift = g(bn + '.bias') - g(bn + '.running_mean') * scale
        parts.append(scale.astype(np.float32))
        parts.append(shift.astype(np.float32))

    conv_bn('conv1', 'bn1')
    for li, nb in enumerate(num_blocks, start=1):
        for b in range(nb):
            p = 'layer%d.%d' % (li, b)
            conv_bn(p + '.conv1', p + '.bn1')
            conv_bn(p + '.conv2', p + '.bn2')
            conv_bn(p + '.conv3', p + '.bn3')
            if (p + '.shortcut.0.weight') in sd:
                conv_bn(p + '.shortcut.0', p + '.shortcut.1')
    parts.append(np.ascontiguousarray(g('embedding.weight').T).ravel())           # [in][embed]
    parts.append(g('embedding.bias'))
    return np.concatenate(parts).astype(np.float32)


# ------------------------------------------------------------------ the plugin ABC (vbx_segmenter.py:205-246)
class VBxExtractor(ABC):
    """VBxExtractor is an abstract class performing xvector extraction."""

    @abstractmethod
    def __init__(self):
        pass

    def __call__(self, basename, fea, duration):
        """One get_embedding() call per planned window (vbx_segmenter.py:217-246): NaN embeddings are dropped with a
        warning, the tail window ends at `duration`, embeddings are returned x10."""
        out = []
        for start, length, is_tail in window_plan(len(fea)):
            stop = start + length
            key = '%s_%08d-%08d' % (basename, start, stop)
            x = self.get_embedding(fea[start:stop])
            if np.isnan(x).any():
                logger.warning('NaN found, not processing: %s%s' % (key, os.linesep))
                continue
            t0 = round(start / 100.0, 3)
            t1 = round(duration, 3) if is_tail else round(start / 100.0 + WINLEN / 100.0, 3)
            out.append((key, (t0, t1), x * 10))
        return out


class B200BackendExtractor(VBxExtractor):
    """ResNet101 x-vector extractor on libiss_b200 (K5)."""

    def __init__(self, state_dict=None, device=0, ctx=None, onnx_path=None):
        """Weights come from (first match): ``state_dict`` (resnet.py layout), ``onnx_path``, the reference's
        production asset ``final.onnx`` (vbx_segmenter.py:249-266) or ``raw_81.pth`` (:271-288) in the model
        directories (models.find_model_file).  The ONNX file is read by onnx_reader (no onnx runtime)."""
        self.ctx = ctx if ctx is not None else Context(device)
        m, feat_dim, embed_dim, num_blocks = M_CHANNELS, FEAT_DIM, EMBED_DIM, NUM_BLOCKS
        if state_dict is None:
            from .models import find_model_file
            onnx_path = onnx_path or find_model_file('final.onnx')
            if onnx_path is not None:
                from .onnx_reader import resnet_blob_from_onnx
                blob, m, feat_dim, embed_dim, num_blocks = resnet_blob_from_onnx(onnx_path)
                if (m, feat_dim, embed_dim, tuple(num_blocks)) != (M_CHANNELS, FEAT_DIM, EMBED_DIM, NUM_BLOCKS):
                    raise ValueError('%s is not the VBx ResNet101 (m=%d, feat=%d, embed=%d, blocks=%r)'
                                     % (onnx_path, m, feat_dim, embed_dim, num_blocks))
            else:
                path = find_model_file('raw_81.pth')
                if path is None:
                    raise FileNotFoundError('neither final.onnx nor raw_81.pth found (the reference fetches them from its '
                                            'GitHub release, remote_utils.py:5,13-14; this build does no network access)')
                state_dict = torch.load(path, map_location='cpu')
                state_dict = state_dict.get('state_dict', state_dict)
        if state_dict is not None:
            blob = resnet_blob_from_state(state_dict)
        blob = np.ascontiguousarray(blob, dtype=np.float32)
        nb = (ctypes.c_int * 4)(*NUM_BLOCKS)
        lib = _lib.load()
        h = ctypes.c_void_p()
        _lib.check(lib.iss_resnet_create(self.ctx.handle, _lib.ptr(blob), blob.size, M_CHANNELS, FEAT_DIM, EMBED_DIM,
                                         ctypes.cast(nb, ctypes.c_void_p), ctypes.byref(h)), 'iss_resnet_create')
        self.handle = h
        self.flops_per_window = lib.iss_resnet_flops_per_window(h, WINLEN)

    def embed_windows(self, fea, starts, win_len, stream=None):
        """fea: CUDA float32 [M, 64]; starts: window start rows -> CUDA float32 [n, 256]."""
        assert fea.is_cuda and fea.dtype == torch.float32 and fea.is_contiguous()
        starts = np.ascontiguousarray(starts, dtype=np.int32)
        n = len(starts)
        emb = torch.empty((n, EMBED_DIM), dtype=torch.float32, device=fea.device)
        if n == 0:
            return emb
        lib = _lib.load()
        work = self.ctx.workspace('resnet', lib.iss_resnet_workspace_bytes(self.handle, n, int(win_len)))
        _lib.check(lib.iss_resnet_embed(self.ctx.handle, self.handle, _lib.ptr(fea), fea.shape[0], _lib.ptr(starts), n,
                                        int(win_len), _lib.ptr(emb), _lib.ptr(work), work.numel(),
                                        _stream_ptr(fea.device, stream)), 'iss_resnet_embed')
        return emb

    @staticmethod
    def _check_range(emb, what=''):
        """On the fp16-split engine, a non-finite embedding means an activation left the fp16 range (|x| < 65504 in the
        split-half words between its layers): that is an error, not a window to drop.  The fp32-range engines keep
        the reference's drop-with-warning.  `what` names the recording in the message."""
        B200BackendExtractor.check_finite(bool(np.isfinite(emb).all()), what)
        return emb

    @staticmethod
    def check_finite(all_finite, what=''):
        """_check_range's error, from whether every x-vector of a call was finite."""
        if _lib.load().iss_get_gemm_mode() == _lib.GEMM_TC_F16 and not all_finite:
            raise _lib.IssError('B200BackendExtractor: the ResNet returned non-finite x-vectors%s: an activation left the '
                                'fp16 range of the default fp16-split GEMM engine; run with ISS_B200_GEMM=tc_ts '
                                '(3xTF32, fp32 range)' % what)

    def get_embedding(self, fea):
        """OnnxBackendExtractor.get_embedding contract (vbx_segmenter.py:262-266): fea [T, 64] -> [256]."""
        t = torch.from_numpy(np.ascontiguousarray(fea, dtype=np.float32)).to(self.ctx.device)
        return self._check_range(self.embed_windows(t, [0], t.shape[0]).cpu().numpy()[0])

    def __call__(self, basename, fea, duration):
        """Same output as VBxExtractor.__call__, windows embedded in GPU batches."""
        if isinstance(fea, np.ndarray):
            fea = torch.from_numpy(np.ascontiguousarray(fea, dtype=np.float32)).to(self.ctx.device)
        M = fea.shape[0]
        plan = window_plan(M)
        reg = [s for s, n, tail in plan if not tail]
        emb = self.embed_windows(fea, reg, WINLEN).cpu().numpy() if reg else np.zeros((0, EMBED_DIM), np.float32)
        tail = lambda start, n: self.embed_windows(fea, [start], n).cpu().numpy()[0]     # noqa: E731
        return self._xvectors(basename, M, duration, plan, emb, tail)

    def _xvectors(self, basename, M, duration, plan, emb, tail, what=''):
        """The per-window bookkeeping of __call__ for one recording of M frames: emb holds the x-vectors of the plan's
        regular windows, in order, and tail(start, n) returns the tail window's."""
        self._check_range(emb, what)
        out = []
        for i, (start, _, _) in enumerate(w for w in plan if not w[2]):
            key = f'{basename}_{start:08}-{(start + WINLEN):08}'
            if np.isnan(emb[i]).any():
                logger.warning(f'NaN found, not processing: {key}{os.linesep}')
                continue
            out.append((key, (round(start / 100.0, 3), round(start / 100.0 + WINLEN / 100.0, 3)), emb[i]))
        for start, n, is_tail in plan:
            if is_tail:
                x = self._check_range(tail(start, n), what)
                key = f'{basename}_{start:08}-{M:08}'
                if np.isnan(x).any():
                    logger.warning(f'NaN found, not processing: {key}{os.linesep}')
                else:
                    out.append((key, (round(start / 100.0, 3), round(duration, 3)), x))
        return [(key, seg, x * 10) for key, seg, x in out]

    def embed_packed(self, fea, plan, stream=None):
        """The x-vectors of every window of the recordings packed in fea (CUDA float32 [rows, 64]) by plan
        (pack.VbxPlan): one embed_windows call for all regular windows, one per distinct tail length, one copy back.
        Returns (regular [len(plan.reg_start), 256], {tail length: [windows, 256]}), numpy float32."""
        parts = [self.embed_windows(fea, plan.reg_start, WINLEN, stream)]
        parts += [self.embed_windows(fea, starts, n, stream) for n, (_, starts) in plan.tails.items()]
        host = torch.cat(parts).cpu().numpy()
        reg, k, tails = host[:len(plan.reg_start)], len(plan.reg_start), {}
        for n, (recs, _) in plan.tails.items():
            tails[n] = host[k:k + len(recs)]
            k += len(recs)
        return reg, tails

    def packed_xvectors(self, plan, emb, i, basename, duration, what=''):
        """__call__'s result for recording i of a pack.VbxPlan, from the embed_packed output emb."""
        reg, tails = emb
        M = int(plan.frames[i])
        tail = lambda start, n: tails[n][plan.tail_pos[i]]     # noqa: E731
        return self._xvectors(basename, M, duration, plan.plans[i], reg[plan.reg_off[i]:plan.reg_off[i + 1]], tail, what)

    def call_packed(self, fea, plan, basenames, durations, stream=None):
        """__call__ on every recording of fea packed by plan (pack.VbxPlan), each with its basename and duration: the same
        lists, in order.  The engine-3 range error names the first failing recording's index."""
        emb = self.embed_packed(fea, plan, stream)
        return [self.packed_xvectors(plan, emb, i, basenames[i], durations[i], ' (signal %d)' % i)
                for i in range(len(plan.frames))]


# ------------------------------------------------------------------ VoiceFemininityScoring (vbx_segmenter.py:28-202)
def _overlap(start, stop, speech):
    """Total duration of [start, stop] covered by the (disjoint) speech intervals: what
    ``Timeline([Segment(start, stop)]).crop(vad_timeline).duration()`` yields (:140)."""
    return sum(max(0.0, min(stop, e) - max(start, b)) for b, e in speech)


def is_mid_speech(start, stop, speech):
    """True if the window's midpoint lies strictly inside a speech segment (:28-37)."""
    m = (start + stop) / 2
    return any(b < m < e for b, e in speech)


def select_windows(ratios, vad_thresh):
    """The windows the score keeps, as indices into `ratios` (the speech-overlap ratios of the windows whose midpoint
    is in speech, in window order), in the order the score takes them: those with ratio >= vad_thresh, then, when
    fewer than 50 % of the windows were kept, the others in decreasing overlap order up to that share (add_needed_vectors,
    :40-52).  (The reference sorts a ragged object array and reads ``Segment.stop``, which pyannote's Segment does not
    define; this implements the documented intent with the same selection rule: sort by overlap ratio descending,
    skip the first len(kept) entries, take the next ``diff``.)"""
    kept = [i for i, r in enumerate(ratios) if r >= vad_thresh]
    min_pred = round(0.5 * len(ratios))
    if len(kept) < min_pred:
        order = np.argsort(np.array(ratios, dtype=np.float64))[::-1]
        kept += [int(i) for i in order[len(kept):min_pred]]
    return kept


def get_femininity_score(g_preds):
    """Share of retained windows predicted feminine (p >= 0.5) (:55-61).  The reference goes through a
    pyannote Annotation keyed by segment, so a later window with identical bounds replaces an earlier one."""
    by_segment = {}
    for start, stop, p in g_preds:
        by_segment[(start, stop)] = bool(np.all(np.asarray(p) >= 0.5))
    return sum(by_segment.values()) / len(by_segment)


def score_kept(segs, preds):
    """(score, nb_vectors) of the kept windows' (start, stop) and their MLP output rows, as __call__ forms them
    (:188-202); ZeroDivisionError when no window was kept."""
    if len(preds) > 1:
        preds = np.squeeze(preds)
    g = [(seg[0], seg[1], p) for seg, p in zip(segs, preds)]
    return get_femininity_score(g), len(g)


class VoiceFemininityScoring:
    """Same contract as the reference class (vbx_segmenter.py:92-202): ``__call__(fpath) ->
    (score, speech_duration, nb_vectors)``.  VAD = this package's ``Segmenter('smn', detect_gender=False)``,
    x-vectors = K4 + K5, the gender MLP runs on device through ``iss_mlp_forward``; the interval
    bookkeeping the reference delegates to pyannote.core is plain Python here.
    Extra optional arguments: ``device``, ``ffmpeg`` and ``models`` = {'vad': (config, weights),
    'mlp': (config, weights), 'resnet': state_dict} to bypass the model-file lookup."""

    def __init__(self, gd_model_criteria="bgc", backend='onnx', device=0, ffmpeg='ffmpeg', models=None):
        assert backend in ['onnx', 'b200'], "Backend should be 'onnx' (served by the GPU extractor) or 'b200'."
        from .engine import MlpModel
        from .models import find_model_file, load_model_file
        from .segmenter import Segmenter
        models = models or {}
        assert gd_model_criteria in ["bgc", "vfp"], "Gender detection model Criteria must be 'bgc' (default) or 'vfp'"
        if gd_model_criteria == "bgc":
            gd_model, self.vad_thresh = "interspeech2023_all.hdf5", 0.7
        else:
            gd_model, self.vad_thresh = "interspeech2023_cvfr.hdf5", 0.62
        self.vad = Segmenter(vad_engine='smn', detect_gender=False, ffmpeg=ffmpeg, device=device,
                             models={'vad': models['vad']} if 'vad' in models else None)
        self.ctx = self.vad.ctx
        self.xvector_model = B200BackendExtractor(state_dict=models.get('resnet'), ctx=self.ctx)
        mlp = models.get('mlp')
        if mlp is None:
            path = find_model_file(gd_model)
            if path is None:
                raise FileNotFoundError('%s not found (reference asset, remote_utils.py:4-15)' % gd_model)
            mlp = load_model_file(path)
        self.gender_detection_mlp_model = MlpModel(self.ctx, mlp[0], mlp[1], EMBED_DIM)
        self.frontend = VbxFrontEnd(self.ctx)
        self.ffmpeg = ffmpeg

    def apply_vad(self, xvectors, speech):
        """vbx_segmenter.py:129-145 with `speech` = [(start, end)] of the 'speech' VAD segments."""
        mid, ratios = [], []
        for key, (start, stop), x in xvectors:
            if is_mid_speech(start, stop, speech):
                ratios.append(_overlap(start, stop, speech) / (stop - start))
                mid.append((key, (start, stop), x))
        return [mid[i] for i in select_windows(ratios, self.vad_thresh)]

    def score_signal(self, sig, basename='signal', sample_rate=16000):
        """The body of __call__ on a decoded signal: 16 kHz mono numpy int16 / float, or, at any other ``sample_rate``
        or channel count, what ``Segmenter.segment_signal`` resamples (then resampled to 16 kHz int16 on the device)."""
        from . import resample
        if not resample.is_native(sig, sample_rate):
            return self._score_16k(resample.to16k(self.ctx, sig, sample_rate), basename)
        sig = np.asarray(sig)
        sig = sig.reshape(-1) if sig.ndim == 2 else sig
        sig = sig if sig.dtype in (np.int16, np.float32) else sig.astype(np.float32)
        return self._score_16k(sig, basename)

    def _score_16k(self, sig, basename):
        """score_signal on 16 kHz mono: a host array, or the int16 CUDA tensor of a resampled recording."""
        pcm = sig if isinstance(sig, torch.Tensor) else None
        duration = len(sig) / SR
        vad_seg = self.vad.segment_signal(sig)
        speech = [(b, e) for lab, b, e in vad_seg if lab == 'speech']
        speech_duration = sum(e - b for b, e in speech)
        if not speech_duration:
            return None, speech_duration, 0
        if pcm is None:
            pcm = torch.from_numpy(np.ascontiguousarray(sig)).to(self.ctx.device)
        features = self.frontend(pcm)
        x_vectors = self.xvector_model(basename, features, duration)
        x_vectors = self.apply_vad(x_vectors, speech)
        x = np.asarray([x for _, _, x in x_vectors])
        gender_pred = self.gender_detection_mlp_model.predict(x, verbose=0)
        score, nb = score_kept([seg for _, seg, _ in x_vectors], gender_pred)
        return score, speech_duration, nb

    def score_signals(self, signals, basename='signal', sample_rates=None):
        """score_signal on each of a list of signals (what score_signal takes, or 1-D int16 / float32 CUDA tensors, read in
        place, at the rate sample_rates[i], 16000 by default) in as few device passes as possible: one
        (score, speech_duration, nb_vectors) per signal, in input order, equal to score_signal(signals[i], basename,
        sample_rates[i]).  Per pass of pack.plan_passes over the 16 kHz lengths, host arrays are staged and uploaded
        once, each (rate, channels, dtype) group is resampled in one launch, the VAD runs as Segmenter.segment_signals,
        the VBx features of the recordings with speech as one K4 launch pair, their x-vectors as one ResNet call for all
        regular windows plus one per tail length, and the MLP once.  Signals of pack.LONG_FRAMES frames or more at
        16 kHz go through score_signal.  If score_signal would raise for some signals, the exception of the first of
        them is raised."""
        from . import resample
        from .segmenter import _pass_input
        rates = resample.check_rates(sample_rates, len(signals))
        sigs = [_pass_input(s, r) for s, r in zip(signals, rates)]
        passes, long_ = resample.plan(sigs, rates)
        out = [None] * len(sigs)
        for idx in passes:
            for i, r in zip(idx, self._score_pass([sigs[i] for i in idx], idx, basename, [rates[i] for i in idx])):
                out[i] = r
        for i in long_:
            sig = signals[i]
            if isinstance(sig, torch.Tensor) and resample.is_native(sig, rates[i]):
                sig = sig.cpu().numpy()
            try:
                out[i] = self.score_signal(sig, basename, rates[i])
            except Exception as e:          # raised below, in input order
                out[i] = e
        for r in out:
            if isinstance(r, Exception):
                raise r
        return out

    def _score_pass(self, sigs, idx, basename, rates):
        """One pass of score_signals over signals whose 16 kHz recordings share one PCM format (idx: their input
        indices).  A recording for which score_signal would raise gets the exception as its result."""
        from .segmenter import _pass_pcms
        pcms = _pass_pcms(self.ctx, sigs, rates)
        speech = [[(b, e) for lab, b, e in segs if lab == 'speech'] for segs in self.vad.segment_signals(pcms)]
        out = [(None, sum(e - b for b, e in sp), 0) for sp in speech]
        live = [k for k, sp in enumerate(speech) if out[k][1]]
        if not live:
            return out
        fea, _ = self.frontend.multi([pcms[k] for k in live])
        plan = pack.VbxPlan([pcms[k].numel() for k in live])
        emb = self.xvector_model.embed_packed(fea, plan)
        kept = {}
        for j, k in enumerate(live):
            try:
                xv = self.xvector_model.packed_xvectors(plan, emb, j, basename, pcms[k].numel() / SR,
                                                        ' (signal %d)' % idx[k])
                kept[k] = self.apply_vad(xv, speech[k])
            except Exception as e:
                out[k] = e
        x = [x for k in kept for _, _, x in kept[k]]
        preds = self.gender_detection_mlp_model.predict(np.asarray(x, dtype=np.float32).reshape(len(x), EMBED_DIM))
        pos = 0
        for k, xv in kept.items():
            gender_pred = preds[pos:pos + len(xv)]
            pos += len(xv)
            try:
                score, nb = score_kept([seg for _, seg, _ in xv], gender_pred)
                out[k] = (score, out[k][1], nb)
            except ZeroDivisionError as e:
                out[k] = e
        return out

    def stream(self, calibration_sec=60.0):
        """Extension: live femininity scores of many streams fed chunk by chunk (``vfs_stream.LiveScores``).  The VAD is
        ``self.vad.stream(calibration_sec)``; a stream's final score is the offline one on its VAD segments."""
        from .vfs_stream import LiveScores
        return LiveScores(self, calibration_sec)

    def __call__(self, fpath):
        """Voice femininity score of a media file (vbx_segmenter.py:147-202)."""
        from .io import media2sig16kmono
        from .segmenter import _device_wav, _wav_to16k
        basename = os.path.splitext(os.path.basename(fpath))[0]
        wav = _device_wav(fpath, None, None, self.ffmpeg)
        if wav is not None:         # a WAV that is not 16 kHz mono, without ffmpeg: decoded on the device
            return self._score_16k(_wav_to16k(self.ctx, wav), basename)
        sig = media2sig16kmono(fpath, ffmpeg=self.ffmpeg, dtype='float32', return_int16=True)
        return self.score_signal(sig, basename)
