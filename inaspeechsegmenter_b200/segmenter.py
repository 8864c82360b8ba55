"""``Segmenter`` -- same public API as the reference (inaSpeechSegmenter/
segmenter.py:207-335) with the per-frame hot path running as sm_90a CUDA
kernels behind the C ABI of libiss_b200.so:

  _media2feats   (:53-67)   -> K1 fused log-mel/log-energy kernel
  _energy_activity (:69-73) -> device reduction + K3 Viterbi (K = 2)
  _get_patches + keras predict (:76-88, :163) -> K2 (patches never materialised)
  viterbi_decoding (:176)   -> K3 batched over segments

Host code only moves bytes (pinned host -> device, small label arrays back),
run-length-encodes label tracks (_binidx2seglist, :91-108) and formats output.
"""
import os
import zlib
import random
import shutil
import sys
import time
import warnings

import numpy as np
import torch

from . import _lib, engine, models, pack, resample
from .export_funcs import seg2csv, seg2textgrid
from .io import media2sig16kmono, wav_data
from .sidekit_mfcc import SidekitFrontEnd

PATCH_W = 68

_state = {}          # per-process lazily created contexts: {'main': Context, 'feat': Context, ...}


def _get_ctx(name, device=0):
    key = (name, device)
    if key not in _state:
        ctx = engine.Context(device)
        _state[key] = ctx
    return _state[key]


def _get_frontend(name='feat', device=0):
    key = ('fe', name, device)
    if key not in _state:
        _state[key] = SidekitFrontEnd(_get_ctx(name, device))
    return _state[key]


def _to_device_pcm(sig, device):
    """Host signal -> device tensor through pinned memory (int16 stays int16)."""
    sig = np.ascontiguousarray(sig)
    if sig.dtype not in (np.int16, np.float32):
        sig = sig.astype(np.float32)
    host = torch.from_numpy(sig)
    try:
        host = host.pin_memory()
    except RuntimeError:
        pass
    return host.to(device, non_blocking=True)


def _pass_input(sig, rate=16000):
    """A signal of segment_signals as a 1-D int16 / float32 numpy array or contiguous CUDA tensor (what
    feats_from_signal would upload); a signal to resample (not 16 kHz mono) as resample.as_input returns it."""
    if not resample.is_native(sig, rate):
        return resample.as_input(sig)
    if isinstance(sig, torch.Tensor):
        if sig.is_cuda:
            if sig.dtype not in (torch.int16, torch.float32):
                raise TypeError('pcm must be int16 or float32, got %s' % sig.dtype)
            return sig.reshape(-1).contiguous()
        sig = sig.numpy()
    sig = np.ascontiguousarray(sig).reshape(-1)
    if sig.dtype not in (np.int16, np.float32):
        sig = sig.astype(np.float32)
    return sig


_TORCH_DTYPE = {np.dtype(np.int16): torch.int16, np.dtype(np.float32): torch.float32}


def _stage_pass(sigs, dev):
    """Device views of the signals of one pass (numpy arrays or CUDA tensors, int16 or float32, any shape, or
    io.WavData): CUDA tensors are used in place; host arrays are copied, and WAV data chunks read, into one pinned
    staging buffer, each 16-byte aligned (vector loads in the kernels), and uploaded in one copy.  A WAV comes back as
    its stored bytes, uint8 [frames, channels, bytes per sample]."""
    host = [i for i, s in enumerate(sigs) if not isinstance(s, torch.Tensor)]
    pcms = list(sigs)
    if host:
        off = np.concatenate(([0], np.cumsum([(sigs[i].nbytes + 15) // 16 * 16 for i in host]))).astype(np.int64)
        try:
            buf = torch.empty(int(off[-1]), dtype=torch.uint8, pin_memory=True)
        except RuntimeError:
            buf = torch.empty(int(off[-1]), dtype=torch.uint8)
        stage = buf.numpy()
        for k, i in enumerate(host):
            a, b = int(off[k]), int(off[k]) + sigs[i].nbytes
            if isinstance(sigs[i], np.ndarray):
                stage[a:b] = sigs[i].reshape(-1).view(np.uint8)
            else:
                sigs[i].readinto(stage[a:b])
            stage[b:off[k + 1]] = 0
        buf = buf.to(dev, non_blocking=True)
        for k, i in enumerate(host):
            v = buf[off[k]:off[k] + sigs[i].nbytes]
            pcms[i] = v.view(_TORCH_DTYPE[sigs[i].dtype]).view(sigs[i].shape) if isinstance(sigs[i], np.ndarray) \
                else v.view(sigs[i].shape)
    return pcms


def _pass_pcms(ctx, sigs, rates):
    """16 kHz mono device recordings of one pass: the signals staged at their own rate, then resampled per group."""
    return resample.resample_pass(ctx, _stage_pass(sigs, ctx.device), rates)


def feats_from_signal(sig, device=0, fft_precision=_lib.FFT_FP64, ctx_name='feat', medianame='<array>'):
    """(mspec, loge, difflen) on the device from a host (or device) 16 kHz mono
    signal: the body of ``_media2feats`` after decoding (segmenter.py:53-67)."""
    dev = torch.device('cuda', device)
    if isinstance(sig, torch.Tensor):
        pcm = sig if sig.is_cuda else sig.to(dev, non_blocking=True)     # pinned host tensors copy asynchronously
    else:
        pcm = _to_device_pcm(sig, dev)
    fe = _get_frontend(ctx_name, device)
    if pcm.numel() < 400:
        raise ValueError('media %s holds %d samples: less than one 25 ms analysis frame' % (medianame, pcm.numel()))
    mspec, loge, stats = fe(pcm, fft_precision)
    difflen = 0
    if len(loge) < PATCH_W:
        # short media: pad with rows of min(mspec) (segmenter.py:60-65)
        difflen = PATCH_W - len(loge)
        warnings.warn("media %s duration is short. Robust results require length of at least 720 milliseconds" % medianame)
        fill = mspec.min() if mspec.numel() else torch.tensor(float('nan'), device=dev)
        mspec = torch.cat((mspec, fill.expand(difflen, 24).to(mspec.dtype)))
    return mspec, loge, difflen


def _device_wav(medianame, start_sec, stop_sec, ffmpeg):
    """The io.WavData of a whole file read without ffmpeg that is a WAV but not 16 kHz mono: the device decodes and
    resamples it (_wav_to16k).  None for every other call, which keeps media2sig16kmono's path and errors."""
    if ffmpeg is not None or start_sec is not None or stop_sec is not None:
        return None
    try:
        wav = wav_data(medianame)
    except Exception:           # not a readable WAV: media2sig16kmono reports it
        return None
    return None if (wav.rate == resample.TARGET_RATE and wav.channels == 1) else wav


def _wav_to16k(ctx, wav):
    """A WAV's data chunk read into the pinned staging buffer, uploaded once and resampled to 16 kHz mono int16 on
    the device: what segment_signal(x, sample_rate=wav.rate) feeds the front ends, for x the file's samples."""
    resample.check_rate(wav.rate)
    if not 1 <= wav.channels <= resample.MAX_CHANNELS:
        raise ValueError('%d channels: 1 to %d are supported' % (wav.channels, resample.MAX_CHANNELS))
    return resample.resample_pass(ctx, _stage_pass([wav], ctx.device), [wav.rate], [wav.encoding])[0]


def _media2feats(medianame, start_sec, stop_sec, ffmpeg, device=0, fft_precision=_lib.FFT_FP64, ctx_name='feat'):
    wav = _device_wav(medianame, start_sec, stop_sec, ffmpeg)
    if wav is not None:
        return feats_from_signal(_wav_to16k(_get_ctx(ctx_name, device), wav), device, fft_precision, ctx_name,
                                 medianame)
    sig = media2sig16kmono(medianame, start_sec, stop_sec, ffmpeg, 'float32', return_int16=True)
    if sig.ndim > 1:
        raise ValueError('expected a mono signal, got shape %r' % (sig.shape,))
    return feats_from_signal(sig, device, fft_precision, ctx_name, medianame)


def _rle(track):
    """_binidx2seglist (segmenter.py:91-108) on a numpy label track -> [(value, start, stop)]."""
    n = len(track)
    if n == 0:
        return [(None, -1, 0)]          # what the reference returns for an empty track
    cut = np.flatnonzero(track[1:] != track[:-1]) + 1
    starts = np.concatenate(([0], cut))
    stops = np.concatenate((cut, [n]))
    return [(track[a].item(), int(a), int(b)) for a, b in zip(starts, stops)]


_binidx2seglist = _rle


class DnnSegmenter:
    """Same contract as the reference's abstract class (segmenter.py:111-179):
    child classes define nmel, viterbi_arg, model_fname, inlabel, outlabels."""

    def __init__(self, batch_size, ctx=None, model=None):
        self.ctx = ctx if ctx is not None else _get_ctx('main')
        self.batch_size = batch_size        # perf knob of keras predict; results never depended on it
        if model is None:
            path = models.find_model_file(self.model_fname)
            if path is None:
                if os.environ.get('ISS_B200_SYNTHETIC_MODELS') == '1':
                    warnings.warn('%s not found: using a SYNTHETIC stand-in network (labels are meaningless)' % self.model_fname)
                    model = models.synthetic_keras_cnn(self.nmel, len(self.outlabels), seed=zlib.crc32(self.model_fname.encode()) % 1000)
                else:
                    raise FileNotFoundError(
                        '%s not found in $%s, /root/.keras/inaSpeechSegmenter or ~/.keras/inaSpeechSegmenter '
                        '(the reference downloads it from its GitHub release, remote_utils.py:4-27; '
                        'this build does no network access)' % (self.model_fname, models.MODEL_DIR_ENV))
            else:
                model = models.load_model_file(path)
        config, weights = model
        self.nn = engine.CnnModel.from_keras(self.ctx, config, weights, self.nmel)
        assert self.nn.n_classes == len(self.outlabels), (self.nn.n_classes, self.outlabels)
        self.last_probs = None

    def _ranges(self, lseg, difflen):
        ranges = [(a, b) for lab, a, b in lseg if lab == self.inlabel]
        if ranges and difflen > 0:
            # patches[:-int(difflen / 2)] (segmenter.py:150-152): ranges never reach the trimmed tail
            limit = (17 + 1 + 16) - int(difflen / 2)
            assert max(b for _, b in ranges) <= limit, (ranges, limit)
        return ranges

    def _decode(self, probs, ranges, lsegs):
        """Viterbi over the posteriors of `ranges` (the inlabel segments of the lseg lists, in order), then the
        relabelled lseg lists."""
        self.last_probs = probs
        seg_off = np.concatenate(([0], np.cumsum([b - a for a, b in ranges]))).astype(np.int64)
        trans = engine.diag_trans_exp(self.viterbi_arg, len(self.outlabels))
        states = engine.viterbi_segments(self.ctx, probs, seg_off, trans)
        # Non-finite posteriors (rows of non-finite patches are already 0.5) mean the network left the range of its GEMM
        # engine: the fp16-split engine carries activations as fp16 hi / lo pairs, |x| < 65504.  The flag is computed on
        # the device and comes back with the states, in the copy that synchronises anyway.
        flag = torch.isfinite(probs).all().to(torch.uint8).view(1)
        states = torch.cat((states, flag)).cpu().numpy()
        if not states[-1]:
            raise _lib.IssError('%s: the CNN returned non-finite posteriors: an activation left the fp16 range of the '
                                'default fp16-split GEMM engine; run with ISS_B200_GEMM=tc_ts (3xTF32, fp32 range)'
                                % type(self).__name__)
        states = states[:-1]
        k = 0
        out = []
        for lseg in lsegs:
            ret = []
            for lab, a, b in lseg:
                if lab != self.inlabel:
                    ret.append((lab, a, b))
                    continue
                pred = states[seg_off[k]:seg_off[k + 1]]
                k += 1
                for lab2, a2, b2 in _rle(pred):
                    ret.append((self.outlabels[int(lab2)], a2 + a, b2 + a))
            out.append(ret)
        return out

    def __call__(self, mspec, lseg, difflen=0, edge_left=True, edge_right=True):
        if isinstance(mspec, np.ndarray):
            mspec = torch.from_numpy(np.ascontiguousarray(mspec, dtype=np.float32)).to(self.ctx.device)
        ranges = self._ranges(lseg, difflen)
        if not ranges:
            return list(lseg)
        probs = self.nn.forward(mspec, ranges, edge_left, edge_right)
        return self._decode(probs, ranges, [lseg])[0]

    def call_packed(self, mspec, layout, lsegs):
        """__call__ over the recordings of one pass: mspec holds recording i at rows layout.row_off[i] .. +
        layout.rows[i] (pack.PassLayout) and lsegs[i] is its segment list.  One CNN call and one Viterbi call for all
        recordings; ``last_probs`` holds the posteriors of all their inlabel segments, in order."""
        ranges, rec = [], []
        for i, lseg in enumerate(lsegs):
            r = self._ranges(lseg, int(layout.difflen[i]))
            ranges += r
            rec += [i] * len(r)
        if not ranges:
            return [list(lseg) for lseg in lsegs]
        probs = self.nn.forward_multi(mspec, layout.row_off, layout.rows, rec, ranges)
        return self._decode(probs, ranges, lsegs)


class SpeechMusic(DnnSegmenter):
    # Voice activity detection: requires energetic activity detection (segmenter.py:182-188)
    outlabels = ('speech', 'music')
    model_fname = 'keras_speech_music_cnn.hdf5'
    inlabel = 'energy'
    nmel = 21
    viterbi_arg = 150


class SpeechMusicNoise(DnnSegmenter):
    # segmenter.py:190-196
    outlabels = ('speech', 'music', 'noise')
    model_fname = 'keras_speech_music_noise_cnn.hdf5'
    inlabel = 'energy'
    nmel = 21
    viterbi_arg = 80


class Gender(DnnSegmenter):
    # Gender segmentation, requires voice activity detection (segmenter.py:198-204)
    outlabels = ('female', 'male')
    model_fname = 'keras_male_female_cnn.hdf5'
    inlabel = 'speech'
    nmel = 24
    viterbi_arg = 80


class Segmenter:
    def __init__(self, vad_engine='smn', detect_gender=True, ffmpeg='ffmpeg', batch_size=32, energy_ratio=0.03,
                 device=0, models=None, fft_precision='fp64'):
        """Same arguments as the reference (segmenter.py:208-248).  Extra,
        optional: ``device`` (CUDA ordinal), ``models`` ({'vad': (config,
        weights), 'gender': (config, weights)} to bypass the model-file lookup)
        and ``fft_precision`` ('fp64' = the reference's precision recipe,
        'fp32' = faster)."""
        if ffmpeg is not None:
            if shutil.which(ffmpeg) is None:
                raise (Exception("""ffmpeg program not found"""))
        self.ffmpeg = ffmpeg
        self.energy_ratio = energy_ratio
        self.device = device
        self.fft_precision = {'fp64': _lib.FFT_FP64, 'fp32': _lib.FFT_FP32}[fft_precision]
        self.ctx = _get_ctx('main', device)
        models = models or {}

        assert vad_engine in ['sm', 'smn']
        if vad_engine == 'sm':
            self.vad = SpeechMusic(batch_size, self.ctx, models.get('vad'))
        elif vad_engine == 'smn':
            self.vad = SpeechMusicNoise(batch_size, self.ctx, models.get('vad'))

        assert detect_gender in [True, False]
        self.detect_gender = detect_gender
        if detect_gender:
            self.gender = Gender(batch_size, self.ctx, models.get('gender'))

    def energy_segments(self, loge):
        """segmenter.py:262-267 on device: [(label, start, stop)] in patch units."""
        if isinstance(loge, np.ndarray):
            host = np.ascontiguousarray(loge, dtype=np.float32)
            loge = torch.from_numpy(host).to(self.ctx.device)
        stats = engine.loge_stats(self.ctx, loge)              # {sum, count} of finite loge: two tiny kernels, fixed order
        track = engine.energy_viterbi(self.ctx, loge, stats, self.energy_ratio, out_stride=2).cpu().numpy()
        return [('noEnergy' if lab == 0 else 'energy', a, b) for lab, a, b in _rle(track)]

    def segment_feats(self, mspec, loge, difflen, start_sec):
        """do segmentation -- input corresponds to a 16 kHz mono signal (segmenter.py:250-276)."""
        lseg = self.energy_segments(loge)
        lseg = self.vad(mspec, lseg, difflen)
        if self.detect_gender:
            lseg = self.gender(mspec, lseg, difflen)
        return [(lab, start_sec + start * .02, start_sec + stop * .02) for lab, start, stop in lseg]

    def __call__(self, medianame, start_sec=None, stop_sec=None):
        """Return segmentation of a given file (segmenter.py:279-294)."""
        mspec, loge, difflen = _media2feats(medianame, start_sec, stop_sec, self.ffmpeg, self.device,
                                            self.fft_precision, 'main')
        if start_sec is None:
            start_sec = 0
        return self.segment_feats(mspec, loge, difflen, start_sec)

    def segment_signal(self, sig, start_sec=0, sample_rate=16000):
        """Extension: segment an in-memory signal (numpy int16/float32 or CUDA tensor).  16 kHz mono ([frames]) goes to
        the front end as it is; any other rate or channel count (``sample_rate`` an integer from 8000 to 192000 Hz,
        int16 or float32 [frames, channels] with 1 to 8 channels) is first resampled to 16 kHz mono int16 on the device
        (``resample``)."""
        if not resample.is_native(sig, sample_rate):
            sig = resample.to16k(self.ctx, sig, sample_rate)
        elif len(resample.shape(sig)) == 2:
            sig = sig.reshape(-1)
        mspec, loge, difflen = feats_from_signal(sig, self.device, self.fft_precision, 'main')
        return self.segment_feats(mspec, loge, difflen, start_sec)

    def segment_signals(self, signals, start_secs=None, sample_rates=None):
        """Extension: segment a list of in-memory signals (each what ``segment_signal`` accepts, at the rate
        ``sample_rates[i]``, 16000 by default) in as few device passes as possible.  Returns one segment list per
        signal, in input order, equal to ``segment_signal(signals[i], start_secs[i], sample_rates[i])``.  Host arrays
        are staged in one pinned buffer per pass; CUDA tensors are read in place.  Signals are grouped and routed by
        their 16 kHz length: those of 65536 frames (10.9 min) or more go through ``segment_signal``."""
        n = len(signals)
        if start_secs is None:
            start_secs = [0] * n
        if len(start_secs) != n:
            raise ValueError('%d signals but %d start times' % (n, len(start_secs)))
        rates = resample.check_rates(sample_rates, n)
        sigs = [_pass_input(s, r) for s, r in zip(signals, rates)]
        passes, long_ = resample.plan(sigs, rates)
        out = [None] * n
        for idx in passes:
            for i, segs in zip(idx, self._segment_pass([sigs[i] for i in idx], [start_secs[i] for i in idx],
                                                       [rates[i] for i in idx])):
                out[i] = segs
        for i in long_:
            out[i] = self.segment_signal(signals[i], start_secs[i], rates[i])
        return out

    def _segment_pass(self, sigs, start_secs, rates):
        """One device pass over signals whose 16 kHz recordings share one PCM format, each shorter than
        pack.LONG_FRAMES frames at 16 kHz."""
        dev = self.ctx.device
        pcms = _pass_pcms(self.ctx, sigs, rates)
        layout = pack.PassLayout([p.shape[0] for p in pcms], pcms[0].element_size())
        mspec, loge, stats = _get_frontend('main', dev.index).multi(pcms, layout, self.fft_precision)
        for i in np.flatnonzero(layout.difflen > 0):
            # short media: pad with rows of min(mspec) (segmenter.py:60-65)
            warnings.warn("media <signal %d> duration is short. Robust results require length of at least 720 "
                          "milliseconds" % i)
            a, L = int(layout.row_off[i]), int(layout.frames[i])
            mspec[a + L:a + pack.PATCH_W] = mspec[a:a + L].min()
        track = engine.energy_viterbi_multi(self.ctx, loge, layout.loge_off, stats, self.energy_ratio,
                                            layout.out_off).cpu().numpy()
        lsegs = [[('noEnergy' if lab == 0 else 'energy', a, b)
                  for lab, a, b in _rle(track[layout.out_off[i]:layout.out_off[i + 1]])] for i in range(len(sigs))]
        lsegs = self.vad.call_packed(mspec, layout, lsegs)
        if self.detect_gender:
            lsegs = self.gender.call_packed(mspec, layout, lsegs)
        return [[(lab, start_sec + start * .02, start_sec + stop * .02) for lab, start, stop in lseg]
                for lseg, start_sec in zip(lsegs, start_secs)]

    def stream(self, calibration_sec=60.0):
        """Extension: live segmentation of many 16 kHz mono streams fed chunk by chunk (``stream.LiveStreams``).  The
        energy threshold of a stream comes from its first ``calibration_sec`` seconds (>= 1); no label is decided
        before that."""
        from .stream import LiveStreams
        return LiveStreams(self, calibration_sec)

    def batch_process(self, linput, loutput, verbose=False, skipifexist=False, nbtry=1, trydelay=2., output_format='csv'):
        """segmenter.py:297-335 -- same return tuple and message codes."""
        if verbose:
            print('batch_processing %d files' % len(linput))

        if output_format == 'csv':
            fexport = seg2csv
        elif output_format == 'textgrid':
            fexport = seg2textgrid
        else:
            raise NotImplementedError()

        t_batch_start = time.time()

        lmsg = []
        fg = featGenerator(linput.copy(), loutput.copy(), self.ffmpeg, skipifexist, nbtry, trydelay,
                           self.device, self.fft_precision)
        i = 0
        for feats, msg in fg:
            lmsg += msg
            i += len(msg)
            if verbose:
                print('%d/%d' % (i, len(linput)), msg)
            if feats is None:
                break
            mspec, loge, difflen = feats
            b = time.time()
            lseg = self.segment_feats(mspec, loge, difflen, 0)
            fexport(lseg, loutput[len(lmsg) - 1])
            lmsg[-1] = (lmsg[-1][0], lmsg[-1][1], 'ok ' + str(time.time() - b))

        t_batch_dur = time.time() - t_batch_start
        nb_processed = len([e for e in lmsg if e[1] == 0])
        if nb_processed > 0:
            avg = t_batch_dur / nb_processed
        else:
            avg = -1
        return t_batch_dur, nb_processed, avg, lmsg


class _FeaturePrefetcher:
    """Depth-1 prefetch of the per-file front-end (decode -> pinned upload -> K1 on a side
    context) while the main thread segments the previous file: the role of the reference's
    ``medialist2feats`` / ``featGenerator`` pair (segmenter.py:338-387), with the same message
    protocol -- one ``(dst, code, text)`` per consumed input, code 0 = features ready,
    1 = output already exists (skipped), 2 = every attempt failed."""

    def __init__(self, sources, destinations, ffmpeg, skipifexist, nbtry, trydelay, device, fft_precision):
        from concurrent.futures import ThreadPoolExecutor
        self._todo = list(zip(sources, destinations))
        self._opt = (ffmpeg, skipifexist, max(1, nbtry), trydelay, device, fft_precision)
        self._pool = ThreadPoolExecutor(max_workers=1, thread_name_prefix='iss-feat')
        self._next = self._pool.submit(self._advance)

    def _extract(self, src):
        ffmpeg, _, nbtry, trydelay, device, fft_precision = self._opt
        last = None
        for attempt in range(nbtry):
            try:
                feats = _media2feats(src, None, None, ffmpeg, device, fft_precision, 'feat')
                torch.cuda.current_stream(feats[0].device).synchronize()      # hand-off to the main thread
                return feats, None
            except BaseException:                                              # same catch-all as the reference (:364)
                last = sys.exc_info()[0]
                if attempt + 1 < nbtry:
                    time.sleep(random.random() * trydelay)
        return None, last

    def _advance(self):
        """Consume inputs until one yields features (or none are left)."""
        skipifexist = self._opt[1]
        log = []
        while self._todo:
            src, dst = self._todo.pop(0)
            if skipifexist and os.path.exists(dst):
                log.append((dst, 1, 'already exists'))
                continue
            parent = os.path.dirname(dst)
            if not os.path.isdir(parent):
                os.makedirs(parent)
            feats, err = self._extract(src)
            if feats is None:
                log.append((dst, 2, 'error: ' + str(err)))
                continue
            log.append((dst, 0, 'ok'))
            return feats, log
        return None, log

    def __iter__(self):
        try:
            while True:
                feats, log = self._next.result()
                more = bool(self._todo)
                if more:
                    self._next = self._pool.submit(self._advance)
                yield feats, log
                if not more:
                    return
        finally:
            self._pool.shutdown(wait=False)


def featGenerator(ilist, olist, ffmpeg='ffmpeg', skipifexist=False, nbtry=1, trydelay=2., device=0,
                  fft_precision=_lib.FFT_FP64):
    """Name kept for users of the reference helper (segmenter.py:377-387)."""
    return iter(_FeaturePrefetcher(ilist, olist, ffmpeg, skipifexist, nbtry, trydelay, device, fft_precision))
