"""Live streams: ``Segmenter.stream()``.  Many audio streams are fed chunk by chunk; each call segments the new audio of
all of them in one device pass and returns the segments whose labels can no longer change.

Definition.  For a stream x of L frames, the concatenation of everything ``feed`` and ``end`` return for it equals
``segment_signal(x)`` when L <= N_cal = round(100 * calibration_sec), and otherwise the offline segmentation with one
change: the energy threshold is computed from the first N_cal loge values only (a causal threshold: the reference's
mean over the whole file cannot be known while the stream is live).

Pipeline of one call (``_run``), every stage over all streams at once:
  K1 on each stream's retained tail (< 400 samples) + new chunk  ->  new log-mel / loge rows
  energy chain (one per calibrated stream, K = 2) continued over the new frames
  VAD chains (one per decided ``energy`` run) over the decided, computable ``energy`` patches
  gender chains (one per decided ``speech`` run) over the decided ``speech`` patches
Each chain is continued from its carried scores and emits the states that are final (``iss_viterbi_online``): the
states up to the latest step where the backtracks from all K current states meet, or all of them when the chain ends.

Streams at another rate or channel count (any integer rate from 8 to 192 kHz, 1 to 8 channels) are first resampled
to 16 kHz mono int16 chunk by chunk (``resample.ready_outputs`` / ``end_outputs`` / ``first_kept``, DESIGN.md "Resampled
streams"): the 16 kHz samples a stream's calls produce concatenate to ``resample.to16k`` on the whole stream, and the
pipeline above runs on them as on a 16 kHz int16 stream.

The device work sits behind a backend object (``CudaBackend``) so that the same orchestration can run against a CPU
oracle in the tests.  The host keeps only small per-stream counters and the decided label tracks not yet returned.
"""
import warnings

import numpy as np
import torch

from . import _lib, engine, pack, resample

PATCH_W, LFILL = pack.PATCH_W, pack.PATCH_LFILL
_UNDECIDED, _PASS = -1, -2         # per-patch output of a stage: not yet known / patch not in the stage's input label


def computable_patches(F):
    """Padded patches whose rows exist once F frames exist (patch p reads frames 2(p-17) .. 2(p-17)+67, clamped at 0)."""
    return 0 if F < PATCH_W else LFILL + (F - PATCH_W) // 2 + 1


class _Chain:
    __slots__ = ('slot', 'next', 'pend')

    def __init__(self, slot, first):
        self.slot, self.next, self.pend = slot, first, 0       # next: first patch (step) not yet decided


class _Track:
    """Per-patch int8 values from absolute index `base` on; the prefix everyone is done with is dropped."""

    def __init__(self):
        self.base, self.a = 0, np.zeros(0, dtype=np.int8)

    def extend(self, n, fill=_UNDECIDED):
        if n > self.base + len(self.a):
            self.a = np.concatenate((self.a, np.full(n - self.base - len(self.a), fill, dtype=np.int8)))

    def __len__(self):
        return self.base + len(self.a)

    def get(self, a, b):
        return self.a[a - self.base:b - self.base]

    def put(self, a, vals):
        self.extend(a + len(vals))
        self.a[a - self.base:a - self.base + len(vals)] = vals

    def first_undecided(self, frm):
        rest = np.flatnonzero(self.a[frm - self.base:] == _UNDECIDED)
        return frm + int(rest[0]) if len(rest) else len(self)

    def drop(self, upto):
        k = upto - self.base
        if k > 0:
            self.a, self.base = self.a[k:].copy(), upto


class _Stage:
    """A CNN + Viterbi stage (VAD or gender) of one stream: one chain per run of `inlabel` in its input track."""

    def __init__(self):
        self.fed = 0                   # patches < fed are either sent to a chain or passed through
        self.dec = 0                   # patches < dec have their output decided
        self.chain = None              # open chain
        self.out = _Track()


class _Stream:
    def __init__(self, key, sid, kind):
        self.key, self.sid, self.kind = key, sid, kind        # kind: (where, dtype, rate, channels)
        self.rate = kind[2] if kind[2:] != (resample.TARGET_RATE, 1) else None    # resampled streams: their rate
        self.frames_in = 0             # frames fed at the stream's own rate (resampled streams)
        self.samples = 0               # 16 kHz samples fed
        self.F = 0                     # frames computed
        self.R0 = 0                    # first frame still retained on the device
        self.calibrated = False
        self.ended = False
        self.e_fed = 0                 # frames fed to the energy chain
        self.e_dec = 0                 # frames decided by it
        self.e_pend = 0
        self.elab = _Track()           # energy state per patch (frame 2p)
        self.vad, self.gen = _Stage(), _Stage()
        self.fin = 0                   # patches whose final label is known
        self.open = None               # (label, start patch) of the run not yet returned


def _kind(chunk, rate):
    """(kind, chunk): the (where, dtype name, rate, channels) of a chunk, and the chunk as the pipeline takes it: 16 kHz
    mono ([frames] or [frames, 1]) 1-D, any other as resample.as_input returns it.  Raises the error a chunk of another
    sort raises."""
    rate = resample.check_rate(rate)
    if not isinstance(chunk, (torch.Tensor, np.ndarray)):
        raise TypeError('a stream chunk is a numpy array or a torch tensor, got %s' % type(chunk).__name__)
    where = 'cuda' if isinstance(chunk, torch.Tensor) and chunk.is_cuda else 'host'
    if resample.is_native(chunk, rate):
        name = str(chunk.dtype).replace('torch.', '')
        if name not in ('int16', 'float32'):
            raise TypeError('stream chunks are int16 or float32, got %s' % chunk.dtype)
        return (where, name, rate, 1), chunk.reshape(-1)
    x = resample.as_input(chunk)
    return (where, str(x.dtype).replace('torch.', ''), rate, resample.channels(x)), x


def _khz(rate):
    return '%g kHz' % (rate / 1000)


def _check_same(key, opened, got):
    if opened[:2] != got[:2]:
        raise TypeError('stream %r was opened with %s %s chunks, got %s %s' % ((key,) + opened[:2] + got[:2]))
    if opened[2] != got[2]:
        raise ValueError('stream %r was opened at %s, got %s' % (key, _khz(opened[2]), _khz(got[2])))
    if opened[3] != got[3]:
        raise ValueError('stream %r was opened with %d channels, got %d' % (key, opened[3], got[3]))


class LiveStreams:
    """Live segmentation of many streams (``Segmenter.stream``).  ``feed({key: chunk})`` returns {key: segments decided
    in this call}; ``end(keys)`` returns {key: its remaining segments} and frees the keys; ``decided_until(key)`` is the
    time (s) up to which the stream's labels are final."""

    def __init__(self, seg, calibration_sec=60.0, backend=None, observer=None):
        """``observer``, if given, is called as observer({key: chunk}) with the 16 kHz chunk of every stream in each
        device pass, before the pass (what ``vfs_stream.LiveScores`` continues its own pipeline from)."""
        if not calibration_sec >= 1.0:
            raise ValueError('calibration_sec must be >= 1.0 (got %r): a stream must hold 68 frames before its '
                             'labels can be decided' % (calibration_sec,))
        self.seg = seg
        self.n_cal = int(round(100 * calibration_sec))
        self.vad_labels = seg.vad.outlabels
        self.gender_labels = seg.gender.outlabels if seg.detect_gender else None
        self.backend = backend if backend is not None else CudaBackend(seg)
        self.observer = observer
        self.streams = {}
        self._free_sids, self._next_sid = [], 0
        self._failed = None            # the error of a call that stopped part way: the object is no longer usable

    # ---- public -------------------------------------------------------------------------------------------------
    def _usable(self):
        if self._failed is not None:
            raise RuntimeError('this LiveStreams object stopped in a failed call (%s: %s); its streams cannot '
                               'continue' % (type(self._failed).__name__, self._failed))

    def _guarded(self, fn, *args):
        """Run a call that changes stream state; if it fails part way, no later call may continue from it."""
        try:
            return fn(*args)
        except BaseException as e:
            self._failed = e
            raise

    def feed(self, chunks, sample_rate=16000):
        """Feed one chunk per key (opening the streams not seen before); returns {key: segments decided now}.
        ``sample_rate`` is the rate of every chunk, or a dict {key: rate}.  A chunk is int16 or float32, [frames] or
        [frames, channels], a numpy array, a CPU tensor or a CUDA tensor; a stream's location, dtype, rate and channel
        count are those of its first chunk.  Streams other than 16 kHz mono are resampled to 16 kHz mono int16 on
        the device, chunk by chunk, as ``segment_signal(x, sample_rate=rate)`` resamples the whole stream.  Invalid
        chunks raise before anything changes.  If the device pass itself fails, the object cannot be used again: every
        later call raises."""
        self._usable()
        if isinstance(sample_rate, dict):
            missing = [k for k in chunks if k not in sample_rate]
            if missing:
                raise ValueError('no sample rate for stream %r in the sample_rate dict' % (missing[0],))
            checked = {k: _kind(c, sample_rate[k]) for k, c in chunks.items()}
        else:
            checked = {k: _kind(c, sample_rate) for k, c in chunks.items()}
        for k, (kind, _) in checked.items():
            st = self.streams.get(k)
            if st is not None:
                _check_same(k, st.kind, kind)
        for k, (kind, _) in checked.items():
            if k not in self.streams:
                self.streams[k] = _Stream(k, self._new_sid(), kind)
        return self._guarded(self._feed, {self.streams[k]: c for k, (_, c) in checked.items()})

    def _feed(self, chunks):
        rs = [st for st in chunks if st.rate is not None]
        if rs:
            got = self.backend.resample({st.sid: chunks[st] for st in rs}, {st.sid: st.rate for st in rs})
            for st in rs:
                st.frames_in += int(chunks[st].shape[0])
                chunks[st] = got[st.sid]
        return self._run(chunks, [])

    @staticmethod
    def _samples_at_end(st):
        """16 kHz samples of a stream once it ends (a resampled stream's last outputs come with the end)."""
        return st.samples if st.rate is None else resample.end_outputs(st.frames_in, st.rate)

    def end(self, keys):
        self._usable()
        keys = list(keys)
        unknown = [k for k in keys if k not in self.streams]
        if unknown:
            raise KeyError('no open stream %r' % (unknown[0],))
        # counted before the resampler's flush, from the count the flush brings a stream to, so that a rejected end
        # leaves the other streams as they were
        short = [k for k in keys if self._samples_at_end(self.streams[k]) < pack.WIN]
        if short:
            st = self._close(self.streams[short[0]])
            raise ValueError('media <array> holds %d samples: less than one 25 ms analysis frame'
                             % self._samples_at_end(st))
        return self._guarded(self._end, [self.streams[k] for k in keys])

    def _end(self, ending):
        out = {st.key: [] for st in ending}
        rs = [st for st in ending if st.rate is not None]
        if rs:
            # flush the resampler first: its last outputs (those that read the zeros past the end) are the stream's
            # last 16 kHz samples, and may complete its calibration
            last = self.backend.resample({}, {st.sid: st.rate for st in rs}, [st.sid for st in rs])
            for k, v in self._run({st: last[st.sid] for st in rs}, []).items():
                out[k] += v
        offline = [st for st in ending if not st.calibrated]
        for st in offline:
            with warnings.catch_warnings():
                warnings.simplefilter('ignore')
                out[st.key] += self.backend.offline(st.sid, st.F)
        live = [st for st in ending if st.calibrated]
        for st in live:
            st.ended = True
        if live:
            for k, v in self._run({}, live).items():
                out[k] += v
        for st in ending:
            self._close(st)
        return {st.key: out[st.key] for st in ending}

    def decided_until(self, key):
        self._usable()
        return self.streams[key].fin * .02

    # ---- one device pass ----------------------------------------------------------------------------------------
    def _new_sid(self):
        if self._free_sids:
            return self._free_sids.pop()
        self._next_sid += 1
        return self._next_sid - 1

    def _close(self, st):
        del self.streams[st.key]
        for stage, name in ((st.vad, 'vad'), (st.gen, 'gender')):
            if stage.chain is not None:
                self.backend.free_slot(name, stage.chain.slot)
        self.backend.release(st.sid)
        self._free_sids.append(st.sid)
        return st

    def _run(self, chunks, ending):
        be = self.backend
        if self.observer is not None and chunks:
            self.observer({st.key: c for st, c in chunks.items()})
        for st, c in chunks.items():
            st.samples += len(c)
        keep = {st.sid: st.R0 for st in self.streams.values()}
        be.ingest({st.sid: c for st, c in chunks.items()}, keep)
        for st in chunks:
            st.F = pack.num_frames(st.samples)
        # calibration: threshold from the first N_cal loge values
        cal = [st for st in chunks if not st.calibrated and st.F >= self.n_cal]
        if cal:
            be.calibrate([st.sid for st in cal], self.n_cal)
            for st in cal:
                st.calibrated = True
        # energy chains
        todo = [st for st in set(chunks) | set(ending) if st.calibrated and (st.F > st.e_fed or st.ended)]
        todo.sort(key=lambda s: s.sid)
        if todo:
            rows = [(st.sid, st.e_fed, st.F - st.e_fed, st.e_pend,
                     (engine.ONLINE_START if st.e_fed == 0 else 0) | (engine.ONLINE_END if st.ended else 0))
                    for st in todo]
            for st, dec in zip(todo, be.energy(rows)):
                st.e_pend += st.F - st.e_fed - len(dec)
                st.e_fed = st.F
                first = st.e_dec
                st.e_dec += len(dec)
                st.elab.put((first + 1) // 2, dec[(first % 2)::2].astype(np.int8))
        # VAD over energy, gender over VAD speech
        self._stage('vad', todo, lambda st: (st.elab, (st.e_dec + 1) // 2, 1))
        if self.gender_labels is not None:
            speech = self.vad_labels.index('speech')
            self._stage('gender', todo, lambda st: (st.vad.out, st.vad.dec, speech))
        out = {st.key: [] for st in chunks}
        for st in todo:
            out[st.key] = self._emit(st)
        for st in todo:
            need = min(st.vad.fed, st.gen.fed if self.gender_labels is not None else st.vad.fed)
            st.R0 = max(0, min(2 * max(need - LFILL, 0), (st.F - PATCH_W - 1) // 2 * 2))
        return out

    def _stage(self, name, streams, source):
        """Plan the chains of one CNN stage for every stream, run them in one backend call, store the decisions."""
        rows, owners = [], []
        for st in streams:
            track, n_in, inlabel = source(st)
            stage = st.vad if name == 'vad' else st.gen
            total = (st.F + 1) // 2
            limit = total if st.ended else computable_patches(st.F)
            p = a = stage.fed
            vals = track.get(p, n_in)
            stage.out.extend(n_in)
            cut = np.flatnonzero(vals[1:] != vals[:-1]) + 1 + p
            for r0, r1 in zip(np.concatenate(([p], cut)).tolist(), np.concatenate((cut, [n_in])).tolist()):
                if r0 >= r1:
                    break
                if vals[r0 - stage.fed] != inlabel:
                    if stage.chain is not None:
                        rows.append((stage.chain.slot, st.sid, a, r0, self._flags(stage, a, True)))
                        owners.append((st, stage, stage.chain))
                        stage.chain = None
                    stage.out.put(r0, np.full(r1 - r0, _PASS, dtype=np.int8))
                    p = a = r1
                    continue
                if r0 >= limit:
                    break
                if stage.chain is None:
                    stage.chain = _Chain(self.backend.new_slot(name), r0)
                    stage.chain.pend = -1           # marks a chain that starts in this call
                    a = r0
                p = min(r1, limit)
                if p < r1:
                    break
            stage.fed = p
            if stage.chain is not None and (p > a or (st.ended and p == total)):
                end = st.ended and p == total
                rows.append((stage.chain.slot, st.sid, a, p, self._flags(stage, a, end)))
                owners.append((st, stage, stage.chain))
                if end:
                    stage.chain = None
        if not rows:
            for st in streams:
                stage = st.vad if name == 'vad' else st.gen
                stage.dec = stage.out.first_undecided(stage.dec)
            return
        chains = [(slot, sid, a, b, flags, ch.pend if ch.pend >= 0 else 0)
                  for (slot, sid, a, b, flags), (_, _, ch) in zip(rows, owners)]
        decided = self.backend.decode(name, chains, {st.sid: (st.F, st.ended) for st in streams})
        for (slot, sid, a, b, flags), (st, stage, ch), dec in zip(rows, owners, decided):
            ch.pend = (ch.pend if ch.pend >= 0 else 0) + (b - a) - len(dec)
            stage.out.put(ch.next, dec.astype(np.int8))
            ch.next += len(dec)
            if flags & engine.ONLINE_END:
                self.backend.free_slot(name, slot)
        for st in streams:
            stage = st.vad if name == 'vad' else st.gen
            stage.dec = stage.out.first_undecided(stage.dec)

    @staticmethod
    def _flags(stage, a, end):
        ch = stage.chain
        return (engine.ONLINE_START if ch.pend == -1 and ch.next == a else 0) | (engine.ONLINE_END if end else 0)

    def _emit(self, st):
        """Segments whose labels are final, in patch units -> seconds; the last run stays open until it is complete."""
        e_n = (st.e_dec + 1) // 2
        lim = min(e_n, st.vad.dec) if e_n else 0
        if self.gender_labels is not None:
            lim = min(lim, st.gen.dec)
        # patches < lim: energy, VAD and gender outputs are all decided (or passed through)
        segs = []
        if lim > st.fin:
            # one code per patch: -1 noEnergy, VAD class k, 16 + gender class
            code = np.where(st.elab.get(st.fin, lim) == 0, -1, st.vad.out.get(st.fin, lim)).astype(np.int16)
            if self.gender_labels is not None:
                g = st.gen.out.get(st.fin, lim)
                code = np.where(g >= 0, 16 + g, code)
            cut = (np.flatnonzero(code[1:] != code[:-1]) + 1).tolist()
            for r0, r1 in zip([0] + cut, cut + [len(code)]):
                c = int(code[r0])
                nm = 'noEnergy' if c < 0 else (self.gender_labels[c - 16] if c >= 16 else self.vad_labels[c])
                p = st.fin + r0
                if st.open is None:
                    st.open = (nm, p)
                elif st.open[0] != nm:
                    segs.append((st.open[0], 0 + st.open[1] * .02, 0 + p * .02))
                    st.open = (nm, p)
            st.fin = lim
        total = (st.F + 1) // 2
        if st.ended and st.fin == total and st.open is not None:
            segs.append((st.open[0], 0 + st.open[1] * .02, 0 + total * .02))
            st.open = None
        low = min(st.fin, st.vad.fed, st.gen.fed if self.gender_labels is not None else st.fin)
        for t in (st.elab, st.vad.out, st.gen.out):
            t.drop(min(low, st.fin))
        return segs


class CudaBackend:
    """The device side of LiveStreams: sample tails, retained log-mel / loge rows and the chains' scores and histories,
    each packed across streams in one buffer that is rebuilt or grown, never allocated per stream."""

    def __init__(self, seg):
        from .segmenter import _get_frontend, _stage_pass
        self.seg, self.ctx, self.dev = seg, seg.ctx, seg.ctx.device
        self.fe = _get_frontend('main', self.dev.index)
        self._stage_pass = _stage_pass
        self.tails = {}                # sid -> CUDA tensor: samples from 160 * F on
        self.rows = {}                 # sid -> (first retained frame, rows in store)
        self.frames = {}               # sid -> frames computed
        self.mspec = torch.empty((0, 24), dtype=torch.float32, device=self.dev)
        self.loge = torch.empty((0,), dtype=torch.float32, device=self.dev)
        self.off = {}                  # sid -> first store row
        self.stats = torch.zeros((0, 2), dtype=torch.float64, device=self.dev)
        self.e_scores = torch.zeros((0, 4), dtype=torch.float64, device=self.dev)
        self.e_hist = torch.zeros((0, 256), dtype=torch.uint8, device=self.dev)
        self.chain = {n: [torch.zeros((0, 4), dtype=torch.float64, device=self.dev),
                          torch.zeros((0, 256), dtype=torch.uint8, device=self.dev)] for n in ('vad', 'gender')}
        self.free = {'vad': [], 'gender': []}
        self.nslot = {'vad': 0, 'gender': 0}
        self.rs = {}                   # sid -> _RsTail of a resampled stream

    # slots of CNN chains
    def new_slot(self, name):
        if self.free[name]:
            return self.free[name].pop()
        self.nslot[name] += 1
        return self.nslot[name] - 1

    def free_slot(self, name, slot):
        self.free[name].append(slot)

    def release(self, sid):
        self.rs.pop(sid, None)
        self.tails.pop(sid, None)
        self.rows.pop(sid, None)
        self.frames.pop(sid, None)

    @staticmethod
    def _grow(scores, hist, nslot, need):
        """Tables with room for nslot slots and histories of `need` steps (doubling), contents kept."""
        cap = hist.shape[1]
        while cap < need:
            cap *= 2
        rows = max(nslot, scores.shape[0])
        if rows > scores.shape[0]:
            rows = max(rows, 2 * scores.shape[0], 64)
        if rows == scores.shape[0] and cap == hist.shape[1]:
            return scores, hist
        s2 = torch.zeros((rows, 4), dtype=scores.dtype, device=scores.device)
        h2 = torch.zeros((rows, cap), dtype=hist.dtype, device=hist.device)
        s2[:scores.shape[0]] = scores
        h2[:hist.shape[0], :hist.shape[1]] = hist
        return s2, h2

    def resample(self, chunks, rates, final=()):
        """{sid: the 16 kHz int16 samples that become final}: chunks {sid: the stream's next frames, as _kind returns
        them} at rates[sid], and for the streams in `final` (which have ended) all their remaining samples.  Each
        stream keeps its raw input from resample.first_kept on; its tail and new chunk are one window.  Host chunks go
        up in one pinned copy; each (rate, channels, dtype) group is one concatenation and one launch, into one int16
        buffer whose views are returned."""
        sids = sorted(set(chunks) | set(final))
        fed = [s for s in sids if s in chunks]
        staged = dict(zip(fed, self._stage_pass([chunks[s] for s in fed], self.dev))) if fed else {}
        groups, n_out, pos = {}, {}, 0
        for sid in sids:
            t = self.rs.get(sid)
            if t is None:
                c = staged[sid]
                t = self.rs[sid] = _RsTail(rates[sid], resample.channels(c), c.dtype)
            n = t.n + (int(staged[sid].shape[0]) if sid in staged else 0)
            k_to = (resample.end_outputs if sid in final else resample.ready_outputs)(n, t.rate)
            n_out[sid] = (pos, k_to - t.k)
            pos += k_to - t.k
            groups.setdefault((t.rate, t.C, t.dtype), []).append((sid, n, k_to))
        out = torch.empty(pos, dtype=torch.int16, device=self.dev)
        for (rate, C, _), items in groups.items():
            pieces = []
            for sid, _, _ in items:
                t = self.rs[sid]
                pieces += [p for p in (t.tail, staged[sid].reshape(-1) if sid in staged else None) if p is not None]
            big = torch.cat(pieces)
            wins, rows, tails, at = [], [], [], 0
            for sid, n, k_to in items:
                t = self.rs[sid]
                win = big[at:at + (n - t.f0) * C]
                at += win.numel()
                wins.append(win.view(-1, C))
                rows.append((t.f0, n, t.k, k_to - t.k, n_out[sid][0], _lib.RESAMPLE_END if sid in final else 0))
                keep = min(resample.first_kept(k_to, rate), n)
                tails.append(win[(keep - t.f0) * C:])
                t.f0, t.n, t.k = keep, n, k_to
            resample.window_multi(self.ctx, wins, np.array(rows, dtype=np.int64), rate, out)
            # the tails (a few ms each) get a buffer of their own, so that `big` is freed after this call
            tb, at = torch.cat(tails), 0
            for (sid, _, _), tl in zip(items, tails):
                self.rs[sid].tail = tb[at:at + tl.numel()]
                at += tl.numel()
        return {sid: out[a:a + k] for sid, (a, k) in n_out.items()}

    def ingest(self, chunks, keep):
        """Append each chunk to its stream, compute the new frames (K1 on tail + chunk) and rebuild the store with the
        rows from keep[sid] on, for every open stream."""
        sids = sorted(chunks)
        staged = self._stage_pass([c.reshape(-1) if isinstance(c, torch.Tensor) and c.is_cuda else
                                   (c.numpy() if isinstance(c, torch.Tensor) else np.ascontiguousarray(c))
                                   for c in (chunks[s] for s in sids)], self.dev) if sids else []
        new_rows = {}
        # tail + chunk of every stream of one sample type in one concatenation
        bydt = {}
        for sid, c in zip(sids, staged):
            tail = self.tails.get(sid)
            bydt.setdefault(c.dtype, []).append((sid, [c] if tail is None else [tail, c]))
        groups = {}
        for dtype, items in bydt.items():
            big = torch.cat([piece for _, pieces in items for piece in pieces])
            pos, tails = 0, []
            for sid, pieces in items:
                n = sum(p.numel() for p in pieces)
                pcm = big[pos:pos + n]
                pos += n
                nf = pack.num_frames(n)
                tails.append(pcm[nf * pack.HOP:] if nf else pcm)
                self.frames[sid] = self.frames.get(sid, 0) + nf
                if nf:
                    groups.setdefault(dtype, []).append((sid, pcm[:(nf - 1) * pack.HOP + pack.WIN], nf))
            # the tails (< 400 samples each) get a buffer of their own, so that `big` is freed after this call
            tb, pos = torch.cat(tails), 0
            for (sid, _), t in zip(items, tails):
                self.tails[sid] = tb[pos:pos + t.numel()]
                pos += t.numel()
        for dtype, items in groups.items():
            nfs = np.array([nf for _, _, nf in items], dtype=np.int64)
            lay = _Layout(nfs)
            m, l, _ = self.fe.multi([p for _, p, _ in items], lay, self.seg.fft_precision)
            for i, (sid, _, nf) in enumerate(items):
                a = int(lay.row_off[i])
                new_rows[sid] = (m[a:a + nf], l[a:a + nf])
        # rebuild the store: per stream, its retained old rows then its new rows, gathered by ranges (first source row,
        # length) of the concatenation [old store, new rows ...]
        src_m, src_l, rng, off, pos = [self.mspec], [self.loge], [], {}, 0
        base = self.mspec.shape[0]
        for sid in sorted(keep):
            F = self.frames.get(sid, 0)
            R0 = keep[sid]
            old = self.rows.get(sid)
            nnew = new_rows[sid][0].shape[0] if sid in new_rows else 0
            off[sid] = pos
            if old is not None:
                a0, n0 = old
                take = a0 + n0 - R0
                if take > 0:
                    rng.append((self.off[sid] + (R0 - a0), take))
                    pos += take
            if nnew:
                m, l = new_rows[sid]
                rng.append((base, nnew))
                src_m.append(m)
                src_l.append(l)
                base += nnew
                pos += nnew
            self.rows[sid] = (R0 if old is not None else F - nnew, pos - off[sid])
        self.off = off
        if pos:
            r = np.array(rng, dtype=np.int64).reshape(-1, 2)
            dst = np.concatenate(([0], np.cumsum(r[:, 1])[:-1]))
            shift = torch.from_numpy(r[:, 0] - dst).to(self.dev, non_blocking=True)
            lens = torch.from_numpy(r[:, 1].copy()).to(self.dev, non_blocking=True)
            ix = torch.arange(pos, device=self.dev) + torch.repeat_interleave(shift, lens, output_size=pos)
            self.mspec = torch.cat(src_m).index_select(0, ix)
            self.loge = torch.cat(src_l).index_select(0, ix)
        else:
            self.mspec, self.loge = self.mspec[:0], self.loge[:0]

    def _row(self, sid, frame):
        a0, n0 = self.rows[sid]
        assert a0 <= frame <= a0 + n0, (sid, frame, a0, n0)
        return self.off[sid] + frame - a0

    def calibrate(self, sids, n_cal):
        st = engine.loge_stats_multi(self.ctx, self.loge, [self._row(s, 0) for s in sids], [n_cal] * len(sids))
        nmax = max(sids) + 1
        if self.stats.shape[0] < nmax:
            s2 = torch.zeros((max(nmax, 2 * self.stats.shape[0], 64), 2), dtype=torch.float64, device=self.dev)
            s2[:self.stats.shape[0]] = self.stats
            self.stats = s2
        self.stats[torch.as_tensor(sids, device=self.dev)] = st

    def energy(self, rows):
        """rows: (sid, first frame, frames, undecided steps, flags) -> decided frame states per row."""
        need = max(p + n for _, _, n, p, _ in rows)
        self.e_scores, self.e_hist = self._grow(self.e_scores, self.e_hist, max(r[0] for r in rows) + 1, need)
        ch = np.array([(self._row(sid, f0), n, sid, p, 0, fl) for sid, f0, n, p, fl in rows], dtype=np.int64)
        ch[:, 4] = np.concatenate(([0], np.cumsum(ch[:, 1] + ch[:, 3])[:-1]))
        buf = engine.viterbi_online(self.ctx, ch, self.loge, self.e_scores, self.e_hist, int((ch[:, 1] + ch[:, 3]).sum()),
                                    stats=self.stats, energy_ratio=self.seg.energy_ratio)
        return self._split(buf, ch)

    @staticmethod
    def _split(buf, ch):
        host = buf.cpu().numpy()
        nd, states = engine.split_online(host, len(ch))
        return [states[o:o + k].copy() for o, k in zip(ch[:, 4], nd)]

    def decode(self, name, chains, info):
        """chains: (slot, sid, first patch, stop patch, flags, undecided steps): the network of stage `name` on the
        patches, then the chains continued over their posteriors -> decided states per chain."""
        net = self.seg.vad if name == 'vad' else self.seg.gender
        sids = sorted({c[1] for c in chains})
        rec = {sid: i for i, sid in enumerate(sids)}
        row_off = [self.off[sid] for sid in sids]
        lens = [self.rows[sid][1] for sid in sids]
        ranges, rrec = [], []
        for slot, sid, a, b, fl, p in chains:
            if b > a:
                r0 = self.rows[sid][0] // 2          # the store starts at an even frame: patch p is patch p - r0 there
                ranges.append((a - r0, b - r0))
                rrec.append(rec[sid])
        probs = net.nn.forward_multi(self.mspec, row_off, lens, rrec, ranges) if ranges else \
            torch.empty((0, net.nn.n_classes), dtype=torch.float32, device=self.dev)
        scores, hist = self.chain[name]
        need = max(p + b - a for _, _, a, b, _, p in chains)
        scores, hist = self._grow(scores, hist, self.nslot[name], need)
        self.chain[name] = [scores, hist]
        ch = np.zeros((len(chains), 6), dtype=np.int64)
        pos = 0
        for i, (slot, sid, a, b, fl, p) in enumerate(chains):
            ch[i] = (pos, b - a, slot, p, 0, fl)
            pos += b - a
        ch[:, 4] = np.concatenate(([0], np.cumsum(ch[:, 1] + ch[:, 3])[:-1]))
        K = len(net.outlabels)
        buf = engine.viterbi_online(self.ctx, ch, probs, scores, hist, int((ch[:, 1] + ch[:, 3]).sum()), K=K,
                                    trans=engine.diag_trans_exp(net.viterbi_arg, K))
        # non-finite posteriors are an error, as in the offline path; the flag travels with the decided states
        flag = torch.isfinite(probs).all().to(torch.uint8).view(1)
        host = torch.cat((buf, flag)).cpu().numpy()
        if not host[-1]:
            raise _lib.IssError('%s: the CNN returned non-finite posteriors: an activation left the fp16 range of the '
                                'default fp16-split GEMM engine; run with ISS_B200_GEMM=tc_ts (3xTF32, fp32 range)'
                                % type(net).__name__)
        nd, states = engine.split_online(host[:-1], len(ch))
        return [states[o:o + k].copy() for o, k in zip(ch[:, 4], nd)]

    def offline(self, sid, F):
        """The offline segmentation of a stream that ended before calibration (all its rows are still retained)."""
        from .segmenter import PATCH_W as W
        a = self.off[sid]
        mspec, loge = self.mspec[a:a + F], self.loge[a:a + F]
        difflen = 0
        if F < W:
            difflen = W - F
            mspec = torch.cat((mspec, mspec.min().expand(difflen, 24)))
        return self.seg.segment_feats(mspec.contiguous(), loge.contiguous(), difflen, 0)


class _RsTail:
    """The resampler state of a stream: its raw samples of frames [f0, n) (flattened) and its next output k."""
    __slots__ = ('rate', 'C', 'dtype', 'tail', 'f0', 'n', 'k')

    def __init__(self, rate, C, dtype):
        self.rate, self.C, self.dtype = rate, C, dtype
        self.tail, self.f0, self.n, self.k = None, 0, 0, 0


class _Layout:
    """Offsets of K1 outputs packed back to back (pack.PassLayout without the 68-row reservation)."""

    def __init__(self, frames):
        self.row_off = np.concatenate(([0], np.cumsum(frames)[:-1])).astype(np.int64)
        self.loge_off = np.concatenate(([0], np.cumsum(frames))).astype(np.int64)
        self.total_rows = int(frames.sum())
