"""Device operators: thin, typed wrappers over the C ABI (torch tensors are
only device-memory containers and stream handles here -- no torch.nn, no
torch math on the hot path)."""
import ctypes

import numpy as np
import torch

from . import _lib
from .models import LoweredModel, lower_keras_model


def _stream_ptr(dev, stream=None):
    st = stream if stream is not None else torch.cuda.current_stream(dev)
    return ctypes.c_void_p(st.cuda_stream)


class Context:
    """One libiss_b200 context = one CUDA device + one in-flight stream of work."""

    def __init__(self, device=0):
        if not torch.cuda.is_available():
            raise _lib.IssError('inaspeechsegmenter_b200 needs a CUDA device (H100, sm_90a); there is no CPU path')
        self.device = torch.device('cuda', device if isinstance(device, int) else torch.device(device).index or 0)
        lib = _lib.load()
        h = ctypes.c_void_p()
        _lib.check(lib.iss_ctx_create(self.device.index, ctypes.byref(h)), 'iss_ctx_create')
        self.handle = h
        self._work = {}

    def workspace(self, key, nbytes):
        """Grow-only scratch buffers (device), one per use so stages never alias."""
        buf = self._work.get(key)
        if buf is None or buf.numel() < nbytes:
            buf = torch.empty(int(nbytes * 1.25) + 256, dtype=torch.uint8, device=self.device)
            self._work[key] = buf
        return buf

    def close(self):
        if self.handle:
            _lib.load().iss_ctx_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class CnnModel:
    """The ``keras.Model.predict`` seam (segmenter.py:131-133,163) on device,
    fused with ``_get_patches`` (:76-88) and the 0.5 override (:175)."""

    def __init__(self, ctx, lowered: LoweredModel):
        self.ctx, self.lowered = ctx, lowered
        lib = _lib.load()
        descs = lowered.c_descs()
        blob = np.ascontiguousarray(lowered.blob, dtype=np.float32)
        h = ctypes.c_void_p()
        _lib.check(lib.iss_cnn_create(ctx.handle, descs, len(lowered.descs), _lib.ptr(blob), blob.size,
                                      lowered.in_h, lowered.in_w, ctypes.byref(h)), 'iss_cnn_create')
        self.handle = h
        self.n_classes = lib.iss_cnn_num_classes(h)
        self.flops_per_patch = lib.iss_cnn_flops_per_patch(h)
        self.nmel = lowered.in_w

    @classmethod
    def from_keras(cls, ctx, config, weights, nmel):
        return cls(ctx, lower_keras_model(config, weights, 68, nmel))

    def forward(self, mspec, ranges, edge_left=True, edge_right=True, stream=None):
        """mspec: CUDA float32 [L, ld]; ranges: list of (start, stop) padded-patch
        index ranges.  Returns CUDA float32 [n, K] probabilities (rows of
        non-finite patches already forced to 0.5)."""
        assert mspec.is_cuda and mspec.dtype == torch.float32 and mspec.is_contiguous()
        L, ld = mspec.shape
        starts = np.ascontiguousarray([a for a, _ in ranges], dtype=np.int32)
        stops = np.ascontiguousarray([b for _, b in ranges], dtype=np.int32)
        n = int((stops - starts).sum()) if len(ranges) else 0
        probs = torch.empty((n, self.n_classes), dtype=torch.float32, device=mspec.device)
        if n == 0:
            return probs
        lib = _lib.load()
        wb = lib.iss_cnn_workspace_bytes(self.handle, n, len(ranges))
        work = self.ctx.workspace('cnn', wb)
        _lib.check(lib.iss_cnn_forward(self.ctx.handle, self.handle, _lib.ptr(mspec), L, ld,
                                       int(bool(edge_left)), int(bool(edge_right)),
                                       _lib.ptr(starts), _lib.ptr(stops), len(ranges),
                                       _lib.ptr(probs), _lib.ptr(work), work.numel(),
                                       _stream_ptr(mspec.device, stream)), 'iss_cnn_forward')
        return probs

    def forward_multi(self, mspec, row_off, lens, rec, ranges, stream=None):
        """Recordings packed in mspec (CUDA float32 [rows, ld]): recording r is rows row_off[r] .. + lens[r]
        (lens[r] >= 68); range s = ranges[s] = (start, stop) padded patches of recording rec[s], both edges
        replicated.  Returns CUDA float32 [n, K] as forward() does."""
        assert mspec.is_cuda and mspec.dtype == torch.float32 and mspec.is_contiguous()
        rows, ld = mspec.shape
        row_off = np.ascontiguousarray(row_off, dtype=np.int64)
        lens = np.ascontiguousarray(lens, dtype=np.int64)
        rec = np.ascontiguousarray(rec, dtype=np.int32)
        starts = np.ascontiguousarray([a for a, _ in ranges], dtype=np.int32)
        stops = np.ascontiguousarray([b for _, b in ranges], dtype=np.int32)
        n = int((stops - starts).sum()) if len(ranges) else 0
        probs = torch.empty((n, self.n_classes), dtype=torch.float32, device=mspec.device)
        if n == 0:
            return probs
        lib = _lib.load()
        work = self.ctx.workspace('cnn', lib.iss_cnn_workspace_bytes(self.handle, n, len(ranges)))
        _lib.check(lib.iss_cnn_forward_multi(self.ctx.handle, self.handle, _lib.ptr(mspec), rows, ld,
                                             _lib.ptr(row_off), _lib.ptr(lens), len(lens), _lib.ptr(rec),
                                             _lib.ptr(starts), _lib.ptr(stops), len(ranges),
                                             _lib.ptr(probs), _lib.ptr(work), work.numel(),
                                             _stream_ptr(mspec.device, stream)), 'iss_cnn_forward_multi')
        return probs

    def close(self):
        if self.handle:
            _lib.load().iss_cnn_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class MlpModel:
    """Dense stack on device: the ``keras.Model.predict`` seam of the gender-detection MLP
    (vbx_segmenter.py:116-124,188-191)."""

    def __init__(self, ctx, config, weights, in_dim):
        self.ctx = ctx
        low = lower_keras_model(config, weights, 1, in_dim, allow_no_head=True)
        self.lowered = low
        blob = np.ascontiguousarray(low.blob, dtype=np.float32)
        h = ctypes.c_void_p()
        _lib.check(_lib.load().iss_mlp_create(ctx.handle, low.c_descs(), len(low.descs), _lib.ptr(blob), blob.size,
                                              in_dim, ctypes.byref(h)), 'iss_mlp_create')
        self.handle, self.in_dim = h, in_dim
        self.out_dim = _lib.load().iss_mlp_out_dim(h)

    def predict(self, x, **_):
        """x: [n, in_dim] numpy or CUDA tensor -> numpy float32 [n, out_dim] (keras predict contract)."""
        return self.forward(x).cpu().numpy()

    def forward(self, x):
        """predict without the copy back: a CUDA float32 [n, out_dim] tensor."""
        t = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
        t = t.to(self.ctx.device).contiguous()
        if t.data_ptr() % 16:                       # a view at an odd offset: iss_mlp_forward needs 16-byte rows
            t = t.clone()
        n = t.shape[0]
        y = torch.empty((n, self.out_dim), dtype=torch.float32, device=self.ctx.device)
        if n:
            lib = _lib.load()
            work = self.ctx.workspace('mlp', lib.iss_mlp_workspace_bytes(self.handle, n))
            _lib.check(lib.iss_mlp_forward(self.ctx.handle, self.handle, _lib.ptr(t), n, _lib.ptr(y), _lib.ptr(work),
                                           work.numel(), _stream_ptr(self.ctx.device)), 'iss_mlp_forward')
        return y

    def close(self):
        if self.handle:
            _lib.load().iss_mlp_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ---- Viterbi operators (pyannote_viterbi.py:118-224 + viterbi_utils.py:29-49) ------------

def log_trans_exp(exp, cost0=0, cost1=0):
    """viterbi_utils.py:36-42 (host constants; numpy so the doubles match the reference's)."""
    cost = -exp * np.log(10)
    ret = np.ones((2, 2)) * cost
    ret[0, 0] = cost0
    ret[1, 1] = cost1
    return ret


def diag_trans_exp(exp, dim):
    """viterbi_utils.py:44-49."""
    cost = -exp * np.log(10)
    ret = np.ones((dim, dim)) * cost
    for i in range(dim):
        ret[i, i] = 0
    return ret


def loge_stats(ctx, loge, stream=None):
    """{sum, count} of the finite entries of a CUDA float32 loge array (segmenter.py:70),
    bit-identical to the reduction fused into the K1 kernel."""
    stats = torch.empty((2,), dtype=torch.float64, device=loge.device)
    _lib.check(_lib.load().iss_loge_stats(ctx.handle, _lib.ptr(loge), loge.numel(), _lib.ptr(stats),
                                          _stream_ptr(loge.device, stream)), 'iss_loge_stats')
    return stats


_EMIS = np.log(np.array([1 - 1e-10, 1e-10]))          # pred2logemission, viterbi_utils.py:29-34


def _energy_consts(energy_ratio):
    """(transition matrix, prior log(1/2), log(energy_ratio)) of the energy Viterbi (segmenter.py:69-73)."""
    trans = np.ascontiguousarray(log_trans_exp(150, cost0=-5), dtype=np.float64)
    return trans, float(np.log(np.ones(2) / 2)[0]), float(np.log(energy_ratio))


def energy_viterbi(ctx, loge, stats, energy_ratio, out_stride=2, stream=None):
    """``_energy_activity(loge, ratio)[::out_stride]`` (segmenter.py:69-73,262) -> CUDA uint8."""
    L = loge.numel()
    nout = (L + out_stride - 1) // out_stride
    states = torch.empty((nout,), dtype=torch.uint8, device=loge.device)
    if L == 0:
        return states
    lib = _lib.load()
    work = ctx.workspace('vit_energy', lib.iss_viterbi_work_bytes(L, 1))
    trans, prior, lr = _energy_consts(energy_ratio)
    _lib.check(lib.iss_energy_viterbi(ctx.handle, _lib.ptr(loge), L, _lib.ptr(stats), lr,
                                      _lib.ptr(_EMIS), _lib.ptr(trans), prior, int(out_stride),
                                      _lib.ptr(states), _lib.ptr(work), _stream_ptr(loge.device, stream)),
               'iss_energy_viterbi')
    return states


def energy_viterbi_multi(ctx, loge, loge_off, stats, energy_ratio, out_off, out_stride=2, stream=None):
    """energy_viterbi on each recording of a packed loge: recording r is loge[loge_off[r]:loge_off[r+1]] with
    statistics stats[r] (CUDA float64 [n, 2]); its track goes to states[out_off[r]:out_off[r+1]] -> CUDA uint8."""
    loge_off = np.ascontiguousarray(loge_off, dtype=np.int64)
    out_off = np.ascontiguousarray(out_off, dtype=np.int64)
    n_rec = len(loge_off) - 1
    states = torch.empty((int(out_off[-1]),), dtype=torch.uint8, device=loge.device)
    lib = _lib.load()
    work = ctx.workspace('vit_energy', lib.iss_viterbi_work_bytes(int(loge_off[-1]), n_rec))
    trans, prior, lr = _energy_consts(energy_ratio)
    _lib.check(lib.iss_energy_viterbi_multi(ctx.handle, _lib.ptr(loge), _lib.ptr(loge_off), n_rec, _lib.ptr(stats), lr,
                                            _lib.ptr(_EMIS), _lib.ptr(trans), prior, int(out_stride), _lib.ptr(out_off),
                                            _lib.ptr(states), _lib.ptr(work), _stream_ptr(loge.device, stream)),
               'iss_energy_viterbi_multi')
    return states


def viterbi_segments(ctx, probs, seg_off, trans, stream=None):
    """Per-segment ``viterbi_decoding(np.log(r), trans)`` (segmenter.py:176) -> CUDA uint8 [n]."""
    n, K = probs.shape
    states = torch.empty((n,), dtype=torch.uint8, device=probs.device)
    if n == 0:
        return states
    lib = _lib.load()
    seg_off = np.ascontiguousarray(seg_off, dtype=np.int64)
    nseg = len(seg_off) - 1
    work = ctx.workspace('vit_seg', lib.iss_viterbi_work_bytes(n, nseg))
    trans = np.ascontiguousarray(trans, dtype=np.float64)
    prior = float(np.log(np.ones(K) / K)[0])
    _lib.check(lib.iss_viterbi_segments(ctx.handle, _lib.ptr(probs), K, _lib.ptr(seg_off), nseg,
                                        _lib.ptr(trans), prior, _lib.ptr(states), _lib.ptr(work),
                                        _stream_ptr(probs.device, stream)), 'iss_viterbi_segments')
    return states


# ---- partial energy chains for time-sharded recordings (shard.py) ---------------------------------
def energy_transfer(ctx, loge, stats, energy_ratio, stream=None):
    """2x2 max-plus transfer matrix (numpy float64, M[j, i]) of this slice of the energy chain."""
    lib = _lib.load()
    L = loge.numel()
    trans, _, lr = _energy_consts(energy_ratio)
    work = ctx.workspace('vit_energy', lib.iss_viterbi_work_bytes(L, 1))
    M = np.zeros(4, dtype=np.float64)
    _lib.check(lib.iss_energy_transfer(ctx.handle, _lib.ptr(loge), L, _lib.ptr(stats), lr, _lib.ptr(_EMIS), _lib.ptr(trans),
                                       _lib.ptr(M), _lib.ptr(work), _stream_ptr(loge.device, stream)), 'iss_energy_transfer')
    return M.reshape(2, 2)


def energy_forward(ctx, loge, stats, energy_ratio, vin=None, stream=None):
    """True forward pass over this slice; returns (vout[2] float64, backmap[2] uint8)."""
    lib = _lib.load()
    L = loge.numel()
    trans, prior, lr = _energy_consts(energy_ratio)
    work = ctx.workspace('vit_energy', lib.iss_viterbi_work_bytes(L, 1))
    vout = np.zeros(2, dtype=np.float64)
    bmap = np.zeros(2, dtype=np.uint8)
    vin_arr = None if vin is None else np.ascontiguousarray(vin, dtype=np.float64)
    _lib.check(lib.iss_energy_forward(ctx.handle, _lib.ptr(loge), L, _lib.ptr(stats), lr, _lib.ptr(_EMIS), _lib.ptr(trans), prior,
                                      _lib.ptr(vin_arr), _lib.ptr(vout), _lib.ptr(bmap), _lib.ptr(work),
                                      _stream_ptr(loge.device, stream)), 'iss_energy_forward')
    return vout, bmap


def energy_emit(ctx, loge, end_state, out_stride=2, stream=None):
    """Backtrack the slice decoded by the preceding energy_forward (same context) -> CUDA uint8 track."""
    lib = _lib.load()
    L = loge.numel()
    states = torch.empty(((L + out_stride - 1) // out_stride,), dtype=torch.uint8, device=loge.device)
    work = ctx.workspace('vit_energy', lib.iss_viterbi_work_bytes(L, 1))
    _lib.check(lib.iss_energy_emit(ctx.handle, L, int(end_state), int(out_stride), _lib.ptr(states), _lib.ptr(work),
                                   _stream_ptr(loge.device, stream)), 'iss_energy_emit')
    return states


# ---- live streams (stream.py) ------------------------------------------------------------------------------------
def loge_stats_multi(ctx, loge, offs, lens, stream=None):
    """loge_stats of each sequence loge[offs[i]:offs[i] + lens[i]] of one CUDA float32 buffer -> CUDA float64 [n, 2]."""
    offs = np.ascontiguousarray(offs, dtype=np.int64)
    lens = np.ascontiguousarray(lens, dtype=np.int64)
    stats = torch.empty((len(offs), 2), dtype=torch.float64, device=loge.device)
    _lib.check(_lib.load().iss_loge_stats_multi(ctx.handle, _lib.ptr(loge), _lib.ptr(offs), _lib.ptr(lens), len(offs),
                                                _lib.ptr(stats), _stream_ptr(loge.device, stream)), 'iss_loge_stats_multi')
    return stats


ONLINE_START, ONLINE_END = 1, 2


def viterbi_online(ctx, chains, src, scores, hist, out_len, K=2, trans=None, stats=None, energy_ratio=None, stream=None):
    """One call of many online Viterbi chains (iss_viterbi_online).  chains: int64 [n, 6] rows {src, n, slot, pend, out,
    flags}; src: CUDA float32 loge (energy mode: `stats` CUDA float64 [slots, 2] and `energy_ratio` given) or posteriors
    [rows, K] (CNN mode: `trans` the K x K transition matrix); scores (CUDA float64 [slots, 4]) and hist (CUDA uint8
    [slots, cap]) carry the chains from call to call.  Returns one CUDA uint8 buffer: n int64 decided counts, then
    out_len decided states, so that the host reads both back in one copy."""
    chains = np.ascontiguousarray(chains, dtype=np.int64).reshape(-1, 6)
    n = len(chains)
    buf = torch.empty((8 * n + max(int(out_len), 1),), dtype=torch.uint8, device=src.device)
    if n == 0:
        return buf
    lib = _lib.load()
    work = ctx.workspace('vit_online', lib.iss_viterbi_online_work_bytes(n))
    if stats is not None:
        t, prior, lr = _energy_consts(energy_ratio)
        emis, K = _EMIS, 2
    else:
        t, prior, lr, emis = np.ascontiguousarray(trans, dtype=np.float64), float(np.log(np.ones(K) / K)[0]), 0.0, None
    n_slots = min(scores.shape[0], hist.shape[0], stats.shape[0] if stats is not None else scores.shape[0])
    _lib.check(lib.iss_viterbi_online(ctx.handle, int(K), n, _lib.ptr(chains), _lib.ptr(src), src.shape[0],
                                      _lib.ptr(stats), lr, _lib.ptr(emis), _lib.ptr(t), prior, _lib.ptr(scores),
                                      _lib.ptr(hist), n_slots, hist.shape[1],
                                      _lib.ptr(buf[8 * n:]), buf.numel() - 8 * n,
                                      _lib.ptr(buf[:8 * n].view(torch.int64)), _lib.ptr(work),
                                      _stream_ptr(src.device, stream)), 'iss_viterbi_online')
    return buf


def split_online(host_buf, n):
    """(decided counts int64 [n], decided states uint8) of a viterbi_online buffer copied to the host."""
    host_buf = np.asarray(host_buf)
    return host_buf[:8 * n].view(np.int64), host_buf[8 * n:]
