"""CPU stand-ins for the device side of live streams (test infrastructure): ``online_step``, the numpy model of one
call of one chain of ``iss_viterbi_online``, and ``OracleStreamBackend``, which gives ``stream.LiveStreams`` the
front end of ``oracle/sidekit_oracle.py``, the patches of ``oracle/segmenter_oracle.py`` and a CNN callable."""
import numpy as np

from oracle import segmenter_oracle as so
from oracle import sidekit_oracle as sk
from oracle import viterbi_oracle as vo


def online_step(emis, trans, prior, V, hist, start, end):
    """numpy model of one call of one chain of ``iss_viterbi_online``: emis [n, K] float64 log emissions of the new
    steps, V the carried scores, hist the back-pointers of the undecided steps (int array [P, K]).  Returns
    (decided states, V, hist) with the same arithmetic and tie rules as the kernel."""
    K = trans.shape[0]
    V = None if start else np.array(V, dtype=np.float64)
    bps = [hist] if len(hist) else []
    cols = np.arange(K)
    new = np.zeros((len(emis), K), dtype=np.int64)
    for t, e in enumerate(emis):
        if V is None:
            V = e + prior
            new[t] = cols
            continue
        cand = V[:, None] + trans
        new[t] = np.argmax(cand, axis=0)
        V = e + cand[new[t], cols]
    bps.append(new)
    h = np.concatenate(bps) if bps else np.zeros((0, K), dtype=np.int64)
    P = len(h)
    if end:
        m, x = P - 1, int(np.argmax(V)) if P else 0
    else:
        m, x, cur = -1, 0, cols.copy()
        for i in range(P - 1, -1, -1):
            if np.all(cur == cur[0]):
                m, x = i, int(cur[0])
                break
            if i == 0:
                break
            cur = h[i][cur]
    out = np.zeros(m + 1, dtype=np.uint8)
    for r in range(m, -1, -1):
        out[r] = x
        if r > 0:
            x = int(h[r][x])
    return out, V, (h[:0] if end else h[m + 1:])


class OracleStreamBackend:
    """The CudaBackend interface on the CPU.  Each stream keeps its sample tail and its rows from the first retained
    frame R0 on; patch p of a stream is taken as padded patch p - R0/2 of ``get_patches`` on those rows, the addressing
    the device backend relies on."""

    def __init__(self, energy_ratio, nets):
        self.ratio, self.nets = energy_ratio, nets       # nets: {'vad': (predict, nmel, outlabels, viterbi_arg), ...}
        self.tails, self.rows, self.thr, self.chains = {}, {}, {}, {}
        self.free, self.nslot = {'vad': [], 'gender': []}, {'vad': 0, 'gender': 0}

    def new_slot(self, name):
        if self.free[name]:
            return self.free[name].pop()
        self.nslot[name] += 1
        return self.nslot[name] - 1

    def free_slot(self, name, slot):
        self.free[name].append(slot)
        self.chains.pop((name, slot), None)

    def release(self, sid):
        for d in (self.tails, self.rows, self.thr):
            d.pop(sid, None)
        self.chains.pop(('energy', sid), None)

    def ingest(self, chunks, keep):
        for sid, c in chunks.items():
            x = np.asarray(c)
            x = x.astype(np.float32) / np.float32(32768) if x.dtype == np.int16 else x.astype(np.float32)
            pcm = np.concatenate((self.tails.get(sid, np.zeros(0, np.float32)), x))
            nf = sk.num_frames(len(pcm))
            R0, M, L = self.rows.get(sid, (0, np.zeros((0, 24), np.float32), np.zeros(0, np.float32)))
            if nf:
                m, l = sk.logmel_loge(pcm[:(nf - 1) * 160 + 400])
                M, L = np.concatenate((M, m)), np.concatenate((L, l))
            self.rows[sid] = (R0, M, L)
            self.tails[sid] = pcm[nf * 160:]
        for sid, R1 in keep.items():
            R0, M, L = self.rows[sid]
            assert R1 >= R0 and R1 % 2 == 0, (R0, R1)
            self.rows[sid] = (R1, M[R1 - R0:], L[R1 - R0:])

    def calibrate(self, sids, n_cal):
        for sid in sids:
            R0, _, L = self.rows[sid]
            assert R0 == 0
            g = L[:n_cal]
            self.thr[sid] = np.mean(g[np.isfinite(g)]) + np.log(self.ratio)         # segmenter.py:70 on the prefix

    def _step(self, key, emis, trans, flags, pend):
        K = trans.shape[0]
        V, hist = self.chains.get(key, (None, np.zeros((0, K), np.int64)))
        assert len(hist) == pend, (key, len(hist), pend)
        dec, V, hist = online_step(emis, trans, np.log(np.ones(K) / K)[0], V, hist, bool(flags & 1), bool(flags & 2))
        self.chains[key] = (V, hist)
        return dec

    def energy(self, rows):
        out = []
        for sid, f0, n, pend, flags in rows:
            R0, _, L = self.rows[sid]
            em = vo.pred2logemission(L[f0 - R0:f0 - R0 + n] > self.thr[sid])
            out.append(self._step(('energy', sid), em, vo.log_trans_exp(150, cost0=-5), flags, pend))
        return out

    def decode(self, name, chains, info):
        predict, nmel, outlabels, arg = self.nets[name]
        out = []
        for slot, sid, a, b, flags, pend in chains:
            R0, M, _ = self.rows[sid]
            emis = np.zeros((0, len(outlabels)))
            if b > a:
                patches, finite = so.get_patches(M[:, :nmel])
                idx = np.arange(a, b) - R0 // 2
                assert idx.min() >= 0 and idx.max() < len(patches) and (R0 == 0 or idx.min() >= 17)
                r = np.array(predict(patches[idx][..., None].astype(np.float32)), dtype=np.float32)
                r[~finite[idx]] = 0.5
                with np.errstate(divide='ignore'):
                    emis = np.log(r).astype(np.float64)
            out.append(self._step((name, slot), emis, vo.diag_trans_exp(arg, len(outlabels)), flags, pend))
        return out

    def offline(self, sid, F):
        R0, M, L = self.rows[sid]
        assert R0 == 0 and len(L) == F
        return segment_reference(M, L, None, self.ratio, self.nets)


def segment_reference(mspec, loge, n_cal, ratio, nets):
    """oracle.segmenter_oracle.segment_feats on (mspec, loge), short recordings padded as media2feats pads them, with
    the energy threshold of the first n_cal loge values (n_cal None: all of them, the reference's threshold)."""
    difflen = 0
    if len(loge) < so.PATCH_W:
        difflen = so.PATCH_W - len(loge)
        mspec = np.concatenate((mspec, np.ones((difflen, 24)) * np.min(mspec)))
    g = loge if n_cal is None else loge[:n_cal]
    thr = np.mean(g[np.isfinite(g)]) + np.log(ratio)
    track = vo.viterbi_decoding(vo.pred2logemission(loge > thr), vo.log_trans_exp(150, cost0=-5))[::2]
    lseg = [('noEnergy' if lab == 0 else 'energy', a, b) for lab, a, b in so.binidx2seglist(track)]
    for name in ('vad', 'gender'):
        if name in nets:
            predict, nmel, outlabels, arg = nets[name]
            inlabel = 'energy' if name == 'vad' else 'speech'
            lseg = so.DnnSegmenterOracle(predict, nmel, arg, inlabel, outlabels)(mspec, lseg, difflen)
    return [(lab, 0 + a * .02, 0 + b * .02) for lab, a, b in lseg]
