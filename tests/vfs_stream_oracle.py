"""CPU stand-in for the device side of live femininity scores (test infrastructure): ``OracleVfsBackend`` gives
``vfs_stream.LiveScores`` the VBx front end of ``oracle/vbx_oracle.py`` computed window by window from what a stream
retains, a deterministic stand-in embedding and the MLP of ``oracle/vfs_oracle.py``.  It keeps only what the host asks
it to keep and checks every window it is handed against it, so a retention or finality rule that is off by one row
fails here."""
import numpy as np

from oracle import vbx_oracle as vx
from oracle import vfs_oracle
from inaspeechsegmenter_b200 import vfs_stream as vs


def standin_embedding(fea):
    """fea [T, 64] float32 -> [256] float32: per-band mean, standard deviation, maximum and minimum."""
    fea = np.asarray(fea, dtype=np.float32)
    return np.concatenate((fea.mean(0), fea.std(0), fea.max(0), fea.min(0))).astype(np.float32)


class StandinNet:
    """vbx_oracle.extract_xvectors' `net` with the stand-in embedding."""

    def get_embedding(self, fea):
        return standin_embedding(fea)


def raw_rows(x, s_base, n, r_first, rows):
    """Raw fbank rows r_first .. r_first + rows - 1 of a stream of n samples from its samples [s_base, n) (quantised
    and dithered): the arithmetic of vbx_oracle.raw_fbank on frames gathered through the mirror padding."""
    p = (np.arange(r_first, r_first + rows) * 160)[:, None] + np.arange(vx.FRAME)[None, :]
    src = np.where(p < 120, 119 - p, np.where(p < 120 + n, p - 120, 2 * n + 119 - p))
    assert src.min() >= s_base and src.max() < n, (src.min(), s_base, src.max(), n)
    fr = x[src - s_base].copy()
    fr -= fr.mean(axis=1)[:, np.newaxis]
    fr = fr - np.c_[fr[..., :1], fr[..., :-1]] * 0.97
    fr *= vx.povey_window()
    sp = np.fft.rfft(fr, vx.NFFT)
    return np.log(np.maximum(1.0, np.dot(sp.real ** 2 + sp.imag ** 2, vx.mel_bank())))


def cmvn_rows(raw, r_base, M, t_first, rows):
    """CMVN rows t_first .. + rows - 1 from raw rows [r_base, ...) with window length min(M, 300), as the kernel computes
    them: each 128-row chunk of the whole-recording grid from its direct sum, then one add and one subtract per row."""
    wl = min(M, 300)
    ws_of = lambda t: max(min(t - 150, M - wl), 0)      # noqa: E731
    out = np.zeros((rows, raw.shape[1]))
    t = t_first
    while t < t_first + rows:
        t0 = t // 128 * 128
        ws = ws_of(t0)
        assert ws >= r_base, (ws, r_base)
        s = np.zeros(raw.shape[1])
        for r in range(ws, ws + wl):
            s = s + raw[r - r_base]
        for u in range(t0, min(t0 + 128, t_first + rows)):
            nws = ws_of(u)
            if nws != ws:
                s = s + (raw[nws + wl - 1 - r_base] - raw[ws - r_base])
                ws = nws
            if u >= t_first:
                out[u - t_first] = raw[u - r_base] - s / wl
        t = min(t0 + 128, t_first + rows)
    return out


def whole_features(sig):
    """The features the window-by-window computation must reproduce: the kernel's CMVN arithmetic on the whole
    recording's raw rows, float32."""
    raw = vx.raw_fbank(sig)
    return cmvn_rows(raw, 0, len(raw), 0, len(raw)).astype(np.float32)


class OracleVfsBackend:
    """The vfs_stream.CudaBackend interface on the CPU."""

    def __init__(self, mlp):
        self.mlp = mlp                               # (config, weights) of the Keras MLP
        self.rng, self.x, self.raw, self.fea = {}, {}, {}, {}     # sid -> RandomState / (first index, rows)
        self.computed = {}                           # sid -> every feature row computed, in order (kept after release)

    def open(self, sid):
        self.rng[sid] = np.random.RandomState(3)
        self.x[sid] = (0, np.zeros(0))
        self.raw[sid] = (0, np.zeros((0, 64)))
        self.fea[sid] = (0, np.zeros((0, 64), np.float32))
        self.computed[sid] = []

    def release(self, sid):
        for d in (self.rng, self.x, self.raw, self.fea):
            d.pop(sid, None)

    def features(self, rows, keep):
        for sid, (c, n, (r0, nr), (t0, nt), end, (s_keep, _, _)) in rows.items():
            base, x = self.x[sid]
            if c is not None and len(c):
                c = np.asarray(c)
                q = c.astype(np.float64) if c.dtype == np.int16 else np.trunc(c.astype(np.float64) * 32768)
                x = np.concatenate((x, q + 8 * (self.rng[sid].rand(len(c)) * 2 - 1)))
            assert base + len(x) == n
            a0, raw = self.raw[sid]
            if nr:
                assert a0 + len(raw) == r0
                raw = np.concatenate((raw, raw_rows(x, base, n, r0, nr)))
            self.raw[sid] = (a0, raw)
            f0, fea = self.fea[sid]
            if nt:
                assert f0 + len(fea) == t0
                new = cmvn_rows(raw, a0, a0 + len(raw), t0, nt).astype(np.float32)
                self.computed[sid].append(new)
                fea = np.concatenate((fea, new))
            self.fea[sid] = (f0, fea)
            self.x[sid] = (s_keep, x[s_keep - base:])
        for sid, (_, r_keep, t_keep) in keep.items():
            a0, raw = self.raw[sid]
            k = max(r_keep, a0)
            self.raw[sid] = (k, raw[k - a0:])
            f0, fea = self.fea[sid]
            k = max(t_keep, f0)
            self.fea[sid] = (k, fea[k - f0:])

    def embed(self, wins):
        emb = []
        for sid, start, n in wins:
            f0, fea = self.fea[sid]
            assert f0 <= start and start + n <= f0 + len(fea), (f0, start, n, len(fea))
            emb.append(standin_embedding(fea[start - f0:start + n - f0]))
        emb = np.asarray(emb, dtype=np.float32)
        return vfs_oracle.mlp_numpy(*self.mlp, emb * 10), np.isnan(emb).any(1)
