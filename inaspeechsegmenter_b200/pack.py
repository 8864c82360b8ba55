"""Packing plan of ``Segmenter.segment_signals``: which recordings share a device pass and where each one's samples,
log-mel rows, loge entries and energy track live in the pass's packed buffers.  Pure host arithmetic (no device, no
library), so it can be checked on its own."""
import numpy as np

WIN, HOP = 400, 160                # analysis frame and hop in samples (sidekit_mfcc.py:254)
PATCH_W = 68                       # frames per CNN patch (segmenter.py:149)
PATCH_LFILL = 17                   # left replicas of the first patch (segmenter.py:83)
FEAT_TILE = 48                     # frames per CTA tile of the K1 kernel (feat_sidekit.cu FR)
LONG_FRAMES = 4 * 16384            # recordings this long are decoded chunk-parallel by the single-recording path
STAGE_ALIGN = 16                   # bytes: each staged recording starts 16-byte aligned (vector loads in K1)

# Frames of audio per device pass (2^18 frames = 43.7 min of 16 kHz audio).  It must hold the longest packed recording
# (LONG_FRAMES).  On an H100 80GB HBM3 at a 400 W limit (tools/pack_times.py, 1 h of 2 s clips from host memory), budgets
# from 2^16 to 2^22 frames showed no trend (2.34-2.95 audio-hours/s over two rounds); 2^18 keeps a pass's log-mel buffer
# at 25 MB while needing 14 passes per audio-hour.
PASS_FRAMES = 1 << 18


def num_frames(n_samples):
    """Frames of a recording of n_samples samples (iss_sidekit_num_frames)."""
    return (n_samples - WIN) // HOP + 1 if n_samples >= WIN else 0


def check_lengths(n_samples):
    """ValueError naming the first recording shorter than one analysis frame, as segment_signal raises it."""
    for i, n in enumerate(n_samples):
        if n < WIN:
            raise ValueError('media <signal %d> holds %d samples: less than one 25 ms analysis frame' % (i, n))


def plan_passes(n_samples, kinds, budget=None):
    """Split recordings into device passes.  Recordings of LONG_FRAMES frames or more go to the single-recording path
    (returned as `long`).  The others are grouped per kind (PCM format), in input order, greedily: a pass is closed when
    the next recording would take it past `budget` frames.  Returns (passes, long), passes a list of index lists."""
    budget = PASS_FRAMES if budget is None else budget
    long_, passes, open_ = [], [], {}
    for i, (n, kind) in enumerate(zip(n_samples, kinds)):
        L = num_frames(n)
        if L >= LONG_FRAMES:
            long_.append(i)
            continue
        cur = open_.get(kind)
        if cur is not None and cur[1] + L > budget:
            cur = None
        if cur is None:
            cur = open_[kind] = [[], 0]
            passes.append(cur[0])
        cur[0].append(i)
        cur[1] += L
    return passes, long_


class PassLayout:
    """Offsets of the recordings of one pass in its packed buffers (int64 numpy arrays, one entry per recording plus the
    total where a table has one):
      frames    L_i;  rows  max(L_i, 68) mspec rows reserved (short recordings are padded with min(mspec) rows)
      row_off   first mspec row;  loge_off  first loge entry (n + 1);  out_off  first entry of the [::2] energy track (n + 1)
      tile_off  first K1 tile (n + 1);  stage_off  first element in the staging buffer of `itemsize`-byte samples
    """

    def __init__(self, n_samples, itemsize=2):
        n_samples = np.asarray(n_samples, dtype=np.int64)
        self.n_samples = n_samples
        self.frames = np.array([num_frames(int(n)) for n in n_samples], dtype=np.int64)
        self.rows = np.maximum(self.frames, PATCH_W)
        self.row_off = _starts(self.rows)
        self.loge_off = _starts(self.frames, total=True)
        self.out_off = _starts((self.frames + 1) // 2, total=True)
        self.tile_off = _starts((self.frames + FEAT_TILE - 1) // FEAT_TILE, total=True)
        step = STAGE_ALIGN // itemsize
        self.stage_off = _starts((n_samples + step - 1) // step * step, total=True)
        self.total_rows = int(self.rows.sum())
        self.difflen = self.rows - self.frames


def _starts(sizes, total=False):
    off = np.concatenate(([0], np.cumsum(sizes, dtype=np.int64))).astype(np.int64)
    return off if total else off[:-1]


def patch_row0(L, p):
    """First frame of padded patch p of a recording of L >= 68 frames (patch_index_kernel with both edges replicated):
    the 17 left replicas repeat window 0, the 16 + L % 2 right ones window U - 1."""
    U = (L - PATCH_W) // 2 + 1
    return 2 * min(max(p - PATCH_LFILL, 0), U - 1)


def num_patches(L):
    """Padded patches of a recording of L >= 68 frames: 17 + U + 16 + L % 2."""
    return PATCH_LFILL + (L - PATCH_W) // 2 + 1 + PATCH_LFILL - 1 + L % 2


# ---- VBx x-vector windows of VoiceFemininityScoring.score_signals ---------------------------------------------------
VBX_PADL, VBX_PADR = 120, 200      # mirror padding of get_features (feat_vbx.cu VPADL / VPADR)
VBX_STEP, VBX_WINLEN = 24, 144     # x-vector window hop and length in frames (vbx_segmenter.STEP / WINLEN)
VBX_MIN_TAIL = 10                  # a shorter remainder gets no tail window


def vbx_num_frames(n_samples):
    """VBx feature frames of a recording of n_samples samples (iss_vbx_num_frames): 0 below 200 samples."""
    return (n_samples + VBX_PADL + VBX_PADR - WIN) // HOP + 1 if n_samples >= VBX_PADR else 0


def window_plan(M):
    """(start, length, is_tail) for every window of VBxExtractor.__call__ on M feature frames (vbx_segmenter.py:222-243):
    regular windows every 24 frames while one more fits strictly inside, then a tail from the next hop to the end if it
    holds at least 10 frames."""
    plan, start = [], 0
    for start in range(0, M - VBX_WINLEN, VBX_STEP):
        plan.append((start, VBX_WINLEN, False))
    if M - start - VBX_STEP >= VBX_MIN_TAIL:
        plan.append((start + VBX_STEP, M - (start + VBX_STEP), True))
    return plan


class VbxPlan:
    """Where the VBx features and x-vector windows of a list of recordings live when their features are packed in one
    [fea_off[-1], 64] buffer (int64 numpy arrays):
      frames    M_i;  fea_off  first feature row of recording i (n + 1)
      reg_start packed first row of every regular 144-frame window, recordings in order and each one's windows in order;
      reg_rec   its recording;  reg_off  first regular window of recording i (n + 1)
      tails     {length: (recordings, packed starts)}: the tail windows grouped by length, in recording order;
      tail_pos  position of recording i's tail in its length group, -1 if it has none
    """

    def __init__(self, n_samples):
        self.frames = np.array([vbx_num_frames(int(n)) for n in n_samples], dtype=np.int64)
        self.fea_off = _starts(self.frames, total=True)
        self.plans = [window_plan(int(M)) for M in self.frames]
        reg = [[s for s, _, tail in p if not tail] for p in self.plans]
        self.reg_off = _starts([len(r) for r in reg], total=True)
        self.reg_start = np.array([self.fea_off[i] + s for i, r in enumerate(reg) for s in r], dtype=np.int64)
        self.reg_rec = np.repeat(np.arange(len(reg), dtype=np.int64), [len(r) for r in reg])
        groups = {}
        self.tail_pos = np.full(len(self.plans), -1, dtype=np.int64)
        for i, p in enumerate(self.plans):
            for s, n, tail in p:
                if tail:
                    g = groups.setdefault(n, ([], []))
                    self.tail_pos[i] = len(g[0])
                    g[0].append(i)
                    g[1].append(self.fea_off[i] + s)
        self.tails = {n: (np.array(r, dtype=np.int64), np.array(s, dtype=np.int64)) for n, (r, s) in sorted(groups.items())}
