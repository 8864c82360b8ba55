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
