"""Packing plan of Segmenter.segment_signals (inaspeechsegmenter_b200/pack.py): offsets, tiling, patch rows and pass
splitting, checked against the single-recording arithmetic on the host."""
import numpy as np
import pytest

from inaspeechsegmenter_b200 import pack

# sample counts around the frame and patch boundaries: 400 / 560 / 720 samples are 1 / 2 / 3 frames, 0.5 s is 48 frames
# (< 68: padded), then odd and even L and a multi-tile recording
LENGTHS = [400, 559, 560, 719, 720, 8000, 16000, 16160, 32000, 160000, 48 * 160 + 240, 47 * 160 + 240]


def single_patch_row0(L, p):
    """patch_index_kernel of iss_cnn_forward on one recording (both edges replicated)."""
    U = (L - 68) // 2 + 1
    j = p - 17
    j = max(j, 0)
    j = min(j, U - 1)
    return 2 * j


def test_offsets():
    lay = pack.PassLayout(LENGTHS, itemsize=2)
    frames = [pack.num_frames(n) for n in LENGTHS]
    assert frames[:5] == [1, 1, 2, 2, 3]
    assert list(lay.frames) == frames
    rows = [max(L, 68) for L in frames]
    assert list(lay.rows) == rows
    assert list(lay.row_off) == list(np.cumsum([0] + rows[:-1]))
    assert list(lay.loge_off) == list(np.cumsum([0] + frames))
    assert list(lay.out_off) == list(np.cumsum([0] + [(L + 1) // 2 for L in frames]))
    assert lay.total_rows == sum(rows)
    assert list(lay.difflen) == [r - L for r, L in zip(rows, frames)]


@pytest.mark.parametrize('itemsize', [2, 4])
def test_staging_is_aligned_and_disjoint(itemsize):
    lay = pack.PassLayout(LENGTHS, itemsize=itemsize)
    for i, n in enumerate(LENGTHS):
        assert (lay.stage_off[i] * itemsize) % 16 == 0
        assert lay.stage_off[i] + n <= lay.stage_off[i + 1]


def test_tiles_cover_each_recording_from_its_first_frame():
    lay = pack.PassLayout(LENGTHS)
    for i, L in enumerate(lay.frames):
        tiles = range(lay.tile_off[i], lay.tile_off[i + 1])
        covered = []
        for t in tiles:
            f0 = (t - lay.tile_off[i]) * pack.FEAT_TILE            # sidekit_features_kernel: tile's first frame
            covered += list(range(f0, min(f0 + pack.FEAT_TILE, L)))
            assert f0 < L
        assert covered == list(range(L))
    # the kernel's binary search maps every global tile to its recording
    for t in range(int(lay.tile_off[-1])):
        i = int(np.searchsorted(lay.tile_off, t, side='right')) - 1
        while lay.tile_off[i + 1] == lay.tile_off[i]:
            i += 1
        assert lay.tile_off[i] <= t < lay.tile_off[i + 1]


def test_patch_rows_match_the_single_recording():
    lay = pack.PassLayout(LENGTHS)
    for i, L in enumerate(lay.rows):
        L = int(L)
        P = pack.num_patches(L)
        assert P == 17 + (L - 68) // 2 + 1 + 16 + L % 2
        # the energy track has ceil(frames / 2) entries, and ranges stop there: never past the padded patches
        assert (int(lay.frames[i]) + 1) // 2 <= P
        for p in range(P):
            r0 = pack.patch_row0(L, p)
            assert r0 == single_patch_row0(L, p)
            absolute = lay.row_off[i] + r0
            # no patch reads rows of another recording
            assert lay.row_off[i] <= absolute and absolute + 68 <= lay.row_off[i] + lay.rows[i]
        # left replicas repeat window 0, the 16 + L % 2 right ones window U - 1
        U = (L - 68) // 2 + 1
        assert [pack.patch_row0(L, p) for p in range(17)] == [0] * 17
        assert [pack.patch_row0(L, p) for p in range(17 + U - 1, P)] == [2 * (U - 1)] * (17 + L % 2)


def test_pass_splitting_respects_budget_and_order():
    rng = np.random.default_rng(3)
    n = list(rng.integers(400, 16000 * 60, size=300))
    kinds = ['int16'] * 300
    budget = 1 << 17
    passes, long_ = pack.plan_passes(n, kinds, budget)
    assert long_ == []
    assert [i for p in passes for i in p] == list(range(300))
    for p in passes:
        assert sum(pack.num_frames(n[i]) for i in p) <= budget
    # greedy: the first recording of the next pass would not have fitted
    for p, q in zip(passes, passes[1:]):
        assert sum(pack.num_frames(n[i]) for i in p) + pack.num_frames(n[q[0]]) > budget


def test_mixed_formats_get_their_own_passes():
    n = [16000] * 6
    kinds = ['int16', 'float32', 'int16', 'float32', 'float32', 'int16']
    passes, long_ = pack.plan_passes(n, kinds)
    assert passes == [[0, 2, 5], [1, 3, 4]]
    assert long_ == []


def test_long_recordings_are_routed_to_the_single_path():
    edge = (pack.LONG_FRAMES - 1) * 160 + 400                        # exactly 65536 frames
    n = [16000, edge, edge - 160, 32000, edge + 10 ** 6]
    passes, long_ = pack.plan_passes(n, ['int16'] * 5)
    assert pack.num_frames(edge) == 65536
    assert long_ == [1, 4]
    assert passes == [[0, 2, 3]]


def test_default_budget_fits_every_routed_recording():
    assert pack.PASS_FRAMES >= pack.LONG_FRAMES


def test_short_recording_error_names_its_index():
    with pytest.raises(ValueError, match=r'<signal 2> holds 399 samples'):
        pack.check_lengths([400, 16000, 399, 10])
    pack.check_lengths([400])
