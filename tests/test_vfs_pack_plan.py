"""VBx window plan of VoiceFemininityScoring.score_signals (inaspeechsegmenter_b200/pack.py VbxPlan): frame counts,
packed window starts and tail groups, checked against each recording's own window_plan on the host."""
import numpy as np
import pytest

from inaspeechsegmenter_b200 import pack


def samples_for(M, extra=0):
    """Sample counts with exactly M VBx frames: 80 + 160 (M - 1) .. + 159."""
    return 80 + 160 * (M - 1) + extra


# 200 / 201 / 399 / 400 samples; M = 33, 34, 35 (no regular window, tail of 9 / 10 / 11 frames from frame 24);
# M = 143 .. 170 (first regular window and the tails around it); 300 / 301 frames (the CMVN window); K4 tiles (16 frames)
# and CMVN chunks (128 frames) at and around their boundaries; under 200 samples (no frames); 2 s, 5 s and 10 s
M_CASES = [33, 34, 35] + list(range(143, 171)) + [300, 301, 15, 16, 17, 31, 32, 127, 128, 129, 255, 256, 257]
LENGTHS = [200, 201, 399, 400, 0, 199, 32000, 80000, 160000] + [samples_for(M) for M in M_CASES] + \
    [samples_for(M, 159) for M in (34, 144, 300)]


def ref_num_frames(n):
    """iss_vbx_num_frames (feat_vbx.cu): mirror padding 120 / 200, frames 400 / 160, none under 200 samples."""
    return 0 if n < 200 else (n + 320 - 400) // 160 + 1


def test_frame_counts():
    plan = pack.VbxPlan(LENGTHS)
    assert [int(M) for M in plan.frames] == [ref_num_frames(n) for n in LENGTHS]
    assert [pack.vbx_num_frames(n) for n in (199, 200, 201, 399, 400)] == [0, 1, 1, 2, 3]
    for M in M_CASES:
        assert pack.vbx_num_frames(samples_for(M)) == M == pack.vbx_num_frames(samples_for(M, 159))
        assert pack.vbx_num_frames(samples_for(M, 160)) == M + 1
    assert list(plan.fea_off) == list(np.cumsum([0] + [ref_num_frames(n) for n in LENGTHS]))


def test_frame_counts_match_the_library():
    lib = pytest.importorskip('inaspeechsegmenter_b200._lib').load()
    for n in LENGTHS + [1, 2 ** 20 + 7]:
        assert lib.iss_vbx_num_frames(n) == pack.vbx_num_frames(n), n


def test_window_plan_is_the_extractors():
    from oracle import vbx_oracle as vx
    for M in sorted(set(M_CASES + [0, 5, 9, 10, 200, 1464])):
        assert pack.window_plan(M) == vx.window_plan(M), M
    vb = pytest.importorskip('inaspeechsegmenter_b200.vbx_segmenter')
    assert vb.window_plan is pack.window_plan
    assert (vb.STEP, vb.WINLEN) == (pack.VBX_STEP, pack.VBX_WINLEN)


def test_regular_windows_are_each_recordings_own_shifted():
    plan = pack.VbxPlan(LENGTHS)
    for i, M in enumerate(plan.frames):
        own = [s for s, n, tail in pack.window_plan(int(M)) if not tail]
        a, b = plan.reg_off[i], plan.reg_off[i + 1]
        assert list(plan.reg_start[a:b] - plan.fea_off[i]) == own
        assert list(plan.reg_rec[a:b]) == [i] * len(own)
        # every regular window lies inside its recording's rows
        assert all(plan.fea_off[i] <= s and s + pack.VBX_WINLEN <= plan.fea_off[i + 1] for s in plan.reg_start[a:b])
    assert plan.reg_off[-1] == len(plan.reg_start) == len(plan.reg_rec)


def test_tail_groups_cover_each_tail_once():
    plan = pack.VbxPlan(LENGTHS)
    want = {}
    for i, M in enumerate(plan.frames):
        for s, n, tail in pack.window_plan(int(M)):
            if tail:
                want[i] = (n, int(plan.fea_off[i] + s))
    got = {}
    for n, (recs, starts) in plan.tails.items():
        assert len(recs) == len(starts) > 0
        assert list(recs) == sorted(recs)
        for pos, (i, s) in enumerate(zip(recs, starts)):
            assert int(i) not in got
            got[int(i)] = (n, int(s))
            assert plan.tail_pos[i] == pos
            assert plan.fea_off[i] <= s and s + n == plan.fea_off[i + 1]          # a tail ends at its recording's end
    assert got == want
    assert [i for i in range(len(LENGTHS)) if plan.tail_pos[i] < 0] == [i for i in range(len(LENGTHS)) if i not in want]
    assert list(plan.tails) == sorted(plan.tails)
    # the boundary lengths give tails from 10 frames up: M = 33 has none, 34 / 35 have 10 / 11 frames from frame 24
    assert pack.window_plan(33) == [] and pack.window_plan(34) == [(24, 10, True)] and pack.window_plan(35) == [(24, 11, True)]


def test_empty_and_frameless_lists():
    plan = pack.VbxPlan([])
    assert list(plan.fea_off) == [0] and len(plan.reg_start) == 0 and plan.tails == {}
    plan = pack.VbxPlan([0, 199, 100])
    assert list(plan.frames) == [0, 0, 0] and list(plan.reg_off) == [0, 0, 0, 0] and plan.tails == {}
