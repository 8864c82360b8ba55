"""The two feature front ends against their float64 reference (oracle/frontend_ref.py) -- on the GPU.

K1 (feat_sidekit.cu) runs in both FFT precisions and K4 (feat_vbx.cu) with and without dither, each fixture from int16
and from float32 PCM.  Every output must lie within C_BOUND times the bound frontend_ref carries for the kernel's
recipe; K4's float32 outputs must be faithfully rounded from a value within C_BOUND times the float64 term.  One
SidekitFrontEnd.multi and one VbxFrontEnd.multi call then pack all fixtures and are held to the same bounds.

The fixtures are what a fixed tolerance cannot take: tones on and between bins, below the first filter and near
Nyquist, at full scale and at a few LSB (their quiet bands are rounding noise), DC, impulses at frame edges and tile
seams, full-scale squares and clipping, digital silence across tile seams, a chirp, the lengths around one frame and one
48-frame tile, and for K4 the lengths where the mirror pads cover most of the recording and the frame counts around the
16-frame tile, the 128-frame CMVN chunk and the 300-frame CMVN window.  Float input below about 1e-20 is outside the
reference's domain (it decodes through pcm_s16le, and its float32 squares underflow there): it is checked against the
float64 values only.

With ISS_B200_REPORT_DIR set, the module writes frontend_report.json there: the worst ratio per kernel, precision and
fixture."""
import json
import os

import numpy as np
import pytest

from conftest import synth_audio

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')

from oracle import frontend_ref as fr          # noqa: E402

REPORT = {}
C_BOUND = 2.0
FS = 16000
FULL = 32767


# ------------------------------------------------------------------ fixtures (seeded, built here)
def _tone(f, amp, n=8000, phase=0.3):
    t = np.arange(n) / FS
    return np.clip(np.round(amp * np.sin(2 * np.pi * f * t + phase)), -32768, 32767).astype(np.int16)


def _impulses(positions, n=16000):
    x = np.zeros(n, dtype=np.int16)
    for i, p in enumerate(positions):
        x[p] = FULL if i % 2 == 0 else -FULL
    return x


def k1_fixtures():
    """name -> int16 PCM; each also runs as float32 (samples / 32768)."""
    rng = np.random.default_rng(20261016)
    fx = {}
    for f, tag in ((1000.0, 'bin'), (1015.625, 'between'), (60.0, 'low'), (7968.75, 'nyquist')):
        fx['tone_%s_full' % tag] = _tone(f, FULL)
        fx['tone_%s_3lsb' % tag] = _tone(f, 3.0)
        fx['tone_%s_1lsb' % tag] = _tone(f, 1.0)
    fx['dc_half'] = np.full(4000, 16384, dtype=np.int16)
    fx['dc_min'] = np.full(4000, -32768, dtype=np.int16)
    fx['impulse_first'] = _impulses([160 * k for k in (5, 11, 30, 47, 71)])            # a frame's first sample
    fx['impulse_last'] = _impulses([160 * k + 399 for k in (3, 12, 33, 60, 85)])       # a frame's last sample
    fx['impulse_seam'] = _impulses([7680, 15360], n=16400)                             # 48-frame tile seams
    fx['square_nyquist'] = np.tile(np.array([FULL, -32768], dtype=np.int16), 4000)
    fx['noise_clipped'] = np.clip(np.round(rng.standard_normal(16000) * 30000), -32768, 32767).astype(np.int16)
    fx['noise_1lsb'] = rng.integers(-1, 2, size=16000).astype(np.int16)
    s = synth_audio(2, seed=7)
    for a, b in ((7000, 8700), (15000, 16400), (22500, 23300)):                       # across the seams 7680, 15360, 23040
        s[a:b] = 0
    fx['silence_runs'] = s
    t = np.arange(2 * FS) / FS
    fx['chirp'] = np.round(20000 * np.sin(2 * np.pi * (8000 / 4) * t ** 2)).astype(np.int16)      # 0 -> 8 kHz in 2 s
    base = synth_audio(1, seed=9)
    for n in (400, 401, 559, 560, 7919, 7920, 7921):
        fx['len%d' % n] = base[:n].copy()
    return fx


def k1_float_fixtures():
    """name -> float32 PCM with no int16 counterpart: amplitudes below the reference's float32 range (float64 only)."""
    rng = np.random.default_rng(5)
    g = rng.standard_normal(8000)
    return {'tiny_1e-20': (g * 1e-20).astype(np.float32), 'tiny_1e-25': (g * 1e-25).astype(np.float32)}


def _n_for(M, k=0):
    """A sample count with M VBx frames: n + 320 - 400 = 160 (M - 1) + r, 0 <= r < 160 (and n >= 200 for the pads)."""
    return 160 * (M - 1) + 80 + (37 * k) % 160 if M > 1 else 200 + (37 * k) % 40


def k4_fixtures():
    """name -> (signal float64, int16 PCM or None, dither)."""
    rng = np.random.default_rng(31)
    fx = {}

    def add(name, s16, dither=True):
        fx[name] = (s16.astype(np.float64) / 32768, s16, dither)

    speech = synth_audio(6, seed=11)
    add('speech', speech[:3 * FS])
    add('speech_nodither', speech[:3 * FS], dither=False)
    add('silence_nodither', np.zeros(FS, dtype=np.int16), dither=False)
    add('silence', np.zeros(FS, dtype=np.int16))
    add('tone_full', _tone(1000.0, FULL, n=FS))
    add('tone_full_nodither', _tone(1015.625, FULL, n=FS), dither=False)
    add('tone_3lsb_nodither', _tone(440.0, 3.0, n=FS), dither=False)
    add('square_full', np.tile(np.array([FULL, -32768], dtype=np.int16), FS // 2), dither=False)
    add('noise_clipped', np.clip(np.round(rng.standard_normal(FS) * 30000), -32768, 32767).astype(np.int16))
    for n in (200, 201, 359, 360, 361):
        add('n%d' % n, speech[FS:FS + n].copy())
    for k, M in enumerate((1, 2, 15, 16, 17, 127, 128, 129, 299, 300, 301, 450, 451)):
        add('M%d' % M, speech[:_n_for(M, k)].copy())
    # float input only: above full scale, and fractions of an LSB of both signs (trunc toward zero, not round)
    loud = (speech[:FS].astype(np.float64) / 32768 * 1.7).astype(np.float32)
    fx['float_above_1'] = (loud.astype(np.float64), None, True)
    frac = ((rng.integers(-40, 41, size=FS) + rng.choice([-0.75, -0.5, -0.25, 0.25, 0.5, 0.75], size=FS)) / 32768)
    frac = frac.astype(np.float32)
    fx['float_fractions'] = (frac.astype(np.float64), None, False)
    fx['float_fractions_dither'] = (frac.astype(np.float64), None, True)
    return fx


K1_FIX = k1_fixtures()
K1_FLOAT = k1_float_fixtures()
K4_FIX = k4_fixtures()


# ------------------------------------------------------------------ harness
@pytest.fixture(scope='module')
def rt():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from inaspeechsegmenter_b200 import _lib, engine
    from inaspeechsegmenter_b200.sidekit_mfcc import SidekitFrontEnd
    from inaspeechsegmenter_b200.vbx_segmenter import VbxFrontEnd
    ctx = engine.Context(0)
    return dict(ctx=ctx, k1=SidekitFrontEnd(ctx), k4=VbxFrontEnd(ctx), lib=_lib)


@pytest.fixture(scope='module', autouse=True)
def _dump_report():
    yield
    out = os.environ.get('ISS_B200_REPORT_DIR')
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, 'frontend_report.json'), 'w') as f:
            json.dump(REPORT, f, indent=1, sort_keys=True)


def _note(kernel, variant, name, worst):
    e = REPORT.setdefault(kernel, {}).setdefault(variant, {})
    e[name] = max(float(worst), e.get(name, 0.0))


def _pcm(fmt, s16=None, f32=None):
    a = s16 if fmt == 's16' else (f32 if f32 is not None else s16.astype(np.float32) / np.float32(32768))
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _f32(s16):
    return s16.astype(np.float32) / np.float32(32768)


def _check_k1(ref, mspec, loge, stats, prec, tag):
    """mspec, loge within C_BOUND of the bound of the recipe; stats = (sum, count) of the finite loge."""
    Em, El = ref.bound(prec)
    assert mspec.shape == ref.mspec.shape and loge.shape == ref.loge.shape, tag
    rm, rl = fr.ratio(mspec, ref.mspec, Em), fr.ratio(loge, ref.loge, El)
    worst = max(float(rm.max()) if rm.size else 0.0, float(rl.max()) if rl.size else 0.0)
    assert worst <= C_BOUND, (tag, np.unravel_index(np.argmax(rm), rm.shape) if rm.size else None,
                              float(rm.max()) if rm.size else 0.0, float(rl.max()) if rl.size else 0.0)
    fin = np.isfinite(loge)
    assert stats[1] == fin.sum(), tag
    s = loge[fin].astype(np.float64)
    assert abs(stats[0] - s.sum()) <= 1e-12 * np.abs(s).sum(), tag
    return worst


def _k1(rt, pcm, prec):
    lib = rt['lib']
    mspec, loge, stats = rt['k1'](pcm, lib.FFT_FP64 if prec == 'fp64' else lib.FFT_FP32)
    torch.cuda.synchronize()
    return mspec.cpu().numpy(), loge.cpu().numpy(), stats.cpu().numpy()


# ------------------------------------------------------------------ K1
@pytest.mark.parametrize('prec', ['fp64', 'fp32'])
@pytest.mark.parametrize('name', sorted(K1_FIX))
def test_k1_fixture_within_bound(rt, name, prec):
    s16 = K1_FIX[name]
    ref = fr.K1Ref(_f32(s16))
    for fmt in ('s16', 'f32'):
        got = _k1(rt, _pcm(fmt, s16), prec)
        _note('k1', '%s_%s' % (prec, fmt), name, _check_k1(ref, *got, prec, (name, prec, fmt)))


@pytest.mark.parametrize('prec', ['fp64', 'fp32'])
@pytest.mark.parametrize('name', sorted(K1_FLOAT))
def test_k1_tiny_float_input_within_float64_bound(rt, name, prec):
    """Below the reference's float32 range: the kernel against float64 only (not reference parity)."""
    x = K1_FLOAT[name]
    ref = fr.K1Ref(x)
    got = _k1(rt, _pcm('f32', f32=x), prec)
    _note('k1', '%s_f32' % prec, name, _check_k1(ref, *got, prec, (name, prec)))


@pytest.mark.parametrize('prec', ['fp64', 'fp32'])
def test_k1_two_byte_aligned_views(rt, prec):
    """The scalar staging path: int16 views 2 bytes past a 16-byte boundary, at the lengths around one frame and one
    48-frame tile."""
    s16 = synth_audio(1, seed=9)
    base = torch.from_numpy(np.concatenate((np.zeros(1, np.int16), s16))).cuda()
    for n in (400, 401, 559, 560, 7919, 7920, 7921):
        ref = fr.K1Ref(_f32(s16[:n]))
        got = _k1(rt, base[1:1 + n], prec)
        _note('k1', '%s_s16_view' % prec, 'len%d' % n, _check_k1(ref, *got, prec, (n, prec)))


@pytest.mark.parametrize('prec', ['fp64', 'fp32'])
@pytest.mark.parametrize('fmt', ['s16', 'f32'])
def test_k1_multi_packs_all_fixtures_within_bound(rt, prec, fmt):
    from inaspeechsegmenter_b200 import pack
    names = sorted(K1_FIX)
    sigs = [K1_FIX[k] for k in names]
    pcms = [_pcm(fmt, s) for s in sigs]
    layout = pack.PassLayout([len(s) for s in sigs], itemsize=2 if fmt == 's16' else 4)
    lib = rt['lib']
    mspec, loge, stats = rt['k1'].multi(pcms, layout, lib.FFT_FP64 if prec == 'fp64' else lib.FFT_FP32)
    torch.cuda.synchronize()
    mspec, loge, stats = mspec.cpu().numpy(), loge.cpu().numpy(), stats.cpu().numpy()
    worst = 0.0
    for i, (name, s) in enumerate(zip(names, sigs)):
        L = int(layout.frames[i])
        r0, l0 = int(layout.row_off[i]), int(layout.loge_off[i])
        worst = max(worst, _check_k1(fr.K1Ref(_f32(s)), mspec[r0:r0 + L], loge[l0:l0 + L], stats[i], prec, (name, 'multi')))
    _note('k1', '%s_%s' % (prec, fmt), 'multi', worst)


# ------------------------------------------------------------------ K4
def _check_k4(ref, got, tag):
    assert got.shape == ref.fea.shape, (tag, got.shape, ref.fea.shape)
    ok, r = ref.check(got, C_BOUND)
    bad = np.argwhere(~ok)
    assert ok.all(), (tag, len(bad), bad[:4].tolist(), [(float(got[i, j]), float(ref.fea[i, j])) for i, j in bad[:4]])
    return float(r.max()) if r.size else 0.0


@pytest.mark.parametrize('name', sorted(K4_FIX))
def test_k4_fixture_faithfully_rounded(rt, name):
    sig, s16, dither = K4_FIX[name]
    ref = fr.K4Ref(sig, dither)
    fmts = ('s16', 'f32') if s16 is not None else ('f32',)
    for fmt in fmts:
        pcm = _pcm(fmt, s16, None if s16 is not None else sig.astype(np.float32))
        got = rt['k4'](pcm, dither=dither)
        torch.cuda.synchronize()
        _note('k4', fmt, name, _check_k4(ref, got.cpu().numpy(), (name, fmt)))


@pytest.mark.parametrize('dither', [True, False])
@pytest.mark.parametrize('fmt', ['s16', 'f32'])
def test_k4_multi_packs_all_fixtures(rt, fmt, dither):
    names = [k for k in sorted(K4_FIX) if K4_FIX[k][1] is not None or fmt == 'f32']
    sigs = [K4_FIX[k][0] for k in names]
    pcms = [_pcm(fmt, K4_FIX[k][1], None if K4_FIX[k][1] is not None else K4_FIX[k][0].astype(np.float32)) for k in names]
    fea, off = rt['k4'].multi(pcms, dither=dither)
    torch.cuda.synchronize()
    fea = fea.cpu().numpy()
    worst = 0.0
    for i, (name, sig) in enumerate(zip(names, sigs)):
        worst = max(worst, _check_k4(fr.K4Ref(sig, dither), fea[off[i]:off[i + 1]], (name, fmt, dither, 'multi')))
    _note('k4', fmt, 'multi_%s' % ('dither' if dither else 'nodither'), worst)
