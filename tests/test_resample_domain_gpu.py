"""The resampler (resample.cu) over its whole domain on the device (run with -m gpu on an H100): every rate of
resample_fixtures.RATES with 1 to 8 channels, every WAV encoding at odd frame sizes, the smallest tile's seams past
2^31 in k * down, live streams and the window check at awkward rates, all against oracle/resample_ref.py.  At an
output the oracle flags as a near tie, either integer around y * 32768 is accepted; each test prints its count."""
import warnings

import numpy as np
import pytest

from conftest import synth_audio
from oracle import resample_ref as rr
from resample_fixtures import RATES, check, frames_for, lengths, reach, reference, tile_for
from test_sample_rates_gpu import _recording
from wav_fixtures import decode, domain_fixtures, encode, signal

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')

WAV_RATES = (88200, 176400, 191999)
WAV_ENCODINGS = ('u8', 's24', 's32', 'f64')
WAV_CHANNELS = (3, 5, 7, 8)
STREAMS = [(191999, 8, 'float32'), (11025, 5, 'int16'), (15999, 1, 'float32')]


@pytest.fixture(scope='module')
def rt():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from inaspeechsegmenter_b200 import _lib, engine, io, resample, segmenter, stream
    return dict(lib=_lib, engine=engine, io=io, resample=resample, segmenter=segmenter, stream=stream,
                ctx=engine.Context(0))


def _misaligned(x):
    """A CUDA view of x one sample past a 16-byte boundary (scalar staging; one frame past would be aligned with 8
    int16 or 4 float32 channels)."""
    flat = np.ascontiguousarray(x).reshape(-1)
    d = torch.from_numpy(np.concatenate([flat[:1], flat])).cuda()[1:].view(x.shape)
    assert d.data_ptr() % 16 != 0
    return d


@pytest.mark.parametrize('rate', RATES)
@pytest.mark.parametrize('fmt', ['int16', 'float32'])
def test_in_memory_every_channel_count(rt, rate, fmt):
    """1 to 8 channels at the boundary lengths of each tile: host arrays (one call each) against the oracle, and CUDA
    tensors, misaligned views and one packed call against those calls."""
    resample, ctx = rt['resample'], rt['ctx']
    flagged = outputs = 0
    for C in range(1, 9):
        xs = [_recording(rate, n, C, fmt, seed=rate + 7 * n + C) for n in lengths(rate, C, 2 if fmt == 'int16' else 4)]
        singles = [resample.to16k(ctx, x if C > 1 else x[:, 0], rate) for x in xs]
        for x, s in zip(xs, singles):
            what = (rate, fmt, C, len(x))
            flagged += check(s.cpu().numpy(), x, rate, what + ('host',))
            outputs += len(s)
            assert torch.equal(resample.to16k(ctx, torch.from_numpy(x).cuda(), rate), s), what + ('cuda',)
            assert torch.equal(resample.to16k(ctx, _misaligned(x), rate), s), what + ('view',)
        packed = resample.resample_pass(ctx, [torch.from_numpy(x).cuda() for x in xs], [rate] * len(xs))
        for x, s, p in zip(xs, singles, packed):
            assert torch.equal(s, p), (rate, fmt, C, len(x), 'packed')
    print('%d Hz %s: %d flagged near ties in %d outputs' % (rate, fmt, flagged, outputs))


@pytest.fixture(scope='module')
def domain_wavs(tmp_path_factory):
    return domain_fixtures(str(tmp_path_factory.mktemp('domain_wavs')), WAV_ENCODINGS, WAV_CHANNELS, WAV_RATES,
                           frames=6001)


def _stored(w):
    with open(w.path, 'rb') as f:
        f.seek(w.start)
        return f.read(w.nbytes)


@pytest.mark.parametrize('rate', WAV_RATES)
def test_wav_encodings_at_odd_frame_sizes(rt, domain_wavs, rate):
    """u8, s24, s32 and f64 with 3, 5, 7 and 8 channels (frames of 3 to 64 bytes, 9-, 15- and 21-byte ones among
    them): the file route against the oracle, the stored bytes 1 to 15 bytes past a 16-byte boundary and one packed
    pass against the file route."""
    io, resample, segmenter, ctx = rt['io'], rt['resample'], rt['segmenter'], rt['ctx']
    ws = {name: io.wav_data(path) for name, (path, _, _, r) in domain_wavs.items() if r == rate}
    assert len(ws) == len(WAV_ENCODINGS) * len(WAV_CHANNELS)
    flagged, singles = 0, {}
    for name, w in ws.items():
        raw = _stored(w)
        singles[name] = segmenter._wav_to16k(ctx, w)
        flagged += check(singles[name].cpu().numpy(), decode(raw, w.encoding, w.channels), rate, (name, 'file'))
        src = torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()
        out = torch.empty(resample.num_frames(w.frames, rate), dtype=torch.int16, device='cuda')
        for shift in range(1, 16):
            buf = torch.zeros(w.nbytes + 32, dtype=torch.uint8, device='cuda')
            view = buf[16 - buf.data_ptr() % 16 + shift:][:w.nbytes]
            assert view.data_ptr() % 16 == shift
            view.copy_(src)
            out.fill_(0x5555)
            resample.to16k_multi(ctx, [view.view(w.shape)], rate, out, [0], encoding=w.encoding)
            assert torch.equal(out, singles[name]), (name, shift)
    names = sorted(ws)
    pcms = segmenter._stage_pass([ws[n] for n in names], ctx.device)
    packed = resample.resample_pass(ctx, pcms, [rate] * len(names), [ws[n].encoding for n in names])
    for n, p in zip(names, packed):
        assert torch.equal(p, singles[n]), n
    print('%d Hz WAV: %d flagged near ties over %d files' % (rate, flagged, len(ws)))


@pytest.mark.parametrize('rate', [176400, 191999, 192000])
def test_smallest_tile_seams(rt, rate):
    """8 channels of float64, the widest frame: 64 outputs per CTA, so outputs 62 .. 65 and 126 .. 129 sit on tile
    seams.  30001 outputs, every one checked; at 191999 Hz k * down passes 2^31 (k = 11185) and 2^32 (k = 22370)."""
    resample, ctx = rt['resample'], rt['ctx']
    assert tile_for(rate, 8, 8) == 64
    up, down = rr.factors(rate)
    n = frames_for(rate, 30001)
    x = signal(n, 8, rate, seed=rate)
    raw = np.frombuffer(encode(x, 'f64'), dtype=np.uint8)
    dev = torch.from_numpy(raw.copy()).cuda().view(n, 8, 8)
    out = torch.empty(resample.num_frames(n, rate), dtype=torch.int16, device='cuda')
    resample.to16k_multi(ctx, [dev], rate, out, [0], encoding='f64')
    got = out.cpu().numpy()
    assert len(got) == 30001
    if rate == 191999:
        assert (len(got) - 1) * down >= 2 ** 32
    flagged = check(got, decode(raw, 'f64', 8), rate, (rate, 'f64 8ch'))
    print('%d Hz f64 8ch: %d flagged near ties in %d outputs' % (rate, flagged, len(got)))


def _random_parts(n, rng, longest):
    out, pos = [], 0
    while pos < n:
        m = int(rng.integers(1, longest + 1))
        out.append((pos, min(pos + m, n)))
        pos += m
    return out


@pytest.mark.parametrize('rate,C,fmt', STREAMS)
def test_streams_equal_whole_recording(rt, synth_models, rate, C, fmt):
    """A live stream's 16 kHz samples, over three random chunkings (host chunks, and CUDA chunks in the third), are
    resample.to16k of the whole stream bit for bit; that equals the oracle (past 2^31 in k * down at 191999 Hz)."""
    resample, segmenter = rt['resample'], rt['segmenter']
    seg = segmenter.Segmenter(vad_engine='smn', detect_gender=True, ffmpeg=None,
                              models={'vad': synth_models['smn'], 'gender': synth_models['gender']})
    x = _recording(rate, 2 * rate + 333, C, fmt, seed=rate + C)
    x = x[:, 0] if C == 1 else x
    whole = resample.to16k(seg.ctx, x, rate)
    flagged = check(whole.cpu().numpy(), x, rate, (rate, C, fmt, 'whole'))
    rng = np.random.default_rng(rate)
    for i, longest in enumerate((rate // 50, rate // 3, 2 * rate)):
        be = rt['stream'].CudaBackend(seg)
        got = []
        for a, b in _random_parts(len(x), rng, longest):
            c = x[a:b] if i < 2 else torch.from_numpy(np.ascontiguousarray(x[a:b])).cuda()
            got.append(be.resample({0: c}, {0: rate})[0])
        got.append(be.resample({}, {0: rate}, [0])[0])
        assert torch.equal(torch.cat(got), whole), (rate, C, fmt, i)
    print('%d Hz %d channels %s: %d flagged near ties in %d outputs' % (rate, C, fmt, flagged, len(whole)))


@pytest.mark.parametrize('rate,C,fmt', STREAMS)
def test_window_boundary_matches_first_kept(rt, rate, C, fmt):
    """iss_resample_window_multi takes a window of one output k that starts at the first frame k reads,
    ceil((k down - H) / up), and refuses one that starts a frame later, over 64 consecutive k of every phase offset;
    resample.first_kept(k) is that frame where k's phase reads from s_min, and never after it."""
    lib, resample, ctx = rt['lib'], rt['resample'], rt['ctx']
    L = lib.load()
    resample._ensure_taps(ctx, rate)
    up, down = rr.factors(rate)
    H = 10 * max(up, down)
    s_min, e_max = reach(rate)
    k0 = 2 ** 31 // down - 20 if rate == 191999 else 5 * up - 3
    dt = torch.int16 if fmt == 'int16' else torch.float32
    x = torch.zeros(((e_max - s_min + 2) * C,), dtype=dt, device='cuda')
    out = torch.empty(1, dtype=torch.int16, device='cuda')
    ptrs = (lib._c.c_void_p * 1)(x.data_ptr())
    pcm = lib.PCM_S16 if fmt == 'int16' else lib.PCM_F32

    def call(f_base, k):
        n_known = k * down // up + e_max
        w = np.array([[f_base, n_known, k, 1, 0, 0]], dtype=np.int64)
        c0 = L.iss_launch_count()
        rc = L.iss_resample_window_multi(ctx.handle, 1, ptrs, lib.ptr(w), C, rate, pcm, lib.ptr(out), None)
        if rc != 0:
            assert L.iss_launch_count() == c0 and b'before the window' in L.iss_last_error(), (rate, k, f_base)
        return rc

    at_kept = 0
    for k in range(k0, k0 + 64):
        first = -((H - k * down) // up)
        kept = resample.first_kept(k, rate)
        assert 0 < kept <= first, (rate, k, kept, first)
        assert call(first, k) == 0 and call(first + 1, k) == -1, (rate, k, first)
        at_kept += kept == first
    assert at_kept > 0
    if rate == 191999:
        assert k0 * down < 2 ** 31 <= (k0 + 63) * down
    torch.cuda.synchronize()


def test_segment_signal_191999_8ch_equals_reference_pcm(rt, synth_models):
    """segment_signal of 20 s of 8-channel audio at 191999 Hz equals segment_signal of the oracle's 16 kHz int16."""
    seg = rt['segmenter'].Segmenter(vad_engine='smn', detect_gender=True, ffmpeg=None,
                                    models={'vad': synth_models['smn'], 'gender': synth_models['gender']})
    rate = 191999
    base = [synth_audio(20, seed=80 + c, sr=rate) for c in range(3)]
    x = np.stack([base[c % 3] // (1 + c // 3) for c in range(8)], axis=1)
    q, tie, _, _ = reference(x, rate)
    assert not tie.any()
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        got = seg.segment_signal(x, sample_rate=rate)
        assert got == seg.segment_signal(q)
    assert got[-1][2] == pytest.approx(20.0, abs=0.03)
