"""WAV files of any rate, channel count and PCM encoding without ffmpeg, host side: io.wav_data's header reading
against read_wav (the host decoder), the tests' sample conversions (wav_fixtures.decode, which the device tests
feed to oracle/resample_ref.py), and which files the device route takes."""
import os

import numpy as np
import pytest

from wav_fixtures import decode, encode, fixtures, signal, write_wav

from inaspeechsegmenter_b200 import io as iss_io


@pytest.fixture(scope='module')
def wavs(tmp_path_factory):
    return fixtures(str(tmp_path_factory.mktemp('wavs')))


def _bytes(w):
    with open(w.path, 'rb') as f:
        f.seek(w.start)
        return f.read(w.stop - w.start)


def test_layout_and_decode_equal_read_wav(wavs):
    """For every fixture, the reported byte range through wav_fixtures.decode is read_wav's float64 signal, exactly."""
    for name, (path, enc, C, rate) in wavs.items():
        w = iss_io.wav_data(path)
        assert (w.encoding, w.channels, w.rate) == (enc, C, rate), name
        assert w.stop - w.start == w.frames * C * iss_io.BYTES[enc] and w.shape == (w.frames, C, iss_io.BYTES[enc])
        ref, sr = iss_io.read_wav(path, 'float64')
        assert sr == rate
        got = decode(_bytes(w), enc, C)
        assert got.shape == (len(ref), C), name
        assert np.array_equal(got, ref.reshape(len(ref), -1)), name


def test_encoding_extremes():
    """The conversions at the ends of each integer range and at the sign boundary of 24-bit samples."""
    ints = {'u8': ([0, 128, 255], np.uint8), 's16': ([-32768, 0, 32767], '<i2'), 's32': ([-2 ** 31, -1, 2 ** 31 - 1], '<i4')}
    for enc, (v, dt) in ints.items():
        got = decode(np.array(v, dtype=dt).tobytes(), enc, 1)[:, 0]
        scale = {'u8': 128.0, 's16': 32768.0, 's32': 2.0 ** 31}[enc]
        assert list(got) == [((s - 128) if enc == 'u8' else s) / scale for s in v]
    s24 = bytes([0x00, 0x00, 0x80, 0xFF, 0xFF, 0xFF, 0xFF, 0xFF, 0x7F, 0x01, 0x00, 0x00])
    assert list(decode(s24, 's24', 1)[:, 0]) == [-1.0, -2.0 ** -23, 1 - 2.0 ** -23, 2.0 ** -23]


def test_header_forms(tmp_path):
    x = signal(1000, 2, 48000, seed=5)
    data = encode(x, 's24')
    base = iss_io.wav_data(write_wav(str(tmp_path / 'a.wav'), data, 's24', 2, 48000))
    assert base.start == 44 and base.frames == 1000
    odd = iss_io.wav_data(write_wav(str(tmp_path / 'b.wav'), data, 's24', 2, 48000, pre_chunks=((b'junk', b'abc'),)))
    assert odd.start == 44 + 8 + 4 and odd.frames == 1000
    ext = iss_io.wav_data(write_wav(str(tmp_path / 'c.wav'), data, 's24', 2, 48000, extensible=True))
    assert ext.encoding == 's24' and ext.start == 68
    valid24 = iss_io.wav_data(write_wav(str(tmp_path / 'd.wav'), encode(x, 's32'), 's32', 2, 48000, extensible=True,
                                        valid_bits=24))
    assert valid24.encoding == 's32'
    pipe = iss_io.wav_data(write_wav(str(tmp_path / 'e.wav'), data, 's24', 2, 48000, unknown_size=True, tail=b'\x07'))
    assert pipe.frames == 1000 and pipe.stop == pipe.start + 6000
    # a partial frame of whole samples is dropped too (read_wav itself cannot reshape such a file)
    part = iss_io.wav_data(write_wav(str(tmp_path / 'f.wav'), data, 's24', 2, 48000, tail=data[:3]))
    assert part.frames == 1000 and part.stop == part.start + 6000
    short = iss_io.wav_data(write_wav(str(tmp_path / 'g.wav'), b'', 'u8', 1, 8000))
    assert short.frames == 0 and short.nbytes == 0
    buf = np.zeros(pipe.nbytes, np.uint8)
    pipe.readinto(buf)
    assert buf.tobytes() == data


def test_header_errors(tmp_path):
    with open(tmp_path / 'x.wav', 'wb') as f:
        f.write(b'not a wav file at all')
    with pytest.raises(ValueError, match='RIFF'):
        iss_io.wav_data(str(tmp_path / 'x.wav'))
    p = write_wav(str(tmp_path / 'mulaw.wav'), b'\x00' * 100, 'u8', 1, 8000)
    with open(p, 'r+b') as f:                            # format tag 7 (mu-law)
        f.seek(20)
        f.write(b'\x07\x00')
    with pytest.raises(NotImplementedError):
        iss_io.wav_data(p)


def test_parse_wav_unchanged(media):
    """wav_data and read_wav (built on the same chunk walk) agree on the golden media: 16 kHz mono int16 / float32."""
    for name in ('musanmix.wav', 'lamartine.wav', 'silence2sec.wav'):
        p = os.path.join(media, name)
        w = iss_io.wav_data(p)
        raw, sr = iss_io.read_wav(p, 'float32', return_int16=True)
        assert w.encoding in ('s16', 'f32') and (w.channels, w.rate, sr) == (1, 16000, 16000)
        assert w.frames == len(raw) and _bytes(w) == raw.tobytes()


def test_route_choice(wavs, tmp_path):
    """Only whole files read without ffmpeg that are WAVs but not 16 kHz mono take the device route."""
    from inaspeechsegmenter_b200 import segmenter
    for name, (path, enc, C, rate) in wavs.items():
        w = segmenter._device_wav(path, None, None, None)
        assert (w is None) == (rate == 16000 and C == 1), name
        assert segmenter._device_wav(path, None, None, 'ffmpeg') is None
        assert segmenter._device_wav(path, 1.0, None, None) is None
        assert segmenter._device_wav(path, None, 2.0, None) is None
    with open(tmp_path / 'x.wav', 'wb') as f:
        f.write(b'garbage')
    assert segmenter._device_wav(str(tmp_path / 'x.wav'), None, None, None) is None
    assert segmenter._device_wav(str(tmp_path / 'missing.wav'), None, None, None) is None
    assert segmenter._device_wav('http://host/x.wav', None, None, None) is None


def test_start_stop_without_ffmpeg_still_refused(wavs):
    """start_sec / stop_sec with ffmpeg=None raise the reference's NotImplementedError, for any WAV."""
    from inaspeechsegmenter_b200 import segmenter
    path = wavs['s24_2ch_48000'][0]
    with pytest.raises(NotImplementedError, match='start_sec'):
        segmenter._media2feats(path, 1.0, None, None)
    with pytest.raises(NotImplementedError, match='stop_sec'):
        segmenter._media2feats(path, None, 2.0, None)


def test_cli_text():
    from inaspeechsegmenter_b200 import cli
    help_b = next(a.help for a in cli.build_parser()._actions if '-b' in a.option_strings)
    assert 'WAV input only' in help_b and '16 kHz' not in help_b
