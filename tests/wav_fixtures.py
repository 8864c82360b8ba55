"""WAV files written with numpy for the WAV-input tests: every encoding the device route reads, and the header forms
a WAV file can take (WAVE_FORMAT_EXTENSIBLE, chunks before `data`, ffmpeg's data size 0xFFFFFFFF, a trailing partial
frame)."""
import os
import struct

import numpy as np

ENCODINGS = ('u8', 's16', 's24', 's32', 'f32', 'f64')
CHANNELS = (1, 2, 6)
RATES = (8000, 16000, 44100, 48000, 192000)
_TAG_BITS = {'u8': (1, 8), 's16': (1, 16), 's24': (1, 24), 's32': (1, 32), 'f32': (3, 32), 'f64': (3, 64)}


def encode(x, encoding):
    """The stored bytes of float64 samples x in [-1, 1] ([frames] or [frames, channels], interleaved) in `encoding`;
    integers round to nearest and saturate."""
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    if encoding == 'u8':
        return (np.clip(np.round(x * 128), -128, 127) + 128).astype(np.uint8).tobytes()
    if encoding == 's16':
        return np.clip(np.round(x * 32768), -32768, 32767).astype('<i2').tobytes()
    if encoding == 's24':
        v = np.clip(np.round(x * 2 ** 23), -2 ** 23, 2 ** 23 - 1).astype(np.int64) & 0xFFFFFF
        return np.stack([v & 255, (v >> 8) & 255, v >> 16], axis=1).astype(np.uint8).tobytes()
    if encoding == 's32':
        return np.clip(np.round(x * 2 ** 31), -2 ** 31, 2 ** 31 - 1).astype('<i4').tobytes()
    return x.astype('<f4' if encoding == 'f32' else '<f8').tobytes()


def decode(raw, encoding, channels):
    """float64 [frames, channels] of the samples a WAV stores in the bytes `raw` (whole frames): step 1 of the
    resampler's definition for every encoding, u8 (s - 128) / 128, s16 s / 2^15, s24 (3 bytes little-endian, two's
    complement) s / 2^23, s32 s / 2^31, f32 and f64 as is.  Each value is exact in float64, so
    oracle.resample_ref.reference takes the result as it is.  Written apart from read_wav, which the tests hold it
    against."""
    b = np.frombuffer(bytes(raw), dtype=np.uint8)
    if encoding == 'u8':
        v = (b.astype(np.int64) - 128) * 2.0 ** -7
    elif encoding == 's24':
        t = b.reshape(-1, 3).astype(np.int64)
        u = t[:, 0] + 256 * t[:, 1] + 65536 * t[:, 2]
        v = (u - (u >= 2 ** 23) * 2 ** 24) * 2.0 ** -23
    else:
        dt, scale = {'s16': ('<i2', 2.0 ** -15), 's32': ('<i4', 2.0 ** -31), 'f32': ('<f4', 1.0),
                     'f64': ('<f8', 1.0)}[encoding]
        v = b.view(dt).astype(np.float64) * scale
    return v.reshape(-1, channels)


def write_wav(path, data, encoding, channels, rate, extensible=False, valid_bits=None, pre_chunks=(),
              unknown_size=False, tail=b'', channel_mask=0):
    """Writes a RIFF/WAVE file whose data chunk holds the bytes `data` (then `tail`, e.g. a partial frame).
    extensible: WAVE_FORMAT_EXTENSIBLE with the sub-format of `encoding`, valid_bits (the container's by default) and
    channel_mask; pre_chunks: (id, body) chunks written between fmt and data, odd bodies padded; unknown_size: data
    size 0xFFFFFFFF and RIFF size 0xFFFFFFFF, as ffmpeg writes to a pipe."""
    tag, bits = _TAG_BITS[encoding]
    block = channels * bits // 8
    fmt = struct.pack('<HHIIHH', 0xFFFE if extensible else tag, channels, rate, rate * block, block, bits)
    if extensible:
        guid_tail = b'\x00\x00\x00\x00\x10\x00\x80\x00\x00\xaa\x00\x38\x9b\x71'
        fmt += struct.pack('<HHI', 22, valid_bits or bits, channel_mask) + struct.pack('<H', tag) + guid_tail
    body = b'WAVE' + b'fmt ' + struct.pack('<I', len(fmt)) + fmt
    for cid, chunk in pre_chunks:
        body += cid + struct.pack('<I', len(chunk)) + chunk + (b'\x00' if len(chunk) & 1 else b'')
    payload = data + tail
    body += b'data' + struct.pack('<I', 0xFFFFFFFF if unknown_size else len(payload)) + payload
    riff = 0xFFFFFFFF if unknown_size else len(body)
    with open(path, 'wb') as f:
        f.write(b'RIFF' + struct.pack('<I', riff) + body)
    return path


def signal(frames, channels, rate, seed):
    """float64 [frames, channels] in [-1, 1]: noise, a tone per channel, full-scale samples of both signs (the
    extremes of every integer encoding) and a clipped square on channel 0."""
    rng = np.random.default_rng(seed)
    t = np.arange(frames) / rate
    x = rng.standard_normal((frames, channels)) * 0.2 + 0.3 * np.sin(2 * np.pi * (440 + 97 * np.arange(channels)) * t[:, None])
    x[::max(frames // 7, 1)] = 1.0
    x[1::max(frames // 5, 1)] = -1.0
    x[frames // 2:, 0] = np.where(np.sin(2 * np.pi * 1234 * t[frames // 2:]) >= 0, 1.0, -1.0)
    return np.clip(x, -1, 1)


def fixtures(directory, frames=3001):
    """{name: (path, encoding, channels, rate)}: every encoding x channel count x rate, plus the header forms."""
    out = {}
    for enc in ENCODINGS:
        for C in CHANNELS:
            for rate in RATES:
                name = '%s_%dch_%d' % (enc, C, rate)
                x = signal(frames, C, rate, seed=len(out))
                out[name] = (write_wav(os.path.join(directory, name + '.wav'), encode(x, enc), enc, C, rate), enc, C,
                             rate)
    x = signal(frames, 2, 48000, seed=101)
    forms = {
        'ext_s24_2ch_48000': (dict(extensible=True), 's24', 2),
        'ext_s32_valid24_2ch_48000': (dict(extensible=True, valid_bits=24), 's32', 2),
        'ext_f32_2ch_48000': (dict(extensible=True), 'f32', 2),
        'oddchunk_s16_2ch_48000': (dict(pre_chunks=((b'LIST', b'INFOabcde'), (b'bext', b'x' * 7))), 's16', 2),
        'ffmpegsize_s16_2ch_48000': (dict(unknown_size=True), 's16', 2),
        'partial_s24_1ch_48000': (dict(tail=b'\x01\x02'), 's24', 1),
        'partial_s32_1ch_48000': (dict(tail=b'\x01\x02\x03'), 's32', 1),
        'partial_f64_1ch_48000': (dict(tail=b'\x00' * 5), 'f64', 1),
    }
    for name, (kw, enc, C) in forms.items():
        path = os.path.join(directory, name + '.wav')
        out[name] = (write_wav(path, encode(x[:, :C], enc), enc, C, 48000, **kw), enc, C, 48000)
    return out


# dwChannelMask of WAVE_FORMAT_EXTENSIBLE for each channel count over 2: front left / right / centre, LFE, back
# left / right, side left / right (3.0, quad, 5.0, 5.1, 6.1, 7.1)
CHANNEL_MASKS = {3: 0x7, 4: 0x33, 5: 0x37, 6: 0x3F, 7: 0x70F, 8: 0x63F}
DOMAIN_CHANNELS = (3, 4, 5, 7, 8)
DOMAIN_RATES = (11025, 32000, 88200, 96000, 176400, 191999)


def domain_fixtures(directory, encodings=ENCODINGS, channels=DOMAIN_CHANNELS, rates=DOMAIN_RATES, frames=2001):
    """{name: (path, encoding, channels, rate)}: every encoding x channel count x rate given, as a multichannel file
    is written: WAVE_FORMAT_EXTENSIBLE with the channel mask of its layout over 2 channels, the plain header below."""
    out = {}
    for enc in encodings:
        for C in channels:
            for rate in rates:
                name = '%s_%dch_%d' % (enc, C, rate)
                x = signal(frames, C, rate, seed=1000 + len(out))
                kw = dict(extensible=True, channel_mask=CHANNEL_MASKS[C]) if C > 2 else {}
                out[name] = (write_wav(os.path.join(directory, name + '.wav'), encode(x, enc), enc, C, rate, **kw),
                             enc, C, rate)
    return out
