"""Audio ingest: ``media2sig16kmono`` (inaSpeechSegmenter/io.py:32-79).

Behaviour kept: with ``ffmpeg=None`` the file is read directly and must be
16 kHz (same NotImplementedError / assertion messages, io.py:37-55); with an
ffmpeg binary the reference command line is used verbatim (io.py:60-77).
``soundfile`` is replaced by a small RIFF reader (PCM16 / PCM8 / PCM24 / PCM32 /
float32 / float64) with soundfile's integer scaling (value / 2**(bits-1)).

Additionally ``return_int16=True`` hands back the raw int16 samples when the
source is PCM16 so that the device front-end can ingest 2 bytes/sample (the
conversion s/32768 then happens in the kernel, bit-identical to soundfile's).

``wav_data`` reads a WAV header alone: with ffmpeg disabled, a WAV that is not
16 kHz mono is uploaded as stored and decoded by the device resampler
(segmenter._media2feats).
"""
import mmap
import struct
import subprocess
from collections import namedtuple
from tempfile import TemporaryFile

import numpy as np


def _wav_chunks(raw):
    """(fmt, start, stop) of a RIFF/WAVE image (bytes, or an mmap: only the fmt chunk is copied): the fmt fields
    (tag, channels, rate, byte rate, block align, bits) and the byte range of the data chunk, cut at the end of raw."""
    if raw[:4] != b'RIFF' or raw[8:12] != b'WAVE':
        raise ValueError('not a RIFF/WAVE file')
    pos, fmt, data = 12, None, None
    while pos + 8 <= len(raw):
        cid = raw[pos:pos + 4]
        size = struct.unpack('<I', raw[pos + 4:pos + 8])[0]
        if cid == b'fmt ':
            body = raw[pos + 8:pos + 8 + size]
            fmt = struct.unpack('<HHIIHH', body[:16])
            if fmt[0] == 0xFFFE and len(body) >= 26:        # WAVE_FORMAT_EXTENSIBLE: sub-format tag
                fmt = (struct.unpack('<H', body[24:26])[0],) + fmt[1:]
        elif cid == b'data':
            stop = len(raw) if size == 0xFFFFFFFF else min(pos + 8 + size, len(raw))   # ffmpeg pipes write size -1
            data = (pos + 8, stop)
            break
        pos += 8 + size + (size & 1)
    if fmt is None or data is None:
        raise ValueError('missing fmt/data chunk')
    return (fmt,) + data


def _parse_wav(raw):
    fmt, start, stop = _wav_chunks(raw)
    return fmt, raw[start:stop]


# encoding of a WAV by (format tag, container bits): what read_wav decodes, named as resample.PCM_FORMATS
_ENCODINGS = {(1, 8): 'u8', (1, 16): 's16', (1, 24): 's24', (1, 32): 's32', (3, 32): 'f32', (3, 64): 'f64'}
BYTES = {'u8': 1, 's16': 2, 's24': 3, 's32': 4, 'f32': 4, 'f64': 8}


class WavData(namedtuple('WavData', 'path encoding channels rate frames start stop')):
    """The layout of a WAV file (wav_data): its samples are the bytes [start, stop) of the file, `frames` frames of
    `channels` interleaved samples of `encoding` at `rate` Hz."""

    @property
    def shape(self):
        """[frames, channels, bytes per sample]: the stored bytes as a uint8 array."""
        return (self.frames, self.channels, BYTES[self.encoding])

    @property
    def nbytes(self):
        return self.stop - self.start

    def readinto(self, buf):
        """Reads the samples into the writable buffer buf (nbytes long) with no intermediate copy."""
        view = memoryview(buf).cast('B')
        with open(self.path, 'rb', buffering=0) as f:
            f.seek(self.start)
            done = 0
            while done < len(view):
                n = f.readinto(view[done:])
                if not n:
                    raise EOFError('%s ends inside its data chunk' % self.path)
                done += n


def wav_data(path):
    """WavData of the WAV file at `path`, read from its header alone.  Handles WAVE_FORMAT_EXTENSIBLE, chunks before
    `data` (odd sizes padded) and a data size of 0xFFFFFFFF (to the end of the file), as read_wav does.  The container
    bit depth decides the encoding (24 valid bits in 32 is s32, as read_wav reads it), and a trailing partial frame is
    dropped.  ValueError for a file that is not a RIFF/WAVE, NotImplementedError for an encoding read_wav lacks."""
    with open(path, 'rb') as f:
        with mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ) as raw:
            (tag, nch, sr, _, _, bits), start, stop = _wav_chunks(raw)
    enc = _ENCODINGS.get((tag, bits))
    if enc is None:
        raise NotImplementedError('WAV format tag %d with %d bits' % (tag, bits))
    if nch < 1:
        raise ValueError('WAV header with %d channels' % nch)
    frames = (stop - start) // (nch * BYTES[enc])
    return WavData(path, enc, nch, sr, frames, start, start + frames * nch * BYTES[enc])


def read_wav(path_or_file, dtype='float64', return_int16=False):
    """-> (signal, sample_rate); multi-channel data is [frames, channels]."""
    if hasattr(path_or_file, 'read'):
        raw = path_or_file.read()
    else:
        with open(path_or_file, 'rb') as f:
            raw = f.read()
    (tag, nch, sr, _, _, bits), data = _parse_wav(raw)
    if tag == 1:
        if bits == 16:
            ints = np.frombuffer(data[:len(data) // 2 * 2], dtype='<i2')
            if return_int16:
                sig = ints
            else:
                sig = ints.astype(dtype) / np.dtype(dtype).type(32768)
        elif bits == 8:
            sig = (np.frombuffer(data, dtype=np.uint8).astype(dtype) - 128) / np.dtype(dtype).type(128)
        elif bits == 24:
            b = np.frombuffer(data[:len(data) // 3 * 3], dtype=np.uint8).reshape(-1, 3).astype(np.int32)
            ints = (b[:, 0] | (b[:, 1] << 8) | (b[:, 2] << 16))
            ints = np.where(ints >= 1 << 23, ints - (1 << 24), ints)
            sig = ints.astype(dtype) / np.dtype(dtype).type(1 << 23)
        elif bits == 32:
            sig = np.frombuffer(data[:len(data) // 4 * 4], dtype='<i4').astype(dtype) / np.dtype(dtype).type(2 ** 31)
        else:
            raise NotImplementedError('PCM %d bits' % bits)
    elif tag == 3:
        src = '<f4' if bits == 32 else '<f8'
        sig = np.frombuffer(data[:len(data) // (bits // 8) * (bits // 8)], dtype=src).astype(dtype)
    else:
        raise NotImplementedError('WAV format tag %d' % tag)
    if nch > 1:
        sig = sig.reshape(-1, nch)
    return sig, sr


def media2sig16kmono(medianame, start_sec=None, stop_sec=None, ffmpeg='ffmpeg', dtype='float64',
                     return_int16=False):
    """Convert media to 16 kHz mono and return the signal (io.py:32-79)."""
    if ffmpeg is None:
        if start_sec is not None or stop_sec is not None:
            raise NotImplementedError(
                f'start_sec={start_sec} and stop_sec={stop_sec} cannot be set '
                f' when running inaSpeechSegmenter without ffmpeg. Please cut '
                f'down your audio files beforehand or use ffmpeg.')
        if medianame.startswith('http://') or medianame.startswith('https://'):
            raise NotImplementedError(
                f'Without ffmpeg you cannot process media content on http '
                f'servers. You need to download your audio files beforehand '
                f'or use ffmpeg. You gave medianame={medianame}.')
        sig, sr = read_wav(medianame, dtype=dtype, return_int16=return_int16)
        assert sr == 16_000, \
            f'Without ffmpeg, inaSpeechSegmenter can only take files sampled ' \
            f'at 16000 Hz. The file {medianame} is sampled at {sr} Hz.'
        return sig

    cmd = [ffmpeg, '-i', medianame, '-f', 'wav', '-acodec', 'pcm_s16le', '-ar', '16000', '-ac', '1']
    if start_sec is None:
        start_sec = 0
    else:
        cmd += ['-ss', '%f' % start_sec]
    if stop_sec is not None:
        cmd += ['-to', '%f' % stop_sec]
    cmd += ['pipe:1']
    with TemporaryFile() as out, TemporaryFile() as err:
        ret = subprocess.run(cmd, stdout=out, stderr=err)
        if ret.returncode != 0:
            err.seek(0)
            raise Exception(err.read())
        out.seek(0)
        wav_data, fs = read_wav(out, dtype=dtype, return_int16=return_int16)
    assert fs == 16000
    return wav_data
