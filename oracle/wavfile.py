"""CPU restatement of librosa.load(path, sr=None, mono=True)'s samples for WAV files (tools/utils.py:46-48,
evaluation_proc/metrics.py:33-34), the reference of vf_decode_pcm_varlen.  TEST INFRASTRUCTURE.

librosa 0.8 reads through soundfile (libsndfile) as float32, transposes to [C, N] and averages the channels (to_mono:
np.mean(y, axis=0), a reduction over each frame's contiguous run of C values).  Neither soundfile nor librosa is in this
image, so both steps are restated with numpy.  Parity status: the conversion follows libsndfile's float read as recalled
(below); the downmix is numpy's own arithmetic, pinned by tests/test_wavfile_cpu.py against numpy's x.mean(axis=1).

Conversion (libsndfile's *2f readers with normalisation on, soundfile's default):
* u8: (b - 128) * (1 / 128);  s16: v * 2^-15;  s24: sign-extended v * 2^-23;  s32: float32(v) * 2^-31, the int rounded to
  float32 to nearest first;  f32: unchanged, NaN and Inf included;  f64: rounded to float32 to nearest.
* channel 0 in float64 (speechmetrics' soundfile.read, dtype float64): the exact quotient v / 2^(bits - 1) (u8: (b - 128)
  / 128) for the integer formats, the stored value for the float formats.
Downmix (numpy's float32 add.reduce over C values, pairwise_sum within one block of at most 128):
* C < 8: one running sum from 0, in channel order.  C >= 8: r[j] = x[j] (j < 8), then r[j] += x[i + j] for each further
  whole block of 8, res = ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), then the remaining C % 8 values one by one;
  the reduction adds res to its identity 0.  Then one float32 division by C.
* C == 1: the channel itself.  librosa's to_mono leaves a 1-D signal alone; x.mean(axis=1) would add it to 0, which
  differs only in the sign of a zero sample (-0.0 becomes +0.0).
"""
import numpy as np

from voicefixer_main_b200 import wavfile as W


def samples(data, channels: int, fmt: int) -> np.ndarray:
    """libsndfile's float32 values of the interleaved little-endian `data` -> [frames, channels]."""
    raw = np.frombuffer(data, dtype=np.uint8)
    frames = raw.size // (channels * W.WIDTH[fmt])
    raw = raw[:frames * channels * W.WIDTH[fmt]]
    if fmt == W.U8:
        x = (raw.astype(np.int32) - 128).astype(np.float32) * np.float32(1 / 128)
    elif fmt == W.S16:
        x = raw.view("<i2").astype(np.float32) * np.float32(2.0 ** -15)
    elif fmt == W.S24:
        b = raw.reshape(-1, 3).astype(np.int32)
        v = ((b[:, 0] << 8) | (b[:, 1] << 16) | (b[:, 2] << 24)) >> 8
        x = v.astype(np.float32) * np.float32(2.0 ** -23)
    elif fmt == W.S32:
        x = raw.view("<i4").astype(np.float32) * np.float32(2.0 ** -31)
    elif fmt == W.F32:
        x = raw.view("<f4").copy()
    else:
        x = raw.view("<f8").astype(np.float32)
    return x.reshape(frames, channels)


def first64(data, channels: int, fmt: int) -> np.ndarray:
    """Channel 0 as soundfile reads it in float64 -> [frames]."""
    raw = np.frombuffer(data, dtype=np.uint8)
    frames = raw.size // (channels * W.WIDTH[fmt])
    raw = raw[:frames * channels * W.WIDTH[fmt]]
    if fmt == W.U8:
        v = raw.astype(np.float64) - 128
        return v.reshape(frames, channels)[:, 0] / 128.0
    if fmt == W.S24:
        b = raw.reshape(-1, 3).astype(np.int32)
        v = ((b[:, 0] << 8) | (b[:, 1] << 16) | (b[:, 2] << 24)) >> 8
        return v.reshape(frames, channels)[:, 0].astype(np.float64) / 2.0 ** 23
    dtype, scale = {W.S16: ("<i2", 2.0 ** 15), W.S32: ("<i4", 2.0 ** 31), W.F32: ("<f4", 1.0), W.F64: ("<f8", 1.0)}[fmt]
    return raw.view(dtype).reshape(frames, channels)[:, 0].astype(np.float64) / scale


def downmix(x: np.ndarray) -> np.ndarray:
    """librosa 0.8's to_mono of soundfile's [frames, C] float32 array, in numpy's add.reduce order (module docstring)."""
    n, c = x.shape
    if c == 1:
        return x[:, 0].copy()
    if c < 8:
        res = np.zeros(n, np.float32)
        for j in range(c):
            res = res + x[:, j]
    else:
        r = [x[:, j].copy() for j in range(8)]
        i = 8
        while i < c - c % 8:
            for j in range(8):
                r[j] = r[j] + x[:, i + j]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for k in range(i, c):
            res = res + x[:, k]
        res = np.zeros(n, np.float32) + res
    return res / np.float32(c)


def random_data(rng, frames: int, channels: int, fmt: int) -> np.ndarray:
    """Seeded interleaved samples [frames, channels] of `fmt` covering its whole range: integers (u8 as uint8, s24 as int32
    in -2^23 .. 2^23 - 1) with both extremes, floats over many magnitudes with +-0 and a few values beyond +-1."""
    if fmt in (W.F32, W.F64):
        x = rng.standard_normal((frames, channels)) * np.exp2(rng.integers(-30, 3, (frames, channels)))
        x.flat[::7] = 0.0
        x.flat[3::11] = -0.0
        return x.astype(np.float32 if fmt == W.F32 else np.float64)
    lo, hi = {W.U8: (0, 255), W.S16: (-2 ** 15, 2 ** 15 - 1), W.S24: (-2 ** 23, 2 ** 23 - 1), W.S32: (-2 ** 31, 2 ** 31 - 1)}[fmt]
    x = rng.integers(lo, hi, (frames, channels), endpoint=True, dtype=np.int64)
    x.flat[::5] = lo
    x.flat[2::9] = hi
    return x


def encode(x: np.ndarray, fmt: int) -> bytes:
    """The little-endian data chunk bytes of random_data's samples x [frames, channels]."""
    if fmt == W.S24:
        v = x.astype("<i4").reshape(-1, 1).view(np.uint8)
        return v[:, :3].tobytes()
    dtype = {W.U8: "u1", W.S16: "<i2", W.S32: "<i4", W.F32: "<f4", W.F64: "<f8"}[fmt]
    return x.astype(dtype).tobytes()


def wav_bytes(data: bytes, rate: int, channels: int, fmt: int, extensible: bool = False, valid_bits: int = None,
              before=(), after=(), tag: int = None, block_align: int = None, data_size: int = None) -> bytes:
    """A RIFF WAVE file around a data chunk: `before` / `after` are (id, payload) chunks around it (odd payloads get their pad
    byte); extensible writes WAVE_FORMAT_EXTENSIBLE with `valid_bits`; tag, block_align and data_size override the header's
    fields to build malformed files."""
    width, bits = W.WIDTH[fmt], 8 * W.WIDTH[fmt]
    code = tag if tag is not None else (W.TAG_FLOAT if fmt in (W.F32, W.F64) else W.TAG_PCM)
    align = block_align if block_align is not None else channels * width
    if extensible:
        sub = code.to_bytes(2, "little") + b"\x00\x00\x00\x00\x10\x00\x80\x00\x00\xaa\x00\x38\x9b\x71"
        fmt_body = (W.TAG_EXTENSIBLE.to_bytes(2, "little") + channels.to_bytes(2, "little") + rate.to_bytes(4, "little")
                    + (rate * align).to_bytes(4, "little") + align.to_bytes(2, "little") + bits.to_bytes(2, "little")
                    + (22).to_bytes(2, "little") + (valid_bits or bits).to_bytes(2, "little") + (0).to_bytes(4, "little")
                    + sub)
    else:
        fmt_body = (code.to_bytes(2, "little") + channels.to_bytes(2, "little") + rate.to_bytes(4, "little")
                    + (rate * align).to_bytes(4, "little") + align.to_bytes(2, "little") + bits.to_bytes(2, "little"))

    def chunk(cid, payload, size=None):
        n = len(payload) if size is None else size
        return cid + n.to_bytes(4, "little") + payload + (b"\x00" if len(payload) % 2 else b"")

    body = b"WAVE" + b"".join(chunk(c, p) for c, p in before) + chunk(b"fmt ", fmt_body) + chunk(b"data", data, data_size) \
        + b"".join(chunk(c, p) for c, p in after)
    return b"RIFF" + len(body).to_bytes(4, "little") + body


def load(path):
    """(mono float32, rate, channel 0 float64) of a WAV file as librosa.load(path, sr=None, mono=True) and soundfile give
    them, parsed by voicefixer_main_b200.wavfile."""
    w = W.parse(path)
    return downmix(samples(w.data, w.channels, w.format)), w.rate, first64(w.data, w.channels, w.format)
