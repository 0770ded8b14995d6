"""The RIFF / WAVE container of the files librosa.load reads (tools/utils.py:46-48, evaluation_proc/metrics.py:33-34).

`parse(path)` reads a file's chunks and returns its rate, channel count, sample format, frame count and a view of its data
chunk's bytes; it converts no sample (vf_decode_pcm_varlen does, on the GPU).  What soundfile (libsndfile) accepts among
uncompressed WAVs is accepted: format tag 1 (PCM: unsigned 8-bit, signed 16-, 24- and 32-bit), tag 3 (IEEE float: 32- and
64-bit) and tag 0xFFFE (WAVE_FORMAT_EXTENSIBLE) with the PCM or IEEE-float subformat GUID, 1 to 64 channels.  Other chunks
(LIST, fact, bext, cue, ...) are skipped with their pad byte.  Anything else raises ValueError naming the file and what it
found: a compressed format tag (ADPCM, mu-law, A-law, ...), RF64 or RIFX, a missing `fmt ` or `data` chunk, a block align
that is not channels x sample width, a sample width the tag does not define.

Choices where libsndfile's behaviour could not be run and checked:
* A data chunk whose declared size runs past the end of the file (a recorder that died before it patched the header, or
  a streaming writer's 0xFFFFFFFF) is cut to the bytes the file holds, as libsndfile logs and truncates it.
* A data chunk that is not a whole number of frames: the trailing partial frame is not read (libsndfile's frame count is
  the data length over the block align).
* WAVE_FORMAT_EXTENSIBLE with fewer valid bits than container bits (20 bits in 24, 24 in 32): samples are read at the
  container width, the padding bits included, as libsndfile reads them; the channel mask is ignored (librosa averages every
  channel).
* The first `data` chunk is the audio; chunks after it are skipped.  A `fmt ` chunk may come before or after it.
* A sample rate of 0 is rejected.
"""
import struct
from collections import namedtuple

# sample formats, the VF_PCM_* codes of include/b200vf.h
U8, S16, S24, S32, F32, F64 = range(6)
NAMES = ("u8", "s16", "s24", "s32", "f32", "f64")
WIDTH = (1, 2, 3, 4, 4, 8)

TAG_PCM, TAG_FLOAT, TAG_EXTENSIBLE = 0x0001, 0x0003, 0xFFFE
_GUID_TAIL = b"\x00\x00\x00\x00\x10\x00\x80\x00\x00\xaa\x00\x38\x9b\x71"   # KSDATAFORMAT_SUBTYPE_* after the 2-byte tag
_COMPRESSED = {0x0002: "MS ADPCM", 0x0006: "A-law", 0x0007: "mu-law", 0x0011: "IMA ADPCM", 0x0031: "GSM 6.10",
               0x0050: "MPEG", 0x0055: "MP3"}
_FORMATS = {(TAG_PCM, 8): U8, (TAG_PCM, 16): S16, (TAG_PCM, 24): S24, (TAG_PCM, 32): S32, (TAG_FLOAT, 32): F32,
            (TAG_FLOAT, 64): F64}

WavInfo = namedtuple("WavInfo", "path rate channels format frames data")
WavInfo.__doc__ = """A parsed WAV file: rate (Hz), channels, format (U8 .. F64), frames, and data, a memoryview of the
frames * channels * WIDTH[format] bytes of interleaved little-endian samples."""


def _tag_name(tag):
    return f"0x{tag:04X}" + (f" ({_COMPRESSED[tag]})" if tag in _COMPRESSED else "")


def parse(path) -> WavInfo:
    """The WavInfo of the WAV file at `path`, or ValueError naming the file and what is wrong with it."""
    with open(path, "rb") as f:
        raw = f.read()
    head = raw[:4]
    if head == b"RF64":
        raise ValueError(f"{path}: RF64 WAV is not supported (need a RIFF WAVE file)")
    if head == b"RIFX":
        raise ValueError(f"{path}: big-endian RIFX WAV is not supported (need a RIFF WAVE file)")
    if len(raw) < 12 or head != b"RIFF" or raw[8:12] != b"WAVE":
        raise ValueError(f"{path}: not a RIFF WAVE file")
    fmt = data = None
    pos = 12
    while pos + 8 <= len(raw) and (fmt is None or data is None):
        cid, size = raw[pos:pos + 4], struct.unpack_from("<I", raw, pos + 4)[0]
        body = pos + 8
        if cid == b"fmt " and fmt is None:
            fmt = raw[body:body + size]
        elif cid == b"data" and data is None:
            data = (body, min(size, len(raw) - body))        # cut to the bytes the file holds
        pos = body + size + (size & 1)
    if fmt is None:
        raise ValueError(f"{path}: no 'fmt ' chunk")
    if data is None:
        raise ValueError(f"{path}: no 'data' chunk")
    if len(fmt) < 16:
        raise ValueError(f"{path}: 'fmt ' chunk of {len(fmt)} bytes (need at least 16)")
    tag, channels, rate, _, block_align, bits = struct.unpack_from("<HHIIHH", fmt)
    if tag == TAG_EXTENSIBLE:
        if len(fmt) < 40:
            raise ValueError(f"{path}: extensible 'fmt ' chunk of {len(fmt)} bytes (need 40)")
        guid = fmt[24:40]
        if guid[2:] != _GUID_TAIL:
            raise ValueError(f"{path}: extensible WAV with subformat GUID {guid.hex()} (need PCM or IEEE float)")
        tag = struct.unpack_from("<H", guid)[0]
    if tag not in (TAG_PCM, TAG_FLOAT):
        what = "compressed " if tag in _COMPRESSED else ""
        raise ValueError(f"{path}: {what}format tag {_tag_name(tag)} is not supported (need PCM (1) or IEEE float (3))")
    if (tag, bits) not in _FORMATS:
        raise ValueError(f"{path}: {bits}-bit {'PCM' if tag == TAG_PCM else 'IEEE float'} is not supported")
    form = _FORMATS[tag, bits]
    if not 1 <= channels <= 64:
        raise ValueError(f"{path}: {channels} channels (need 1 .. 64)")
    if block_align != channels * WIDTH[form]:
        raise ValueError(f"{path}: block align {block_align} is not {channels} channels x {WIDTH[form]} bytes")
    if rate == 0:
        raise ValueError(f"{path}: sample rate 0")
    start, size = data
    frames = size // block_align
    return WavInfo(path, rate, channels, form, frames, memoryview(raw)[start:start + frames * block_align])
