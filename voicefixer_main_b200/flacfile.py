"""The FLAC container (RFC 9639) of the files librosa.load reads through soundfile (tools/utils.py:46-48,
evaluation_proc/metrics.py:33-34), and the drop-in for the reference's FLAC-to-WAV conversion (tools/file/wav.py:176-195).

`parse(path)` reads a file's metadata and returns its STREAMINFO facts and a view of its audio region, from the first
frame's sync code to the end of the file; it decodes no frame (vf_decode_flac_varlen does, on the GPU).  An ID3v2 tag
before `fLaC` is skipped as libsndfile skips it (10 header bytes, the syncsafe size, 10 more with the footer flag).  Every
metadata block after STREAMINFO (padding, application, seek table, Vorbis comment, cue sheet, picture, reserved types) is
skipped.  Accepted: 1 to 8 channels of 8-, 16- or 24-bit samples at any rate, fixed or variable blocking with block sizes up
to 65535.  The decoded samples are libsndfile's float read, v / 2^(bits - 1), which for these depths equals the WAV path's
value of the same integer sample, so a FLAC file and a WAV file holding the same samples load to the same bits.

Rejected with ValueError naming the file and the reason (choices made where libsndfile's own behaviour could not be run and
checked): Ogg FLAC; bit depths other than 8, 16 and 24; a STREAMINFO total of 0 samples (unknown length); STREAMINFO
missing or not the first block; truncated metadata; and, on the GPU, every reserved or forbidden code in a frame, a frame
that disagrees with STREAMINFO, a CRC-8 or CRC-16 mismatch, invalid partitioning, a sample outside the bit depth's range and
frames whose sample counts do not add up to the total.  When libsndfile fails on a file, librosa 0.8 falls back to
audioread; that fallback is not reproduced.  The STREAMINFO MD5 is not checked on the load path (libsndfile does not check
it either); `convert_flac_to_wav` checks it.
"""
import glob
import hashlib
import os
import struct
import wave
from collections import namedtuple

import numpy as np

# the messages of the VF_FLAC_E* codes of include/b200vf.h
ERRORS = {1: "no frame sync code where a frame must start", 2: "a reserved or forbidden code in a frame header",
          3: "a frame header disagrees with STREAMINFO (channels, bit depth, rate or blocking strategy)",
          4: "frame header CRC-8 mismatch",
          5: "a reserved or forbidden subframe code (type, LPC precision, negative shift or residual coding)",
          6: "invalid residual partitioning", 7: "a frame runs past the end of the file", 8: "frame CRC-16 mismatch",
          9: "a decoded sample outside the bit depth's range",
          10: "a frame or sample number out of sequence, or a short fixed-blocking frame before the last",
          11: "the frames' sample counts do not add up to STREAMINFO's total samples",
          12: "too many frame candidates (more than one per 8 bytes)"}

FlacInfo = namedtuple("FlacInfo", "path rate channels bits total min_block max_block md5 variable first_block audio_start "
                                  "audio")
FlacInfo.__doc__ = """A parsed FLAC file: rate (Hz), channels, bits, total samples per channel, STREAMINFO's min / max block
size and MD5 (16 bytes), the blocking strategy (variable: 0 fixed, 1 variable) and block size of the first frame, the file
offset of the first frame, and audio, a memoryview of the bytes from the first frame to the end of the file."""


def is_flac(head: bytes) -> bool:
    """Whether a file starting with `head` (at least 4 bytes) goes to `parse`: `fLaC`, an ID3v2 tag before it, or an Ogg
    stream (`OggS`), which `parse` rejects with its reason rather than the WAV parser calling it a bad RIFF file."""
    return head[:4] in (b"fLaC", b"OggS") or head[:3] == b"ID3"


def _first_block(path, raw, pos):
    """(blocking strategy, block size) of the frame header at raw[pos] (RFC 9639 §9.1.1, §9.1.5, §9.1.6)."""
    if len(raw) < pos + 6 or raw[pos] != 0xFF or raw[pos + 1] & 0xFE != 0xF8:
        raise ValueError(f"{path}: no frame sync code after the metadata (byte {pos})")
    code = raw[pos + 2] >> 4
    lead = raw[pos + 4]                       # the coded number's continuation bytes (§9.1.5)
    extra = next(n for n, top in enumerate((0x80, 0xE0, 0xF0, 0xF8, 0xFC, 0xFE, 0x100)) if lead < top)
    at = pos + 5 + extra
    if code == 0:
        raise ValueError(f"{path}: reserved block size code 0000 in the first frame (byte {pos})")
    if code == 1:
        block = 192
    elif code <= 5:
        block = 576 << (code - 2)
    elif code in (6, 7):
        if len(raw) < at + code - 5:
            raise ValueError(f"{path}: the first frame's header is cut off (byte {pos})")
        block = int.from_bytes(raw[at:at + code - 5], "big") + 1
    else:
        block = 256 << (code - 8)
    return raw[pos + 1] & 1, block


def parse(path) -> FlacInfo:
    """The FlacInfo of the FLAC file at `path`, or ValueError naming the file and what is wrong with it."""
    with open(path, "rb") as f:
        raw = f.read()
    pos = 0
    if raw[:3] == b"ID3":                     # ID3v2: 10 header bytes + syncsafe size (+ 10 footer bytes)
        if len(raw) < 10:
            raise ValueError(f"{path}: truncated ID3v2 tag")
        size = (raw[6] & 0x7F) << 21 | (raw[7] & 0x7F) << 14 | (raw[8] & 0x7F) << 7 | (raw[9] & 0x7F)
        pos = 10 + size + (10 if raw[5] & 0x10 else 0)
    if raw[pos:pos + 4] == b"OggS":               # Ogg FLAC's first packet starts 0x7F "FLAC" after the 28-byte page header
        what = "Ogg FLAC" if raw[pos + 28:pos + 33] == b"\x7fFLAC" else "an Ogg stream"
        raise ValueError(f"{path}: {what} is not supported (need native FLAC or WAV)")
    if raw[pos:pos + 4] != b"fLaC":
        raise ValueError(f"{path}: not a FLAC file")
    pos += 4
    info = None
    last = False
    while not last:                           # metadata blocks (§8.1): last flag, 7-bit type, 24-bit length
        if pos + 4 > len(raw):
            raise ValueError(f"{path}: truncated metadata (block header at byte {pos})")
        last, kind, size = raw[pos] >> 7, raw[pos] & 0x7F, int.from_bytes(raw[pos + 1:pos + 4], "big")
        body = pos + 4
        if body + size > len(raw):
            raise ValueError(f"{path}: truncated metadata (block of type {kind} at byte {pos} needs {size} bytes)")
        if info is None:
            if kind != 0:
                raise ValueError(f"{path}: STREAMINFO missing or not the first metadata block (found type {kind})")
            if size != 34:
                raise ValueError(f"{path}: STREAMINFO of {size} bytes (need 34)")
            info = raw[body:body + 34]
        elif kind == 127:
            raise ValueError(f"{path}: forbidden metadata block type 127 at byte {pos}")
        pos = body + size
    # STREAMINFO (§8.2): u16 min / max block, u24 min / max frame, u20 rate, u3 channels - 1, u5 bits - 1, u36 total, MD5
    min_block, max_block = struct.unpack_from(">HH", info)
    packed = int.from_bytes(info[10:18], "big")
    rate, channels, bits, total = packed >> 44, (packed >> 41 & 7) + 1, (packed >> 36 & 31) + 1, packed & (1 << 36) - 1
    if bits not in (8, 16, 24):
        raise ValueError(f"{path}: {bits}-bit FLAC is not supported (need 8, 16 or 24)")
    if total == 0:
        raise ValueError(f"{path}: STREAMINFO total samples 0 (unknown length) is not supported")
    if rate == 0:
        raise ValueError(f"{path}: sample rate 0")
    variable, first_block = _first_block(path, raw, pos)
    return FlacInfo(path, rate, channels, bits, total, min_block, max_block, bytes(info[18:34]), variable, first_block, pos,
                    memoryview(raw)[pos:])


def pcm_bytes_md5(pcm: np.ndarray, bits: int) -> bytes:
    """The MD5 STREAMINFO holds for the WAV data bytes `pcm` of a file of `bits` bits: over the samples as signed
    little-endian integers, so 8-bit data has its +128 offset undone."""
    data = pcm.tobytes() if bits != 8 else (pcm ^ np.uint8(0x80)).tobytes()
    return hashlib.md5(data).digest()


CONVERT_CHUNK_BYTES = 256 << 20       # FLAC bytes per convert_flac_to_wav decode call; a larger file goes alone


def convert_flac_to_wav(root, engine, chunk_bytes=CONVERT_CHUNK_BYTES):
    """The drop-in for tools/file/wav.py:176-195: every *.flac of root/, root/*/, root/*/*/, root/*/*/*/ and root/*/*/*/*/
    (the five depths the reference globs) becomes path[:-5] + ".wav" with the FLAC's rate, channels and bit depth, written
    by the standard `wave` module from the bytes the GPU decodes.  The files go through packed decode calls
    (vf_decode_flac_varlen) of at most `chunk_bytes` of FLAC each, in path order, so host and device memory stay bounded
    on a whole corpus.  Per chunk: every file is parsed and decoded, a non-zero STREAMINFO MD5 is checked with hashlib,
    each WAV is written and read back, and only then are the chunk's FLACs deleted, as the reference deletes each FLAC
    after converting it.  On any error the failing chunk's FLACs are kept and the error is raised; earlier chunks stay
    converted.  -> the WAV paths written.  The header bytes are not claimed to match sox's; the samples read back are the
    same."""
    paths = sorted(set(p for depth in range(5) for p in glob.glob(os.path.join(root, *["*"] * depth, "*.flac"))))
    chunks, size = [], 0
    for p in paths:
        n = os.path.getsize(p)
        if not chunks or size + n > chunk_bytes:
            chunks.append([])
            size = 0
        chunks[-1].append(p)
        size += n
    written = []
    for chunk in chunks:
        infos = [parse(p) for p in chunk]
        pcms = engine.decode_flac_pcm(infos)
        for w, pcm in zip(infos, pcms):
            if any(w.md5) and pcm_bytes_md5(pcm, w.bits) != w.md5:
                raise ValueError(f"{w.path}: decoded audio does not match the STREAMINFO MD5")
        for w, pcm in zip(infos, pcms):
            out = w.path[:-5] + ".wav"
            with wave.open(out, "wb") as f:
                f.setnchannels(w.channels)
                f.setsampwidth(w.bits // 8)
                f.setframerate(w.rate)
                f.writeframes(pcm.tobytes())
            with wave.open(out, "rb") as f:
                back = f.readframes(f.getnframes())
            if back != pcm.tobytes():
                raise ValueError(f"{out}: the written WAV does not read back to the decoded samples")
            written.append(out)
        for p in chunk:
            os.remove(p)
    return written
