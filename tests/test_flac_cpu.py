"""The FLAC oracle (oracle/flac.py) against its encoder and against a hand-assembled stream, and the host side of FLAC
reading (voicefixer_main_b200/flacfile.py): metadata, ID3v2, rejections and the engine= rule."""
import numpy as np
import pytest

from oracle import flac as F
from voicefixer_main_b200 import flacfile as FF


def test_round_trip_over_the_feature_matrix():
    for name, raw, x, bits, rate in F.feature_matrix(seed=0):
        info, y = F.decode(raw, name)
        assert (info["rate"], info["channels"], info["bits"], info["total"]) == (rate, x.shape[1], bits, x.shape[0]), name
        assert y.shape == x.shape and np.array_equal(y, x), name
        assert info["md5"] == F.md5_of(x, bits), name


def _crc8(data):                                   # RFC 9639 §9.1.8, written out again for the hand-assembled stream
    c = 0
    for b in data:
        c ^= b
        for _ in range(8):
            c = ((c << 1) ^ 0x07) & 0xFF if c & 0x80 else (c << 1) & 0xFF
    return c


def _crc16(data):                                  # §9.3
    c = 0
    for b in data:
        c ^= b << 8
        for _ in range(8):
            c = ((c << 1) ^ 0x8005) & 0xFFFF if c & 0x8000 else (c << 1) & 0xFFFF
    return c


def test_hand_assembled_left_side_frame(tmp_path):
    head = bytes.fromhex("664c6143")                              # "fLaC" (§6)
    meta = bytes([0x80, 0, 0, 34])                                  # last block, STREAMINFO, 34 bytes (§8.1)
    meta += (4).to_bytes(2, "big") + (4).to_bytes(2, "big")         # min / max block size 4 (§8.2)
    meta += bytes(6)                                                # min / max frame size unknown
    meta += (8000 << 44 | 1 << 41 | 7 << 36 | 4).to_bytes(8, "big")  # 8000 Hz, 2 channels, 8 bits, 4 samples
    meta += bytes(16)                                               # MD5 not set
    hdr = bytes([0xFF, 0xF8,                                        # sync code, fixed blocking (§9.1)
                 0x60,                                              # block size 0110: 8-bit size - 1 follows; rate 0000
                 0x82,                                              # left/side 1000, 8 bits 001, reserved 0
                 0x00,                                              # frame number 0, one byte (§9.1.5)
                 0x03])                                             # block size 4 (§9.1.6)
    hdr += bytes([_crc8(hdr)])                                      # §9.1.8
    bits = (
        "0" "001010" "0"              # left: FIXED order 2, no wasted bits (§9.2.1, §9.2.5)
        "00001010" "00001100"         # warm-up 10, 12 (8 bits)
        "00" "0000"                   # Rice 4-bit parameters, partition order 0 (§9.2.7)
        "1111" "00011"                # escape, 3-bit raw residuals (§9.2.7.1)
        "001" "110"                   # residuals 1, -2
        "0" "100010" "1"              # side: LPC order 3, wasted bits flag (§9.2.6, §9.2.2)
        "1"                           # k - 1 = 0 zeros then 1: one wasted bit; side is 9 - 1 = 8 bits
        "00000010" "11111111" "00000011"   # warm-up 2, -1, 3
        "0011"                        # precision 4 bits
        "00010"                       # shift 2
        "0010" "1111" "0001"          # coefficients 2, -1, 1
        "00" "0000" "0001"            # Rice, partition order 0, parameter 1
        "001" "1"                     # quotient 2, low bit 1: u = 5, residual -3 (zigzag, §9.2.7.3)
    )
    bits += "0" * (-len(bits) % 8)                                   # zero padding to a byte (§9.3)
    body = hdr + int(bits, 2).to_bytes(len(bits) // 8, "big")
    frame = body + _crc16(body).to_bytes(2, "big")
    # left: 10, 12, then 1 + (2*12 - 10) = 15, -2 + (2*15 - 12) = 16
    # side (before the shift): 2, -1, 3, then -3 + ((2*3 + -1*-1 + 1*2) >> 2) = -1; shifted: 4, -2, 6, -2
    # right = left - side: 6, 14, 9, 18
    want = np.array([[10, 6], [12, 14], [15, 9], [16, 18]])
    info, got = F.decode(head + meta + frame, "hand")
    assert np.array_equal(got, want)
    p = tmp_path / "hand.flac"
    p.write_bytes(head + meta + frame)
    w = FF.parse(str(p))
    assert (w.rate, w.channels, w.bits, w.total, w.variable, w.first_block) == (8000, 2, 8, 4, 0, 4)
    assert bytes(w.audio) == frame


@pytest.mark.parametrize("nbytes", range(1, 8))
def test_coded_numbers_of_every_length(nbytes):
    lo = [0, 1 << 7, 1 << 11, 1 << 16, 1 << 21, 1 << 26, 1 << 31][nbytes - 1]
    hi = [1 << 7, 1 << 11, 1 << 16, 1 << 21, 1 << 26, 1 << 31, 1 << 36][nbytes - 1] - 1
    for v in (lo, hi, (lo + hi) // 2):
        b = F.coded(v)
        assert len(b) == nbytes
        assert F.coded_number(b + bytes(8), 0) == (v, nbytes)
        info = dict(variable=1, channels=1, bits=16, rate=44100)
        head = bytearray([0xFF, 0xF9, 0x80, 0x08]) + b          # 256-sample block, mono, 16 bits
        head.append(F.crc8(head))
        h = F.parse_header(bytes(head) + bytes(4), 0, info)
        assert (h["number"], h["len"], h["block"]) == (v, 5 + nbytes, 256)


def test_every_rejection_raises_naming_the_file():
    for name, raw, code in F.rejections():
        with pytest.raises(ValueError, match=name) as e:
            F.decode(raw, name)
        if isinstance(e.value, F.FlacError):
            assert e.value.code == code, name


def _stream(**kw):
    return F.encode(F.signal(np.random.default_rng(0), 600, 2, 16), 44100, 16, blocks=256, **kw)


def test_host_rejections(tmp_path):
    raw = _stream()
    si = raw.index(b"fLaC") + 4

    def info(bits, total=600):                     # the stream with another STREAMINFO
        return raw[:si + 4] + F.streaminfo(44100, 2, bits, total, 256, 256, bytes(16)) + raw[si + 4 + 34:]

    cases = {
        "ogg": (b"OggS" + bytes(24) + b"\x7fFLAC" + raw, "Ogg FLAC"),
        "bits12": (info(12), "12-bit FLAC"),
        "bits20": (info(20), "20-bit FLAC"),
        "bits32": (info(32), "32-bit FLAC"),
        "total0": (info(16, 0), "total samples 0"),
        "nostreaminfo": (raw[:si] + bytes([0x84]) + raw[si + 1:], "STREAMINFO missing"),
        "truncated": (raw[:si + 20], "truncated metadata"),
        "notflac": (b"RIFF" + raw[4:], "not a FLAC file"),
    }
    for name, (data, why) in cases.items():
        p = tmp_path / f"{name}.flac"
        p.write_bytes(data)
        with pytest.raises(ValueError, match=f"{name}.flac: .*{why}"):
            FF.parse(str(p))


def test_id3_and_metadata_blocks_are_skipped(tmp_path):
    x = F.signal(np.random.default_rng(1), 700, 2, 24)
    plain = F.encode(x, 48000, 24, blocks=300)
    for footer in (False, True):
        raw = F.encode(x, 48000, 24, blocks=300, id3=(b"TALB" + bytes(30), footer),
                       metadata=[(1, bytes(64)), (4, b"\x03\x00\x00\x00abc" + bytes(4)), (6, bytes(50)), (9, b"x")])
        p = tmp_path / f"t{footer}.flac"
        p.write_bytes(raw)
        w = FF.parse(str(p))
        assert bytes(w.audio) == plain[plain.index(b"\xff\xf8"):]
        assert raw[w.audio_start:w.audio_start + 2] == b"\xff\xf8"
        assert (w.rate, w.channels, w.bits, w.total, w.md5) == (48000, 2, 24, 700, F.md5_of(x, 24))
        _, y = F.decode(raw, "t")
        assert np.array_equal(y, x)


def test_flac_needs_an_engine_and_is_chosen_by_content(tmp_path):
    from voicefixer_main_b200.handler import decode_wavs
    p = tmp_path / "named.wav"                                      # a FLAC under a .wav name is still FLAC
    p.write_bytes(_stream())
    with pytest.raises(ValueError, match="named.wav: FLAC decodes on the GPU .*engine="):
        decode_wavs([str(p)])


def test_ogg_is_rejected_with_its_reason_on_the_load_path(tmp_path):
    from voicefixer_main_b200.handler import decode_wavs
    page = b"OggS" + bytes(24)                                      # a 28-byte page header (its fields unused here)
    for stem, packet, what in (("flac", b"\x7fFLAC\x01\x00", "Ogg FLAC"), ("vorbis", b"\x01vorbis", "an Ogg stream")):
        p = tmp_path / f"{stem}.ogg"
        p.write_bytes(page + packet + bytes(64))
        with pytest.raises(ValueError, match=f"{stem}.ogg: {what} is not supported"):
            decode_wavs([str(p)])
