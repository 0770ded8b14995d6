"""FLAC (RFC 9639) restated from the RFC for the tests: an integer decoder, and an encoder able to emit every feature
vf_decode_flac_varlen decodes.  Test infrastructure only; the library reads FLAC with voicefixer_main_b200/flacfile.py and
csrc/flac.cu.

decode(raw, name) -> (FlacInfo-like dict, int64 samples [total, channels]) follows the same rules and rejections as the
library (ValueError naming `name`; FlacError with the VF_FLAC_E* reason for a frame), with its own metadata parser
(`metadata`) and frame decoder, independent of voicefixer_main_b200/flacfile.py.  Sections cited are RFC 9639's.

encode(x, rate, bits, ...) writes a stream from int samples x [n, channels] with per-frame and per-subframe choices
(every subframe type and order, wasted bits, channel assignments, both Rice codings, escapes, partition orders, block size
and rate codes, fixed or variable blocking, metadata blocks, an ID3v2 tag).  encode_fast(x, rate, bits) is a vectorised
FIXED-2 encoder with per-partition Rice parameters, for realistic sets of files.
"""
import hashlib

import numpy as np

RATES = {1: 88200, 2: 176400, 3: 192000, 4: 8000, 5: 16000, 6: 22050, 7: 24000, 8: 32000, 9: 44100, 10: 48000, 11: 96000}
BITS = {1: 8, 2: 12, 4: 16, 5: 20, 6: 24, 7: 32}
FIXED = ((), (1,), (2, -1), (3, -3, 1), (4, -6, 4, -1))        # §9.2.5

# VF_FLAC_E* of include/b200vf.h
ENOSYNC, ERESERVED, EMISMATCH, ECRC8, ESUBFRAME, EPARTITION, ETRUNCATED, ECRC16, ERANGE, ESEQUENCE, ELENGTH = range(1, 12)


# ------------------------------------------------------------------------------------------------------------ checksums
def crc8(data) -> int:
    """§9.1.8: polynomial 0x07, initial value 0."""
    c = 0
    for b in bytes(data):
        c ^= b
        for _ in range(8):
            c = ((c << 1) ^ (0x07 if c & 0x80 else 0)) & 0xFF
    return c


def _crc16_tables():
    t0 = np.zeros(256, np.int64)
    for i in range(256):
        c = i << 8
        for _ in range(8):
            c = ((c << 1) ^ (0x8005 if c & 0x8000 else 0)) & 0xFFFF
        t0[i] = c
    tables = [t0]                               # tables[d][b]: the CRC of byte b followed by d zero bytes
    for _ in range(255):
        t = tables[-1]
        tables.append(((t << 8) & 0xFFFF) ^ t0[t >> 8])
    return np.stack(tables)


_T16 = None


def crc16(data) -> int:
    """§9.3: polynomial 0x8005, initial value 0, vectorised over 256-byte blocks (leading zero bytes do not change it)."""
    global _T16
    if _T16 is None:
        _T16 = _crc16_tables()
    m = np.frombuffer(bytes(data), np.uint8)
    m = np.concatenate([np.zeros((-len(m)) % 256, np.uint8), m]).reshape(-1, 256)
    blocks = np.bitwise_xor.reduce(_T16[np.arange(255, -1, -1)[None, :], m], axis=1)
    c = 0
    for b in blocks.tolist():
        c = int(_T16[255][c >> 8] ^ _T16[254][c & 0xFF]) ^ b
    return c


def md5_of(x, bits) -> bytes:
    """The STREAMINFO MD5 of int samples x [n, channels]: signed little-endian, bits / 8 bytes each, interleaved."""
    w = bits // 8
    v = np.asarray(x, np.int64).reshape(-1) & ((1 << bits) - 1)
    b = np.stack([(v >> (8 * i)) & 0xFF for i in range(w)], axis=1).astype(np.uint8)
    return hashlib.md5(b.tobytes()).digest()


def wav_bytes(x, bits) -> bytes:
    """The WAV data chunk of int samples x [n, channels]: u8 as v + 128, s16 / s24 little-endian."""
    v = np.asarray(x, np.int64).reshape(-1) + (128 if bits == 8 else 0)
    v &= (1 << bits) - 1
    return np.stack([(v >> (8 * i)) & 0xFF for i in range(bits // 8)], axis=1).astype(np.uint8).tobytes()


# -------------------------------------------------------------------------------------------------------------- decoder
class _Bits:
    def __init__(self, raw, pos_bits, limit_bits):
        self.raw, self.pos, self.limit = raw, pos_bits, limit_bits

    def read(self, n):
        if n == 0:
            return 0
        if self.pos + n > self.limit:
            raise EOFError
        b0, b1 = self.pos >> 3, (self.pos + n + 7) >> 3
        v = int.from_bytes(self.raw[b0:b1], "big")
        v >>= (b1 * 8) - (self.pos + n)
        self.pos += n
        return v & ((1 << n) - 1)

    def signed(self, n):
        v = self.read(n)
        return v - (1 << n) if n and v >> (n - 1) else v

    def unary(self):                            # zeros ended by a 1
        q = 0
        while True:
            if self.pos >= self.limit:
                raise EOFError
            if self.pos & 7 == 0 and self.raw[self.pos >> 3] == 0:
                q += 8
                self.pos += 8
                continue
            if self.read(1):
                return q
            q += 1


class FlacError(ValueError):
    def __init__(self, name, code, at):
        self.code, self.at = code, at
        super().__init__(f"{name}: FLAC error {code} at byte {at}")


def coded_number(raw, pos):
    """§9.1.5: the UTF-8-style number at raw[pos] -> (value, length) or None when it is not well formed."""
    b0 = raw[pos]
    for extra, top, mask in ((0, 0x80, 0x7F), (1, 0xE0, 0x1F), (2, 0xF0, 0x0F), (3, 0xF8, 0x07), (4, 0xFC, 0x03),
                             (5, 0xFE, 0x01), (6, 0xFF, 0x00)):
        if b0 < top:
            break
    else:
        return None
    if 0x80 <= b0 < 0xC0 or pos + 1 + extra > len(raw):
        return None
    v = b0 & mask
    for c in raw[pos + 1:pos + 1 + extra]:
        if c & 0xC0 != 0x80:
            return None
        v = (v << 6) | (c & 0x3F)
    return v, 1 + extra


def parse_header(raw, pos, info):
    """§9.1: the frame header at raw[pos] -> dict (block, channels, assign, number, len) or raise _Reject(code)."""
    if len(raw) - pos < 6:
        raise _Reject(ETRUNCATED)
    if raw[pos] != 0xFF or raw[pos + 1] & 0xFE != 0xF8:
        raise _Reject(ENOSYNC)
    if raw[pos + 1] & 1 != info["variable"]:
        raise _Reject(EMISMATCH)
    bs_code, rate_code = raw[pos + 2] >> 4, raw[pos + 2] & 15
    ch_code, bits_code = raw[pos + 3] >> 4, (raw[pos + 3] >> 1) & 7
    if bs_code == 0 or rate_code == 15 or ch_code > 10 or bits_code == 3 or raw[pos + 3] & 1:
        raise _Reject(ERESERVED)
    num = coded_number(raw, pos + 4)
    if num is None:
        raise _Reject(ERESERVED if len(raw) - pos - 4 > 7 else ETRUNCATED)
    number, n = num[0], 4 + num[1]
    tail = {6: 1, 7: 2}.get(bs_code, 0) + (1 if rate_code == 12 else 2 if rate_code in (13, 14) else 0)
    if len(raw) < pos + n + tail + 1:
        raise _Reject(ETRUNCATED)
    p = pos + n
    if bs_code == 1:
        block = 192
    elif bs_code <= 5:
        block = 576 << (bs_code - 2)
    elif bs_code == 6:
        block, p = raw[p] + 1, p + 1
    elif bs_code == 7:
        block, p = int.from_bytes(raw[p:p + 2], "big") + 1, p + 2
    else:
        block = 256 << (bs_code - 8)
    rate = 0
    if 1 <= rate_code <= 11:
        rate = RATES[rate_code]
    elif rate_code == 12:
        rate, p = raw[p] * 1000, p + 1
    elif rate_code == 13:
        rate, p = int.from_bytes(raw[p:p + 2], "big"), p + 2
    elif rate_code == 14:
        rate, p = int.from_bytes(raw[p:p + 2], "big") * 10, p + 2
    if crc8(raw[pos:p]) != raw[p]:
        raise _Reject(ECRC8)
    channels = ch_code + 1 if ch_code < 8 else 2
    if (channels != info["channels"] or (bits_code and BITS[bits_code] != info["bits"]) or (rate_code and rate != info["rate"])
            or block > 65535):
        raise _Reject(EMISMATCH)
    return dict(block=block, channels=channels, assign=ch_code, number=number, len=p + 1 - pos)


class _Reject(Exception):
    def __init__(self, code):
        self.code = code


def _fits(v, bits):
    return -(1 << (bits - 1)) <= v < (1 << (bits - 1))


def decode_subframe(r, block, bps):
    """§9.2: one subframe -> (samples before the wasted-bits shift, wasted bits k)."""
    head = r.read(8)
    if head & 0x80:
        raise _Reject(ESUBFRAME)
    kind = (head >> 1) & 0x3F
    k = 0
    if head & 1:                                       # §9.2.2
        k = r.unary() + 1
        if k >= bps:
            raise _Reject(ESUBFRAME)
    bps -= k
    if kind == 0:                                      # CONSTANT §9.2.3
        return [r.signed(bps)] * block, k
    if kind == 1:                                      # VERBATIM §9.2.4
        return [r.signed(bps) for _ in range(block)], k
    if 8 <= kind <= 12:
        order, coefs, shift = kind - 8, None, 0
    elif kind >= 32:
        order = kind - 31
    else:
        raise _Reject(ESUBFRAME)
    if order > block:
        raise _Reject(EPARTITION)
    s = [r.signed(bps) for _ in range(order)]
    if kind >= 32:                                     # LPC §9.2.6
        precision = r.read(4) + 1
        if precision == 16:
            raise _Reject(ESUBFRAME)
        shift = r.signed(5)
        if shift < 0:
            raise _Reject(ESUBFRAME)
        coefs = [r.signed(precision) for _ in range(order)]
    else:
        coefs = list(FIXED[order])
    method = r.read(2)                                 # §9.2.7
    if method > 1:
        raise _Reject(ESUBFRAME)
    pbits, escape = (5, 31) if method else (4, 15)
    porder = r.read(4)
    if block % (1 << porder) or (block >> porder) < order:
        raise _Reject(EPARTITION)
    per = block >> porder
    for part in range(1 << porder):
        n = per - (order if part == 0 else 0)
        param = r.read(pbits)
        if param == escape:
            width = r.read(5)
            s.extend(r.signed(width) for _ in range(n))
        else:
            for _ in range(n):
                u = (r.unary() << param) | r.read(param)
                if u >> 32:
                    raise _Reject(ERANGE)
                s.append((u >> 1) ^ -(u & 1))
    for i in range(order, block):
        acc = sum(c * s[i - 1 - j] for j, c in enumerate(coefs))
        v = s[i] + (acc >> shift)
        if not _fits(v, bps):
            raise _Reject(ERANGE)
        s[i] = v
    return s, k


def decode_frame(raw, pos, info, h):
    """The frame at raw[pos] with header h -> (int samples [block, channels], end byte)."""
    r = _Bits(raw, 8 * (pos + h["len"]), 8 * len(raw))
    side = {8: 1, 9: 0, 10: 1}.get(h["assign"], -1)
    ch = []
    try:
        for c in range(h["channels"]):
            s, k = decode_subframe(r, h["block"], info["bits"] + (c == side))
            ch.append([v << k for v in s])
    except EOFError:
        raise _Reject(ETRUNCATED)
    end = ((r.pos + 7) >> 3) + 2
    if end > len(raw):
        raise _Reject(ETRUNCATED)
    if crc16(raw[pos:end - 2]) != int.from_bytes(raw[end - 2:end], "big"):
        raise _Reject(ECRC16)
    x = np.array(ch, dtype=np.int64).T.copy()
    if h["assign"] == 8:                               # left / side
        x[:, 1] = x[:, 0] - x[:, 1]
    elif h["assign"] == 9:                             # side / right
        x[:, 0] = x[:, 0] + x[:, 1]
    elif h["assign"] == 10:                            # mid / side
        mid = (x[:, 0] << 1) | (x[:, 1] & 1)
        x[:, 0], x[:, 1] = (mid + x[:, 1]) >> 1, (mid - x[:, 1]) >> 1
    if not all(_fits(int(v), info["bits"]) for v in (x.min(), x.max())):
        raise _Reject(ERANGE)
    return x, end


def metadata(raw, name="<stream>"):
    """§8, restated apart from the library's parser: skip an ID3v2 tag (10 bytes, the syncsafe size, 10 more with the
    footer flag), check `fLaC`, walk the metadata blocks and read STREAMINFO -> (info dict, offset of the first frame).
    ValueError naming `name` for what the host side rejects."""
    pos = 0
    if raw[:3] == b"ID3":
        if len(raw) < 10:
            raise ValueError(f"{name}: truncated ID3v2 tag")
        pos = 10 + sum((raw[6 + i] & 0x7F) << (21 - 7 * i) for i in range(4)) + (10 if raw[5] & 0x10 else 0)
    if raw[pos:pos + 4] == b"OggS":
        raise ValueError(f"{name}: Ogg is not supported")
    if raw[pos:pos + 4] != b"fLaC":
        raise ValueError(f"{name}: not a FLAC file")
    pos += 4
    si, last = None, 0
    while not last:
        if pos + 4 > len(raw):
            raise ValueError(f"{name}: truncated metadata")
        last, kind, size = raw[pos] >> 7, raw[pos] & 0x7F, int.from_bytes(raw[pos + 1:pos + 4], "big")
        if pos + 4 + size > len(raw):
            raise ValueError(f"{name}: truncated metadata")
        if si is None:
            if kind != 0 or size != 34:
                raise ValueError(f"{name}: STREAMINFO missing or not the first metadata block")
            si = raw[pos + 4:pos + 38]
        elif kind == 127:
            raise ValueError(f"{name}: forbidden metadata block type 127")
        pos += 4 + size
    v = int.from_bytes(si[10:18], "big")
    info = dict(min_block=int.from_bytes(si[0:2], "big"), max_block=int.from_bytes(si[2:4], "big"), rate=v >> 44,
                channels=(v >> 41 & 7) + 1, bits=(v >> 36 & 31) + 1, total=v & ((1 << 36) - 1), md5=bytes(si[18:34]))
    if info["bits"] not in (8, 16, 24):
        raise ValueError(f"{name}: {info['bits']}-bit FLAC is not supported")
    if info["total"] == 0:
        raise ValueError(f"{name}: total samples 0 (unknown length) is not supported")
    if info["rate"] == 0:
        raise ValueError(f"{name}: sample rate 0")
    if len(raw) < pos + 2 or raw[pos] != 0xFF or raw[pos + 1] & 0xFE != 0xF8:
        raise ValueError(f"{name}: no frame sync code after the metadata")
    info["variable"] = raw[pos + 1] & 1
    return info, pos


def decode(raw, name="<stream>"):
    """(info, int64 samples [total, channels]) of the FLAC stream `raw`; ValueError naming `name` for what the host side
    rejects, FlacError (a ValueError) with the VF_FLAC_E* code and the byte of the first bad frame for what the device
    rejects."""
    raw = bytes(raw)
    info, start = metadata(raw, name)
    audio = raw[start:]
    try:
        info["first_block"] = parse_header(audio, 0, info)["block"]
    except _Reject as e:
        raise FlacError(name, e.code, start) from None
    total, variable, first_block = info["total"], info["variable"], info["first_block"]
    out, pos, done, k = [], 0, 0, 0
    while done < total:
        if pos >= len(audio):
            raise FlacError(name, ELENGTH, start + pos)
        try:
            h = parse_header(audio, pos, info)
            x, end = decode_frame(audio, pos, info, h)
        except _Reject as e:
            raise FlacError(name, e.code, start + pos) from None
        if h["number"] != (done if variable else k):
            raise FlacError(name, ESEQUENCE, start + pos)
        if not variable and (h["block"] > first_block or (h["block"] < first_block and done + h["block"] < total)):
            raise FlacError(name, ESEQUENCE, start + pos)
        if done + h["block"] > total:
            raise FlacError(name, ELENGTH, start + pos)
        out.append(x)
        done += h["block"]
        pos = end
        k += 1
    return info, np.concatenate(out)


# -------------------------------------------------------------------------------------------------------------- encoder
def pack_bits(values, widths) -> bytes:
    """Big-endian bit fields (value, width >= 0, width <= 64, value already < 2^width) -> bytes, zero-padded to a byte."""
    v = np.asarray(values, dtype=np.uint64)
    w = np.asarray(widths, dtype=np.int64)
    keep = w > 0
    v, w = v[keep], w[keep]
    total = int(w.sum())
    if total == 0:
        return b""
    starts = np.cumsum(w) - w
    rep_v = np.repeat(v, w)
    j = np.arange(total, dtype=np.int64) - np.repeat(starts, w)
    sh = (np.repeat(w, w) - 1 - j).astype(np.uint64)
    bits = ((rep_v >> sh) & np.uint64(1)).astype(np.uint8)
    return np.packbits(bits).tobytes()


class _Writer:
    def __init__(self):
        self.v, self.w = [], []

    def put(self, value, width):
        self.v.append(int(value) & ((1 << width) - 1) if width else 0)
        self.w.append(width)

    def unary(self, q):                            # q zeros then a 1
        while q >= 63:
            self.put(0, 63)
            q -= 63
        self.put(1, q + 1)

    def put_arrays(self, values, widths):
        self.v.extend(np.asarray(values, np.uint64).tolist())
        self.w.extend(np.asarray(widths, np.int64).tolist())

    def bytes(self):
        return pack_bits(np.array(self.v, dtype=np.uint64), np.array(self.w, dtype=np.int64))


def coded(value, nbytes=None) -> bytes:
    """§9.1.5: value as a UTF-8-style number of the shortest length (or of `nbytes` bytes)."""
    if nbytes is None:
        nbytes = next(n for n, lim in enumerate((7, 11, 16, 21, 26, 31, 36), 1) if value < 1 << lim)
    if nbytes == 1:
        return bytes([value])
    lead_bits = 7 - nbytes if nbytes < 7 else 0
    out = []
    for _ in range(nbytes - 1):
        out.append(0x80 | (value & 0x3F))
        value >>= 6
    assert value < 1 << max(lead_bits, 0) or (nbytes == 7 and value == 0)
    lead = ((0xFF << (8 - nbytes)) & 0xFF) | value
    return bytes([lead] + out[::-1])


def _residual(w, r, order, block, method=0, porder=0, params=None, escape=None):
    """§9.2.7: residuals r (block - order values) with `porder` partitions; params: per-partition Rice parameters (None:
    the best of each partition); escape: {partition: raw bit width} for escaped partitions."""
    escape = escape or {}
    assert block % (1 << porder) == 0 and block >> porder >= order, "invalid partitioning"
    pbits, esc = (5, 31) if method else (4, 15)
    w.put(method, 2)
    w.put(porder, 4)
    per = block >> porder
    i = 0
    for part in range(1 << porder):
        n = per - (order if part == 0 else 0)
        seg = np.asarray(r[i:i + n], np.int64)
        i += n
        if part in escape:
            w.put(esc, pbits)
            w.put(escape[part], 5)
            for v in seg.tolist():
                w.put(v, escape[part])
            continue
        u = ((seg << 1) ^ (seg >> 63)).astype(np.uint64)      # zigzag
        if params is None:
            k = best_param(u, esc - 1)
        else:
            k = params[part]
        w.put(k, pbits)
        q = (u >> np.uint64(k)).astype(np.int64)
        if len(u) and q.max() < 60 - k:
            w.put_arrays((np.uint64(1) << np.uint64(k)) | (u & np.uint64((1 << k) - 1)), q + 1 + k)
        else:
            for uu in u.tolist():
                w.unary(uu >> k)
                w.put(uu & ((1 << k) - 1), k)


def best_param(u, kmax):
    """The Rice parameter of least cost for zigzag values u."""
    if len(u) == 0:
        return 0
    u = u.astype(np.float64)
    costs = [(u / (1 << k)).astype(np.int64).sum() + len(u) * (1 + k) for k in range(kmax + 1)]
    return int(np.argmin(costs))


def _subframe(w, s, bps, spec):
    """§9.2: one subframe of int samples s (the channel, before any wasted-bits removal) at sample size bps."""
    kind = spec.get("type", "fixed")
    k = spec.get("wasted", 0)
    s = np.asarray(s, np.int64)
    if k:
        assert not (s & ((1 << k) - 1)).any()
        s = s >> k
    b = bps - k
    block = len(s)
    codes = {"constant": 0, "verbatim": 1}
    if kind in codes:
        code = codes[kind]
    elif kind == "fixed":
        code = 8 + spec.get("order", min(2, block))
    else:
        code = 31 + spec["order"]
    w.put(code << 1 | (1 if k else 0), 8)
    if k:
        w.unary(k - 1)
    if kind == "constant":
        assert (s == s[0]).all()
        w.put(s[0], b)
        return
    if kind == "verbatim":
        for v in s.tolist():
            w.put(v, b)
        return
    order = spec.get("order", min(2, block))
    for v in s[:order].tolist():
        w.put(v, b)
    if kind == "fixed":
        coefs, shift = FIXED[order], 0
    else:
        precision, shift, coefs = spec["precision"], spec["shift"], spec["coefs"]
        w.put(precision - 1, 4)
        w.put(shift, 5)
        for c in coefs:
            w.put(c, precision)
    acc = np.zeros(block - order, np.int64)
    for j, c in enumerate(coefs):
        acc += c * s[order - 1 - j:block - 1 - j]
    r = s[order:] - (acc >> shift)
    _residual(w, r, order, block, spec.get("method", 0), spec.get("porder", 0), spec.get("params"), spec.get("escape"))


def frame_bytes(x, number, bits, assign=None, subframes=None, variable=False, bs_code=None, rate_code=0, rate=None,
                bits_code=None, number_bytes=None):
    """One frame (§9) of int samples x [block, channels]: its header codes (None: the usual choice) and subframe specs."""
    block, C = x.shape
    if assign is None:
        assign = C - 1
    if bs_code is None:
        common = {192: 1, 576: 2, 1152: 3, 2304: 4, 4608: 5, 256: 8, 512: 9, 1024: 10, 2048: 11, 4096: 12, 8192: 13,
                  16384: 14, 32768: 15}
        bs_code = common.get(block, 6 if block <= 256 else 7)
    if bits_code is None:
        bits_code = {8: 1, 16: 4, 24: 6}[bits]
    head = bytearray([0xFF, 0xF8 | int(variable), bs_code << 4 | rate_code, assign << 4 | bits_code << 1])
    head += coded(number, number_bytes)
    if bs_code == 6:
        head += bytes([block - 1])
    elif bs_code == 7:
        head += (block - 1).to_bytes(2, "big")
    if rate_code == 12:
        head += bytes([rate // 1000])
    elif rate_code == 13:
        head += rate.to_bytes(2, "big")
    elif rate_code == 14:
        head += (rate // 10).to_bytes(2, "big")
    head.append(crc8(head))
    ch = [x[:, c].astype(np.int64) for c in range(C)]
    side = -1
    if assign == 8:
        ch[1], side = ch[0] - ch[1], 1
    elif assign == 9:
        ch[0], side = ch[0] - ch[1], 0
    elif assign == 10:
        ch[0], ch[1], side = (ch[0] + ch[1]) >> 1, ch[0] - ch[1], 1
    w = _Writer()
    subframes = subframes or [{}] * C
    for c in range(C):
        _subframe(w, ch[c], bits + (c == side), subframes[c])
    body = bytes(head) + w.bytes()
    return body + crc16(body).to_bytes(2, "big")


def streaminfo(rate, channels, bits, total, min_block, max_block, md5, min_frame=0, max_frame=0) -> bytes:
    """§8.2: the 34-byte STREAMINFO block body."""
    packed = rate << 44 | (channels - 1) << 41 | (bits - 1) << 36 | total
    return (min_block.to_bytes(2, "big") + max_block.to_bytes(2, "big") + min_frame.to_bytes(3, "big") +
            max_frame.to_bytes(3, "big") + packed.to_bytes(8, "big") + md5)


def container(frames, rate, channels, bits, total, min_block, max_block, md5, metadata=(), id3=None) -> bytes:
    """fLaC, STREAMINFO, then `metadata` blocks (type, body), then the frames; optionally an ID3v2 tag first
    (id3 = (body bytes, footer flag))."""
    blocks = [(0, streaminfo(rate, channels, bits, total, min_block, max_block, md5))] + list(metadata)
    out = bytearray()
    if id3 is not None:
        body, footer = id3
        n = len(body)
        out += b"ID3\x04\x00" + bytes([0x10 if footer else 0]) + bytes([(n >> 21) & 0x7F, (n >> 14) & 0x7F, (n >> 7) & 0x7F,
                                                                        n & 0x7F]) + body
        if footer:
            out += b"3DI\x04\x00\x10" + out[6:10]
    out += b"fLaC"
    for i, (kind, body) in enumerate(blocks):
        out += bytes([(0x80 if i == len(blocks) - 1 else 0) | kind]) + len(body).to_bytes(3, "big") + body
    return bytes(out) + b"".join(frames)


def encode(x, rate, bits, blocks=4096, variable=False, frame=None, metadata=(), id3=None, md5=True, rate_code=0):
    """A FLAC stream of int samples x [n, channels].  blocks: a block size or a list of them (summing to n); frame(k,
    start, block) -> frame_bytes keyword overrides for frame k (assign, subframes, bs_code, rate_code, bits_code, ...)."""
    x = np.asarray(x, np.int64)
    n, C = x.shape
    if isinstance(blocks, int):
        blocks = [blocks] * (n // blocks) + ([n % blocks] if n % blocks else [])
    assert sum(blocks) == n
    frames, start = [], 0
    for k, b in enumerate(blocks):
        opts = dict(rate_code=rate_code, rate=rate)
        if frame is not None:
            opts.update(frame(k, start, b) or {})
        frames.append(frame_bytes(x[start:start + b], start if variable else k, bits, variable=variable, **opts))
        start += b
    digest = md5_of(x, bits) if md5 else bytes(16)
    return container(frames, rate, C, bits, n, min(blocks), max(blocks), digest, metadata, id3)


def encode_fast(x, rate, bits, block=4096, porder=4):
    """A fixed-blocking stream of independent FIXED-2 subframes with per-partition Rice parameters, vectorised per frame."""
    x = np.asarray(x, np.int64)
    n, C = x.shape
    frames = []
    for k, start in enumerate(range(0, n, block)):
        seg = x[start:start + block]
        b = len(seg)
        po = porder
        while po and (b % (1 << po) or (b >> po) < 2):
            po -= 1
        frames.append(frame_bytes(seg, k, bits, subframes=[{"type": "fixed", "order": 2, "porder": po}] * C))
    return container(frames, rate, C, bits, n, min(block, n), block, md5_of(x, bits))


# --------------------------------------------------------------------------------------------------------- test streams
def signal(rng, n, channels, bits, k=0):
    """Seeded int samples [n, channels] of `bits` bits: a clipped random walk with its low k bits zero (wasted bits)."""
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    step = max(1, 1 << max(0, bits - 7))
    x = np.cumsum(rng.integers(-step, step + 1, (n, channels)), axis=0) + rng.integers(lo // 4, hi // 4 + 1, (1, channels))
    x = np.clip(x, lo, hi)
    return (x >> k) << k


def _lpc(rng, order, precision, shift, bits):
    """LPC coefficients of `precision` bits small enough that a prediction of `bits`-bit samples fits 31 bits."""
    lim = min((1 << (precision - 1)) - 1, max(1, (1 << (29 + shift - bits)) // order))
    c = rng.integers(-lim, lim + 1, order)
    if precision > 1 and order == 1 and lim == (1 << (precision - 1)) - 1:
        c[0] = -(1 << (precision - 1))                 # the most negative coefficient
    return c.tolist()


def feature_matrix(seed=0):
    """Seeded streams over every feature the decoder supports -> list of (name, raw, x, bits, rate)."""
    rng = np.random.default_rng(seed)
    out = []

    def add(name, x, rate, bits, **kw):
        out.append((name, encode(x, rate, bits, **kw), x, bits, rate))

    # every subframe type and order, with and without wasted bits, at each depth
    for bits in (8, 16, 24):
        specs = [{"type": "constant"}, {"type": "verbatim"}] + [{"type": "fixed", "order": o} for o in range(5)] + \
                [{"type": "lpc", "order": o, "precision": 12, "shift": 9} for o in (1, 2, 3, 8, 17, 32)]
        for k in (0, 2):
            x = signal(rng, 300 * len(specs), 1, bits, k)
            for i, s in enumerate(specs):
                if s["type"] == "constant":
                    x[i * 300:(i + 1) * 300] = x[i * 300]
                if s["type"] == "lpc":
                    s["coefs"] = _lpc(rng, s["order"], s["precision"], s["shift"], bits)
            add(f"subframes-{bits}bit-wasted{k}", x, 44100, bits, blocks=300,
                frame=lambda f, st, b, specs=specs, k=k: {"subframes": [dict(specs[f], wasted=k)]})
    # LPC precisions 1 .. 15 with shifts 0 .. 15
    combos = [(p, sh) for p in range(1, 16) for sh in range(16)]
    x = signal(rng, 64 * len(combos), 1, 16)
    add("lpc-precision-shift", x, 16000, 16, blocks=64, frame=lambda f, st, b: {"subframes": [
        {"type": "lpc", "order": 2, "precision": combos[f][0], "shift": combos[f][1],
         "coefs": _lpc(np.random.default_rng(f), 2, combos[f][0], combos[f][1], 16), "porder": 1}]})
    # Rice and Rice2, escapes (0-bit ones included), partition orders 0 .. 8
    res = []
    for method in (0, 1):
        for po in range(9):
            res.append({"type": "fixed", "order": 1, "method": method, "porder": po})
        res.append({"type": "fixed", "order": 2, "method": method, "porder": 3, "escape": {0: 17, 5: 9}})
        res.append({"type": "verbatim"})
    x = signal(rng, 512 * len(res), 1, 16)
    for i, s in enumerate(res):
        if s.get("escape"):
            x[i * 512 + 5 * 64 - 1:i * 512 + 6 * 64] = x[i * 512 + 5 * 64 - 1]   # FIXED-1 residuals of 0: a 0-bit escape
            s = dict(s, type="fixed", order=1, escape={0: 17, 5: 0})
            res[i] = s
    add("residual-codings", x, 22050, 16, blocks=512, frame=lambda f, st, b: {"subframes": [res[f]]})
    # channel assignments: independent 1 .. 8 channels, left/side, side/right, mid/side, with wasted bits and LPC
    for c in range(1, 9):
        add(f"independent-{c}ch", signal(rng, 1500, c, 24), 48000, 24, blocks=576)
    for assign in (8, 9, 10):
        for bits in (8, 16, 24):
            x = signal(rng, 2000, 2, bits, 2)              # multiples of 4: mid and side keep one wasted bit
            x[:, 1] = np.clip(x[:, 0] + (signal(rng, 2000, 1, bits, 2)[:, 0] >> 5 << 2), -(1 << (bits - 1)),
                              (1 << (bits - 1)) - 4)
            add(f"assign{assign}-{bits}bit", x, 44100, bits, blocks=700, frame=lambda f, st, b, a=assign, bits=bits: {
                "assign": a, "subframes": [{"type": "fixed", "order": 2, "wasted": 1},
                                           {"type": "lpc", "order": 4, "precision": 10, "shift": 8, "wasted": 1,
                                            "coefs": _lpc(np.random.default_rng(f), 4, 10, 8, bits + 1)}]})
    # every block size code (uncommon 8- and 16-bit sizes, a short last frame) and every rate code, fixed and variable
    sizes = [192, 576, 1152, 2304, 4608, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 100, 300, 65535, 77]
    x = signal(rng, sum(sizes), 2, 16)
    add("block-codes-variable", x, 44100, 16, blocks=sizes, variable=True)
    add("block-sizes-explicit", x[:1000], 44100, 16, blocks=[256, 256, 256, 232],
        frame=lambda f, st, b: {"bs_code": 6 if f % 2 else 7})
    rates = {0: 12345, 1: 88200, 2: 176400, 3: 192000, 4: 8000, 5: 16000, 6: 22050, 7: 24000, 8: 32000, 9: 44100,
             10: 48000, 11: 96000, 12: 37000, 13: 65535, 14: 123450}
    for code, rate in rates.items():
        add(f"rate-code{code}", signal(rng, 700, 1, 8), rate, 8, blocks=256, rate_code=code, frame=lambda f, st, b: {
            "bits_code": 0 if f == 1 else None})
    # metadata blocks and an ID3v2 tag before fLaC
    add("metadata-id3", signal(rng, 1000, 2, 16), 44100, 16, blocks=512,
        metadata=[(1, bytes(100)), (2, b"abcd" + bytes(8)), (3, bytes(18)), (4, b"\x05\x00\x00\x00vf-fx\x00\x00\x00\x00"),
                  (5, bytes(30)), (6, bytes(40)), (100, b"reserved")], id3=(b"TIT2" + bytes(20), True))
    return out


def _one_frame(x, bits, subframes=None, **kw):
    """A one-frame stream of int samples x [block, channels] -> (raw, offset of the frame, its header length)."""
    raw = encode(x, 8000, bits, blocks=[len(x)], frame=lambda k, s, b: dict(kw, subframes=subframes))
    at = raw.index(b"\xff\xf8")
    return bytearray(raw), at, parse_header(raw[at:], 0, dict(variable=0, channels=x.shape[1], bits=bits, rate=8000))["len"]


def _refresh(raw, at, hlen):
    """Recompute the CRC-8 and CRC-16 of the one frame at raw[at:] after a patch."""
    raw[at + hlen - 1] = crc8(raw[at:at + hlen - 1])
    raw[-2:] = crc16(raw[at:-2]).to_bytes(2, "big")
    return bytes(raw)


def rejections(seed=0):
    """Streams every frame-level rejection applies to -> list of (name, raw, VF_FLAC_E* code).  Each is one bad thing
    in an otherwise valid stream, its checksums recomputed unless the checksum is the bad thing."""
    rng = np.random.default_rng(seed)
    x = signal(rng, 100, 1, 8)
    out = []

    def patched(name, code, byte, value, mask=0xFF, spec=None, sub=False):
        """Bits `mask` of byte `byte` of the frame (of its first subframe with sub=True) set to `value`."""
        raw, at, hlen = _one_frame(x, 8, subframes=[spec or {"type": "verbatim"}])
        i = at + byte + (hlen if sub else 0)
        raw[i] = (raw[i] & ~mask & 0xFF) | value
        out.append((name, _refresh(raw, at, hlen), code))

    patched("block-size-0000", ERESERVED, 2, 0x00, 0xF0)
    patched("rate-1111", ERESERVED, 2, 0x0F, 0x0F)
    for ch in range(11, 16):
        patched(f"channels-{ch:04b}", ERESERVED, 3, ch << 4, 0xF0)
    patched("bits-011", ERESERVED, 3, 0b0110, 0x0E)
    patched("header-reserved-bit", ERESERVED, 3, 1, 1)
    patched("frame-channels", EMISMATCH, 3, 0x10, 0xF0)
    patched("frame-bits", EMISMATCH, 3, 0b1000, 0x0E)
    patched("frame-rate", EMISMATCH, 2, 0x04, 0x0F)              # 8 kHz is STREAMINFO's; code 0100 says 8 kHz ...
    out.pop()
    patched("frame-rate", EMISMATCH, 2, 0x05, 0x0F)              # ... 0101 says 16 kHz
    for t in (2, 4, 7, 13, 31):
        patched(f"subframe-type-{t}", ESUBFRAME, 0, t << 1, 0x7E, sub=True)
    patched("subframe-zero-bit", ESUBFRAME, 0, 0x80, 0x80, sub=True)
    lpc = {"type": "lpc", "order": 1, "precision": 4, "shift": 3, "coefs": [5]}
    patched("lpc-precision-1111", ESUBFRAME, 2, 0xF0, 0xF0, spec=lpc, sub=True)   # after the 8-bit warm-up sample
    patched("lpc-negative-shift", ESUBFRAME, 2, 0x08, 0x08, spec=lpc, sub=True)   # the shift's sign bit
    for m in (2, 3):
        patched(f"residual-coding-{m:02b}", ESUBFRAME, 1, m << 6, 0xC0, spec={"type": "fixed", "order": 0}, sub=True)
    patched("partition-order", EPARTITION, 1, 0b00001100, 0x3C, spec={"type": "fixed", "order": 0}, sub=True)  # 100 % 8
    # a wasted-bits flag before 72 zero bits: k = 73 wasted bits of an 8-bit subframe
    raw, at, hlen = _one_frame(np.concatenate([np.zeros((9, 1), np.int64), x[9:] | 1]), 8, subframes=[{"type": "verbatim"}])
    raw[at + hlen] |= 1
    out.append(("wasted-run", _refresh(raw, at, hlen), ESUBFRAME))
    raw, at, hlen = _one_frame(x, 8)
    raw[at + hlen - 1] ^= 1
    out.append(("crc8", bytes(raw), ECRC8))
    raw, at, hlen = _one_frame(x, 8, subframes=[{"type": "verbatim"}])
    raw[-10] ^= 1
    out.append(("crc16", bytes(raw), ECRC16))
    # left / side: left 127 VERBATIM, side CONSTANT; patching side's 9-bit value to -100 decodes right = 227
    raw, at, hlen = _one_frame(np.array([[127, 127]] * 16), 8, subframes=[{"type": "verbatim"}, {"type": "constant"}],
                               assign=8)
    side = at + hlen + 1 + 16                            # the side subframe's header byte
    v = int.from_bytes(raw[side + 1:side + 3], "big") & 0x7F | ((-100 & 0x1FF) << 7)
    raw[side + 1:side + 3] = v.to_bytes(2, "big")
    out.append(("range", _refresh(raw, at, hlen), ERANGE))
    good = encode(x, 8000, 8, blocks=25)
    info = streaminfo(8000, 1, 8, 101, 25, 25, md5_of(x, 8))
    start = good.index(b"fLaC") + 8
    out.append(("too-few-frames", good[:start] + info + good[start + 34:], ELENGTH))
    info = streaminfo(8000, 1, 8, 99, 25, 25, md5_of(x, 8))
    out.append(("too-many-samples", good[:start] + info + good[start + 34:], ELENGTH))
    frames = [frame_bytes(x[i * 25:(i + 1) * 25], n, 8) for i, n in enumerate((0, 2, 1, 3))]
    out.append(("sequence", container(frames, 8000, 1, 8, 100, 25, 25, bytes(16)), ESEQUENCE))
    return out
