// FLAC audio decoded on the device (RFC 9639), as libsndfile's read of a FLAC file returns it, into the bytes of a WAV
// data chunk holding the same samples; vf_decode_pcm_varlen then converts those as it converts a WAV's.  See kernels.cuh,
// include/b200vf.h and oracle/flac.py.  Frames are not indexed in FLAC, so the device finds them:
//   flac_sync_kernel    one thread per byte: a sync code of the row's blocking strategy whose header parses, passes CRC-8
//                       and agrees with STREAMINFO becomes a candidate frame;
//   flac_walk_kernel    one thread per candidate: walk its subframes without writing samples, giving its end and CRC-16;
//   flac_chain_kernel   one thread per row: from the first frame, the next frame is the candidate that starts exactly at
//                       the current one's end, so a header-shaped pattern inside a frame never changes the result;
//   flac_decode_kernel  one thread per chained frame: entropy decode, prediction, wasted bits, stereo decorrelation, PCM.
#include <algorithm>

#include "../../include/b200vf.h"
#include "kernels.cuh"

namespace vf {
namespace {

struct Row {          // the STREAMINFO facts a frame must agree with
  int channels, bits, rate, first_block;
  bool variable;
  int64_t nbytes;
};

__device__ __forceinline__ Row row_of(const FlacParams& p, int b) {
  return {p.channels[b], p.bits[b], p.rate[b], p.first_block[b], p.variable[b] != 0, p.scan_off[b + 1] - p.scan_off[b]};
}

__device__ __forceinline__ void fail(const FlacParams& p, int b, int64_t at, int code) {
  atomicMin(p.status + b, ((unsigned long long)at << 8) | (unsigned)code);
}

// CRC-8, polynomial x^8 + x^2 + x + 1 (0x07), initial value 0, over the header from the sync code (RFC 9639 §9.1.8)
__device__ __forceinline__ uint32_t crc8(const uint8_t* p, int n) {
  uint32_t c = 0;
  for (int i = 0; i < n; ++i) {
    c ^= p[i];
    for (int k = 0; k < 8; ++k) c = ((c << 1) ^ ((c & 0x80) ? 0x07u : 0u)) & 0xFF;
  }
  return c;
}

// sample rate codes 0001 .. 1011 (§9.1.2) and bit depth codes 000 .. 111 (§9.1.4; 0: STREAMINFO's or reserved)
__constant__ int kRates[11] = {88200, 176400, 192000, 8000, 16000, 22050, 24000, 32000, 44100, 48000, 96000};
__constant__ int kBits[8] = {0, 8, 12, 0, 16, 20, 24, 32};

struct Header {
  int block, channels, assign, len;   // assign: the channel assignment code (0 .. 10)
  int64_t number;                     // frame number (fixed blocking) or first sample number (variable blocking)
};

// The frame header at p (avail bytes readable; p[0] == 0xFF and p[1] is the row's sync byte) -> 0 or VF_FLAC_E*.
// RFC 9639 §9.1: block size (§9.1.1), sample rate (§9.1.2), channels (§9.1.3), bit depth (§9.1.4), coded number
// (§9.1.5), uncommon block size (§9.1.6), uncommon rate (§9.1.7), CRC-8 (§9.1.8).
__device__ int parse_header(const uint8_t* p, int64_t avail, const Row& r, Header& h) {
  if (avail < 6) return VF_FLAC_ETRUNCATED;
  const int bs_code = p[2] >> 4, rate_code = p[2] & 15, ch_code = p[3] >> 4, bits_code = (p[3] >> 1) & 7;
  if (bs_code == 0 || rate_code == 15 || ch_code > 10 || bits_code == 3 || (p[3] & 1)) return VF_FLAC_ERESERVED;
  int n = 4;
  const uint32_t b0 = p[n++];
  int extra;                                           // continuation bytes of the UTF-8-style number
  uint64_t v;
  if (b0 < 0x80) { extra = 0; v = b0; }
  else if (b0 < 0xC0) return VF_FLAC_ERESERVED;
  else if (b0 < 0xE0) { extra = 1; v = b0 & 0x1F; }
  else if (b0 < 0xF0) { extra = 2; v = b0 & 0x0F; }
  else if (b0 < 0xF8) { extra = 3; v = b0 & 0x07; }
  else if (b0 < 0xFC) { extra = 4; v = b0 & 0x03; }
  else if (b0 < 0xFE) { extra = 5; v = b0 & 0x01; }
  else if (b0 == 0xFE) { extra = 6; v = 0; }
  else return VF_FLAC_ERESERVED;
  const int tail = (bs_code == 6 ? 1 : bs_code == 7 ? 2 : 0) + (rate_code == 12 ? 1 : rate_code >= 13 ? 2 : 0);
  if (avail < n + extra + tail + 1) return VF_FLAC_ETRUNCATED;
  for (int i = 0; i < extra; ++i) {
    const uint32_t c = p[n++];
    if ((c & 0xC0) != 0x80) return VF_FLAC_ERESERVED;
    v = (v << 6) | (c & 0x3F);
  }
  h.number = (int64_t)v;
  int block;
  if (bs_code == 1) block = 192;
  else if (bs_code <= 5) block = 576 << (bs_code - 2);
  else if (bs_code == 6) block = p[n++] + 1;
  else if (bs_code == 7) { block = ((p[n] << 8) | p[n + 1]) + 1; n += 2; }
  else block = 256 << (bs_code - 8);
  int rate = 0;                                        // 0: STREAMINFO's
  if (rate_code >= 1 && rate_code <= 11) rate = kRates[rate_code - 1];
  else if (rate_code == 12) rate = p[n++] * 1000;
  else if (rate_code == 13) { rate = (p[n] << 8) | p[n + 1]; n += 2; }
  else if (rate_code == 14) { rate = ((p[n] << 8) | p[n + 1]) * 10; n += 2; }
  if (crc8(p, n) != p[n]) return VF_FLAC_ECRC8;
  const int channels = ch_code < 8 ? ch_code + 1 : 2;
  if (channels != r.channels || (bits_code && kBits[bits_code] != r.bits) || (rate_code && rate != r.rate) || block > 65535)
    return VF_FLAC_EMISMATCH;
  h.block = block;
  h.channels = channels;
  h.assign = ch_code;
  h.len = n + 1;
  return 0;
}

// Big-endian bit reader over a row's region (8-byte aligned at base, limit bits long): a 64-bit window at any bit from
// two aligned words, reloaded only when the position crosses into another word.  Words past the region read as 0.
struct Bits {
  const unsigned long long* base;
  int64_t nwords, limit, pos;
  int64_t cw;
  uint64_t hi, lo;

  __device__ Bits(const uint8_t* region, int64_t nbytes, int64_t start_bit)
      : base(reinterpret_cast<const unsigned long long*>(region)), nwords((nbytes + 7) / 8), limit(nbytes * 8), pos(start_bit),
        cw(-2), hi(0), lo(0) {}
  __device__ __forceinline__ uint64_t word(int64_t w) const {
    if (w >= nwords) return 0;
    const uint64_t x = base[w];
    return ((uint64_t)__byte_perm((uint32_t)x, 0, 0x0123) << 32) | __byte_perm((uint32_t)(x >> 32), 0, 0x0123);
  }
  __device__ __forceinline__ uint64_t peek() {
    const int64_t w = pos >> 6;
    if (w != cw) {
      hi = w == cw + 1 ? lo : word(w);
      lo = word(w + 1);
      cw = w;
    }
    const int sh = pos & 63;
    return sh ? (hi << sh) | (lo >> (64 - sh)) : hi;
  }
  __device__ __forceinline__ uint32_t read(int n) {          // 0 <= n <= 32
    if (n == 0) return 0;
    const uint32_t v = (uint32_t)(peek() >> (64 - n));
    pos += n;
    return v;
  }
  __device__ __forceinline__ int32_t read_signed(int n) {    // two's complement of n <= 32 bits
    if (n == 0) return 0;
    return (int32_t)(read(n) << (32 - n)) >> (32 - n);
  }
  // One Rice-coded residual with parameter k (RFC 9639 §9.2.7.3): a unary quotient (zeros ended by a 1), k low bits, then
  // the zigzag fold (u >> 1) ^ -(u & 1).  false: it runs past the region or does not fit 32 bits.
  __device__ __forceinline__ bool rice(int k, int32_t& r) {
    uint64_t w = peek();
    uint64_t q = 0;
    while (w == 0) {
      q += 64;
      pos += 64;
      if (pos > limit) return false;
      w = peek();
    }
    const int z = __clzll((long long)w);
    q += z;
    uint32_t low;
    if (k == 0) { low = 0; pos += z + 1; }
    else if (z + 1 + k <= 64) { low = (uint32_t)((w << (z + 1)) >> (64 - k)); pos += z + 1 + k; }
    else { pos += z + 1; low = read(k); }
    if (q >> (32 - k)) return false;
    const uint32_t u = (uint32_t)(q << k) | low;
    r = (int32_t)(u >> 1) ^ -(int32_t)(u & 1);
    return true;
  }
};

// The fixed predictors' coefficients, orders 0 .. 4 (RFC 9639 §9.2.5)
__device__ __forceinline__ int64_t fixed_predict(const int32_t* s, int n, int order) {
  switch (order) {
    case 0: return 0;
    case 1: return s[n - 1];
    case 2: return 2 * (int64_t)s[n - 1] - s[n - 2];
    case 3: return 3 * (int64_t)s[n - 1] - 3 * (int64_t)s[n - 2] + s[n - 3];
    default: return 4 * (int64_t)s[n - 1] - 6 * (int64_t)s[n - 2] + 4 * (int64_t)s[n - 3] - s[n - 4];
  }
}

__device__ __forceinline__ bool fits(int64_t v, int bits) {   // v is a two's complement value of `bits` bits
  return ((v + ((int64_t)1 << (bits - 1))) >> bits) == 0;
}

// One subframe (RFC 9639 §9.2) of `block` samples of sample size `bps` (the frame's bit depth, + 1 for a side channel).
// WRITE: its samples before the wasted-bits shift go to out[0 .. block), and *wasted receives the shift; else it is only
// walked.  -> 0 or VF_FLAC_E*.
template <bool WRITE>
__device__ __forceinline__ int subframe(Bits& in, int block, int bps, int32_t* out, int* wasted) {
  if (in.pos + 8 > in.limit) return VF_FLAC_ETRUNCATED;
  const uint32_t head = in.read(8);
  if (head & 0x80) return VF_FLAC_ESUBFRAME;              // the zero bit before the type (§9.2.1)
  const int type = (head >> 1) & 0x3F;
  int k = 0;
  if (head & 1) {                                        // wasted bits: k - 1 zeros then a 1 (§9.2.2)
    uint64_t w = in.peek();
    int64_t zeros = 0;
    while (w == 0) {                                     // a run past the window: too many, unless the data ends first
      zeros += 64;
      in.pos += 64;
      if (in.pos > in.limit) return VF_FLAC_ETRUNCATED;
      w = in.peek();
    }
    const int z = __clzll((long long)w);
    in.pos += z + 1;
    if (in.pos > in.limit) return VF_FLAC_ETRUNCATED;
    if (zeros + z + 1 >= bps) return VF_FLAC_ESUBFRAME;
    k = z + 1;
  }
  if (WRITE) *wasted = k;
  bps -= k;
  if (type == 0) {                                       // CONSTANT (§9.2.3)
    const int32_t v = in.read_signed(bps);
    if (WRITE)
      for (int i = 0; i < block; ++i) out[i] = v;
    return in.pos > in.limit ? VF_FLAC_ETRUNCATED : 0;
  }
  if (type == 1) {                                       // VERBATIM (§9.2.4)
    if (!WRITE) in.pos += (int64_t)block * bps;
    else
      for (int i = 0; i < block; ++i) out[i] = in.read_signed(bps);
    return in.pos > in.limit ? VF_FLAC_ETRUNCATED : 0;
  }
  int order, precision = 0, shift = 0;
  int32_t coef[32];
  if (type >= 8 && type <= 12) order = type - 8;          // FIXED (§9.2.5)
  else if (type >= 32) order = type - 31;                 // LPC (§9.2.6)
  else return VF_FLAC_ESUBFRAME;
  if (order > block) return VF_FLAC_EPARTITION;
  if (!WRITE) in.pos += (int64_t)order * bps;
  else
    for (int i = 0; i < order; ++i) out[i] = in.read_signed(bps);
  if (type >= 32) {
    precision = (int)in.read(4) + 1;
    if (precision == 16) return VF_FLAC_ESUBFRAME;
    shift = in.read_signed(5);
    if (shift < 0) return VF_FLAC_ESUBFRAME;
    for (int j = 0; j < order; ++j) {
      const int32_t c = in.read_signed(precision);
      if (WRITE) coef[j] = c;
    }
  }
  // residual (§9.2.7): the coding method, the partition order, then each partition's parameter and samples
  if (in.pos + 6 > in.limit) return VF_FLAC_ETRUNCATED;
  const int method = (int)in.read(2);
  if (method > 1) return VF_FLAC_ESUBFRAME;
  const int pbits = method ? 5 : 4, escape = method ? 31 : 15;
  const int porder = (int)in.read(4);
  const int parts = 1 << porder;
  if (block % parts || (block >> porder) < order) return VF_FLAC_EPARTITION;
  const int per = block >> porder;
  int i = order;
  for (int part = 0; part < parts; ++part) {
    const int end = (part + 1) * per;
    const int param = (int)in.read(pbits);
    if (param == escape) {
      const int width = (int)in.read(5);
      if (!WRITE) { in.pos += (int64_t)(end - i) * width; i = end; }
      else
        for (; i < end; ++i) out[i] = in.read_signed(width);
    } else {
      for (; i < end; ++i) {
        int32_t r;
        if (!in.rice(param, r)) return in.pos > in.limit ? VF_FLAC_ETRUNCATED : VF_FLAC_ERANGE;
        if (WRITE) out[i] = r;
      }
    }
    if (in.pos > in.limit) return VF_FLAC_ETRUNCATED;
  }
  // prediction: s[n] = r[n] + (sum_j c[j] s[n - 1 - j] >> shift) for LPC (§9.2.6), the binomial predictors for FIXED,
  // accumulated in int64
  for (int n = order; WRITE && n < block; ++n) {
    int64_t pred;
    if (type < 32) pred = fixed_predict(out, n, order);
    else {
      int64_t acc = 0;
      for (int j = 0; j < order; ++j) acc += (int64_t)coef[j] * out[n - 1 - j];
      pred = acc >> shift;
    }
    const int64_t s = out[n] + pred;
    if (!fits(s, bps)) return VF_FLAC_ERANGE;
    out[n] = (int32_t)s;
  }
  return 0;
}

__device__ __forceinline__ int side_channel(int assign) {   // the channel that carries side (§9.1.3), or -1
  return assign == 8 ? 1 : assign == 9 ? 0 : assign == 10 ? 1 : -1;
}

// Row b's candidate slots: [cand_base(b), cand_base(b + 1)), at least nbytes / 8 + 1 of them, with their own counter
// p.count[b], so a row full of header-shaped bytes can run out of slots only for itself.
__device__ __forceinline__ int64_t cand_base(const FlacParams& p, int b) { return (p.scan_off[b] >> 3) + 2 * (int64_t)b; }

// The row that owns candidate slot `slot` (< cand_base(batch)), and whether the slot holds a candidate
__device__ __forceinline__ int cand_row(const FlacParams& p, int64_t slot, bool& used) {
  int lo = 0, hi = p.batch;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (cand_base(p, mid) <= slot) lo = mid; else hi = mid;
  }
  const int64_t n = min((int64_t)p.count[lo], cand_base(p, lo + 1) - cand_base(p, lo));
  used = slot - cand_base(p, lo) < n;
  return lo;
}

// -------------------------------------------------------------------------------------------------------------- kernels
__global__ void __launch_bounds__(256) flac_sync_kernel(const __grid_constant__ FlacParams p) {
  const int64_t g = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (g >= p.scan_off[p.batch]) return;
  const int b = packed_row(p.scan_off, p.batch, g);
  const Row r = row_of(p, b);
  const int64_t j = g - p.scan_off[b];
  const uint8_t* q = p.bytes + p.byte_off[b] + j;
  int32_t e = 0;
  if (j + 1 < r.nbytes && q[0] == 0xFF && (q[1] & 0xFE) == 0xF8) {
    Header h;
    const int rc = (q[1] & 1) != (int)r.variable ? VF_FLAC_EMISMATCH : parse_header(q, r.nbytes - j, r, h);
    if (rc) e = -rc;
    else {
      const int64_t k = atomicAdd(p.count + b, 1);
      if (k < cand_base(p, b + 1) - cand_base(p, b)) {
        const int64_t idx = cand_base(p, b) + k;
        p.cand_at[idx] = g;
        p.chained[idx] = 0;
        e = (int32_t)(idx + 1);
      } else {
        e = -VF_FLAC_ECANDIDATES;
      }
    }
  }
  p.ends[g] = e;
}

__global__ void __launch_bounds__(128) flac_walk_kernel(const __grid_constant__ FlacParams p) {
  __shared__ uint16_t crc16[256];                        // CRC-16, polynomial 0x8005, initial value 0 (§9.3)
  for (int i = threadIdx.x; i < 256; i += 128) {
    uint32_t c = (uint32_t)i << 8;
    for (int k = 0; k < 8; ++k) c = (c << 1) ^ ((c & 0x8000) ? 0x8005u : 0u);
    crc16[i] = (uint16_t)c;
  }
  __syncthreads();
  for (int64_t idx = (int64_t)blockIdx.x * 128 + threadIdx.x; idx < p.cap; idx += (int64_t)gridDim.x * 128) {
    bool used;
    const int b = cand_row(p, idx, used);
    if (!used) continue;
    const int64_t g = p.cand_at[idx];
    const Row r = row_of(p, b);
    const int64_t j = g - p.scan_off[b];
    const uint8_t* region = p.bytes + p.byte_off[b];
    Header h;
    parse_header(region + j, r.nbytes - j, r, h);        // passed in flac_sync_kernel
    Bits in(region, r.nbytes, (j + h.len) * 8);
    const int side = side_channel(h.assign);
    int rc = 0;
    for (int c = 0; c < h.channels && !rc; ++c) rc = subframe<false>(in, h.block, r.bits + (c == side), nullptr, nullptr);
    int64_t end = ((in.pos + 7) >> 3) + 2;               // zero padding to a byte, then the CRC-16 (§9.3)
    if (!rc && end > r.nbytes) rc = VF_FLAC_ETRUNCATED;
    if (!rc) {
      uint32_t c = 0;
      for (int64_t k = j; k < end - 2; ++k) c = ((c << 8) & 0xFFFF) ^ crc16[(c >> 8) ^ region[k]];
      if (c != (((uint32_t)region[end - 2] << 8) | region[end - 1])) rc = VF_FLAC_ECRC16;
    }
    p.cand_len[idx] = rc ? -rc : (int32_t)(end - j);
  }
}

__global__ void flac_chain_kernel(const __grid_constant__ FlacParams p) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= p.batch) return;
  const Row r = row_of(p, b);
  const int64_t total = p.total[b];
  const uint8_t* region = p.bytes + p.byte_off[b];
  int64_t pos = 0, done = 0, k = 0;
  while (done < total) {
    if (pos >= r.nbytes) return fail(p, b, pos, VF_FLAC_ELENGTH);
    const int32_t e = p.ends[p.scan_off[b] + pos];
    if (e <= 0) return fail(p, b, pos, e ? -e : VF_FLAC_ENOSYNC);
    const int32_t len = p.cand_len[e - 1];
    if (len <= 0) return fail(p, b, pos, -len);
    Header h;
    parse_header(region + pos, r.nbytes - pos, r, h);
    if (h.number != (r.variable ? done : k)) return fail(p, b, pos, VF_FLAC_ESEQUENCE);
    if (!r.variable && (h.block > r.first_block || (h.block < r.first_block && done + h.block < total)))
      return fail(p, b, pos, VF_FLAC_ESEQUENCE);           // fixed blocking: only the last frame may be shorter
    if (done + h.block > total) return fail(p, b, pos, VF_FLAC_ELENGTH);
    p.chained[e - 1] = 1;
    done += h.block;
    pos += len;
    ++k;
  }
}

__global__ void __launch_bounds__(128) flac_decode_kernel(const __grid_constant__ FlacParams p) {
  for (int64_t idx = (int64_t)blockIdx.x * 128 + threadIdx.x; idx < p.cap; idx += (int64_t)gridDim.x * 128) {
    bool used;
    const int b = cand_row(p, idx, used);
    if (!used || !p.chained[idx]) continue;            // chained frames before a chain failure are decoded too, so
    const int64_t g = p.cand_at[idx];                  // an earlier bad sample still names the first bad frame
    const Row r = row_of(p, b);
    const int64_t j = g - p.scan_off[b];
    const uint8_t* region = p.bytes + p.byte_off[b];
    Header h;
    parse_header(region + j, r.nbytes - j, r, h);
    const int64_t t0 = r.variable ? h.number : h.number * r.first_block;   // checked by flac_chain_kernel
    const int C = h.channels, B = h.block, side = side_channel(h.assign);
    int32_t* s = p.smp + p.smp_off[b] + t0 * C;          // channel c's samples at s[c * B ..]
    Bits in(region, r.nbytes, (j + h.len) * 8);
    int wasted[8];
    int rc = 0;
    for (int c = 0; c < C && !rc; ++c) rc = subframe<true>(in, B, r.bits + (c == side), s + c * B, wasted + c);
    if (rc) { fail(p, b, j, rc); continue; }
    // wasted bits (§9.2.2), then the stereo decorrelation (§9.1.3; mid/side: mid = (mid << 1) | (side & 1),
    // L = (mid + side) >> 1, R = (mid - side) >> 1), then the WAV data chunk's bytes: u8 as v + 128, s16 and s24 little-endian
    const int W = (r.bits + 7) / 8;
    uint8_t* out = p.pcm + p.pcm_off[b] + t0 * C * W;
    bool ok = true;
    for (int i = 0; i < B; ++i) {
      int64_t v[8];
      for (int c = 0; c < C; ++c) v[c] = (int64_t)s[c * B + i] << wasted[c];
      if (h.assign == 8) v[1] = v[0] - v[1];
      else if (h.assign == 9) v[0] = v[0] + v[1];
      else if (h.assign == 10) {
        const int64_t mid = (v[0] * 2) | (v[1] & 1), sd = v[1];
        v[0] = (mid + sd) >> 1;
        v[1] = (mid - sd) >> 1;
      }
      for (int c = 0; c < C; ++c) {
        ok &= fits(v[c], r.bits);
        const uint32_t u = (uint32_t)v[c] + (W == 1 ? 128u : 0u);
        uint8_t* o = out + ((int64_t)i * C + c) * W;
        o[0] = (uint8_t)u;
        if (W > 1) o[1] = (uint8_t)(u >> 8);
        if (W > 2) o[2] = (uint8_t)(u >> 16);
      }
    }
    if (!ok) fail(p, b, j, VF_FLAC_ERANGE);
  }
}

}  // namespace

cudaError_t launch_decode_flac(const FlacParams& p, cudaStream_t stream) {
  const int64_t n = p.scan_off[p.batch];
  if (n == 0) return cudaSuccess;
  cudaError_t e = cudaMemsetAsync(p.count, 0, sizeof(int) * p.batch, stream);
  if (e != cudaSuccess) return e;
  flac_sync_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(p);
  const unsigned grid = (unsigned)std::min<int64_t>((p.cap + 127) / 128, 2048);
  flac_walk_kernel<<<grid, 128, 0, stream>>>(p);
  flac_chain_kernel<<<(p.batch + 127) / 128, 128, 0, stream>>>(p);
  flac_decode_kernel<<<grid, 128, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace vf
