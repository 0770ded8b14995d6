// Flat-shift multi-tap GEMM: the one contraction every conv on the VoiceFixer hot path maps to.
//
//   D[m, n] = sum_taps sum_c  A_src(tap)[img, m + a_off(tap), c_off(tap) + c] * W[n, k_off(tap) + c]
//
// Activations live in HBM as "rows x channels" fp16 planes (channels innermost): rows are flattened
// (h, w) pixels with one shared zero pad column per image row for the 2-D UNet (row pitch Wp = W + 1),
// or time steps for the 1-D vocoder.  A conv tap is then a constant row offset; zero padding above /
// below an image is the TMA out-of-bounds fill.  Each fp32 value a is stored as the pair
// hi = fp16(a), lo = fp16(a - hi); the product uses the three terms hi*hi + hi*lo + lo*hi with fp32
// accumulation (error ~2^-22, measured 5e-6 max on the full UNet - see DESIGN.md), or hi*hi only
// (terms = 1) where the stage tolerance allows.
//
// Reference ops covered (file:line in /root/reference):
//   Conv2d 3x3 pad 1 no bias          models/components/modules.py:235-243   9 taps
//   1x1 shortcut Conv2d + bias        models/components/modules.py:245-247   +1 tap, fused in the same accumulator
//   ConvTranspose2d k3 s2             models/components/modules.py:192-194   4 taps, N = 4 phases x Cout
//   Conv1d / ConvTranspose1d          vocoder restatement (oracle/vf_oracle.py:vocoder_generator)
// The epilogue fuses everything the reference does between two convs: bias, residual add
// (modules.py:268-271), eval-mode BatchNorm as a per-channel affine + LeakyReLU/ReLU/ELU of the
// *consumer* (modules.py:263-266, 213), prune/concat placement (modules.py:205-215), the 1x1 head
// with the log-mel residual (unet.py:96-100, gsr_voicefixer.py:90) and the fp16 hi/lo split.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace vf {

constexpr int GEMM_BM = 128;
constexpr int GEMM_MAX_TAPS = 12;

enum { ACT_NONE = 0, ACT_LRELU = 1, ACT_ELU = 2 };
enum { MAP_PLAIN = 0, MAP_CONVT2D = 1, MAP_CONVT1D = 2 };
enum { ERR_FP16_OVERFLOW = 100, ERR_NAN_PHASE = 101, ERR_NONFINITE_INPUT = 102, ERR_PIPE_PRODUCER = 201, ERR_PIPE_MMA = 202, ERR_PIPE_EPILOGUE = 203 };

struct GemmTap {
  int a_off;   // row offset of the tap's window relative to the output row
  int src;     // which A source (0/1)
  int c_off;   // first channel inside the source
  int k_off;   // first column of the tap's segment in the packed weight matrix
  int nch;     // channels contracted by the tap (multiple of the kernel's BK)
};

struct OutPlane {
  __half* hi;
  __half* lo;
  int ld;      // row stride in elements
  int c_off;   // channel offset (concat placement)
};

struct GemmEpilogue {
  int map;             // MAP_*
  int rows_in;         // valid GEMM rows per image
  int Wp;              // 2-D row pitch (pad column = Wp-1); 0 for 1-D data
  int cout;            // channels per phase (N = phases * cout)
  int out_img_rows;    // rows per image in the output allocations
  int out_row0;        // row offset of output row 0 (slack for reflection padding)
  int out_rows_valid;  // MAP_CONVT1D: rows [0, out_rows_valid) exist
  int ct_stride, ct_pad;
  int ct_out_wp;       // MAP_CONVT2D: row pitch of the output level (2*Wp for the mel UNet, modules.py:209 prunes time only;
                       // 2*Wp - 1 for unet_v2's both=True pruning, modules.py:207-208: the column past the pitch is dropped)
  const float* bias;   // [N] or null
  const float* resid;  // fp32 [n_img * rows_in, resid_ld] or null (MAP_PLAIN only)
  int resid_ld;
  const __half* resid_hi;  // residual given as hi/lo planes [n_img * rows_in, resid_ld] (the residual stream of the
  const __half* resid_lo;  // vocoder stacks: separate hi/lo planes of x, or the (a, r) pair below)
  float* out_raw;      // fp32 or null
  int raw_ld;
  OutPlane out_r;      // raw value split hi/lo (consumed by 1x1 shortcut taps)
  OutPlane out_a;      // act(scale * v + shift) split hi/lo (consumed by the next conv)
  const float* a_scale;  // [cout] or null (identity)
  const float* a_shift;
  int act;
  float slope;
  const float* head_w;   // fused 1x1 head over the 32 channels of the row, or null
  float head_b;
  const float* head_in;  // residual input [n_img, head_T, Wp] added to the head (log-mel, gsr_voicefixer.py:90), or null
  float* head_out;       // [n_img, head_T, Wp]: bins 0..Wp-2 = head + bias (+ head_in), bin Wp-1 = 0 (+ head_in): F.pad, unet.py:99
  int head_T;
  // (a, r) residual stream of the hi-only vocoder stacks: x is kept as a = fp16(lrelu_s(x)) - the plane the next conv reads
  // anyway - and r = fp16(x - U(a)), U(a) = min(a, a * inv) the inverse of the LeakyReLU (inv = fp16(1 / s), 0 < s <= 1, in
  // both halves of these words; 0 = off).  Same ~22 significant bits as a hi/lo split of x itself, but a stack moves 4
  // instead of 6 bytes per element out of every residual layer (no separate hi plane of x).
  uint32_t resid_ar;     // the residual planes (resid_hi, resid_lo) hold (a, r): add U(a) + r
  uint32_t out_ar;       // out_a is written as (hi plane = a, lo plane = r); 1-term kernels, ACT_LRELU, no affine
  int tma_out;           // 1: MAP_CONVT1D out_a leaves the staging tiles by TMA store through a 5-D map (see gemm_tc.cu).
                         // MAP_PLAIN outputs always do (GemmTcParams::o_raw / o_r / o_a)
  // Clips of different lengths in one plan (vf_restore_varlen): per image, the count of valid rows - GEMM rows for MAP_PLAIN /
  // MAP_CONVT2D, output rows for MAP_CONVT1D.  Rows past it are written as zeros in every output, like the pad column, so the
  // next conv reads the zero padding it would see past the end of a clip-sized tensor.  nullptr: every row is valid.
  const int* row_valid;
  const int* head_valid;   // per image, frames the fused head writes (t < head_valid[img]); nullptr: head_T
  int* err;
};

// Per image valid-row limit of a varlen plan, or "no limit".
__device__ __forceinline__ int valid_rows(const int* row_valid, int img) {
  return row_valid ? __ldg(row_valid + img) : 0x7fffffff;
}
// A tile of a varlen plan whose rows are all past its image's valid rows: the GEMM issues no loads and no MMAs for it and only
// stores its zeros.  The producer and the consumers evaluate the same predicate, so the operand ring stays in step.
__device__ __forceinline__ bool tile_is_empty(const GemmEpilogue& e, int img, int m0) {
  if (!e.row_valid) return false;
  const int v = __ldg(e.row_valid + img);
  return e.map == MAP_CONVT1D ? (long)m0 * e.ct_stride - e.ct_pad >= v : m0 >= v;
}

struct GemmProblem {
  int n_img;
  int m_tiles;   // ceil(rows_in / 128)
  int N;
  int ntaps;
  int terms;     // 1 or 3
  GemmTap taps[GEMM_MAX_TAPS];
  GemmEpilogue epi;
};

struct GemmTcParams {
  CUtensorMap a_hi[2];            // [C, rows, n_img] fp16 (3-term: [C, rows, n_img, 2], the hi and lo planes)
  CUtensorMap b_hi, b_lo;         // [Ktot, N] fp16 (K-major)
  CUtensorMap i_res;              // epilogue residual by TMA load (MAP_PLAIN only): fp32 [resid_ld, rows_in, n_img] box 32 x 32 x 1
                                  // SWIZZLE_128B (3-term), or fp16 planes [resid_ld, rows_in, n_img, 2] box 32 x 32 x 1 x 2 SWIZZLE_64B
                                  // (3-term) / box min(BN, 64) x 16 x 1 x 2 (hi-only: one warp's fragment rows, gemm_tc.cu)
  int resid_tma;                  // separate residual tiles in flight per 3-term epilogue warp (4 KB and an mbarrier each): 1 or 2;
                                  // 0 without a residual and in hi-only kernels (the residual lands in the staging tile)
  int stg_warp;                   // staging bytes per epilogue warp: 4096, or 16 rows x BN x planes fp16 for a hi-only MAP_PLAIN layer
  CUtensorMap o_raw;              // MAP_PLAIN epilogue TMA stores: fp32 [raw_ld, rows, n_img], box 32 x 32 x 1, SWIZZLE_128B
  CUtensorMap o_r, o_a;           // fp16 [ld, rows, n_img, planes], box 32 x 32 x 1 x planes, SWIZZLE_64B (o_a: also see tma_out);
                                  // hi-only MAP_PLAIN: box min(BN, 64) x 16 x 1 x planes, as i_res
  int stages;
  int tile_chunks; // BK-wide K chunks per output tile
  int seg_chunks;  // 3-term mode: chunks per accumulation segment (promotion to registers in between)
  int grid;        // persistent CTAs
  uint32_t magic_n, magic_m;   // gemm_tc_magic() of N / BN and m_tiles: division-free tile decoding
  GemmProblem prob;
};

// Fused residual pair of the C = 64 vocoder stacks (pair_tc.cu): x_new = x + conv_b(lrelu(conv_a(xa) + bias_a)) + bias_b, with the
// residual stream x kept as the (a, r) pair of GemmEpilogue
struct PairParams {
  CUtensorMap a_map;             // activated input plane lrelu(x), hi: [C, L, clips], box 64 x 128 x 1, SWIZZLE_128B
  CUtensorMap wa_map, wb_map;    // packed K-major hi weights [K >= 3C, C], box 64 x C
  CUtensorMap xin_map;           // the correction plane of the source (box 64 x 126 x 1); its activated plane comes with the centre tap
  CUtensorMap xo_map;            // the correction plane of the destination (box 64 x 126 x 1); unused when ar_out == 0
  CUtensorMap ao_map;            // lrelu(x_new, slope_out), hi plane [C, out_row0 + L, clips] (box 64 x 126 x 1)
  const float* bias_a;
  const float* bias_b;
  uint32_t ar_in, ar_out;        // fp16(1 / slope) words of the (a, r) stream; ar_out = 0 on the last pair of a stack
  int L, n_img, C, dil, out_img_rows, out_row0, tiles_per_img, grid;
  uint32_t magic_t;              // gemm_tc_magic(tiles_per_img, ...)
  float slope_h, slope_out;
  const int* row_valid;          // varlen plans: per clip valid rows (<= L); rows past it are written as zeros.  nullptr: L
  int* err;
};

// The fp16 range guard's running max |v|: max.NaN.f32 returns NaN when either operand is NaN (fmaxf would return the other
// one), so one NaN output keeps the running max NaN and the final !(amax <= 65504) flags it as it flags an overflow
__device__ __forceinline__ float fmax_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

// n / d with the host's multiply-high magic number (gemm_tc_magic): a handful of instructions instead of an integer division
__device__ __forceinline__ uint32_t fast_div(uint32_t n, uint32_t d, uint32_t magic) {
  if (magic == 0u) return n;                    // d == 1
  if (magic == 0xffffffffu) return n / d;       // range too large for the 32-bit magic (host decides)
  return __umulhi(n, magic);
}

__device__ __forceinline__ void split_store8(__half* hi, __half* lo, size_t idx, const float* a) {
  __align__(16) __half h[8];
  __align__(16) __half l[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    h[i] = __float2half_rn(a[i]);
    l[i] = __float2half_rn(a[i] - __half2float(h[i]));
  }
  *reinterpret_cast<uint4*>(hi + idx) = *reinterpret_cast<const uint4*>(h);
  *reinterpret_cast<uint4*>(lo + idx) = *reinterpret_cast<const uint4*>(l);
}

// unet.py:96-100 + gsr_voicefixer.py:90: out = head(x) padded with a zero bin, plus the input log-mel;
// unet_v2.py:125-132: the same head without the residual (the output is the magnitude itself).
__device__ __forceinline__ void epilogue_head(const GemmEpilogue& e, int img, int r, float head_acc) {
  if (!e.head_w || r >= e.rows_in) return;
  const int t = r / e.Wp, f = r - t * e.Wp;
  if (t >= e.head_T || (e.head_valid && t >= __ldg(e.head_valid + img))) return;
  const size_t idx = ((size_t)img * e.head_T + t) * e.Wp + f;
  const float y = (f < e.Wp - 1) ? head_acc + e.head_b : 0.f;
  e.head_out[idx] = e.head_in ? y + __ldg(e.head_in + idx) : y;
}

}  // namespace vf
