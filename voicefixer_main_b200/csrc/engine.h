// Declarations shared by the host translation units of libb200vf.so: engine.cu (context, plan cache, run machinery, C ABI),
// pack.cu (weight ingestion and packing) and plan.cu (launch plans).  No kernels are declared or defined here.
#pragma once

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <unordered_map>
#include <vector>

#include "../../include/b200vf.h"
#include "gemm.cuh"
#include "kernels.cuh"

namespace vf {
cudaError_t launch_gemm_tc(const GemmTcParams& p, int bn, int bk, cudaStream_t stream);
size_t gemm_tc_smem_bytes(int bn, int bk, int stages, int planes_a, int terms, int tile_chunks, int resid_tma);
int gemm_tc_max_bn(int terms);
cudaError_t launch_pair_tc(const PairParams& p, cudaStream_t stream);
size_t pair_tc_smem_bytes(int C);
uint32_t gemm_tc_magic(uint32_t d, uint64_t nmax);
cudaError_t launch_gemm_simt(const GemmSimtParams& p, cudaStream_t stream);

struct HostT {
  std::vector<float> v;
  std::vector<int64_t> shape;
};

struct GemmW {
  __half* hi = nullptr;
  __half* lo = nullptr;
  float* bias = nullptr;
  int N = 0, K = 0;
  int k_tail = 0;      // trailing identity block (pack_conv1d): a GEMM may contract the K - k_tail columns before it only
};
struct Affine {
  float* scale = nullptr;
  float* shift = nullptr;
};
struct Planes {
  PlanePtr p{nullptr, nullptr};
  int C = 0;
  int img_rows = 0;   // allocated rows per image
  size_t plane_stride = 0;   // elements from the hi plane to the lo plane (same allocation)
};
struct ASrc {
  Planes pl;
  int rows;           // valid rows per image (TMA bound / SIMT bound)
  int row0;           // first valid row inside the allocation (reflection slack), usually 0
};

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

enum OpKind { OP_GEMM, OP_FIRST, OP_POOL, OP_COND, OP_REFLECT, OP_TAIL, OP_FINALIZE, OP_MEMSET32, OP_PAIR };

struct Op {
  OpKind kind;
  int bn = 0, bk = 0;
  double flops = 0, bytes = 0;   // algorithmic work of this launch (reference op counts), for the roofline
  double exec_flops = 0;         // tensor-core flops actually issued (3 MMAs per product in 3-term mode, K / phase padding,
                                 // identity taps): numerator of the "executed" tensor fraction
  char label[48] = {0};
  GemmTcParams tc;
  GemmSimtParams simt;
  PairParams pair;
  UnetFirstParams first;
  PoolParams pool;
  VocCondParams cond;
  struct { PlanePtr pl; int batch, L, C, pad; const int* vl_L; } refl;
  VocTailParams tail;
  FinalizeParams fin;
  struct { void* p; size_t bytes; } ms;
};

struct ConvBlockW {
  GemmW conv1, conv2;     // conv2 carries the 1x1 shortcut as an extra K segment when present
  Affine bn1, bn2;
  bool has_sc = false;
  int cin = 0, cout = 0;
};

// One analysis ResUNet (models/components/unet.py / unet_small.py / unet_v2.py share the block structure and key names)
struct UnetW {
  bool loaded = false;
  ConvBlockW enc[6][4], bott, dec[6][4], post;
  GemmW dec_up[6];
  Affine dec_bn1[6];
  float first_bn1_scale = 1, first_bn1_shift = 0;
  float* d_first_w1 = nullptr;
  float* d_first_wsc = nullptr;
  float* d_first_bsc = nullptr;
  float* d_head_w = nullptr;
  float head_b = 0;
};

// PLAN_VARLEN: the GSR path for clips of different lengths (vf_restore_varlen), keyed by (batch, bucket): T = the bucket, a
// multiple of 64 frames (the UNet's time granularity) that holds the call's longest clip.  PLAN_SSR_VARLEN: the same for
// the SSR / GSR-UNet path (vf_ssr_restore_varlen)
enum PlanKind { PLAN_GSR = 0, PLAN_SSR = 1, PLAN_VARLEN = 2, PLAN_SSR_VARLEN = 3 };
// Plans of these kinds run unet_v2 + ISTFT (build_ssr); the others run the mel UNet + vocoder
inline bool is_ssr_plan(int kind) { return kind == PLAN_SSR || kind == PLAN_SSR_VARLEN; }
// Plans of these kinds own a lengths table (kernels.cuh)
inline bool is_varlen_plan(int kind) { return kind == PLAN_VARLEN || kind == PLAN_SSR_VARLEN; }

struct Plan {
  int kind = PLAN_GSR;
  uint64_t last_use = 0;
  int batch = 0, T = 0;
  // varlen plans: the per-clip lengths table (kernels.cuh), rewritten on the stream by every call; null otherwise
  int64_t* d_vl_off = nullptr;   // [batch + 1] sample offsets of the clips
  int* d_vl_rows = nullptr;      // [VL_ROWS][batch]
  const int* vl(int row) const { return d_vl_rows ? d_vl_rows + (size_t)row * batch : nullptr; }
  long n_samples = 0;
  std::vector<void*> allocs;
  size_t bytes = 0;
  std::vector<Op> frontend, unet, vocoder, tail;
  float* d_wav = nullptr;        // [B, N]   staged input of the host entry points (buffer 0)
  float* d_out = nullptr;        // [B, N]
  float* d_io[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};   // [buffer][in / out]: double-buffered host staging
  cudaEvent_t io_ev[2][4] = {{nullptr, nullptr, nullptr, nullptr}, {nullptr, nullptr, nullptr, nullptr}};   // h2d done, input consumed, compute done, d2h done
  unsigned io_seq = 0;
  // a plan's buffers are shared by every call of its shape: uses on different streams are ordered through this event
  cudaEvent_t ev_last = nullptr;
  cudaStream_t last_stream = nullptr;
  bool used = false;
  float* d_mel = nullptr;        // [B, T, 128] linear mel
  float* d_logmel_in = nullptr;  // [B, T, 128] log10 mel (UNet input)
  float* d_logmel_out = nullptr; // [B, T, 128]
  float* d_voc_wav = nullptr;    // [B, L]
  float* d_band = nullptr;       // [B][2] low-band energy sums (unify_energy)
  unsigned int* d_peak = nullptr;
  long L = 0;
  // SSR plans (unet_v2 + ISTFT)
  float* d_sp = nullptr;         // [B, T, 1025] input magnitude
  float* d_mag = nullptr;        // [B, T, 1025] predicted magnitude
  float* d_frames = nullptr;     // [B, T, 2048] windowed inverse-DFT frames
  // CUDA graphs of the fixed-pointer launch chain (GSR: unet [+ band energy] + vocoder, index = unify flag; SSR: unet),
  // captured on the second use of the plan (the first runs eagerly and sets the kernels' function attributes)
  cudaGraphExec_t graph[2] = {nullptr, nullptr};
  int uses = 0;
  // op slots patched per call
  int fe_op = -1, cond_op = -1, fin_op = -1;
};

}  // namespace vf

using namespace vf;

struct vf_ctx {
  int device = 0;
  vf_config cfg;
  std::string err;
  std::unordered_map<std::string, HostT> host_w;
  std::vector<void*> allocs;
  size_t weight_bytes = 0;
  bool loaded = false;
  EncodeTiledFn encode = nullptr;
  int sm_count = 132;
  int unet_terms = 3, voc_terms = 1, validate_simt = 0, unify_energy = 0;
  int64_t launches = 0;
  int* d_err = nullptr;      // [0] device error code, [1] negative-input count
  // tables
  float* d_window = nullptr;
  float2* d_tw1024 = nullptr;
  float2* d_tw2048 = nullptr;
  int *d_fb_f0 = nullptr, *d_fb_len = nullptr, *d_fb_ofs = nullptr;
  float* d_fb_val = nullptr;
  float* d_melw = nullptr;
  double* d_window64 = nullptr;    // metric STFT (vf_metric_spectrogram, vf_score_varlen): float64 window and twiddles
  double2* d_tw1024d = nullptr;
  double2* d_tw2048d = nullptr;
  // vf_score_varlen scratch (two spectrograms, two mels, SSIM tile sums), stream-ordered allocation grown on demand and
  // freed by vf_destroy; uses on different streams are ordered through score_ev
  void* d_score = nullptr;
  size_t score_bytes = 0;
  cudaEvent_t score_ev = nullptr;
  bool score_used = false;
  // UNet weights: the mel-domain analysis module of VoiceFixer (prefix generator.analysis_module.) and the
  // linear-spectrogram unet_v2 of SSR_UNet / GSR_UNet (prefix generator.unet.); either may be absent
  UnetW gsr, ssr;
  bool voc_loaded = false;
  float* d_win_sq_inv = nullptr;   // ISTFT: 1 / clamp(overlap-added squared window, 1e-11), period hop (steady state)
  // vocoder weights
  std::vector<GemmW> voc_cond;
  GemmW voc_stem;
  std::vector<GemmW> voc_up;
  std::vector<std::vector<GemmW>> voc_res_a, voc_res_b;
  float* d_tail_w = nullptr;
  float tail_b = 0;
  int voc_last_c = 64;
  std::map<std::tuple<int, int, long>, std::unique_ptr<Plan>> plans;   // (kind, batch, frames)
  uint64_t use_clock = 0;
  size_t plan_bytes = 0;               // device bytes held by cached plans
  size_t plan_budget = 0;              // cap for plan_bytes (LRU eviction); 0 = decide at first use from free memory
  int64_t plans_evicted = 0;
  bool use_graphs = true;        // option "graphs"
  cudaStream_t cap_stream = nullptr;   // capture happens on an internal stream (the caller's may be the legacy default stream)
  // host entry points: copies and compute on internal streams, so the H2D of call i+1 and the D2H of call i-1 overlap the
  // compute of call i (option "host_pipeline"); the caller's stream only waits for the call's own D2H
  bool host_pipeline = true;
  cudaStream_t s_in = nullptr, s_comp = nullptr, s_out = nullptr;
  bool op_timing = false;
  struct ProfRec { std::string label; double flops, bytes, exec_flops; int bn, bk, terms; };
  std::vector<ProfRec> prof;
  std::vector<cudaEvent_t> prof_ev;
  bool timing = false;
  cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  bool ev_valid = false;
};

namespace vf {

int fail(vf_ctx* c, int code, const char* fmt, ...);
#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess) return fail(ctx, VF_ECUDA, "%s: %s", #call, cudaGetErrorString(e_));   \
  } while (0)

template <typename T>
int dev_alloc(vf_ctx* ctx, std::vector<void*>& pool, size_t& acct, T** out, size_t count) {
  void* p = nullptr;
  const size_t bytes = std::max<size_t>(count * sizeof(T), 256);
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) return fail(ctx, VF_ECUDA, "cudaMalloc(%zu bytes): %s", bytes, cudaGetErrorString(e));
  pool.push_back(p);
  acct += bytes;
  *out = static_cast<T*>(p);
  return VF_OK;
}

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

// pack.cu
int upload_gemm(vf_ctx* ctx, GemmW* w, const std::vector<float>& m, int N, int K, const std::vector<float>* bias);
int build_tables(vf_ctx* ctx);
int load_all(vf_ctx* ctx);
// PyTorch weight layouts -> packed GEMM operands (upload_gemm), as the loaders pack every conv of the networks
int pack_conv3x3(vf_ctx* ctx, GemmW* out, const HostT& w, const HostT* sc_w, const HostT* sc_b);
int pack_convT2d(vf_ctx* ctx, GemmW* out, const HostT& w);
int pack_conv1d(vf_ctx* ctx, GemmW* out, const HostT& w, const HostT& b, bool identity = false);
int pack_convT1d(vf_ctx* ctx, GemmW* out, const HostT& w, const HostT& b, int s);
// the tail Conv1d(C -> 1, k7) weight [1][C][7] -> the tail kernel's [7][C]
int pack_tail(vf_ctx* ctx, float** out, const HostT& w);
// Residual add of a vocoder stack as an identity tap (through the accumulator, no epilogue loads) up to this channel count;
// above it the epilogue adds the hi/lo planes.  The packer appends the identity block and the plan builder adds the tap.
constexpr int IDENT_MAX_C = 128;

// plan.cu
struct Builder {
  vf_ctx* ctx;
  Plan* plan;
  int rc = VF_OK;
  std::string label;   // name given to the next op (profiling only)

  template <typename T>
  T* alloc(size_t count) {
    T* p = nullptr;
    if (rc) return nullptr;
    rc = dev_alloc(ctx, plan->allocs, plan->bytes, &p, count);
    return p;
  }
  Planes planes(size_t n_img, int img_rows, int C);
  // taps: nch = real channel count; k segments are laid out back to back, each padded to BK.
  void gemm(std::vector<Op>& ops, const GemmW& W, const ASrc& s0, const ASrc* s1, std::vector<GemmTap> taps,
            GemmEpilogue epi, int n_img, int terms);
};
GemmEpilogue epi_plain(int rows_in, int Wp, int cout, int out_img_rows);
// (a, r) residual stream (gemm.cuh): fp16(1 / slope) in both halves of a word, 0 when the LeakyReLU is not invertible that way
uint32_t ar_inv_word(float slope);
// Tap lists of the plans' convs: Conv2d 3x3 pad 1 on rows of pitch Wp; the four (dh, dw) input shifts of ConvTranspose2d
// k3 s2 (pack_convT2d); Conv1d k with dilation, centred (pad (k - 1) / 2 * dil) or not (the caller pads); ConvTranspose1d
// rows q and q - 1 (pack_convT1d)
std::vector<GemmTap> taps3x3(int Wp, int cin);
std::vector<GemmTap> taps_convt2d(int Wp, int cin);
std::vector<GemmTap> taps1d(int k, int dil, int cin, bool centered);
std::vector<GemmTap> taps_convt1d(int cin);
// Fused residual pair (pair_tc.cu) of a C = 64 stack: src / dst hold (a, r) planes of L rows per image; dst's activated
// plane is written from row out_row0; `last`: no correction plane out
int pair_setup(vf_ctx* ctx, PairParams* pp, const Planes& src, const Planes& dst, const GemmW& wa, const GemmW& wb, int n_img,
               int L, int dil, uint32_t ar, bool last, int out_row0, float slope_h, float slope_out, const int* row_valid);
// The non-GEMM ops of the launch chains, set up as the plan builders and the restore paths use them (vf_selftest_op runs the
// same set-up).  LeakyReLU slope of the UNet blocks, modules.py:265-266
constexpr float UNET_SLOPE = 0.01f;
// encoder_block1.conv_block1 on a [batch, T, W0 + 1] input: Tp = T padded to a multiple of 64; blk supplies bn2
Op first_op(vf_ctx* ctx, const UnetW& U, const ConvBlockW& blk, const float* in, int batch, int T, int W0, PlanePtr a2,
            float* sc_raw, const int* vl_T, const int* vl_Tp);
// avg_pool2d(2,2) of an [batch, H * (W + 1), C] level + the consumer's bn1 + LeakyReLU: output pitch (W >> 1) + 1
Op pool_op(vf_ctx* ctx, const float* in, int batch, int H, int W, int C, const Affine& next_bn1, PlanePtr out_r, PlanePtr out_a,
           float* out_raw, const int* row_valid);
// vocoder conditioning of the restored log-mel [batch, T, 128]: Tv = T + T % 2 + voc_tail_base rows per clip
Op cond_op(vf_ctx* ctx, const float* logmel, int batch, int T, PlanePtr out, const int* vl_T, const int* vl_Tv);
inline int voc_frames(const vf_config& c, int T) { return T + T % 2 + c.voc_tail_base; }
// amp_to_original_f (VF_RESTORE_UNIFY_ENERGY): zeroes `sums` and launches the low-band reduction on the stream, then points
// the conditioning op at it
cudaError_t unify_energy(const float* mel_lin, const float* logmel_est, int batch, int T, float* sums, const int* vl_T,
                         VocCondParams* cond, cudaStream_t st);
// ReflectionPad1d(3) of [batch, L + 6, C] planes, the peak memset and the tail conv (the vocoder's last three launches)
Op reflect_op(PlanePtr pl, int batch, int L, int C, const int* vl_L);
Op memset_op(void* p, size_t bytes);
Op tail_op(PlanePtr in, int batch, long L, int C, int terms, const float* w, float bias, int tanh_out, float* wav,
           unsigned int* peak, const int* vl_L);
// peak normalise + trim_center of a [batch, L] vocoder output into [batch, n] (varlen: packed by vl_off, trimmed by vl_L)
int finalize_params(vf_ctx* ctx, FinalizeParams* f, const float* wav, const unsigned int* peak, int batch, long L, long n,
                    float* out, const int64_t* vl_off, const int* vl_L);
// the SSR back end: the predicted magnitude with the phase of `wav`'s STFT -> frames -> overlap-add into out [batch, n]
void istft_params(vf_ctx* ctx, IstftFramesParams* fp, IstftOlaParams* op, const float* mag, const float* wav, int batch, long n,
                  int T, float* frames, float* out, const int64_t* vl_off, const int* vl_T);
int build_plan(vf_ctx* ctx, Plan* plan);

}  // namespace vf
