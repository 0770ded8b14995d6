// Analysis modules bi_gru / dnn of VoiceFixer's Generator (models/gsr_voicefixer.py:54-83): the bidirectional GRU recurrence
// and the hi/lo planes of the modules' input.  Every Linear layer (and the GRU's input projection) is a one-tap conv GEMM.
//
// GRU layer (torch.nn.GRU, batch_first, gate order r, z, n):
//   r = sigma(G_r + W_hr h),  z = sigma(G_z + W_hz h),  n = tanh(G_n + r * (W_hn h + b_hn)),  h' = (1 - z) * n + z * h
// with G = x W_ih^T + b_ih + (b_hr, b_hz, 0) from the GEMM.  One persistent launch per layer; one thread-block cluster of
// GRU_CTAS CTAs per (direction, group of GRU_CLIPS clips).  CTA `rank` owns hidden units [32 rank, 32 rank + 32): the three
// gate rows of W_hh for them (96 x 256 fp32) live in registers for the whole sequence, 64 weights per thread.  Every CTA
// keeps the whole h of its clips in a double-buffered shared tile; after each step a CTA stores its 32 new values into the
// next tile of every CTA of the cluster (distributed shared memory), and one cluster barrier publishes them.
#include <cooperative_groups.h>

#include <algorithm>

#include "gemm.cuh"
#include "kernels.cuh"

namespace cg = cooperative_groups;

namespace vf {
namespace {

constexpr int H = GRU_HIDDEN;            // 256
constexpr int UNITS = H / GRU_CTAS;      // hidden units per CTA: 32
constexpr int ROWS = 3 * UNITS;          // gate rows per CTA: 96
constexpr int THREADS = ROWS * 4;        // a thread per (gate row, K quarter): 384
constexpr int QS = H / 4 + 4;            // padded stride of a K quarter of h: the four quarters a warp reads hit distinct banks
constexpr int HS = 4 * QS;               // h floats per clip
constexpr int DEPTH = 8;                 // G rows prefetched this many steps ahead (cp.async)

struct GruSmem {
  float h[2][GRU_CLIPS][HS];                     // h_t of every clip of the cluster, double-buffered
  float gh[GRU_CLIPS][ROWS];                     // W_hh h for this CTA's gate rows
  float g[DEPTH][GRU_CLIPS * UNITS][4];          // prefetched (G_r, G_z, G_n) of each gate thread's unit and clip
};

__device__ __forceinline__ int hidx(int k) { return (k >> 6) * QS + (k & 63); }
__device__ __forceinline__ void cp_async4(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ void store_split(const PlanePtr& o, size_t i, float y) {
  const __half hi = __float2half_rn(y);
  o.hi[i] = hi;
  o.lo[i] = __float2half_rn(y - __half2float(hi));
}
// the fp16 range guard of a split value (NaN fails the compare)
__device__ __forceinline__ void check_range(float y, int* err) {
  if (!(fabsf(y) <= 65504.f) && err) atomicCAS(err, 0, ERR_FP16_OVERFLOW);
}

}  // namespace

__global__ void __cluster_dims__(GRU_CTAS, 1, 1) __launch_bounds__(THREADS, 1) gru_layer_kernel(const GruParams p) {
  __shared__ __align__(16) GruSmem s;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int dir = blockIdx.y;
  const int c0 = (blockIdx.x / GRU_CTAS) * GRU_CLIPS;
  const int tid = threadIdx.x, lane = tid & 31;
  const int kq = lane & 3, jl = (tid >> 5) * 8 + (lane >> 2);     // K quarter and local gate row of this thread
  const int grow = (jl / UNITS) * H + rank * UNITS + jl % UNITS;   // its row of W_hh: gate * H + unit
  float w[64];
  {
    const float4* wp = reinterpret_cast<const float4*>((dir ? p.w_hh[1] : p.w_hh[0]) + (size_t)grow * H + kq * 64);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float4 q = __ldg(wp + i);
      w[4 * i] = q.x; w[4 * i + 1] = q.y; w[4 * i + 2] = q.z; w[4 * i + 3] = q.w;
    }
  }
  int len[GRU_CLIPS], steps = 0;
#pragma unroll
  for (int c = 0; c < GRU_CLIPS; ++c) {
    const int b = c0 + c;
    len[c] = b < p.batch ? (p.vl_T ? __ldg(p.vl_T + b) : p.T) : 0;
    steps = max(steps, len[c]);
  }
  for (int i = tid; i < 2 * GRU_CLIPS * HS; i += THREADS) (&s.h[0][0][0])[i] = 0.f;

  // gate threads: one per (clip, unit) of this CTA
  const bool gate = tid < GRU_CLIPS * UNITS;
  const int gc = tid / UNITS, gu = tid % UNITS, U = rank * UNITS + gu;
  const int gb = c0 + gc;
  const int glen = (gate && gb < p.batch) ? (p.vl_T ? __ldg(p.vl_T + gb) : p.T) : 0;
  const float bhn = gate ? __ldg((dir ? p.b_hn[1] : p.b_hn[0]) + U) : 0.f;
  const float* gsrc = p.G + (size_t)(gate ? gb : 0) * p.T * (6 * H) + dir * (3 * H) + U;
  // the reverse direction of clip b starts at its own last frame glen - 1
  auto frame = [&](int st) { return dir ? glen - 1 - st : st; };
  auto issue = [&](int st) {
    if (st < glen) {
      const float* src = gsrc + (size_t)frame(st) * (6 * H);
      float* dst = s.g[st % DEPTH][tid];
      cp_async4(dst, src);
      cp_async4(dst + 1, src + H);
      cp_async4(dst + 2, src + 2 * H);
    }
    cp_async_commit();
  };
  for (int st = 0; st < DEPTH - 1; ++st) issue(st);
  cluster.sync();          // every CTA of the cluster runs and has zeroed its tiles before any peer stores into them

  float hprev = 0.f;
  for (int st = 0; st < steps; ++st) {
    const int cur = st & 1;
    issue(st + DEPTH - 1);
    float acc[GRU_CLIPS];
#pragma unroll
    for (int c = 0; c < GRU_CLIPS; ++c) {
      float a = 0.f;
      if (st < len[c]) {
        const float4* hp = reinterpret_cast<const float4*>(&s.h[cur][c][kq * QS]);
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const float4 q = hp[i];
          a = fmaf(w[4 * i], q.x, a);
          a = fmaf(w[4 * i + 1], q.y, a);
          a = fmaf(w[4 * i + 2], q.z, a);
          a = fmaf(w[4 * i + 3], q.w, a);
        }
      }
      acc[c] = a;
    }
    // the four K quarters of a row sit in adjacent lanes: (q0 + q1) + (q2 + q3), the same order on every lane
#pragma unroll
    for (int c = 0; c < GRU_CLIPS; ++c) {
      acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], 1);
      acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], 2);
    }
    if (kq == 0) {
#pragma unroll
      for (int c = 0; c < GRU_CLIPS; ++c) s.gh[c][jl] = acc[c];
    }
    cp_async_wait<DEPTH - 1>();      // this thread's G of step st has landed (each gate thread reads only its own copies)
    __syncthreads();
    if (st < glen) {
      const float* g = s.g[st % DEPTH][tid];
      const float r = sigmoidf_(g[0] + s.gh[gc][gu]);
      const float z = sigmoidf_(g[1] + s.gh[gc][UNITS + gu]);
      const float n = tanhf(g[2] + r * (s.gh[gc][2 * UNITS + gu] + bhn));
      const float hn = (1.f - z) * n + z * hprev;
      hprev = hn;
      float* mine = &s.h[cur ^ 1][gc][hidx(U)];
#pragma unroll
      for (int q = 0; q < GRU_CTAS; ++q) *cluster.map_shared_rank(mine, q) = hn;
      check_range(hn, p.err);          // |h| < 1 unless G holds a NaN or an infinity; h itself, as relu(NaN) would read 0
      store_split(p.out, ((size_t)gb * p.T + frame(st)) * (2 * H) + dir * H + U, p.relu ? fmaxf(hn, 0.f) : hn);
    }
    cluster.sync();        // release / acquire: the next h tile is complete in every CTA
  }
  cp_async_wait<0>();
  // varlen: frames past the clip's end are zeros, like every other layer's rows past row_valid
  if (gate && gb < p.batch)
    for (int t = glen; t < p.T; ++t) store_split(p.out, ((size_t)gb * p.T + t) * (2 * H) + dir * H + U, 0.f);
}

__global__ void affine_planes_kernel(const AffinePlanesParams p) {
  const size_t n = (size_t)p.batch * p.T * p.C;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const size_t row = i / p.C;
    const int b = (int)(row / p.T), t = (int)(row % p.T);
    const bool valid = !p.vl_T || t < __ldg(p.vl_T + b);
    const float y = valid ? fmaf(__ldg(p.in + i), p.scale, p.shift) : 0.f;
    check_range(y, p.err);
    store_split(p.out, i, y);
  }
}

int gru_groups(int batch) { return (batch + GRU_CLIPS - 1) / GRU_CLIPS; }

cudaError_t launch_gru(const GruParams& p, cudaStream_t stream) {
  gru_layer_kernel<<<dim3(GRU_CTAS * gru_groups(p.batch), 2), THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_affine_planes(const AffinePlanesParams& p, cudaStream_t stream) {
  const size_t n = (size_t)p.batch * p.T * p.C;
  const int blocks = (int)std::min<size_t>((n + 255) / 256, 4096);
  affine_planes_kernel<<<blocks, 256, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace vf
