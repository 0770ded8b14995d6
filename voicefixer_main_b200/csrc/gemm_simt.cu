// SIMT fp32 implementation of the flat-shift multi-tap GEMM contract (gemm.cuh).
// VALIDATION KERNEL: it exists so every tensor-core GEMM launch can be cross-checked element by element on the
// device (vf_selftest_layer, and whole plans under the option validate_simt); the product path always runs gemm_tc.cu.
// One thread per output row, 32 output columns per pass; the weight tile is staged in shared memory as
// fp32 (hi + lo), the activation row is read straight from the hi/lo planes.
#include "gemm.cuh"

namespace vf {

__global__ void __launch_bounds__(128) gemm_simt_kernel(const GemmSimtParams P) {
  __shared__ float w_s[32][65];
  const GemmProblem& pr = P.prob;
  const int img = blockIdx.x / pr.m_tiles;
  const int m0 = (blockIdx.x - img * pr.m_tiles) * GEMM_BM;
  const int n0 = blockIdx.y * 32;
  const int r = m0 + threadIdx.x;
  const bool three = pr.terms == 3;
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;

  for (int t = 0; t < pr.ntaps; ++t) {
    const GemmTap tap = pr.taps[t];
    const int row = r + tap.a_off;
    const bool in = row >= 0 && row < P.a_rows[tap.src];
    const size_t abase = ((size_t)img * P.a_img_rows[tap.src] + (in ? row : 0)) * P.a_ld[tap.src] + tap.c_off;
    for (int c0 = 0; c0 < tap.nch; c0 += 64) {
      const int cw = min(64, tap.nch - c0);
      __syncthreads();
      for (int idx = threadIdx.x; idx < 32 * 64; idx += 128) {
        const int n = idx >> 6, k = idx & 63;
        float w = 0.f;
        if (k < cw) {
          const size_t wi = (size_t)(n0 + n) * P.ktot + tap.k_off + c0 + k;
          w = __half2float(P.b_hi[wi]);
          if (three) w += __half2float(P.b_lo[wi]);
        }
        w_s[n][k] = w;
      }
      __syncthreads();
      if (in) {
        for (int k = 0; k < cw; ++k) {
          float a = __half2float(P.a_hi[tap.src][abase + c0 + k]);
          if (three) a += __half2float(P.a_lo[tap.src][abase + c0 + k]);
#pragma unroll
          for (int n = 0; n < 32; ++n) acc[n] = fmaf(a, w_s[n][k], acc[n]);
        }
      }
    }
  }
  float head_acc = 0.f;
  epilogue_chunk(pr.epi, img, r, n0, acc, head_acc);
  epilogue_head(pr.epi, img, r, head_acc);
}

cudaError_t launch_gemm_simt(const GemmSimtParams& p, cudaStream_t stream) {
  dim3 grid(p.prob.n_img * p.prob.m_tiles, p.prob.N / 32);
  gemm_simt_kernel<<<grid, 128, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace vf
