// Scoring a file against its target: the spectrogram and SSIM of AudioMetrics.evaluation (evaluation_proc/metrics.py:37-106).
//   * metric STFT: np.abs(librosa.stft(wav, hop_length=441, n_fft=2048)) as librosa 0.8 computes it - reflect padding by
//     n_fft / 2 (index math on the un-padded clip), float64 periodic hann x float32 samples, float64 FFT (the fp64 Stockham
//     FFT of fft.cuh), the spectrum stored as complex64 and |.| of that.  No power clamp: digital silence gives exact zeros.
//     At 16 kHz (hop_length=160, n_fft=743) the same with a direct float64 DFT of the prime length 743.
//   * SSIM: scikit-image 0.18's structural_similarity(x, y, win_size=7) in float64, deterministic.
// Both are HBM / launch bound; one launch covers a whole set of clips or images of different lengths.
#include "fft.cuh"
#include "kernels.cuh"
#include "reduce.cuh"

namespace vf {

// One CTA per (frame of the set, source).  The clip of a frame is found by bisection of the frame offsets.
__global__ void __launch_bounds__(256) metric_stft_kernel(MetricStftParams p) {
  __shared__ double2 buf0[1024];
  __shared__ double2 buf1[1024];
  const int tid = threadIdx.x, z = blockIdx.y;
  const int64_t g = blockIdx.x;
  const int b = packed_row(p.frame_off, p.batch, g);
  const long t = (long)(g - p.frame_off[b]);
  const float* x = p.wav[z] + p.off[z][b];
  const long n = (long)(p.off[z][b + 1] - p.off[z][b]);
  load_frame_packed<441>(buf0, x, n, t, p.window, tid);
  __syncthreads();
  const double2* Z = fft_forward<5>(buf0, buf1, p.tw1024, tid);
  float* out = p.sp[z] + (size_t)g * 1025;
  for (int k = tid; k <= 1024; k += 256) {
    const double2 X = rfft_split<1024>(Z, p.tw2048, k);
    const float re = (float)X.x, im = (float)X.y;                // complex64 storage
    out[k] = (float)sqrt((double)re * re + (double)im * im);     // numpy's complex64 abs (hypotf); the products are exact
  }
}
cudaError_t launch_metric_stft(const MetricStftParams& p, cudaStream_t stream) {
  metric_stft_kernel<<<dim3((unsigned)p.frame_off[p.batch], p.sources), 256, 0, stream>>>(p);
  return cudaGetLastError();
}

// The 16 kHz geometry (n_fft 743, hop 160, 372 bins).  743 is prime, so each bin is a direct float64 sum over the frame,
// n ascending: X[k] = sum_n w[n] x[n] e^{-2 pi i k n / 743}, with the twiddle index j = k n mod 743 advanced by k per term
// (exact integer arithmetic) into a table staged in shared memory.  One CTA per DFT743_FRAMES consecutive frames of the set
// (each frame finds its clip by bisection, as above) and source, one thread per bin: each twiddle read serves all its
// frames.  A frame's sums do not depend on the frames it is grouped with.
constexpr int DFT743_N = 743, DFT743_BINS = 372, DFT743_THREADS = 384, DFT743_FRAMES = 4;
__global__ void __launch_bounds__(DFT743_THREADS) metric_dft743_kernel(MetricStftParams p) {
  __shared__ double xs[DFT743_FRAMES][DFT743_N];
  __shared__ double2 tw[DFT743_N];
  const int tid = threadIdx.x, z = blockIdx.y;
  const int64_t total = p.frame_off[p.batch], g0 = (int64_t)blockIdx.x * DFT743_FRAMES;
  for (int i = tid; i < DFT743_N; i += DFT743_THREADS) tw[i] = p.tw743[i];
  for (int f = 0; f < DFT743_FRAMES; ++f) {
    const int64_t g = g0 + f;
    if (g >= total) {                                           // past the set: zeros, not stored
      for (int i = tid; i < DFT743_N; i += DFT743_THREADS) xs[f][i] = 0.0;
      continue;
    }
    const int b = packed_row(p.frame_off, p.batch, g);
    const long t = (long)(g - p.frame_off[b]);
    const float* x = p.wav[z] + p.off[z][b];
    const long n = (long)(p.off[z][b + 1] - p.off[z][b]);
    for (int i = tid; i < DFT743_N; i += DFT743_THREADS)     // the reflect-padded frame times the float64 window
      xs[f][i] = (double)__ldg(x + reflect_once(t * 160 + i - DFT743_N / 2, n)) * __ldg(p.window + i);
  }
  __syncthreads();
  if (tid >= DFT743_BINS) return;
  const int k = tid;
  double re[DFT743_FRAMES], im[DFT743_FRAMES];
#pragma unroll
  for (int f = 0; f < DFT743_FRAMES; ++f) re[f] = im[f] = 0.0;
  int j = 0;
  for (int i = 0; i < DFT743_N; ++i) {
    const double2 w = tw[j];
#pragma unroll
    for (int f = 0; f < DFT743_FRAMES; ++f) {
      re[f] = fma(xs[f][i], w.x, re[f]);
      im[f] = fma(xs[f][i], w.y, im[f]);
    }
    j += k;
    if (j >= DFT743_N) j -= DFT743_N;
  }
#pragma unroll
  for (int f = 0; f < DFT743_FRAMES; ++f) {
    if (g0 + f >= total) break;
    const float fr = (float)re[f], fi = (float)im[f];           // complex64 storage
    p.sp[z][(size_t)(g0 + f) * DFT743_BINS + k] = (float)sqrt((double)fr * fr + (double)fi * fi);
  }
}
cudaError_t launch_metric_dft743(const MetricStftParams& p, cudaStream_t stream) {
  const unsigned blocks = (unsigned)((p.frame_off[p.batch] + DFT743_FRAMES - 1) / DFT743_FRAMES);
  metric_dft743_kernel<<<dim3(blocks, p.sources), DFT743_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------- SSIM
// S = ((2 ux uy + C1)(2 vxy + C2)) / ((ux^2 + uy^2 + C1)(vx + vy + C2)) with C1 = (0.01 * 2)^2, C2 = (0.03 * 2)^2 and
// v = 49/48 (E[ab] - E[a] E[b]) over the 7x7 window; the operations are written as rounded intrinsics so that no FMA
// contraction makes the numerator and denominator differ: identical images give exactly 1.
__device__ __forceinline__ double ssim_pixel(double sx, double sy, double sxx, double syy, double sxy) {
  const double C1 = 0.0004, C2 = 0.0036, cov = 49.0 / 48.0;
  const double ux = __ddiv_rn(sx, 49.0), uy = __ddiv_rn(sy, 49.0);
  const double uxx = __ddiv_rn(sxx, 49.0), uyy = __ddiv_rn(syy, 49.0), uxy = __ddiv_rn(sxy, 49.0);
  const double vx = __dmul_rn(cov, __dsub_rn(uxx, __dmul_rn(ux, ux)));
  const double vy = __dmul_rn(cov, __dsub_rn(uyy, __dmul_rn(uy, uy)));
  const double vxy = __dmul_rn(cov, __dsub_rn(uxy, __dmul_rn(ux, uy)));
  const double a1 = __dadd_rn(__dmul_rn(__dmul_rn(2.0, ux), uy), C1);
  const double a2 = __dadd_rn(__dmul_rn(2.0, vxy), C2);
  const double b1 = __dadd_rn(__dadd_rn(__dmul_rn(ux, ux), __dmul_rn(uy, uy)), C1);
  const double b2 = __dadd_rn(__dadd_rn(vx, vy), C2);
  return __ddiv_rn(__dmul_rn(a1, a2), __dmul_rn(b1, b2));
}

__global__ void __launch_bounds__(256) ssim_tile_kernel(SsimParams p) {
  constexpr int R = SSIM_TILE_R, C = SSIM_TILE_C, W = SSIM_TILE_C + 6;
  __shared__ float xs[R + 6][W];
  __shared__ float ys[R + 6][W];
  __shared__ double col[5][R][W];             // vertical 7-sums of x, y, x^2, y^2, xy
  __shared__ double sh[8];
  const int tile = blockIdx.x, tid = threadIdx.x;
  int lo = 0, hi = p.batch;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (p.tile_off[mid] <= tile) lo = mid; else hi = mid;
  }
  const long T = (long)(p.frame_off[lo + 1] - p.frame_off[lo]);
  const int F = p.F;
  const int ctiles = (F - 6 + C - 1) / C;
  const int local = tile - p.tile_off[lo];
  const long r0 = (long)(local / ctiles) * R;  // the tile's output pixels are (r0 + 3 + i, c0 + 3 + j)
  const int c0 = (local % ctiles) * C;
  const size_t base = (size_t)p.frame_off[lo] * F;
  for (int i = tid; i < (R + 6) * W; i += 256) {
    const int r = i / W, c = i % W;
    const bool in = r0 + r < T && c0 + c < F;
    const size_t at = base + (size_t)(r0 + r) * F + c0 + c;
    xs[r][c] = in ? __ldg(p.x + at) : 0.f;
    ys[r][c] = in ? __ldg(p.y + at) : 0.f;
  }
  __syncthreads();
  for (int i = tid; i < R * W; i += 256) {
    const int r = i / W, c = i % W;
    double sx = 0, sy = 0, sxx = 0, syy = 0, sxy = 0;
#pragma unroll
    for (int k = 0; k < 7; ++k) {
      const double a = xs[r + k][c], b = ys[r + k][c];
      sx = __dadd_rn(sx, a);
      sy = __dadd_rn(sy, b);
      sxx = __dadd_rn(sxx, __dmul_rn(a, a));
      syy = __dadd_rn(syy, __dmul_rn(b, b));
      sxy = __dadd_rn(sxy, __dmul_rn(a, b));
    }
    col[0][r][c] = sx; col[1][r][c] = sy; col[2][r][c] = sxx; col[3][r][c] = syy; col[4][r][c] = sxy;
  }
  __syncthreads();
  double acc = 0;
  for (int i = tid; i < R * C; i += 256) {
    const int r = i / C, c = i % C;
    if (r0 + 3 + r >= T - 3 || c0 + 3 + c >= F - 3) continue;
    double s[5];
#pragma unroll
    for (int q = 0; q < 5; ++q) {
      double v = 0;
#pragma unroll
      for (int k = 0; k < 7; ++k) v = __dadd_rn(v, col[q][r][c + k]);
      s[q] = v;
    }
    acc += ssim_pixel(s[0], s[1], s[2], s[3], s[4]);
  }
  const double tot = block_sum(acc, sh);
  if (tid == 0) p.partial[tile] = tot;
}

__global__ void __launch_bounds__(256) ssim_mean_kernel(SsimParams p, double* __restrict__ out, int out_stride) {
  __shared__ double sh[8];
  const int b = blockIdx.x;
  double acc = 0;
  for (int i = p.tile_off[b] + threadIdx.x; i < p.tile_off[b + 1]; i += 256) acc += p.partial[i];
  const double tot = block_sum(acc, sh);
  const double count = (double)(p.frame_off[b + 1] - p.frame_off[b] - 6) * (double)(p.F - 6);
  if (threadIdx.x == 0) out[(size_t)b * out_stride] = tot / count;
}

cudaError_t launch_ssim(const SsimParams& p, double* out, int out_stride, cudaStream_t stream) {
  ssim_tile_kernel<<<p.tile_off[p.batch], 256, 0, stream>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  ssim_mean_kernel<<<p.batch, 256, 0, stream>>>(p, out, out_stride);
  return cudaGetLastError();
}

}  // namespace vf
