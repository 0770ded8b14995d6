// I/O edges of the handler (SURVEY.md 8(f) rows 3 and 4), all HBM-bound one-pass kernels:
//   * polyphase FIR resampling to the model rate (load_wav -> librosa.load(sr=44100), tools/utils.py:46-48; arithmetic of
//     scipy.signal.resample_poly, which the reference itself uses for rate conversion, tools/dsp/lowpass.py:138-141)
//   * the mel metrics handler() reports when a target is given (eval_gsr_voicefixer.py:56-64):
//     AudioMetrics.lsd / .sispec (evaluation_proc/metrics.py:83-95, energy_unify evaluation_proc/utils.py:81-101)
#include "kernels.cuh"
#include "reduce.cuh"
#include "resample.cuh"

namespace vf {

// out[b, m] = sum_i h[m * down - i * up + half] * x[b, i]: zero-phase polyphase resampling by up / down with a symmetric
// FIR of 2 * half + 1 taps (designed on the host: firwin(.., 1 / max(up, down), window = ('kaiser', 5.0)) * up).  The body
// is poly_output (resample.cuh), which the streaming resampler shares.
__global__ void __launch_bounds__(256) resample_poly_kernel(const float* __restrict__ x, long n, int up, int down, const float* __restrict__ h,
                                                            int half, float* __restrict__ out, long n_out) {
  const long m = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (m >= n_out) return;
  out[(size_t)b * n_out + m] = poly_output(FlatInput{x + (size_t)b * n}, m, n, up, down, h, half);
}
cudaError_t launch_resample_poly(const float* x, int batch, long n, int up, int down, const float* h, int half, float* out, long n_out,
                                 cudaStream_t stream) {
  dim3 grid((unsigned)((n_out + 255) / 256), batch);
  resample_poly_kernel<<<grid, 256, 0, stream>>>(x, n, up, down, h, half, out, n_out);
  return cudaGetLastError();
}

// One CTA per (clip, channel) image of T x F values; fixed reduction order (deterministic, block_sum in reduce.cuh).
// AudioMetrics.lsd (metrics.py:83-87): mean_t sqrt(mean_f log10(target^2 / (est + EPS)^2 + EPS)^2), EPS = 1e-12 (metrics.py:15)
// The image at element `base` of est / tgt; the value is returned to every thread.
__device__ __forceinline__ float lsd_image(const float* __restrict__ est, const float* __restrict__ tgt, size_t base, int T, int F) {
  __shared__ double sh[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double acc = 0;
  for (int t = warp; t < T; t += 8) {
    float s = 0.f;
    for (int f = lane; f < F; f += 32) {
      const float e = __ldg(est + base + (size_t)t * F + f) + 1e-12f, g = __ldg(tgt + base + (size_t)t * F + f);
      const float l = log10f((g * g) / (e * e) + 1e-12f);
      s = fmaf(l, l, s);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    acc += (double)sqrtf(s / (float)F);
  }
  const double tot = block_sum(lane == 0 ? acc : 0.0, sh);
  return (float)(tot / T);
}
__global__ void __launch_bounds__(256) lsd_kernel(const float* __restrict__ est, const float* __restrict__ tgt, int T, int F, float* __restrict__ out) {
  const float v = lsd_image(est, tgt, (size_t)blockIdx.x * T * F, T, F);
  if (threadIdx.x == 0) out[blockIdx.x] = v;
}
cudaError_t launch_lsd(const float* est, const float* tgt, int images, int T, int F, float* out, cudaStream_t stream) {
  lsd_kernel<<<images, 256, 0, stream>>>(est, tgt, T, F, out);
  return cudaGetLastError();
}

// AudioMetrics.sispec (metrics.py:89-95) per batch item over its n = C * T * F values:
//   target' = (sum(est * target) * target) / (|target|^2 + 1e-8)        (energy_unify, utils.py:90-93; pow_norm sums dims 2,3
//                                                                        per channel - C = 1 on this path)
//   10 log10(|target'|^2 / (|est - target'|^2 + 1e-12) + 1e-12)
// est_map / tgt_map: 0 identity, 1 to_log (log10(clip(x, 1e-8))), 2 from_log (10^min(x, 5)) applied on the fly, so handler()'s
// three variants (log / non-log, eval_gsr_voicefixer.py:60-62) need no extra pass over the mels.
__device__ __forceinline__ float metric_map(float v, int m) {
  if (m == 1) return log10f(fmaxf(v, 1e-8f));
  if (m == 2) return exp10f(fminf(v, 5.f));
  return v;
}
__device__ __forceinline__ float sispec_image(const float* __restrict__ est, const float* __restrict__ tgt, size_t base, long n, int est_map,
                                              int tgt_map) {
  __shared__ double sh[8];
  double st = 0, tt = 0;
  for (long i = threadIdx.x; i < n; i += 256) {
    const float e = metric_map(__ldg(est + base + i), est_map), g = metric_map(__ldg(tgt + base + i), tgt_map);
    st += (double)(e * g);
    tt += (double)(g * g);
  }
  const float s = (float)block_sum(st, sh);
  const float den = (float)block_sum(tt, sh) + 1e-8f;
  double pn = 0, nn = 0;
  for (long i = threadIdx.x; i < n; i += 256) {
    const float e = metric_map(__ldg(est + base + i), est_map), g = metric_map(__ldg(tgt + base + i), tgt_map);
    const float tp = (s * g) / den;
    const float d = e - tp;
    pn += (double)(tp * tp);
    nn += (double)(d * d);
  }
  const float p = (float)block_sum(pn, sh);
  const float q = (float)block_sum(nn, sh);
  return 10.f * log10f(p / (q + 1e-12f) + 1e-12f);
}
__global__ void __launch_bounds__(256) sispec_kernel(const float* __restrict__ est, const float* __restrict__ tgt, long n, int est_map, int tgt_map,
                                                     float* __restrict__ out) {
  const float v = sispec_image(est, tgt, (size_t)blockIdx.x * n, n, est_map, tgt_map);
  if (threadIdx.x == 0) out[blockIdx.x] = v;
}
cudaError_t launch_sispec(const float* est, const float* tgt, int batch, long n, int est_map, int tgt_map, float* out, cudaStream_t stream) {
  sispec_kernel<<<batch, 256, 0, stream>>>(est, tgt, n, est_map, tgt_map, out);
  return cudaGetLastError();
}

// The same metrics over images of different frame counts, one launch for a set: image b is rows [frame_off[b],
// frame_off[b + 1]) of F bins, with the arithmetic and reduction order of a uniform launch on that image alone.  Results are
// widened to double at out[b * out_stride] (sispec: blockIdx.y = 0 non-log, 1 to_log of both operands, at + blockIdx.y).
__global__ void __launch_bounds__(256) lsd_varlen_kernel(const float* __restrict__ est, const float* __restrict__ tgt, int F, ImageSet s,
                                                         double* __restrict__ out, int out_stride) {
  const int b = blockIdx.x;
  const float v = lsd_image(est, tgt, (size_t)s.frame_off[b] * F, (int)(s.frame_off[b + 1] - s.frame_off[b]), F);
  if (threadIdx.x == 0) out[(size_t)b * out_stride] = (double)v;
}
__global__ void __launch_bounds__(256) sispec_varlen_kernel(const float* __restrict__ est, const float* __restrict__ tgt, int F, ImageSet s,
                                                            double* __restrict__ out, int out_stride) {
  const int b = blockIdx.x, m = blockIdx.y;
  const long n = (long)(s.frame_off[b + 1] - s.frame_off[b]) * F;
  const float v = sispec_image(est, tgt, (size_t)s.frame_off[b] * F, n, m, m);
  if (threadIdx.x == 0) out[(size_t)b * out_stride + m] = (double)v;
}
cudaError_t launch_lsd_varlen(const float* est, const float* tgt, int F, const ImageSet& s, double* out, int out_stride, cudaStream_t stream) {
  lsd_varlen_kernel<<<s.batch, 256, 0, stream>>>(est, tgt, F, s, out, out_stride);
  return cudaGetLastError();
}
cudaError_t launch_sispec_varlen(const float* est, const float* tgt, int F, const ImageSet& s, double* out, int out_stride, cudaStream_t stream) {
  sispec_varlen_kernel<<<dim3(s.batch, 2), 256, 0, stream>>>(est, tgt, F, s, out, out_stride);
  return cudaGetLastError();
}

}  // namespace vf
