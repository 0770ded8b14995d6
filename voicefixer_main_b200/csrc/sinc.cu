// librosa 0.8's resample(res_type = "kaiser_best" / "kaiser_fast"), the rate conversion of librosa.load(path, sr=...)
// (tools/utils.py:46-48, evaluation_proc/metrics.py:33-34): resampy's band-limited sinc interpolation of packed float32 rows,
// each with its own filter table.  See kernels.cuh and oracle/resampy.py.
#include "kernels.cuh"

namespace vf {
namespace {

__device__ __forceinline__ int sinc_row_of(const int64_t* off, int batch, int64_t g) {
  int lo = 0, hi = batch;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (off[mid] <= g) lo = mid; else hi = mid;
  }
  return lo;
}

// One wing of resampy's loop: y += (win[o + i step] + eta delta[o + i step]) * x[src(i)] for i < min(count, (nwin - o) /
// step), with o = int(frac num_table) and eta its remainder.  float64 products and sums, y rounded to float32 per tap.
template <int DIR>
__device__ __forceinline__ float sinc_wing(float y, double frac, int64_t count, const double2* __restrict__ tab, int64_t nwin,
                                           int64_t step, double num_table, const float* __restrict__ x) {
  const double index_frac = __dmul_rn(frac, num_table);
  const int64_t offset = (int64_t)index_frac;
  const double eta = __dsub_rn(index_frac, (double)offset);
  int64_t k_max = (nwin - offset) / step;
  if (count < k_max) k_max = count;
  for (int64_t i = 0; i < k_max; ++i) {
    const double2 wd = __ldg(tab + offset + i * step);
    const double weight = __dadd_rn(wd.x, __dmul_rn(eta, wd.y));
    y = __double2float_rn(__dadd_rn((double)y, __dmul_rn(weight, (double)__ldg(x + DIR * i))));
  }
  return y;
}

// One thread per output sample g of the packed output; row b's slots past n_valid[b] = int(n sample_ratio) are zeros.
__global__ void __launch_bounds__(256) sinc_resample_kernel(const SincParams p) {
  const int64_t g = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (g >= p.out_off[p.batch]) return;
  const int b = sinc_row_of(p.out_off, p.batch, g);
  const int64_t t = g - p.out_off[b];
  float y = 0.f;
  if (t < p.n_valid[b]) {
    const double ratio = p.ratio[b], scale = ratio < 1.0 ? ratio : 1.0, num_table = (double)p.num_table[b];
    const int64_t step = (int64_t)__dmul_rn(scale, num_table), nwin = p.nwin[b];
    const int64_t n_orig = p.in_off[b + 1] - p.in_off[b];
    const float* x = p.x + p.in_off[b];
    const double2* tab = p.tables + p.tab_at[b];
    const double tr = __ddiv_rn((double)t, ratio);                   // t_out[t] = arange(n_out)[t] / sample_ratio
    const int64_t n = (int64_t)tr;
    const double frac = __dmul_rn(scale, __dsub_rn(tr, (double)n));
    y = sinc_wing<-1>(y, frac, n + 1, tab, nwin, step, num_table, x + n);                       // x[n - i]
    y = sinc_wing<1>(y, __dsub_rn(scale, frac), n_orig - n - 1, tab, nwin, step, num_table, x + n + 1);   // x[n + 1 + k]
  }
  p.y[g] = y;
}

}  // namespace

cudaError_t launch_sinc_resample(const SincParams& p, cudaStream_t stream) {
  const int64_t n = p.out_off[p.batch];
  if (n > 0) sinc_resample_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace vf
