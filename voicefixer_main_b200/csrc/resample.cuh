// The per-output-sample arithmetic of the float32 resamplers, shared by the whole-signal kernels (resample_poly_kernel in
// edges.cu, sinc_resample_kernel in sinc.cu) and the streaming one (stream_resample_kernel in stream.cu).  Each body is
// templated on how input sample i is read: FlatInput for a packed row, RingInput for a stream's ring row.  The taps, the
// summation order and every rounding live here once, so a stream resampled in pieces from its ring gives the bits of the
// whole signal resampled at once.
#pragma once
#include <cstdint>

namespace vf {

// Input i of a contiguous row
struct FlatInput {
  const float* x;
  __device__ __forceinline__ float operator()(int64_t i) const { return __ldg(x + i); }
};

// Input i of a stream held in a ring row of `len` positions: absolute position i at row[i mod len].  Every read is at or
// after `a0`, whose ring position is `ph`, and less than `len` positions past it, so one subtraction wraps it.
struct RingInput {
  const float* row;
  int64_t len, a0, ph;
  __device__ __forceinline__ float operator()(int64_t i) const {
    int64_t r = ph + (i - a0);
    if (r >= len) r -= len;
    return __ldg(row + r);
  }
};

// Output m of scipy.signal.resample_poly by up / down of an n-sample signal: sum_i h[m down - i up + half] x[i] over the
// taps of the symmetric FIR of 2 half + 1 taps that land on inputs 0 .. n - 1, ascending i, one fmaf per tap.
template <class X>
__device__ __forceinline__ float poly_output(const X& x, int64_t m, int64_t n, int up, int down, const float* __restrict__ h,
                                             int half) {
  const int64_t c = m * down;
  int64_t i_lo = (c - half + up - 1) / up;       // ceil((c - half) / up) for a non-negative numerator
  if (c - half < 0) i_lo = 0;
  int64_t i_hi = (c + half) / up;
  if (i_hi > n - 1) i_hi = n - 1;
  float acc = 0.f;
  for (int64_t i = i_lo; i <= i_hi; ++i) acc = fmaf(__ldg(h + (c - i * up + half)), x(i), acc);
  return acc;
}

// One wing of resampy's loop: y += (win[o + i step] + eta delta[o + i step]) * x(at + DIR i) for i < min(count, (nwin - o) /
// step), with o = int(frac num_table) and eta its remainder.  float64 products and sums, y rounded to float32 per tap.
template <int DIR, class X>
__device__ __forceinline__ float sinc_wing(float y, double frac, int64_t count, const double2* __restrict__ tab, int64_t nwin,
                                           int64_t step, double num_table, const X& x, int64_t at) {
  const double index_frac = __dmul_rn(frac, num_table);
  const int64_t offset = (int64_t)index_frac;
  const double eta = __dsub_rn(index_frac, (double)offset);
  int64_t k_max = (nwin - offset) / step;
  if (count < k_max) k_max = count;
  for (int64_t i = 0; i < k_max; ++i) {
    const double2 wd = __ldg(tab + offset + i * step);
    const double weight = __dadd_rn(wd.x, __dmul_rn(eta, wd.y));
    y = __double2float_rn(__dadd_rn((double)y, __dmul_rn(weight, (double)x(at + DIR * i))));
  }
  return y;
}

// Output t of resampy's resample of an n_orig-sample signal (t below int(n_orig ratio)): the left wing on x[n], x[n - 1],
// .. and the right wing on x[n + 1], x[n + 2], .., n = int(t / ratio).
template <class X>
__device__ __forceinline__ float sinc_output(const X& x, int64_t t, int64_t n_orig, double ratio, int num_table_i,
                                             const double2* __restrict__ tab, int64_t nwin) {
  const double scale = ratio < 1.0 ? ratio : 1.0, num_table = (double)num_table_i;
  const int64_t step = (int64_t)__dmul_rn(scale, num_table);
  const double tr = __ddiv_rn((double)t, ratio);                     // t_out[t] = arange(n_out)[t] / sample_ratio
  const int64_t n = (int64_t)tr;
  const double frac = __dmul_rn(scale, __dsub_rn(tr, (double)n));
  float y = 0.f;
  y = sinc_wing<-1>(y, frac, n + 1, tab, nwin, step, num_table, x, n);                             // x[n - i]
  y = sinc_wing<1>(y, __dsub_rn(scale, frac), n_orig - n - 1, tab, nwin, step, num_table, x, n + 1);   // x[n + 1 + k]
  return y;
}

}  // namespace vf
