// Degrading clean speech for the super-resolution test sets (tools/dsp/lowpass.py): scipy.signal.sosfiltfilt as an exact
// chunked scan and resample_poly with float64 taps, both in float64 on packed rows of different lengths.  See kernels.cuh.
#include "kernels.cuh"

namespace vf {
namespace {

// Sample i of row b's input to this pass.  Forward: the odd extension 2 x[0] - x[edge - i] / x[i - edge] /
// 2 x[n-1] - x[n - 2 - (i - edge - n)] (scipy's odd_ext, computed in the input's dtype: rounded to float32 for a
// float32 row).  Backward: the forward result reversed.
template <bool BACK>
__device__ __forceinline__ double pass_in(const SosParams& p, int b, int64_t i) {
  const int64_t n = p.off[b + 1] - p.off[b], ne = p.ext_off[b + 1] - p.ext_off[b];
  if (BACK) return p.yf[p.ext_off[b] + ne - 1 - i];
  const double* x = p.x + p.off[b];
  const int64_t e = p.edge[b];
  if (i >= e && i < e + n) return x[i - e];
  const double v = i < e ? __dsub_rn(2.0 * x[0], x[e - i]) : __dsub_rn(2.0 * x[n - 1], x[n - 2 - (i - e - n)]);
  return p.ext_f32[b] ? (double)__double2float_rn(v) : v;
}

// One thread per chunk.  PHASE_C = false: phase A (zero start state, end state -> state[g]; the last chunk of a row has
// nothing to carry and returns).  PHASE_C = true: start from state[g], write the outputs.  The section arithmetic is
// scipy's _sosfilt loop without contraction: x_new = b0 x + z0; z0 = (b1 x - a1 x_new) + z1; z1 = b2 x - a2 x_new.
template <bool BACK, bool PHASE_C>
__global__ void __launch_bounds__(128) sos_chunk_kernel(SosParams p) {
  const int64_t g = (int64_t)blockIdx.x * 128 + threadIdx.x;
  if (g >= p.chunk_off[p.batch]) return;
  const int b = packed_row(p.chunk_off, p.batch, g);
  const int64_t k = g - p.chunk_off[b];
  const int64_t nc = p.chunk_off[b + 1] - p.chunk_off[b];
  if (!PHASE_C && k == nc - 1) return;
  const int ns = p.n_sections[b];
  const double* T = p.table[b];
  double c[IIR_MAX_SECTIONS][5], z[IIR_MAX_SECTIONS][2];
  double* st = p.state + g * IIR_MAX_STATES;
#pragma unroll
  for (int s = 0; s < IIR_MAX_SECTIONS; ++s) {
    if (s < ns) {
      c[s][0] = __ldg(T + 6 * s); c[s][1] = __ldg(T + 6 * s + 1); c[s][2] = __ldg(T + 6 * s + 2);
      c[s][3] = __ldg(T + 6 * s + 4); c[s][4] = __ldg(T + 6 * s + 5);
      z[s][0] = PHASE_C ? st[2 * s] : 0.0;
      z[s][1] = PHASE_C ? st[2 * s + 1] : 0.0;
    }
  }
  const int64_t n = p.off[b + 1] - p.off[b], ne = p.ext_off[b + 1] - p.ext_off[b];
  const int64_t i0 = k * IIR_CHUNK, i1 = i0 + IIR_CHUNK < ne ? i0 + IIR_CHUNK : ne;
  for (int64_t i = i0; i < i1; ++i) {
    double xc = pass_in<BACK>(p, b, i);
#pragma unroll
    for (int s = 0; s < IIR_MAX_SECTIONS; ++s) {
      if (s < ns) {
        const double xn = __dadd_rn(__dmul_rn(c[s][0], xc), z[s][0]);
        z[s][0] = __dadd_rn(__dsub_rn(__dmul_rn(c[s][1], xc), __dmul_rn(c[s][3], xn)), z[s][1]);
        z[s][1] = __dsub_rn(__dmul_rn(c[s][2], xc), __dmul_rn(c[s][4], xn));
        xc = xn;
      }
    }
    if (PHASE_C) {
      if (!BACK) {
        p.yf[p.ext_off[b] + i] = xc;
      } else {
        const int64_t j = ne - 1 - i - p.edge[b];        // crop edge samples from each end of the reversed result
        if (j >= 0 && j < n) p.out[p.off[b] + j] = xc;
      }
    }
  }
  if (!PHASE_C) {
#pragma unroll
    for (int s = 0; s < IIR_MAX_SECTIONS; ++s)
      if (s < ns) { st[2 * s] = z[s][0]; st[2 * s + 1] = z[s][1]; }
  }
}

// Phase B, one warp per row: lane i < 2 n_sections holds row i of M and state component i; the other lanes hold zeros
// (phase A stores only the live components, so they read nothing).  s_0 = zi * (first input sample) as scipy scales it;
// then for each chunk k the slot's end state e_k is read, s_k written in its place, and s_{k+1} = M s_k + e_k (a
// fixed-order 20-term sum per lane).
template <bool BACK>
__global__ void __launch_bounds__(32) sos_carry_kernel(SosParams p) {
  const int b = blockIdx.x, lane = threadIdx.x;
  const double* T = p.table[b];
  const bool live = lane < 2 * p.n_sections[b];
  double m[IIR_MAX_STATES];
#pragma unroll
  for (int j = 0; j < IIR_MAX_STATES; ++j) m[j] = live ? __ldg(T + IIR_M_AT + lane * IIR_MAX_STATES + j) : 0.0;
  double s = live ? __dmul_rn(__ldg(T + IIR_ZI_AT + lane), pass_in<BACK>(p, b, 0)) : 0.0;
  const int64_t c0 = p.chunk_off[b], nc = p.chunk_off[b + 1] - c0;
  double* st = p.state + c0 * IIR_MAX_STATES + lane;
  double e = (live && nc > 1) ? st[0] : 0.0;
  for (int64_t k = 0; k < nc; ++k) {
    const double e_next = (live && k + 2 < nc) ? st[(k + 1) * IIR_MAX_STATES] : 0.0;   // read before slot k + 1 is written
    if (live) st[k * IIR_MAX_STATES] = s;
    double acc = 0.0;
#pragma unroll
    for (int j = 0; j < IIR_MAX_STATES; ++j) acc = fma(m[j], __shfl_sync(0xffffffffu, s, j), acc);
    s = acc + e;
    e = e_next;
  }
}

// The table of filter blockIdx.x (kernels.cuh): sos and zi copied, zero past n_sections, and M, whose column j (thread j)
// is the state after IIR_CHUNK zero samples from unit state j, run with the section arithmetic of sos_chunk_kernel.
// Columns and rows past 2 n_sections are zero.
__global__ void __launch_bounds__(32) iir_design_kernel(IirDesignParams p) {
  const int f = blockIdx.x, j = threadIdx.x, ns = p.n_sections[f];
  double* T = p.tables + (size_t)f * IIR_TABLE;
  for (int i = j; i < IIR_ZI_AT; i += 32) T[i] = i < 6 * ns ? p.sos[f][i] : 0.0;
  if (j < IIR_MAX_STATES) T[IIR_ZI_AT + j] = j < 2 * ns ? p.zi[f][j] : 0.0;
  if (j >= IIR_MAX_STATES) return;
  double z[IIR_MAX_SECTIONS][2];
#pragma unroll
  for (int s = 0; s < IIR_MAX_SECTIONS; ++s) {
    z[s][0] = (2 * s == j && j < 2 * ns) ? 1.0 : 0.0;
    z[s][1] = (2 * s + 1 == j && j < 2 * ns) ? 1.0 : 0.0;
  }
  if (j < 2 * ns) {
    for (int i = 0; i < IIR_CHUNK; ++i) {
      double xc = 0.0;
#pragma unroll
      for (int s = 0; s < IIR_MAX_SECTIONS; ++s) {
        if (s < ns) {
          const double* c = p.sos[f] + 6 * s;
          const double xn = __dadd_rn(__dmul_rn(c[0], xc), z[s][0]);
          z[s][0] = __dadd_rn(__dsub_rn(__dmul_rn(c[1], xc), __dmul_rn(c[4], xn)), z[s][1]);
          z[s][1] = __dsub_rn(__dmul_rn(c[2], xc), __dmul_rn(c[5], xn));
          xc = xn;
        }
      }
    }
  }
#pragma unroll
  for (int s = 0; s < IIR_MAX_SECTIONS; ++s) {
    T[IIR_M_AT + (2 * s) * IIR_MAX_STATES + j] = z[s][0];
    T[IIR_M_AT + (2 * s + 1) * IIR_MAX_STATES + j] = z[s][1];
  }
}

// resample_poly: one thread per output sample, taps j ascending.
__global__ void __launch_bounds__(256) resample_f64_kernel(ResampleF64Params p) {
  const int64_t g = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (g >= p.out_off[p.batch]) return;
  const int b = packed_row(p.out_off, p.batch, g);
  const int64_t m = g - p.out_off[b], n = p.in_off[b + 1] - p.in_off[b];
  const int64_t up = p.up[b], down = p.down[b], half = p.half[b];
  double acc = 0.0;
  if (m < (n * up + down - 1) / down) {
    const double* x = p.x + p.in_off[b];
    const double* h = p.taps + p.tap_at[b];
    const int64_t c = m * down + half;                      // taps index of x[0]
    int64_t j0 = c - 2 * half;                              // first j with c - up j <= 2 half
    j0 = j0 > 0 ? (j0 + up - 1) / up : 0;
    int64_t j1 = c / up;                                    // last j with c - up j >= 0
    if (j1 > n - 1) j1 = n - 1;
    for (int64_t j = j0; j <= j1; ++j) acc = fma(__ldg(x + j), __ldg(h + (c - up * j)), acc);
  }
  p.y[g] = acc;
}

unsigned blocks(int64_t n, int per) { return (unsigned)((n + per - 1) / per); }

}  // namespace

cudaError_t launch_sosfiltfilt(const SosParams& p, cudaStream_t stream) {
  const unsigned gc = blocks(p.chunk_off[p.batch], 128);
  sos_chunk_kernel<false, false><<<gc, 128, 0, stream>>>(p);
  sos_carry_kernel<false><<<p.batch, 32, 0, stream>>>(p);
  sos_chunk_kernel<false, true><<<gc, 128, 0, stream>>>(p);
  sos_chunk_kernel<true, false><<<gc, 128, 0, stream>>>(p);
  sos_carry_kernel<true><<<p.batch, 32, 0, stream>>>(p);
  sos_chunk_kernel<true, true><<<gc, 128, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_iir_design(const IirDesignParams& p, cudaStream_t stream) {
  iir_design_kernel<<<p.n, 32, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_resample_f64(const ResampleF64Params& p, cudaStream_t stream) {
  if (p.out_off[p.batch] > 0) resample_f64_kernel<<<blocks(p.out_off[p.batch], 256), 256, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace vf
