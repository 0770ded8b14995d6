// The time-domain keys of AudioMetrics.evaluation (evaluation_proc/metrics.py:58-64): speechmetrics' sisdr and pystoi
// 0.3.3's stoi(target, estimate, 44100 or 16000, extended=False), restated in oracle/speech_metrics.py (44.1 kHz) and
// tests/oracle_16k.py (16 kHz).  Everything is float64:
// STOI's silent-frame mask is a threshold decision that fp32 rounding could flip.  See kernels.cuh for the pipeline.
#include "fft.cuh"
#include "kernels.cuh"
#include "reduce.cuh"

namespace vf {
namespace {

constexpr double EPS = 2.220446049250313e-16;   // np.finfo(np.float64).eps

// SI-SDR of pair blockIdx.x, r = target, e = estimate, both zero-padded to N: a = (eps + r.e) / (r.r + eps), then
// Sss = sum (a r)^2 and Snn = sum (e - a r)^2 in a second pass (no expansion: it would cancel when e ~ r).
__global__ void __launch_bounds__(256) sisdr_kernel(TimeScoreParams p) {
  __shared__ double sh[8];
  const int b = blockIdx.x;
  const float* e = p.est + p.e_off[b];
  const float* r = p.tgt + p.t_off[b];
  const int64_t ne = p.e_off[b + 1] - p.e_off[b], nt = p.t_off[b + 1] - p.t_off[b], n = ne > nt ? ne : nt;
  double rr = 0, re = 0;
  for (int64_t i = threadIdx.x; i < n; i += 256) {
    const double rv = i < nt ? (double)__ldg(r + i) : 0.0, ev = i < ne ? (double)__ldg(e + i) : 0.0;
    rr += rv * rv;
    re += rv * ev;
  }
  rr = block_sum(rr, sh);
  re = block_sum(re, sh);
  const double a = (EPS + re) / (rr + EPS);
  double ss = 0, nn = 0;
  for (int64_t i = threadIdx.x; i < n; i += 256) {
    const double rv = i < nt ? (double)__ldg(r + i) : 0.0, ev = i < ne ? (double)__ldg(e + i) : 0.0;
    const double t = a * rv, d = ev - t;
    ss += t * t;
    nn += d * d;
  }
  ss = block_sum(ss, sh);
  nn = block_sum(nn, sh);
  if (threadIdx.x == 0) p.out[2 * b] = 10.0 * log10((EPS + ss) / (EPS + nn));
}

// scipy.signal.resample_poly(x, up, down, window=taps / up) of the padded clip: y[m] = sum_j x[j] taps[down m - up j + L]
// over the taps in range, j ascending.  One thread per output sample; blockIdx.y = 0 target, 1 estimate.
__global__ void __launch_bounds__(256) stoi_resample_kernel(TimeScoreParams p) {
  const int z = blockIdx.y;
  const int64_t g = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (g >= p.r_off[p.batch]) return;
  const int b = packed_row(p.r_off, p.batch, g);
  const int64_t m = g - p.r_off[b];
  const int64_t* off = z ? p.e_off : p.t_off;
  const float* x = (z ? p.est : p.tgt) + off[b];
  const int64_t nx = off[b + 1] - off[b];
  const int64_t c = m * p.down + p.half;                      // taps index of x[0]
  int64_t j0 = c - 2 * p.half;                                 // first j with c - up j <= 2L
  j0 = j0 > 0 ? (j0 + p.up - 1) / p.up : 0;
  int64_t j1 = c / p.up;                                        // last j with c - up j >= 0
  if (j1 > nx - 1) j1 = nx - 1;
  double acc = 0;
  for (int64_t j = j0; j <= j1; ++j) acc += (double)__ldg(x + j) * __ldg(p.taps + (c - p.up * j));
  p.rs[(size_t)z * p.r_off[p.batch] + g] = acc;
}

// 20 log10(||w x_frame|| + eps) of the target's frame slots, one warp per frame, lanes summing in a fixed order.
__global__ void __launch_bounds__(256) stoi_energy_kernel(TimeScoreParams p) {
  const int64_t g = ((int64_t)blockIdx.x * 256 + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (g >= p.f_off[p.batch]) return;
  const int b = packed_row(p.f_off, p.batch, g);
  const double* x = p.rs + p.r_off[b] + (g - p.f_off[b]) * STOI_HOP;
  double acc = 0;
#pragma unroll
  for (int q = 0; q < STOI_FRAME / 32; ++q) {
    const double v = __dmul_rn(__ldg(p.window + lane + 32 * q), x[lane + 32 * q]);
    acc += v * v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) p.energy[g] = 20.0 * log10(sqrt(acc) + EPS);
}

// One block per pair: frame i is kept where (max - 40) - energy_i < 0; src[k] = the k-th kept frame, kept[b] = their count.
__global__ void __launch_bounds__(256) stoi_mask_kernel(TimeScoreParams p) {
  __shared__ double shm[8];
  __shared__ int warp_n[8];
  __shared__ int base;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int64_t f0 = p.f_off[b];
  const int nf = (int)(p.f_off[b + 1] - f0);
  double mx = -INFINITY;
  for (int i = tid; i < nf; i += 256) mx = fmax(mx, p.energy[f0 + i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) shm[w] = mx;
  if (tid == 0) base = 0;
  __syncthreads();
  mx = shm[0];
  for (int i = 1; i < 8; ++i) mx = fmax(mx, shm[i]);
  const double thr = mx - 40.0;
  for (int c0 = 0; c0 < nf; c0 += 256) {
    const int i = c0 + tid;
    const bool keep = i < nf && thr - p.energy[f0 + i] < 0.0;
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_n[w] = __popc(bal);
    __syncthreads();
    int k = base + __popc(bal & ((1u << lane) - 1u));
    for (int q = 0; q < w; ++q) k += warp_n[q];
    if (keep) p.src[f0 + k] = i;
    __syncthreads();
    if (tid == 0) for (int q = 0; q < 8; ++q) base += warp_n[q];
    __syncthreads();
  }
  if (tid == 0) p.kept[b] = base;
}

// Overlap-add of the kept windowed frames at hop 128 into (kept + 1) * 128 samples: chunk j = the first half of kept frame j
// plus the second half of kept frame j - 1 (two terms: the order cannot change the bits).  blockIdx.y = signal.
__global__ void __launch_bounds__(256) stoi_compact_kernel(TimeScoreParams p) {
  const int z = blockIdx.y;
  const int64_t g = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (g >= p.r_off[p.batch]) return;
  const int b = packed_row(p.r_off, p.batch, g);
  const int64_t s = g - p.r_off[b];
  const int K = p.kept[b];
  if (s >= (int64_t)(K + 1) * STOI_HOP) return;
  const int j = (int)(s / STOI_HOP), r = (int)(s % STOI_HOP);
  const size_t plane = (size_t)z * p.r_off[p.batch];
  const double* x = p.rs + plane + p.r_off[b];
  const int* src = p.src + p.f_off[b];
  double v0 = 0, v1 = 0;
  if (j < K) v0 = __dmul_rn(__ldg(p.window + r), x[(int64_t)src[j] * STOI_HOP + r]);
  if (j > 0) v1 = __dmul_rn(__ldg(p.window + STOI_HOP + r), x[(int64_t)src[j - 1] * STOI_HOP + STOI_HOP + r]);
  p.cs[plane + g] = __dadd_rn(v0, v1);
}

// STFT of the compacted signals (frames at range(0, len - 256, 128): kept - 1 of them, window w, rfft(n = 512)) and the
// band values sqrt(sum_{bins in band} |X|^2).  Four frame slots per block, 64 threads each; slots past the pair's frame
// count run the passes (the block synchronises) and write nothing.
__global__ void __launch_bounds__(256) stoi_bands_kernel(TimeScoreParams p) {
  __shared__ double2 buf[4][2][256];
  __shared__ double pw[4][257];
  const int grp = threadIdx.x >> 6, tid = threadIdx.x & 63;
  const int64_t g = (int64_t)blockIdx.x * 4 + grp;
  const int64_t F = p.f_off[p.batch];
  bool active = g < F;
  int b = 0;
  int64_t k = 0;
  if (active) {
    b = packed_row(p.f_off, p.batch, g);
    k = g - p.f_off[b];
    active = k < (int64_t)p.kept[b] - 1;
  }
  for (int z = 0; z < 2; ++z) {
    const double* c = p.cs + (size_t)z * p.r_off[p.batch] + p.r_off[b] + k * STOI_HOP;
    for (int j = tid; j < 256; j += 64) {       // z[j] = w[2j] c[2j] + i w[2j+1] c[2j+1]; zeros past the 256-sample frame
      double2 v = make_double2(0.0, 0.0);
      if (active && j < 128)
        v = make_double2(__dmul_rn(__ldg(p.window + 2 * j), c[2 * j]), __dmul_rn(__ldg(p.window + 2 * j + 1), c[2 * j + 1]));
      buf[grp][0][j] = v;
    }
    __syncthreads();
    const double2* Z = fft_forward<4>(buf[grp][0], buf[grp][1], p.tw256, tid);
    for (int q = tid; q <= 256; q += 64) {
      const double2 X = rfft_split<256>(Z, p.tw512, q);
      const double m = sqrt(X.x * X.x + X.y * X.y);      // np.square(np.abs(X))
      pw[grp][q] = m * m;
    }
    __syncthreads();
    if (active && tid < STOI_BANDS) {
      double s = 0;
      for (int q = p.band_lo[tid]; q < p.band_hi[tid]; ++q) s += pw[grp][q];
      p.tob[((size_t)z * F + g) * STOI_BANDS + tid] = sqrt(s);
    }
    __syncthreads();
  }
}

// One thread per (segment, band) of a pair, 256 per tile: the correlation of the normalised, clipped, mean-removed
// 30-frame band envelopes; the tile's sum goes to partial[].  Items past the pair's segment count add zero.
__global__ void __launch_bounds__(256) stoi_corr_kernel(TimeScoreParams p) {
  __shared__ double sh[8];
  const int t = blockIdx.x;
  const int b = packed_row(p.tile_off, p.batch, t);
  const int64_t item = (t - p.tile_off[b]) * 256 + threadIdx.x;
  const int64_t J = (int64_t)p.kept[b] - 1 - (STOI_SEG - 1);
  double rho = 0;
  if (item < J * STOI_BANDS) {
    const int64_t F = p.f_off[p.batch];
    const int64_t seg = item / STOI_BANDS;
    const int band = (int)(item % STOI_BANDS);
    const double* xs = p.tob + (p.f_off[b] + seg) * STOI_BANDS + band;
    const double* ys = xs + F * STOI_BANDS;
    double x[STOI_SEG], y[STOI_SEG];
    double sxx = 0, syy = 0;
#pragma unroll
    for (int i = 0; i < STOI_SEG; ++i) {
      x[i] = xs[i * STOI_BANDS];
      y[i] = ys[i * STOI_BANDS];
      sxx += x[i] * x[i];
      syy += y[i] * y[i];
    }
    const double nc = sqrt(sxx) / (sqrt(syy) + EPS);
    double mx = 0, my = 0;
#pragma unroll
    for (int i = 0; i < STOI_SEG; ++i) {
      y[i] = fmin(y[i] * nc, x[i] * p.clip);
      mx += x[i];
      my += y[i];
    }
    mx /= STOI_SEG;
    my /= STOI_SEG;
    double nx = 0, ny = 0;
#pragma unroll
    for (int i = 0; i < STOI_SEG; ++i) {
      x[i] -= mx;
      y[i] -= my;
      nx += x[i] * x[i];
      ny += y[i] * y[i];
    }
    nx = sqrt(nx) + EPS;
    ny = sqrt(ny) + EPS;
#pragma unroll
    for (int i = 0; i < STOI_SEG; ++i) rho += (y[i] / ny) * (x[i] / nx);
  }
  const double tot = block_sum(rho, sh);
  if (threadIdx.x == 0) p.partial[t] = tot;
}

// One block per pair: d = (sum of its tiles, in order) / (J * 15), or 1e-5 below 30 STFT frames (pystoi's warning case).
__global__ void __launch_bounds__(256) stoi_final_kernel(TimeScoreParams p) {
  __shared__ double sh[8];
  const int b = blockIdx.x;
  const int64_t J = (int64_t)p.kept[b] - 1 - (STOI_SEG - 1);
  const int64_t tiles = J > 0 ? (J * STOI_BANDS + 255) / 256 : 0;
  double acc = 0;
  for (int64_t i = threadIdx.x; i < tiles; i += 256) acc += p.partial[p.tile_off[b] + i];
  const double tot = block_sum(acc, sh);
  if (threadIdx.x == 0) p.out[2 * b + 1] = J > 0 ? tot / (double)(J * STOI_BANDS) : 1e-5;
}

unsigned blocks(int64_t n, int per) { return (unsigned)((n + per - 1) / per); }

}  // namespace

cudaError_t launch_score_time(const TimeScoreParams& p, cudaStream_t stream) {
  const int64_t R = p.r_off[p.batch], F = p.f_off[p.batch], T = p.tile_off[p.batch];
  sisdr_kernel<<<p.batch, 256, 0, stream>>>(p);
  stoi_resample_kernel<<<dim3(blocks(R, 256), 2), 256, 0, stream>>>(p);
  stoi_energy_kernel<<<blocks(F, 8), 256, 0, stream>>>(p);
  stoi_mask_kernel<<<p.batch, 256, 0, stream>>>(p);
  stoi_compact_kernel<<<dim3(blocks(R, 256), 2), 256, 0, stream>>>(p);
  stoi_bands_kernel<<<blocks(F, 4), 256, 0, stream>>>(p);
  if (T > 0) stoi_corr_kernel<<<(unsigned)T, 256, 0, stream>>>(p);
  stoi_final_kernel<<<p.batch, 256, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace vf
