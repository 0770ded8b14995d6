// Shared-memory 1024-point complex FFT used by the STFT front end (frontend.cu) and the ISTFT back end (istft.cu) in fp32,
// and by the metric STFT (metrics.cu) in fp64 through the double2 overloads at the end of this file.  256 threads, five
// radix-4 Stockham passes, natural-order output.  A 2048-point REAL transform is one such FFT on the even/odd-packed frame z[n] = x[2n] + i x[2n+1] plus the real-FFT split (forward) or its inverse (backward).
#pragma once
#include <cuda_runtime.h>

namespace vf {

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// In: buf0[0..1023] (synchronised).  Out: returned pointer (== buf1) holds the forward DFT, e^{-2 pi i jk/1024};
// the block is synchronised on return.  tw1024[j] = e^{-2 pi i j / 1024}.
__device__ __forceinline__ float2* fft1024_forward(float2* buf0, float2* buf1, const float2* __restrict__ tw1024, int tid) {
  float2* src = buf0;
  float2* dst = buf1;
#pragma unroll
  for (int pass = 0; pass < 5; ++pass) {
    const int ns = 1 << (2 * pass);
    const int k = tid & (ns - 1);
    const int tw_step = k * (256 / ns);
    float2 a = src[tid];
    float2 bq = src[tid + 256];
    float2 c = src[tid + 512];
    float2 d = src[tid + 768];
    if (pass > 0) {
      bq = cmul(bq, __ldg(tw1024 + tw_step));
      c = cmul(c, __ldg(tw1024 + 2 * tw_step));
      d = cmul(d, __ldg(tw1024 + 3 * tw_step));
    }
    const float2 s0 = make_float2(a.x + c.x, a.y + c.y), s1 = make_float2(a.x - c.x, a.y - c.y);
    const float2 s2 = make_float2(bq.x + d.x, bq.y + d.y), s3 = make_float2(bq.x - d.x, bq.y - d.y);
    const int o = ((tid - k) << 2) + k;
    dst[o] = make_float2(s0.x + s2.x, s0.y + s2.y);
    dst[o + ns] = make_float2(s1.x + s3.y, s1.y - s3.x);          // s1 - i*s3
    dst[o + 2 * ns] = make_float2(s0.x - s2.x, s0.y - s2.y);
    dst[o + 3 * ns] = make_float2(s1.x - s3.y, s1.y + s3.x);      // s1 + i*s3
    __syncthreads();
    float2* tmp = src; src = dst; dst = tmp;
  }
  return src;   // five passes: buf1
}

// Bin k (0..1024) of the 2048-point real DFT from the packed 1024-point spectrum Z: X[k] = E[k] + e^{-2 pi i k/2048} O[k].
__device__ __forceinline__ float2 rfft_split(const float2* Z, const float2* __restrict__ tw2048, int k) {
  const float2 zk = Z[k & 1023];
  const float2 zr = Z[(1024 - k) & 1023];
  const float2 e = make_float2(0.5f * (zk.x + zr.x), 0.5f * (zk.y - zr.y));      // (Zk + conj Zr)/2
  const float2 o = make_float2(0.5f * (zk.y + zr.y), -0.5f * (zk.x - zr.x));     // -i (Zk - conj Zr)/2
  const float2 wo = cmul(o, __ldg(tw2048 + k));
  return make_float2(e.x + wo.x, e.y + wo.y);
}

// Windowed, reflect-padded (center=True, pad n_fft/2) frame t of x[0..n), packed z[j] = x[2j] + i x[2j+1] into buf.
__device__ __forceinline__ void load_frame_packed(float2* buf, const float* __restrict__ x, long n, int t,
                                                  const float* __restrict__ window, int tid) {
  for (int j = tid; j < 1024; j += 256) {
    float v[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      long g = (long)t * 441 + 2 * j + e - 1024;
      if (g < 0) g = -g;
      if (g >= n) g = 2L * (n - 1) - g;
      v[e] = __ldg(x + g) * __ldg(window + 2 * j + e);
    }
    buf[j] = make_float2(v[0], v[1]);
  }
}

// ---- fp64 twins of fft1024_forward / rfft_split for the metric STFT (metrics.cu), which has librosa's float64 FFT.
// Same passes and data flow; the fp32 functions above stay as they are (the front end keeps its bits).
__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
  return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

__device__ __forceinline__ double2* fft1024_forward(double2* buf0, double2* buf1, const double2* __restrict__ tw1024, int tid) {
  double2* src = buf0;
  double2* dst = buf1;
#pragma unroll
  for (int pass = 0; pass < 5; ++pass) {
    const int ns = 1 << (2 * pass);
    const int k = tid & (ns - 1);
    const int tw_step = k * (256 / ns);
    double2 a = src[tid];
    double2 bq = src[tid + 256];
    double2 c = src[tid + 512];
    double2 d = src[tid + 768];
    if (pass > 0) {
      bq = cmul(bq, __ldg(tw1024 + tw_step));
      c = cmul(c, __ldg(tw1024 + 2 * tw_step));
      d = cmul(d, __ldg(tw1024 + 3 * tw_step));
    }
    const double2 s0 = make_double2(a.x + c.x, a.y + c.y), s1 = make_double2(a.x - c.x, a.y - c.y);
    const double2 s2 = make_double2(bq.x + d.x, bq.y + d.y), s3 = make_double2(bq.x - d.x, bq.y - d.y);
    const int o = ((tid - k) << 2) + k;
    dst[o] = make_double2(s0.x + s2.x, s0.y + s2.y);
    dst[o + ns] = make_double2(s1.x + s3.y, s1.y - s3.x);          // s1 - i*s3
    dst[o + 2 * ns] = make_double2(s0.x - s2.x, s0.y - s2.y);
    dst[o + 3 * ns] = make_double2(s1.x - s3.y, s1.y + s3.x);      // s1 + i*s3
    __syncthreads();
    double2* tmp = src; src = dst; dst = tmp;
  }
  return src;
}

__device__ __forceinline__ double2 rfft_split(const double2* Z, const double2* __restrict__ tw2048, int k) {
  const double2 zk = Z[k & 1023];
  const double2 zr = Z[(1024 - k) & 1023];
  const double2 e = make_double2(0.5 * (zk.x + zr.x), 0.5 * (zk.y - zr.y));
  const double2 o = make_double2(0.5 * (zk.y + zr.y), -0.5 * (zk.x - zr.x));
  const double2 wo = cmul(o, __ldg(tw2048 + k));
  return make_double2(e.x + wo.x, e.y + wo.y);
}

// ---- fp64 256-point complex FFT and the 512-point real split, for STOI's STFT (speech_metrics.cu).  The same radix-4
// Stockham passes with 64 threads per transform (tid 0..63); several transforms may share a block, since every thread of
// the block runs the four passes and their __syncthreads.  tw256[j] = e^{-2 pi i j / 256}.
__device__ __forceinline__ double2* fft256_forward(double2* buf0, double2* buf1, const double2* __restrict__ tw256, int tid) {
  double2* src = buf0;
  double2* dst = buf1;
#pragma unroll
  for (int pass = 0; pass < 4; ++pass) {
    const int ns = 1 << (2 * pass);
    const int k = tid & (ns - 1);
    const int tw_step = k * (64 / ns);
    double2 a = src[tid];
    double2 bq = src[tid + 64];
    double2 c = src[tid + 128];
    double2 d = src[tid + 192];
    if (pass > 0) {
      bq = cmul(bq, __ldg(tw256 + tw_step));
      c = cmul(c, __ldg(tw256 + 2 * tw_step));
      d = cmul(d, __ldg(tw256 + 3 * tw_step));
    }
    const double2 s0 = make_double2(a.x + c.x, a.y + c.y), s1 = make_double2(a.x - c.x, a.y - c.y);
    const double2 s2 = make_double2(bq.x + d.x, bq.y + d.y), s3 = make_double2(bq.x - d.x, bq.y - d.y);
    const int o = ((tid - k) << 2) + k;
    dst[o] = make_double2(s0.x + s2.x, s0.y + s2.y);
    dst[o + ns] = make_double2(s1.x + s3.y, s1.y - s3.x);          // s1 - i*s3
    dst[o + 2 * ns] = make_double2(s0.x - s2.x, s0.y - s2.y);
    dst[o + 3 * ns] = make_double2(s1.x - s3.y, s1.y + s3.x);      // s1 + i*s3
    __syncthreads();
    double2* tmp = src; src = dst; dst = tmp;
  }
  return src;   // four passes: buf0
}

// Bin k (0..256) of the 512-point real DFT from the packed 256-point spectrum Z.  tw512[k] = e^{-2 pi i k / 512}.
__device__ __forceinline__ double2 rfft512_split(const double2* Z, const double2* __restrict__ tw512, int k) {
  const double2 zk = Z[k & 255];
  const double2 zr = Z[(256 - k) & 255];
  const double2 e = make_double2(0.5 * (zk.x + zr.x), 0.5 * (zk.y - zr.y));
  const double2 o = make_double2(0.5 * (zk.y + zr.y), -0.5 * (zk.x - zr.x));
  const double2 wo = cmul(o, __ldg(tw512 + k));
  return make_double2(e.x + wo.x, e.y + wo.y);
}

}  // namespace vf
