// Shared-memory radix-4 Stockham FFT and the real-FFT splits of the STFT kernels, templated on the complex type: float2
// for the front end (frontend.cu) and the ISTFT (istft.cu), double2 for the metric STFT (metrics.cu), STOI (speech_metrics.cu)
// and the pre-filter (prefilter.cu).  A 2N-point REAL transform is one N-point complex FFT on the even/odd-packed frame
// z[n] = x[2n] + i x[2n+1] plus the real-FFT split (forward) or its inverse (backward).  Also the frame loads' two
// centre-padding rules.
#pragma once
#include <cuda_runtime.h>

namespace vf {

template <class C>
using real_of = decltype(C::x);

template <class C>
__device__ __forceinline__ C cmul(C a, C b) {
  return C{a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x};
}

// N = 4^PASSES points on N / 4 threads (tid 0 .. N/4 - 1), natural-order output.  Several transforms may share a block,
// since every thread of the block runs the passes and their __syncthreads.  In: buf0[0..N) (synchronised).  Out: the
// returned pointer (buf1 after an odd number of passes, buf0 after an even one) holds the forward DFT, e^{-2 pi i jk/N};
// the block is synchronised on return.  tw[j] = e^{-2 pi i j / N}.
template <int PASSES, class C>
__device__ __forceinline__ C* fft_forward(C* buf0, C* buf1, const C* __restrict__ tw, int tid) {
  constexpr int Q = 1 << (2 * PASSES - 2);
  C* src = buf0;
  C* dst = buf1;
#pragma unroll
  for (int pass = 0; pass < PASSES; ++pass) {
    const int ns = 1 << (2 * pass);
    const int k = tid & (ns - 1);
    const int tw_step = k * (Q / ns);
    C a = src[tid];
    C bq = src[tid + Q];
    C c = src[tid + 2 * Q];
    C d = src[tid + 3 * Q];
    if (pass > 0) {
      bq = cmul(bq, __ldg(tw + tw_step));
      c = cmul(c, __ldg(tw + 2 * tw_step));
      d = cmul(d, __ldg(tw + 3 * tw_step));
    }
    const C s0 = C{a.x + c.x, a.y + c.y}, s1 = C{a.x - c.x, a.y - c.y};
    const C s2 = C{bq.x + d.x, bq.y + d.y}, s3 = C{bq.x - d.x, bq.y - d.y};
    const int o = ((tid - k) << 2) + k;
    dst[o] = C{s0.x + s2.x, s0.y + s2.y};
    dst[o + ns] = C{s1.x + s3.y, s1.y - s3.x};          // s1 - i*s3
    dst[o + 2 * ns] = C{s0.x - s2.x, s0.y - s2.y};
    dst[o + 3 * ns] = C{s1.x - s3.y, s1.y + s3.x};      // s1 + i*s3
    __syncthreads();
    C* tmp = src; src = dst; dst = tmp;
  }
  return src;
}

// Bin k (0..H) of the 2H-point real DFT from the packed H-point spectrum Z: X[k] = E[k] + e^{-2 pi i k/2H} O[k].
// tw[k] = e^{-2 pi i k / 2H}.
template <int H, class C>
__device__ __forceinline__ C rfft_split(const C* Z, const C* __restrict__ tw, int k) {
  const real_of<C> half = 0.5;
  const C zk = Z[k & (H - 1)];
  const C zr = Z[(H - k) & (H - 1)];
  const C e = C{half * (zk.x + zr.x), half * (zk.y - zr.y)};      // (Zk + conj Zr)/2
  const C o = C{half * (zk.y + zr.y), -half * (zk.x - zr.x)};     // -i (Zk - conj Zr)/2
  const C wo = cmul(o, __ldg(tw + k));
  return C{e.x + wo.x, e.y + wo.y};
}

// The last step of the packed 2048-point real inverse (istft.cu describes it): z = FFT(conj Z) of the packed spectrum Z, and
// the frame's samples 2j, 2j + 1 are conj(z[j]) / 1024 times the window; 256 threads
template <class C>
__device__ __forceinline__ void irfft_unpack(C* out, const C* z, const C* __restrict__ win, int tid) {
  const real_of<C> scale = real_of<C>(1) / real_of<C>(1024);
  for (int j = tid; j < 1024; j += 256) {
    const C v = z[j], w = __ldg(win + j);
    out[j] = C{v.x * scale * w.x, -v.y * scale * w.y};
  }
}

// Centre padding, as an index s (-pad <= s < n + pad) into a clip of n samples.  reflect_once: one reflection at each end
// (torch's and librosa's reflect padding, n > pad).
__device__ __forceinline__ long reflect_once(long s, long n) {
  if (s < 0) s = -s;
  if (s >= n) s = 2L * (n - 1) - s;
  return s;
}

// np.pad(x, 1024, mode="reflect") at padded position s + 1024: the even periodic extension of period 2 (n - 1), which
// is what numpy's repeated reflection makes of a clip of n <= 1024 samples; a one-sample clip pads with itself
__device__ __forceinline__ int64_t reflect_repeated(int64_t s, int64_t n) {
  if (n == 1) return 0;
  const int64_t P = 2 * (n - 1);
  s %= P;
  if (s < 0) s += P;
  return s >= n ? P - s : s;
}

// Windowed, reflect-padded (center=True, pad n_fft/2) frame t (the caller's int or long frame index) of x[0..n) at hop
// HOP, packed z[j] = w[2j] x[2j] + i w[2j+1] x[2j+1] into buf; 256 threads
template <int HOP, class C, class I>
__device__ __forceinline__ void load_frame_packed(C* buf, const float* __restrict__ x, long n, I t,
                                                  const real_of<C>* __restrict__ window, int tid) {
  for (int j = tid; j < 1024; j += 256) {
    real_of<C> v[2];
#pragma unroll
    for (int e = 0; e < 2; ++e)
      v[e] = (real_of<C>)__ldg(x + reflect_once((long)t * HOP + 2 * j + e - 1024, n)) * __ldg(window + 2 * j + e);
    buf[j] = C{v[0], v[1]};
  }
}

}  // namespace vf
