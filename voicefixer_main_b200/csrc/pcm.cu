// librosa.load(path, sr=None, mono=True)'s samples of WAV data chunks (tools/utils.py:46-48, evaluation_proc/metrics.py:33-34):
// soundfile's (libsndfile's) float read of every sample, then librosa 0.8's to_mono, numpy's float32 mean over the channels
// of each frame.  See kernels.cuh and oracle/wavfile.py.
#include "../../include/b200vf.h"
#include "kernels.cuh"

namespace vf {
namespace {

// Sample c of the frame at p: libsndfile's float value, and (exact) the float64 value soundfile's double read gives.
template <int F> struct Pcm;
template <> struct Pcm<VF_PCM_U8> {
  static __device__ __forceinline__ int v(const uint8_t* p, int c) { return (int)p[c] - 128; }
  static __device__ __forceinline__ float sample(const uint8_t* p, int c) { return (float)v(p, c) * 0x1p-7f; }
  static __device__ __forceinline__ double exact(const uint8_t* p, int c) { return (double)v(p, c) * 0x1p-7; }
};
template <> struct Pcm<VF_PCM_S16> {
  static __device__ __forceinline__ int v(const uint8_t* p, int c) { return reinterpret_cast<const int16_t*>(p)[c]; }
  static __device__ __forceinline__ float sample(const uint8_t* p, int c) { return (float)v(p, c) * 0x1p-15f; }
  static __device__ __forceinline__ double exact(const uint8_t* p, int c) { return (double)v(p, c) * 0x1p-15; }
};
template <> struct Pcm<VF_PCM_S24> {   // three byte loads: a 24-bit frame sits at any byte
  static __device__ __forceinline__ int v(const uint8_t* p, int c) {
    const uint8_t* q = p + 3 * c;
    return (int)(((uint32_t)q[0] << 8) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 24)) >> 8;
  }
  static __device__ __forceinline__ float sample(const uint8_t* p, int c) { return (float)v(p, c) * 0x1p-23f; }
  static __device__ __forceinline__ double exact(const uint8_t* p, int c) { return (double)v(p, c) * 0x1p-23; }
};
template <> struct Pcm<VF_PCM_S32> {
  static __device__ __forceinline__ int v(const uint8_t* p, int c) { return reinterpret_cast<const int32_t*>(p)[c]; }
  static __device__ __forceinline__ float sample(const uint8_t* p, int c) { return __int2float_rn(v(p, c)) * 0x1p-31f; }
  static __device__ __forceinline__ double exact(const uint8_t* p, int c) { return (double)v(p, c) * 0x1p-31; }
};
template <> struct Pcm<VF_PCM_F32> {
  static __device__ __forceinline__ float sample(const uint8_t* p, int c) { return reinterpret_cast<const float*>(p)[c]; }
  static __device__ __forceinline__ double exact(const uint8_t* p, int c) { return (double)sample(p, c); }
};
template <> struct Pcm<VF_PCM_F64> {
  static __device__ __forceinline__ double exact(const uint8_t* p, int c) { return reinterpret_cast<const double*>(p)[c]; }
  static __device__ __forceinline__ float sample(const uint8_t* p, int c) { return __double2float_rn(exact(p, c)); }
};

// numpy's float32 x.mean(axis=1) of one frame of C >= 2 samples: add.reduce's pairwise_sum over the contiguous run (below 8
// values one running sum from 0; from 8 on eight running sums, added as a tree, then the rest one by one; C <= 64 stays
// within one 128-value block) added to the reduction's identity 0, then one division by C.  _rn intrinsics: no FMA
// contraction or reassociation.
template <int F>
__device__ __forceinline__ float frame_mean(const uint8_t* p, int C) {
  float res;
  if (C < 8) {
    res = 0.f;
    for (int c = 0; c < C; ++c) res = __fadd_rn(res, Pcm<F>::sample(p, c));
  } else {
    float r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = Pcm<F>::sample(p, j);
    int i = 8;
    for (; i < C - C % 8; i += 8) {
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(r[j], Pcm<F>::sample(p, i + j));
    }
    res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])), __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
    for (; i < C; ++i) res = __fadd_rn(res, Pcm<F>::sample(p, i));
    res = __fadd_rn(0.f, res);
  }
  return __fdiv_rn(res, (float)C);
}

template <int F>
__device__ __forceinline__ void decode_frame(const uint8_t* p, int C, float* mono, double* first) {
  *mono = C == 1 ? Pcm<F>::sample(p, 0) : frame_mean<F>(p, C);
  if (first) *first = Pcm<F>::exact(p, 0);
}

__global__ void __launch_bounds__(256) decode_pcm_kernel(const __grid_constant__ PcmParams p) {
  const int64_t g = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (g >= p.out_off[p.batch]) return;
  const int b = packed_row(p.out_off, p.batch, g);
  const int C = p.channels[b];
  const int64_t t = g - p.out_off[b];
  double* first = p.first ? p.first + g : nullptr;
  float* mono = p.mono + g;
  switch (p.format[b]) {
    case VF_PCM_U8: decode_frame<VF_PCM_U8>(p.bytes + p.byte_off[b] + t * C, C, mono, first); break;
    case VF_PCM_S16: decode_frame<VF_PCM_S16>(p.bytes + p.byte_off[b] + t * 2 * C, C, mono, first); break;
    case VF_PCM_S24: decode_frame<VF_PCM_S24>(p.bytes + p.byte_off[b] + t * 3 * C, C, mono, first); break;
    case VF_PCM_S32: decode_frame<VF_PCM_S32>(p.bytes + p.byte_off[b] + t * 4 * C, C, mono, first); break;
    case VF_PCM_F32: decode_frame<VF_PCM_F32>(p.bytes + p.byte_off[b] + t * 4 * C, C, mono, first); break;
    default: decode_frame<VF_PCM_F64>(p.bytes + p.byte_off[b] + t * 8 * C, C, mono, first); break;
  }
}

}  // namespace

cudaError_t launch_decode_pcm(const PcmParams& p, cudaStream_t stream) {
  const int64_t n = p.out_off[p.batch];
  if (n > 0) decode_pcm_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace vf
