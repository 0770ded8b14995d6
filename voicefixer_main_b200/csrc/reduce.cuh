// Fixed-order (deterministic) block reduction shared by the metric kernels (edges.cu, metrics.cu).
#pragma once
#include <cuda_runtime.h>

namespace vf {

// Sum of v over a CTA of 256 threads (eight warps); every thread receives the sum.
__device__ __forceinline__ double block_sum(double v, double* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += sh[i];
  return s;
}

}  // namespace vf
