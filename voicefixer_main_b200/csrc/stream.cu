// The two data-movement kernels of vf_restore_chunks (include/b200vf.h): the gather that builds a step's packed input from
// the streams' device rings, and the crop that keeps each chunk's centre of the packed restored output.  Between them runs
// the varlen restore chain (engine.cu).  Each is one launch per sub-batch of at most VL_MAX_CLIPS chunks, whatever the
// number of streams: the chunk table is a __grid_constant__ kernel parameter (about 8 KB for the gather at 256 rows), so
// no host memory is read after the call returns and no copy of the table is queued.  One thread per packed sample; a
// warp's threads nearly always fall into one chunk, so the table lookups broadcast.
#include "kernels.cuh"

namespace vf {

namespace {

constexpr int STREAM_THREADS = 256;

// The row c of a packed table with bounds[c] <= i < bounds[c + 1] (bounds increasing, i < bounds[n])
__device__ __forceinline__ int find_row(const int64_t* bounds, int n, int64_t i) {
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (bounds[mid] <= i) lo = mid; else hi = mid;
  }
  return lo;
}

}  // namespace

__global__ void __launch_bounds__(STREAM_THREADS) stream_gather_kernel(const __grid_constant__ ChunkGatherParams p) {
  const int64_t i = (int64_t)blockIdx.x * STREAM_THREADS + threadIdx.x;
  if (i >= p.off[p.rows]) return;
  const int c = find_row(p.off, p.rows, i);
  const int64_t j = i - p.off[c];
  float v = 0.f;                                   // past the stream's end: BoxcarOverlapAdd's zero padding
  if (j < p.n_valid[c]) {
    int64_t r = p.phase[c] + j;                    // j < length <= ring_len, so one subtraction wraps it
    if (r >= p.ring_len) r -= p.ring_len;
    v = __ldg(p.ring + p.src[c] + r);
  }
  p.out[i] = v;
}

__global__ void __launch_bounds__(STREAM_THREADS) stream_crop_kernel(const __grid_constant__ ChunkCropParams p) {
  const int64_t i = (int64_t)blockIdx.x * STREAM_THREADS + threadIdx.x;
  if (i >= p.keep[p.chunks]) return;
  const int c = find_row(p.keep, p.chunks, i);
  p.kept[i] = __ldg(p.restored + p.src[c] + (i - p.keep[c]));
}

cudaError_t launch_stream_gather(const ChunkGatherParams& p, cudaStream_t stream) {
  const int64_t n = p.off[p.rows];
  stream_gather_kernel<<<(unsigned)((n + STREAM_THREADS - 1) / STREAM_THREADS), STREAM_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_stream_crop(const ChunkCropParams& p, cudaStream_t stream) {
  const int64_t n = p.keep[p.chunks];
  stream_crop_kernel<<<(unsigned)((n + STREAM_THREADS - 1) / STREAM_THREADS), STREAM_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace vf
