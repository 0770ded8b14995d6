// The data-movement kernels of the packed and streaming calls (include/b200vf.h).  The row copy moves rows of floats
// between packed buffers, plan buffers and the streams' device rings: the streaming calls' gather of a step's input from
// the rings and crop of each chunk's kept centre, vf_vocoder_varlen's scatter and pack, and the varlen restores' mel
// gathers.  vf_restore_windows instead overlap-adds each synthesis-weighted window into the caller's per-stream accumulators
// and then emits the finished samples; vf_resample_rings resamples the streams' input rings into the restore rings.  Each
// is one launch per sub-batch (the emission: per VL_MAX_CLIPS streams), whatever the number of streams: the tables are
// __grid_constant__ kernel parameters (about 24.6 KB for the row copy, 13 KB for the overlap-add at 256 rows), so no host
// memory is read after the call returns and no copy of a table is queued.  One thread per float copied, accumulated or
// resampled; a warp's threads nearly always fall into one row, so the table lookups broadcast.
#include "kernels.cuh"
#include "resample.cuh"

namespace vf {

namespace {

constexpr int STREAM_THREADS = 256;

}  // namespace

__global__ void __launch_bounds__(STREAM_THREADS) row_copy_kernel(const __grid_constant__ RowCopyParams p) {
  const int64_t i = (int64_t)blockIdx.x * STREAM_THREADS + threadIdx.x;
  if (i >= p.off[p.rows]) return;
  const int c = packed_row(p.off, p.rows, i);
  const int64_t j = i - p.off[c];
  float v = 0.f;                                   // before the lead or past the valid count: the zero padding
  if (j >= p.lead[c] && j < p.n_valid[c]) {
    int64_t r = p.phase[c] + j;
    if (r >= p.ring) r -= p.ring;
    v = __ldg(p.src[c] + r);
  }
  p.dst[c][j] = v;
}

// Ascending window order per position, and the product rounded before the add (no FMA contraction): the bits of F.fold
// (CUDA col2im: each output starts at 0 and adds the windows in ascending order) of the rounded `frames * window` tensor.
// The accumulator carries the partial sum from call to call, so the order holds across sub-batches and steps too.
__global__ void __launch_bounds__(STREAM_THREADS) window_ola_kernel(const __grid_constant__ WindowOlaParams p) {
  const int64_t i = (int64_t)blockIdx.x * STREAM_THREADS + threadIdx.x;
  if (i >= p.pos[p.runs]) return;
  const int r = packed_row(p.pos, p.runs, i);
  const int64_t t = p.lo[r] + (i - p.pos[r]);
  int lo = p.first[r], hi = p.first[r + 1];        // the first window with start + W > t: the earliest that covers t
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (p.start[mid] + p.W <= t) lo = mid + 1; else hi = mid;
  }
  int64_t slot = p.acc_phase[r] + (i - p.pos[r]);  // a run spans at most acc_len positions, so one subtraction wraps it
  if (slot >= p.acc_len) slot -= p.acc_len;
  float* a = p.acc + p.acc_row[r] + slot;
  float v = *a;
  for (int w = lo; w < p.first[r + 1] && p.start[w] <= t; ++w) {
    if (t >= p.end[w]) continue;                   // past the stream's end
    const int64_t j = t - p.start[w];
    v = __fadd_rn(v, __fmul_rn(__ldg(p.synth + j), __ldg(p.restored + p.src[w] + j)));
  }
  *a = v;
}

__global__ void __launch_bounds__(STREAM_THREADS) window_emit_kernel(const __grid_constant__ WindowEmitParams p) {
  const int64_t i = (int64_t)blockIdx.x * STREAM_THREADS + threadIdx.x;
  if (i >= p.off[p.n]) return;
  const int e = packed_row(p.off, p.n, i);
  int64_t r = p.phase[e] + (i - p.off[e]);         // count <= acc_len, so one subtraction wraps it
  if (r >= p.acc_len) r -= p.acc_len;
  float* a = p.acc + p.row[e] + r;
  p.out[i] = *a;
  *a = 0.f;                                        // the slot is free for a later position, or a later stream
}

// vf_resample_rings resamples live streams from their own input rings into the restore rings (or a packed buffer): one
// launch per filter family per RING_RESAMPLE_ROWS rows, its table a __grid_constant__ parameter (about 20 KB for poly, 25 KB
// for sinc at 256 rows), one thread per output sample of the rows of one filter family.  The arithmetic is poly_output /
// sinc_output (resample.cuh), the bodies of the whole-signal kernels, reading the stream's ring row instead of a flat row.
__device__ __forceinline__ float ring_output(const PolyRingParams& p, int r, const RingInput& x, int64_t m) {
  const int up = p.up[r], down = p.down[r];
  return poly_output(x, m, p.r.n[r], up, down, p.taps[r], 10 * (up > down ? up : down));
}
__device__ __forceinline__ float ring_output(const SincRingParams& p, int r, const RingInput& x, int64_t m) {
  if (m >= p.n_valid[r]) return 0.f;              // a closed stream's fix_length zeros
  return sinc_output(x, m, p.r.n[r], p.ratio[r], p.num_table[r], p.tab[r], p.nwin[r]);
}

template <class P>
__global__ void __launch_bounds__(STREAM_THREADS) stream_resample_kernel(const __grid_constant__ P p) {
  const RingResampleRows& q = p.r;
  const int64_t i = (int64_t)blockIdx.x * STREAM_THREADS + threadIdx.x;
  if (i >= q.off[q.rows]) return;
  const int r = packed_row(q.off, q.rows, i);
  const int64_t j = i - q.off[r];
  const float y = ring_output(p, r, RingInput{q.ring + q.src[r], q.in_len, q.a0[r], q.a_ph[r]}, q.m0[r] + j);
  int64_t d = j;
  if (q.d_ph[r] >= 0) {                            // a ring row: j < out_len, so one subtraction wraps it
    d = q.d_ph[r] + j;
    if (d >= q.out_len) d -= q.out_len;
  }
  q.out[q.dst[r] + d] = y;
}

template <class P>
cudaError_t launch_ring_resample(const P& p, cudaStream_t stream) {
  const int64_t n = p.r.off[p.r.rows];
  if (n > 0) stream_resample_kernel<P><<<(unsigned)((n + STREAM_THREADS - 1) / STREAM_THREADS), STREAM_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}
cudaError_t launch_stream_resample(const PolyRingParams& p, cudaStream_t stream) { return launch_ring_resample(p, stream); }
cudaError_t launch_stream_resample(const SincRingParams& p, cudaStream_t stream) { return launch_ring_resample(p, stream); }

cudaError_t launch_row_copy(const RowCopyParams& p, cudaStream_t stream) {
  const int64_t n = p.off[p.rows];
  row_copy_kernel<<<(unsigned)((n + STREAM_THREADS - 1) / STREAM_THREADS), STREAM_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_window_ola(const WindowOlaParams& p, cudaStream_t stream) {
  const int64_t n = p.pos[p.runs];
  window_ola_kernel<<<(unsigned)((n + STREAM_THREADS - 1) / STREAM_THREADS), STREAM_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_window_emit(const WindowEmitParams& p, cudaStream_t stream) {
  const int64_t n = p.off[p.n];
  window_emit_kernel<<<(unsigned)((n + STREAM_THREADS - 1) / STREAM_THREADS), STREAM_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace vf
