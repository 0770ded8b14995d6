// librosa 0.8's resample(res_type = "kaiser_best" / "kaiser_fast"), the rate conversion of librosa.load(path, sr=...)
// (tools/utils.py:46-48, evaluation_proc/metrics.py:33-34): resampy's band-limited sinc interpolation of packed float32 rows,
// each with its own filter table.  See kernels.cuh and oracle/resampy.py.
#include "kernels.cuh"
#include "resample.cuh"

namespace vf {
namespace {

// One thread per output sample g of the packed output; row b's slots past n_valid[b] = int(n sample_ratio) are zeros.  The
// body is sinc_output (resample.cuh), which the streaming resampler shares.
__global__ void __launch_bounds__(256) sinc_resample_kernel(const SincParams p) {
  const int64_t g = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (g >= p.out_off[p.batch]) return;
  const int b = packed_row(p.out_off, p.batch, g);
  const int64_t t = g - p.out_off[b];
  float y = 0.f;
  if (t < p.n_valid[b])
    y = sinc_output(FlatInput{p.x + p.in_off[b]}, t, p.in_off[b + 1] - p.in_off[b], p.ratio[b], p.num_table[b],
                    p.tables + p.tab_at[b], p.nwin[b]);
  p.y[g] = y;
}

}  // namespace

cudaError_t launch_sinc_resample(const SincParams& p, cudaStream_t stream) {
  const int64_t n = p.out_off[p.batch];
  if (n > 0) sinc_resample_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace vf
