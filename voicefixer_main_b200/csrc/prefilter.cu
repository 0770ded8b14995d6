// The VoiceFixer pip package's pre-filter, remove_higher_frequency(wav, ratio) (voicefixer/base.py; restore_inmem's
// mode 1), of packed float32 rows in float64 (oracle/prefilter.py restates it):
//   1. librosa 0.8's stft: reflect padding by 1024 (numpy's repeated reflection when n <= 1024), periodic hann, hop 512,
//      the fp64 Stockham FFT of fft.cuh; the complex spectrum goes to the call's scratch.
//   2. per row, the bins' energies sum_t max(log10(|X| + EPS), 0) and the package's sequential scan for the first bin
//      whose running sum reaches ratio times the total: the cutoff.
//   3. per frame, the bins below the cutoff scaled by |X| / (|X| + EPS) (the package's spec * cos, spec * sin), the
//      inverse real FFT times the window, written over the frame's own spectrum slot.
//   4. librosa 0.8's istft overlap-add and window_sumsquare division, trimmed to 512 (n // 512) samples, one thread per
//      output sample, rounded to float32 once.
// The cutoff is a threshold decision, so every step is float64.  A row's values depend on its own samples only.
#include <cfloat>

#include "fft.cuh"
#include "gemm.cuh"
#include "kernels.cuh"

namespace vf {
namespace {

constexpr double PF_EPS = 1e-8;
constexpr int PF_BINS = 1025, PF_HOP = 512, PF_CUTOFF_THREADS = 1024;

// One CTA per frame of the sub-batch
__global__ void __launch_bounds__(256) prefilter_stft_kernel(const PrefilterParams p) {
  __shared__ double2 buf0[1024];
  __shared__ double2 buf1[1024];
  const int tid = threadIdx.x;
  const int64_t g = blockIdx.x;
  const int b = packed_row(p.frame_off, p.batch, g);
  const int64_t t = g - p.frame_off[b];
  const float* x = p.x + p.in_off[b];
  const int64_t n = p.in_off[b + 1] - p.in_off[b];
  bool finite = true;
  for (int j = tid; j < 1024; j += 256) {       // z[j] = w[2j] x[2j] + i w[2j+1] x[2j+1] of the padded frame
    double v[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const float s = __ldg(x + reflect_repeated(t * PF_HOP + 2 * j + e - 1024, n));
      finite = finite && isfinite(s);
      v[e] = (double)s * __ldg(p.window + 2 * j + e);
    }
    buf0[j] = make_double2(v[0], v[1]);
  }
  if (!finite && p.err) atomicCAS(p.err, 0, ERR_NONFINITE_INPUT);
  __syncthreads();
  const double2* Z = fft_forward<5>(buf0, buf1, p.tw1024, tid);
  double2* out = p.spec + (size_t)g * PF_BINS;
  for (int k = tid; k < PF_BINS; k += 256) out[k] = rfft_split<1024>(Z, p.tw2048, k);
}

// max(log10(|X| + EPS), 0): log10 is negative exactly below 1
__device__ __forceinline__ double pf_feature(double2 X) {
  const double v = hypot(X.x, X.y) + PF_EPS;
  return v >= 1.0 ? log10(v) : 0.0;
}

// One CTA per row: thread k sums bin k over the row's frames in ascending order (thread 0 also bin 1024); thread 0 then
// sums the energies over bins in ascending order and runs the package's scan on the same running sums
__global__ void __launch_bounds__(PF_CUTOFF_THREADS) prefilter_cutoff_kernel(const PrefilterParams p) {
  __shared__ double energy[PF_BINS];
  const int b = blockIdx.x, k = threadIdx.x;
  const int64_t T = p.frame_off[b + 1] - p.frame_off[b];
  const double2* X = p.spec + (size_t)p.frame_off[b] * PF_BINS;
  double acc = 0.0, last = 0.0;
#pragma unroll 4
  for (int64_t t = 0; t < T; ++t) {
    acc += pf_feature(X[t * PF_BINS + k]);
    if (k == 0) last += pf_feature(X[t * PF_BINS + PF_BINS - 1]);
  }
  energy[k] = acc;
  if (k == 0) energy[PF_BINS - 1] = last;
  __syncthreads();
  if (k != 0) return;
  double total = 0.0;
  for (int i = 0; i < PF_BINS; ++i) total += energy[i];
  const double threshold = total * p.ratio;
  // while i < 1025 and cur < threshold: cur += energy[i + 1]; i += 1.  The package would index past bin 1024 when the
  // last running sum still misses the threshold; that needs total * ratio > total, which rounding cannot give for
  // ratio <= 1, and is kept as "remove nothing" (cutoff 1025)
  double cur = energy[0];
  int i = 0;
  while (i < PF_BINS && cur < threshold) {
    if (i + 1 == PF_BINS) { i = PF_BINS; break; }
    cur += energy[i + 1];
    ++i;
  }
  p.cutoff[b] = i;
}

// The kept bin k of spectrum slot X: |X| re / (|X| + EPS) + i |X| im / (|X| + EPS), or 0 at or past the cutoff
__device__ __forceinline__ double2 pf_kept(const double2* X, int k, int cutoff) {
  if (k >= cutoff) return make_double2(0.0, 0.0);
  const double2 v = X[k];
  const double m = hypot(v.x, v.y);
  return make_double2(m * (v.x / (m + PF_EPS)), m * (v.y / (m + PF_EPS)));
}

// One CTA per frame: the masked spectrum's inverse real FFT (irfft: the imaginary parts of bins 0 and 1024 are dropped)
// times the window, as 2048 doubles over the frame's own slot.  See istft.cu for the packed inverse.
__global__ void __launch_bounds__(256) prefilter_istft_kernel(const PrefilterParams p) {
  __shared__ double2 buf0[1024];
  __shared__ double2 buf1[1024];
  const int tid = threadIdx.x;
  const int64_t g = blockIdx.x;
  const int b = packed_row(p.frame_off, p.batch, g);
  const int cutoff = p.cutoff[b];
  double2* slot = p.spec + (size_t)g * PF_BINS;
  for (int k = tid; k < 1024; k += 256) {
    double2 yk = pf_kept(slot, k, cutoff), yr = pf_kept(slot, 1024 - k, cutoff);
    if (k == 0) { yk.y = 0.0; yr.y = 0.0; }
    const double2 e = make_double2(0.5 * (yk.x + yr.x), 0.5 * (yk.y - yr.y));     // (Yk + conj Yr)/2
    const double2 d = make_double2(0.5 * (yk.x - yr.x), 0.5 * (yk.y + yr.y));     // (Yk - conj Yr)/2
    const double2 w = __ldg(p.tw2048 + k);
    const double2 o = cmul(d, make_double2(w.x, -w.y));                            // * e^{+2 pi i k/2048}
    buf0[k] = make_double2(e.x - o.y, -(e.y + o.x));                               // conj(E + i O)
  }
  __syncthreads();                              // every read of the slot is done before the frame overwrites it
  const double2* z = fft_forward<5>(buf0, buf1, p.tw1024, tid);
  irfft_unpack(slot, z, reinterpret_cast<const double2*>(p.window), tid);
}

// One thread per output sample j of the sub-batch: padded position j + 1024 gathers its (at most four) frames in
// ascending order and divides by their window sum of squares where that is above float32 tiny (librosa's
// window_sumsquare test).  Products and sums are rounded one by one, as numpy computes them.
__global__ void __launch_bounds__(256) prefilter_ola_kernel(const PrefilterParams p) {
  const int64_t g = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (g >= p.out_off[p.batch]) return;
  const int b = packed_row(p.out_off, p.batch, g);
  const int64_t pos = g - p.out_off[b] + 1024;
  const int64_t T = p.frame_off[b + 1] - p.frame_off[b];
  const int64_t t_lo = pos > 2047 ? (pos - 2047 + PF_HOP - 1) / PF_HOP : 0;
  const int64_t t_hi = min(pos / PF_HOP, T - 1);
  const double* frames = reinterpret_cast<const double*>(p.spec + (size_t)p.frame_off[b] * PF_BINS);
  double acc = 0.0, ws = 0.0;
  for (int64_t t = t_lo; t <= t_hi; ++t) {
    const int off = (int)(pos - t * PF_HOP);
    acc = __dadd_rn(acc, frames[(size_t)t * 2 * PF_BINS + off]);
    const double w = __ldg(p.window + off);
    ws = __dadd_rn(ws, __dmul_rn(w, w));
  }
  p.y[g] = (float)(ws > (double)FLT_MIN ? acc / ws : acc);
}

}  // namespace

cudaError_t launch_prefilter(const PrefilterParams& p, cudaStream_t stream) {
  const int64_t frames = p.frame_off[p.batch], samples = p.out_off[p.batch];
  prefilter_stft_kernel<<<(unsigned)frames, 256, 0, stream>>>(p);
  prefilter_cutoff_kernel<<<p.batch, PF_CUTOFF_THREADS, 0, stream>>>(p);
  prefilter_istft_kernel<<<(unsigned)frames, 256, 0, stream>>>(p);
  if (samples > 0) prefilter_ola_kernel<<<(unsigned)((samples + 255) / 256), 256, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace vf
