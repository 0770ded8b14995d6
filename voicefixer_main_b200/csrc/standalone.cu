// Host side of libb200vf.so's plan-free entry points (include/b200vf.h): the stand-alone boundary ops, the scoring of
// packed sets, the SR degradations and the element-wise conversions.  None of them uses a plan: each launches on the
// caller's stream with its own arguments, the context's tables and at most one context-owned Scratch.
#include <climits>
#include <cmath>
#include <cstring>

#include "engine.h"

namespace {

// The opening of plan-free entry point `fn`: `ok` is its argument check (`why` is added to its message); then the
// context's device is made current.
int begin_call(vf_ctx* ctx, const char* fn, bool ok, const char* why = "") {
  if (!ctx) return VF_EINVAL;
  if (!ok) return fail(ctx, VF_EINVAL, "%s: bad arguments%s", fn, why);
  CK(cudaSetDevice(ctx->device));
  return VF_OK;
}

// Consecutive sub-batches of a packed set of `batch` items: a sub-batch takes items until it holds max_rows, or until the
// next item's size_of(i) would take its size past `cap`; an item larger than cap runs alone.  -> the first item of every
// sub-batch, then `batch`.
template <typename Size>
std::vector<int> split(int batch, int max_rows, int64_t cap, Size size_of) {
  std::vector<int> starts{0};
  int64_t size = 0;
  for (int i = 0; i < batch; ++i) {
    const int64_t n = size_of(i);
    if (i - starts.back() == max_rows || (i > starts.back() && size + n > cap)) {
      starts.push_back(i);
      size = 0;
    }
    size += n;
  }
  starts.push_back(batch);
  return starts;
}
std::vector<int> split(int batch, int max_rows) { return split(batch, max_rows, INT64_MAX, [](int) { return int64_t(0); }); }

// The scratch a split call needs: the largest sum of bytes_of(i) over the items of one sub-batch of `starts`
template <typename Bytes>
size_t max_bytes(const std::vector<int>& starts, Bytes bytes_of) {
  size_t need = 0;
  for (size_t k = 0; k + 1 < starts.size(); ++k) {
    size_t sum = 0;
    for (int i = starts[k]; i < starts[k + 1]; ++i) sum += bytes_of(i);
    need = std::max(need, sum);
  }
  return need;
}

constexpr int64_t ITEM_MAX = int64_t(1) << 30;   // samples of one clip of a scored set

// Host offsets of a packed set of `batch` items of `fn`: off[0] == 0, and item i = [off[i], off[i + 1]) holds lo .. hi
// samples.  A rejection names the set (`side`: est, target, x, y) and the item in the entry point's word (clip, pair, row).
int check_offsets(vf_ctx* ctx, const char* fn, const char* side, const char* item, const int64_t* off, int batch, int64_t lo,
                  int64_t hi = INT64_MAX) {
  if (!off || off[0] != 0) return fail(ctx, VF_EINVAL, "%s: %s offsets must start at 0", fn, side);
  for (int i = 0; i < batch; ++i) {
    const long n = (long)(off[i + 1] - off[i]);
    if (n >= lo && n <= hi) continue;
    if (hi == INT64_MAX) return fail(ctx, VF_EINVAL, "%s: %s %s %d has %ld samples (need at least %ld)", fn, side, item, i, n, (long)lo);
    return fail(ctx, VF_EINVAL, "%s: %s %s %d has %ld samples (need %ld .. %ld)", fn, side, item, i, n, (long)lo, (long)hi);
  }
  return VF_OK;
}

constexpr long SCORE_CAP_FRAMES = 16384;   // vf_score_varlen sub-batch cap (frames per side), see b200vf.h

// The per-rate geometry of the scoring calls: AudioMetrics.wav_to_spectrogram's branch (metrics.py:38-47) and pystoi's
// resampling ratio to 10 kHz, chosen once per call from its rate.
struct Geometry {
  int rate, n_fft, hop, bins, mels;
  SparseFb fb;                                                   // the mel filterbank [bins, mels]
  const double* window;                                          // the STFT's float64 window [n_fft]
  cudaError_t (*stft)(const MetricStftParams&, cudaStream_t);
  int stoi_up, stoi_down;                                        // rate -> 10 kHz, reduced by their gcd
  int slot;                                                      // index of the rate's STOI tables
  // librosa's center=True frame count 1 + (n + 2 (n_fft / 2) - n_fft) / hop: 1 + n / 441, or 1 + (n - 1) / 160
  long frames(int64_t n) const { return 1 + (long)((n - n_fft % 2) / hop); }
  int64_t min_samples() const { return n_fft / 2 + 1; }          // one reflection of the n_fft / 2 padding
  int64_t len10(int64_t n) const { return stoi_len10(n, stoi_up, stoi_down); }
};

int geometry(vf_ctx* ctx, const char* fn, int rate, Geometry* g) {
  if (rate == 44100) {
    *g = {44100, 2048, 441, 1025, 128, {ctx->d_fb_f0, ctx->d_fb_len, ctx->d_fb_ofs, ctx->d_fb_val}, ctx->d_window64,
          launch_metric_stft, 100, 441, 0};
    return VF_OK;
  }
  if (rate == 16000) {
    *g = {16000, 743, 160, 372, 80, ctx->fb16k, ctx->d_window743, launch_metric_dft743, 5, 8, 1};
    return VF_OK;
  }
  return fail(ctx, VF_EINVAL, "%s: rate %d Hz (need 44100 or 16000)", fn, rate);
}

int need_fb(vf_ctx* ctx, const Geometry& g) {
  if (g.fb.val) return VF_OK;
  if (g.rate == 44100) return fail(ctx, VF_ESTATE, "mel filterbank not loaded (call vf_load_weights first)");
  return fail(ctx, VF_ESTATE, "16 kHz mel filterbank not loaded (pass \"metrics.mel_16k.fb\" [372, 80] to vf_load_weights)");
}

void set_tables(vf_ctx* ctx, const Geometry& g, MetricStftParams& p) {
  p.window = g.window; p.tw1024 = ctx->d_tw1024d; p.tw2048 = ctx->d_tw2048d; p.tw743 = ctx->d_tw743;
}
void set_fb(const Geometry& g, MelParams& m) {
  m.fb_f0 = g.fb.f0; m.fb_len = g.fb.len; m.fb_ofs = g.fb.ofs; m.fb_val = g.fb.val;
}

// d_stoi_tables layout (doubles): taps (2 half + 1, an odd count), window, tw256 (double2), tw512 (double2)
constexpr size_t stoi_win_at(int half) { return 2 * (size_t)half + 2; }
constexpr size_t stoi_tw256_at(int half) { return stoi_win_at(half) + 256; }
constexpr size_t stoi_tw512_at(int half) { return stoi_tw256_at(half) + 2 * 256; }
constexpr size_t stoi_table_doubles(int half) { return stoi_tw512_at(half) + 2 * 257; }

// The float64 tables of vf_score_time_varlen for the rate of `g`, designed once per context on the host:
// * pystoi's resample_oct(x, 10000, rate) window, Octave's resample filter for p / q = up / down (100 / 441 or 5 / 8):
//   L = ceil((60 - 8) / (28.714 * roll_off)) with cut-off 1 / (2 max(p, q)) and roll_off = cut-off / 10 (L = 15973 or 290),
//   h = kaiser(2L + 1, 0.1102 * (60 - 8.7)) x 2 p cut-off sinc(2 cut-off t), t = -L..L; scipy's resample_poly uses
//   window = h / sum(h), times up.
// * np.hanning(258)[1:-1] (0.5 + 0.5 cos(pi n / 257), n = -255, -253, ..., 255) and the 256 / 512-point twiddles.
int stoi_tables(vf_ctx* ctx, const Geometry& g) {
  if (ctx->d_stoi_tables[g.slot]) return VF_OK;
  const double PI = 3.14159265358979323846;
  const double fc = 1.0 / (2.0 * std::max(g.stoi_up, g.stoi_down)), roll_off = fc / 10, rejection_db = 60.0;
  const long L = (long)std::ceil((rejection_db - 8) / (28.714 * roll_off));
  std::vector<double> t(stoi_table_doubles((int)L), 0.0);
  const double beta = 0.1102 * (rejection_db - 8.7), alpha = (double)L, i0_beta = std::cyl_bessel_i(0.0, beta);
  double sum = 0;
  for (long i = 0; i <= 2 * L; ++i) {
    const double r = (i - alpha) / alpha;
    const double kaiser = std::cyl_bessel_i(0.0, beta * std::sqrt(1 - r * r)) / i0_beta;
    const double x = 2 * fc * (double)(i - L), y = PI * (x == 0 ? 1e-20 : x);     // np.sinc
    t[i] = kaiser * (2 * (double)g.stoi_up * fc * (std::sin(y) / y));
    sum += t[i];
  }
  for (long i = 0; i <= 2 * L; ++i) t[i] = t[i] / sum * g.stoi_up;
  const size_t win = stoi_win_at((int)L), tw256 = stoi_tw256_at((int)L), tw512 = stoi_tw512_at((int)L);
  for (int i = 0; i < 256; ++i) t[win + i] = 0.5 + 0.5 * std::cos(PI * (2 * i - 255) / 257.0);
  for (int j = 0; j < 256; ++j) {
    t[tw256 + 2 * j] = std::cos(2 * PI * j / 256.0);
    t[tw256 + 2 * j + 1] = -std::sin(2 * PI * j / 256.0);
  }
  for (int k = 0; k <= 256; ++k) {
    t[tw512 + 2 * k] = std::cos(2 * PI * k / 512.0);
    t[tw512 + 2 * k + 1] = -std::sin(2 * PI * k / 512.0);
  }
  double* d = nullptr;
  CK(cudaMalloc((void**)&d, t.size() * sizeof(double)));
  const cudaError_t e = cudaMemcpy(d, t.data(), t.size() * sizeof(double), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) cudaFree(d);
  CK(e);
  ctx->d_stoi_tables[g.slot] = d;
  ctx->stoi_half[g.slot] = (int)L;
  return VF_OK;
}

// pystoi's thirdoct(10000, 512, 15, 150): band k spans the rfft bins nearest (first of ties) to 150 * 2^((2k -+ 1) / 6)
void stoi_bands(int* lo, int* hi) {
  auto nearest = [](double f) {
    int best = 0;
    double d = INFINITY;
    for (int q = 0; q <= 256; ++q) {
      const double e = (q * (10000.0 / 512) - f) * (q * (10000.0 / 512) - f);
      if (e < d) { d = e; best = q; }
    }
    return best;
  };
  for (int k = 0; k < STOI_BANDS; ++k) {
    lo[k] = nearest(150 * std::pow(2.0, (2 * k - 1) / 6.0));
    hi[k] = nearest(150 * std::pow(2.0, (2 * k + 1) / 6.0));
  }
}

// The input windows of the float32 resamplers as resample.cuh computes them, on the host: [*first, *last] are the inputs
// output m reads of an n-input signal (n = VF_RESAMPLE_OPEN while a stream is open: no clamp at its end); first > last when
// it reads none.  The sinc arithmetic is the kernel's float64 arithmetic, operation for operation.
void poly_window(int64_t m, int64_t n, int up, int down, int64_t* first, int64_t* last) {
  const int64_t half = 10 * (int64_t)std::max(up, down), c = m * down;
  *first = c - half < 0 ? 0 : (c - half + up - 1) / up;
  *last = std::min((c + half) / up, n - 1);
}
struct SincGeom {
  double ratio, scale, num_table;
  int64_t step, nwin;
  int64_t wing(double frac) const { return (nwin - (int64_t)(frac * num_table)) / step; }    // a wing's length bound
  int64_t kmax() const { return nwin / step; }                                              // its largest value
  void window(int64_t t, int64_t n, int64_t* first, int64_t* last) const {
    const double tr = (double)t / ratio;
    const int64_t nt = (int64_t)tr;
    const double frac = scale * (tr - (double)nt);
    const int64_t kl = std::min(nt + 1, wing(frac)), kr = std::min(n - nt - 1, wing(scale - frac));
    *first = kl > 0 ? nt - kl + 1 : nt + 1;
    *last = kr > 0 ? nt + kr : kl > 0 ? nt : nt - 1;
  }
};

// vf_resample_rings' checks of one row.  -> why it is refused, or nullptr with the first input it may read (a0) and, for a
// sinc row, its count of non-zero outputs.
struct RingRow {
  int64_t a0, n_valid;
};
const char* ring_row(const vf_resample_row& w, int n_streams, int64_t in_len, int n_out_streams, int64_t out_len, RingRow* c) {
  static thread_local char msg[192];
  if (w.stream < 0 || w.stream >= n_streams) return "stream out of range";
  if (w.m0 < 0 || w.m1 < w.m0) return "bad output range (need 0 <= m0 <= m1)";
  const bool open = w.n == VF_RESAMPLE_OPEN;
  if (!open && (w.n < 1 || w.n > (int64_t(1) << 40))) return "input count n must be 1 .. 2^40, or VF_RESAMPLE_OPEN";
  if (w.avail < 0 || (!open && w.avail > w.n)) return "avail must be 0 .. n";
  if (w.out_stream >= 0) {
    if (w.out_stream >= n_out_streams || out_len < 1) return "out_stream is not a row of the output ring";
    if (w.m1 - w.m0 > out_len) return "more outputs than the output ring holds";
  } else if (w.out_stream != -1 || w.out_offset < 0) {
    return "out_stream must be a ring row or -1 (packed, out_offset >= 0)";
  }
  int64_t out_n = INT64_MAX;                         // the signal's output length once closed
  int64_t first = 0, last = -1;                      // the inputs the row reads
  c->n_valid = INT64_MAX;
  if (w.family == VF_RESAMPLE_POLY) {
    if (!w.taps || w.table || w.up < 1 || w.down < 1 || w.up > (1 << 20) || w.down > (1 << 20))
      return "a poly row needs taps, no table and up, down in 1 .. 2^20";
    if (!open) out_n = (w.n * w.up + w.down - 1) / w.down;
    if (w.m1 > out_n) return "output range past the signal's ceil(n up / down) outputs";
    if (w.m1 > w.m0) {
      int64_t f, l;
      poly_window(w.m0, w.n, w.up, w.down, &first, &l);
      poly_window(w.m1 - 1, w.n, w.up, w.down, &f, &last);
    }
  } else if (w.family == VF_RESAMPLE_SINC) {
    if (!w.table || w.taps || reinterpret_cast<uintptr_t>(w.table) % alignof(double2) != 0)
      return "a sinc row needs a 16-byte aligned table and no taps";
    if (!(w.ratio > 0.0) || !std::isfinite(w.ratio) || w.num_table < 1 || w.nwin <= w.num_table || w.nwin > (int64_t(1) << 30))
      return "a sinc row needs ratio > 0, num_table >= 1 and more than num_table table entries";
    const double scale = std::min(w.ratio, 1.0);
    const SincGeom g{w.ratio, scale, (double)w.num_table, (int64_t)(scale * (double)w.num_table), w.nwin};
    if (g.step < 1) return "the sinc index step int(min(1, ratio) num_table) is 0";
    if (!open) {
      c->n_valid = (int64_t)((double)w.n * w.ratio);
      out_n = (int64_t)std::ceil((double)w.n * w.ratio);
      if (c->n_valid < 1) return "too few inputs to resample (int(n ratio) is 0)";
    }
    if (w.m1 > out_n) return "output range past the signal's ceil(n ratio) outputs";
    const int64_t m_end = std::min(w.m1, c->n_valid);          // outputs that read inputs
    if (m_end > w.m0) {
      first = std::max<int64_t>(0, (int64_t)((double)w.m0 / w.ratio) - (g.kmax() - 1));
      // the last input: exact per output from the end down, until no earlier output can read further
      for (int64_t t = m_end - 1; t >= w.m0; --t) {
        int64_t f, l;
        g.window(t, w.n, &f, &l);
        last = std::max(last, l);
        if ((int64_t)((double)t / w.ratio) + g.kmax() <= last) break;
      }
      if (last < first) last = first - 1;
    }
  } else {
    return "unknown family";
  }
  if (first <= last) {
    if (last > w.avail - 1) {
      snprintf(msg, sizeof msg, "outputs %ld .. %ld read input %ld, past the %ld inputs in the ring", (long)w.m0, (long)w.m1 - 1,
               (long)last, (long)w.avail);
      return msg;
    }
    if (first < w.avail - in_len) {
      snprintf(msg, sizeof msg, "outputs from %ld read input %ld, which the ring of %ld no longer holds", (long)w.m0, (long)first,
               (long)in_len);
      return msg;
    }
  }
  c->a0 = std::max<int64_t>(first, 0);
  return nullptr;
}

}  // namespace

extern "C" {

VF_API int vf_istft(vf_ctx* ctx, const float* real, const float* imag, int batch, int frames, int64_t length, float* wav_out, void* stream) {
  const int rc = begin_call(ctx, "vf_istft", real && imag && wav_out && batch > 0 && batch <= 65535 && frames > 0 && length > 0,
                            " (batch must be 1 .. 65535)");
  if (rc) return rc;
  if (length + 1024 > (int64_t)(frames - 1) * ctx->cfg.hop + 2048)
    return fail(ctx, VF_EINVAL, "vf_istft: %d frames cover %ld samples, fewer than length %ld + n_fft/2", frames, (long)(frames - 1) * ctx->cfg.hop + 2048, (long)length);
  cudaStream_t st = (cudaStream_t)stream;
  float* frames_buf = nullptr;           // stream-ordered scratch: no plan is tied to a bare ISTFT
  CK(cudaMallocAsync((void**)&frames_buf, (size_t)batch * frames * 2048 * 4, st));
  IstftFramesParams fp;
  memset(&fp, 0, sizeof fp);
  fp.real = real; fp.imag = imag; fp.batch = batch; fp.T = frames;
  fp.window = ctx->d_window; fp.tw1024 = ctx->d_tw1024; fp.tw2048 = ctx->d_tw2048; fp.frames = frames_buf;
  cudaError_t e1 = launch_istft_frames(fp, st);
  IstftOlaParams op;
  memset(&op, 0, sizeof op);
  op.frames = frames_buf; op.batch = batch; op.T = frames; op.length = (long)length; op.window = ctx->d_window;
  op.out = wav_out; op.out_ld = (long)length;
  cudaError_t e2 = e1 == cudaSuccess ? launch_istft_ola(op, st) : e1;
  cudaFreeAsync(frames_buf, st);
  if (e2 != cudaSuccess) return fail(ctx, VF_ECUDA, "istft launch: %s", cudaGetErrorString(e2));
  ctx->launches += 2;
  return VF_OK;
}

// ---------------------------------------------------------------------------------------------- stand-alone boundary ops
VF_API int vf_mel(vf_ctx* ctx, const float* specgram, int64_t n_outer, int64_t frames, int64_t stride_outer, int64_t stride_freq,
                  int64_t stride_time, float* mel_out, void* stream) {
  const int rc = begin_call(ctx, "vf_mel", specgram && mel_out && n_outer > 0 && frames > 0 && n_outer <= 65535);
  if (rc) return rc;
  if (!ctx->d_fb_val) return fail(ctx, VF_ESTATE, "mel filterbank not loaded (call vf_load_weights first)");
  MelParams p;
  memset(&p, 0, sizeof p);
  p.in = specgram; p.n_outer = (long)n_outer; p.T = (long)frames; p.so = (long)stride_outer; p.sf = (long)stride_freq; p.st = (long)stride_time;
  p.out = mel_out; p.fb_f0 = ctx->d_fb_f0; p.fb_len = ctx->d_fb_len; p.fb_ofs = ctx->d_fb_ofs; p.fb_val = ctx->d_fb_val;
  CK(launch_mel(p, (cudaStream_t)stream));
  ctx->launches++;
  return VF_OK;
}

VF_API int vf_resample_poly(vf_ctx* ctx, const float* wav, int batch, int64_t n, int up, int down, const float* taps, int n_taps,
                            float* out, int64_t n_out, void* stream) {
  const int rc = begin_call(ctx, "vf_resample_poly", wav && taps && out && batch > 0 && n > 0 && up > 0 && down > 0 && n_taps >= 1 &&
                                                         (n_taps & 1), " (n_taps must be odd)");
  if (rc) return rc;
  if (n_out != (n * up + down - 1) / down) return fail(ctx, VF_EINVAL, "vf_resample_poly: n_out must be ceil(n * up / down) = %ld", (long)((n * up + down - 1) / down));
  CK(launch_resample_poly(wav, batch, (long)n, up, down, taps, n_taps / 2, out, (long)n_out, (cudaStream_t)stream));
  ctx->launches++;
  return VF_OK;
}

VF_API int vf_amp_to_original_f(vf_ctx* ctx, const float* mel_est, const float* mel_target, int batch, int frames, float* mel_out, void* stream) {
  const int rc = begin_call(ctx, "vf_amp_to_original_f", mel_est && mel_target && mel_out && batch > 0 && frames > 0);
  if (rc) return rc;
  CK(launch_amp_to_original(mel_est, mel_target, batch, frames, mel_out, (cudaStream_t)stream));
  ctx->launches++;
  return VF_OK;
}

VF_API int vf_lsd(vf_ctx* ctx, const float* est, const float* target, int images, int frames, int bins, float* out, void* stream) {
  const int rc = begin_call(ctx, "vf_lsd", est && target && out && images > 0 && frames > 0 && bins > 0);
  if (rc) return rc;
  CK(launch_lsd(est, target, images, frames, bins, out, (cudaStream_t)stream));
  ctx->launches++;
  return VF_OK;
}

VF_API int vf_sispec(vf_ctx* ctx, const float* est, const float* target, int batch, int64_t n, int est_map, int target_map, float* out, void* stream) {
  const int rc = begin_call(ctx, "vf_sispec", est && target && out && batch > 0 && n > 0 && est_map >= 0 && est_map <= 2 &&
                                                  target_map >= 0 && target_map <= 2);
  if (rc) return rc;
  CK(launch_sispec(est, target, batch, (long)n, est_map, target_map, out, (cudaStream_t)stream));
  ctx->launches++;
  return VF_OK;
}

// ---------------------------------------------------------------------------------------------------------------- scoring
VF_API int vf_metric_spectrogram_ex(vf_ctx* ctx, const float* wav, const int64_t* offsets, int batch, float* sp_out,
                                    float* mel_out, int rate, void* stream) {
  static const char* fn = "vf_metric_spectrogram";
  Geometry g;
  int rc = begin_call(ctx, fn, wav && sp_out && batch > 0);
  if (!rc) rc = geometry(ctx, fn, rate, &g);
  if (!rc) rc = check_offsets(ctx, fn, "wav", "clip", offsets, batch, g.min_samples(), ITEM_MAX);
  if (!rc && mel_out) rc = need_fb(ctx, g);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const std::vector<int> starts = split(batch, SCORE_MAX_IMAGES);
  long rows = 0;
  for (size_t k = 0; k + 1 < starts.size(); ++k) {
    const int s = starts[k];
    MetricStftParams p;
    memset(&p, 0, sizeof p);
    p.batch = starts[k + 1] - s;
    p.sources = 1;
    p.wav[0] = wav; p.sp[0] = sp_out + (size_t)rows * g.bins;
    set_tables(ctx, g, p);
    for (int i = 0; i <= p.batch; ++i) p.off[0][i] = offsets[s + i];
    for (int i = 0; i < p.batch; ++i) p.frame_off[i + 1] = p.frame_off[i] + g.frames(offsets[s + i + 1] - offsets[s + i]);
    CK(g.stft(p, st));
    ctx->launches++;
    rows += (long)p.frame_off[p.batch];
  }
  if (mel_out) {
    MelParams m;
    memset(&m, 0, sizeof m);
    m.in = sp_out; m.n_outer = 1; m.T = rows; m.so = 0; m.sf = 1; m.st = g.bins;
    m.out = mel_out;
    set_fb(g, m);
    CK(launch_mel(m, st, g.bins, g.mels));
    ctx->launches++;
  }
  return VF_OK;
}
VF_API int vf_metric_spectrogram(vf_ctx* ctx, const float* wav, const int64_t* offsets, int batch, float* sp_out, float* mel_out,
                                 void* stream) {
  return vf_metric_spectrogram_ex(ctx, wav, offsets, batch, sp_out, mel_out, 44100, stream);
}

VF_API int vf_ssim(vf_ctx* ctx, const float* est, const float* target, int images, int frames, int bins, double* out, void* stream) {
  const int rc = begin_call(ctx, "vf_ssim", est && target && out && images > 0);
  if (rc) return rc;
  if (frames < 7 || bins < 7) return fail(ctx, VF_EINVAL, "vf_ssim: a %d x %d image is smaller than the 7 x 7 window", frames, bins);
  cudaStream_t st = (cudaStream_t)stream;
  const int per = ssim_tiles(frames, bins);
  double* partial = nullptr;                 // stream-ordered scratch
  CK(cudaMallocAsync((void**)&partial, (size_t)per * std::min(images, SCORE_MAX_IMAGES) * sizeof(double), st));
  const std::vector<int> starts = split(images, SCORE_MAX_IMAGES);
  cudaError_t e = cudaSuccess;
  for (size_t k = 0; k + 1 < starts.size() && e == cudaSuccess; ++k) {
    const int s = starts[k];
    SsimParams p;
    memset(&p, 0, sizeof p);
    p.batch = starts[k + 1] - s;
    const size_t off = (size_t)s * frames * bins;
    p.x = est + off; p.y = target + off; p.F = bins; p.partial = partial;
    for (int i = 0; i <= p.batch; ++i) { p.frame_off[i] = (int64_t)i * frames; p.tile_off[i] = i * per; }
    e = launch_ssim(p, out + s, 1, st);
    ctx->launches += 2;
  }
  cudaFreeAsync(partial, st);
  if (e != cudaSuccess) return fail(ctx, VF_ECUDA, "ssim launch: %s", cudaGetErrorString(e));
  return VF_OK;
}

VF_API int vf_score_varlen_ex(vf_ctx* ctx, const float* est, const int64_t* est_offsets, const float* target,
                              const int64_t* target_offsets, int batch, double* out, int rate, void* stream) {
  static const char* fn = "vf_score_varlen";
  Geometry g;
  int rc = begin_call(ctx, fn, est && target && out && batch > 0);
  if (!rc) rc = geometry(ctx, fn, rate, &g);
  if (!rc) rc = check_offsets(ctx, fn, "est", "clip", est_offsets, batch, g.min_samples(), ITEM_MAX);
  if (!rc) rc = check_offsets(ctx, fn, "target", "clip", target_offsets, batch, g.min_samples(), ITEM_MAX);
  if (rc) return rc;
  std::vector<long> T(batch);
  for (int i = 0; i < batch; ++i) {
    T[i] = g.frames(est_offsets[i + 1] - est_offsets[i]);
    const long tt = g.frames(target_offsets[i + 1] - target_offsets[i]);
    if (T[i] != tt) return fail(ctx, VF_EINVAL, "vf_score_varlen: pair %d: est has %ld frames, target %ld", i, T[i], tt);
    if (T[i] < 7) return fail(ctx, VF_EINVAL, "vf_score_varlen: pair %d has %ld frames, fewer than SSIM's 7", i, T[i]);
  }
  rc = need_fb(ctx, g);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int B = g.bins, M = g.mels;
  // sub-batches of at most SCORE_MAX_IMAGES pairs and SCORE_CAP_FRAMES frames per side.  Scratch per pair: two
  // spectrograms, two mels, its SSIM tile sums.
  const std::vector<int> starts = split(batch, SCORE_MAX_IMAGES, SCORE_CAP_FRAMES, [&](int i) { return (int64_t)T[i]; });
  rc = acquire_scratch(ctx, ctx->score, max_bytes(starts, [&](int i) {
    return (size_t)T[i] * (2 * B + 2 * M) * 4 + (size_t)(ssim_tiles(T[i], B) + ssim_tiles(T[i], M)) * 8;
  }), st);
  if (rc) return rc;
  cudaError_t e = cudaSuccess;
  for (size_t k = 0; k + 1 < starts.size() && e == cudaSuccess; ++k) {
    const int s = starts[k], nb = starts[k + 1] - starts[k];
    MetricStftParams p;
    memset(&p, 0, sizeof p);
    ImageSet set;
    memset(&set, 0, sizeof set);
    p.batch = set.batch = nb;
    p.sources = 2;
    for (int i = 0; i <= nb; ++i) { p.off[0][i] = est_offsets[s + i]; p.off[1][i] = target_offsets[s + i]; }
    for (int i = 0; i < nb; ++i) p.frame_off[i + 1] = set.frame_off[i + 1] = p.frame_off[i] + T[s + i];
    const long F = (long)p.frame_off[nb];
    float* sp_e = static_cast<float*>(ctx->score.p);
    float* sp_t = sp_e + (size_t)F * B;
    float* mel_e = sp_t + (size_t)F * B;
    float* mel_t = mel_e + (size_t)F * M;
    double* partial = reinterpret_cast<double*>(mel_t + (size_t)F * M);   // F * (2306 or 904) floats: 8-byte aligned
    p.wav[0] = est; p.wav[1] = target; p.sp[0] = sp_e; p.sp[1] = sp_t;
    set_tables(ctx, g, p);
    e = g.stft(p, st);
    MelParams m;                              // both spectrograms in one launch: outer index 0 = est, 1 = target
    memset(&m, 0, sizeof m);
    m.in = sp_e; m.n_outer = 2; m.T = F; m.so = F * B; m.sf = 1; m.st = B;
    m.out = mel_e;
    set_fb(g, m);
    if (e == cudaSuccess) e = launch_mel(m, st, B, M);
    double* o = out + (size_t)s * 8;
    const float* img[2][2] = {{sp_e, sp_t}, {mel_e, mel_t}};
    const int bins[2] = {B, M};
    for (int r = 0; r < 2 && e == cudaSuccess; ++r) {        // keys 0-3 on the spectrogram, 4-7 on the mel
      e = launch_lsd_varlen(img[r][0], img[r][1], bins[r], set, o + 4 * r, 8, st);
      if (e == cudaSuccess) e = launch_sispec_varlen(img[r][0], img[r][1], bins[r], set, o + 4 * r + 1, 8, st);
      SsimParams q;
      memset(&q, 0, sizeof q);
      q.x = img[r][0]; q.y = img[r][1]; q.F = bins[r]; q.batch = nb; q.partial = partial;
      for (int i = 0; i <= nb; ++i) q.frame_off[i] = set.frame_off[i];
      for (int i = 0; i < nb; ++i) q.tile_off[i + 1] = q.tile_off[i] + ssim_tiles(T[s + i], bins[r]);
      if (e == cudaSuccess) e = launch_ssim(q, o + 4 * r + 3, 8, st);
    }
    ctx->launches += 10;
  }
  rc = mark_use(ctx, ctx->score.order, st);
  if (e != cudaSuccess) return fail(ctx, VF_ECUDA, "score launch: %s", cudaGetErrorString(e));
  return rc;
}
VF_API int vf_score_varlen(vf_ctx* ctx, const float* est, const int64_t* est_offsets, const float* target, const int64_t* target_offsets,
                           int batch, double* out, void* stream) {
  return vf_score_varlen_ex(ctx, est, est_offsets, target, target_offsets, batch, out, 44100, stream);
}

VF_API int vf_score_time_varlen_ex(vf_ctx* ctx, const float* est, const int64_t* est_offsets, const float* target,
                                   const int64_t* target_offsets, int batch, double* out, int rate, void* stream) {
  static const char* fn = "vf_score_time_varlen";
  Geometry g;
  int rc = begin_call(ctx, fn, est && target && out && batch > 0);
  if (!rc) rc = geometry(ctx, fn, rate, &g);
  if (!rc) rc = check_offsets(ctx, fn, "est", "pair", est_offsets, batch, 1, ITEM_MAX);
  if (!rc) rc = check_offsets(ctx, fn, "target", "pair", target_offsets, batch, 1, ITEM_MAX);
  if (rc) return rc;
  std::vector<int64_t> N(batch);
  for (int i = 0; i < batch; ++i) {
    N[i] = std::max(est_offsets[i + 1] - est_offsets[i], target_offsets[i + 1] - target_offsets[i]);
    if (g.len10(N[i]) <= STOI_FRAME)
      return fail(ctx, VF_EINVAL, "vf_score_time_varlen: pair %d: %ld samples give %ld at 10 kHz, STOI needs more than %d", i,
                  (long)N[i], (long)g.len10(N[i]), STOI_FRAME);
  }
  rc = stoi_tables(ctx, g);
  if (rc) return rc;
  const int half = ctx->stoi_half[g.slot];
  const double* tables = ctx->d_stoi_tables[g.slot];
  cudaStream_t st = (cudaStream_t)stream;
  // sub-batches of at most SCORE_MAX_IMAGES pairs and SCORE_CAP_FRAMES * hop padded samples: at either rate at most
  // SCORE_CAP_FRAMES * 100 samples at 10 kHz.  Scratch per pair: resampled and compacted signals, energies, band values,
  // tile sums (doubles), then kept-frame indices and a count (ints).
  const std::vector<int> starts = split(batch, SCORE_MAX_IMAGES, SCORE_CAP_FRAMES * g.hop, [&](int i) { return N[i]; });
  rc = acquire_scratch(ctx, ctx->time_score, max_bytes(starts, [&](int i) {
    const int64_t n10 = g.len10(N[i]), nf = stoi_frames(n10);
    return (size_t)(4 * n10 + (1 + 2 * STOI_BANDS) * nf + stoi_tiles(nf)) * 8 + (size_t)(nf + 1) * 4;
  }), st);
  if (rc) return rc;
  cudaError_t e = cudaSuccess;
  for (size_t k = 0; k + 1 < starts.size() && e == cudaSuccess; ++k) {
    const int s = starts[k], nb = starts[k + 1] - starts[k];
    TimeScoreParams p;
    memset(&p, 0, sizeof p);
    p.batch = nb;
    p.est = est + est_offsets[s];
    p.tgt = target + target_offsets[s];
    for (int i = 0; i <= nb; ++i) {
      p.e_off[i] = est_offsets[s + i] - est_offsets[s];
      p.t_off[i] = target_offsets[s + i] - target_offsets[s];
    }
    for (int i = 0; i < nb; ++i) {
      const int64_t n10 = g.len10(N[s + i]), nf = stoi_frames(n10);
      p.r_off[i + 1] = p.r_off[i] + n10;
      p.f_off[i + 1] = p.f_off[i] + nf;
      p.tile_off[i + 1] = p.tile_off[i] + stoi_tiles(nf);
    }
    stoi_bands(p.band_lo, p.band_hi);
    p.clip = 1 + std::pow(10.0, 15.0 / 20);
    p.up = g.stoi_up; p.down = g.stoi_down; p.half = half;
    p.taps = tables;
    p.window = tables + stoi_win_at(half);
    p.tw256 = reinterpret_cast<const double2*>(tables + stoi_tw256_at(half));
    p.tw512 = reinterpret_cast<const double2*>(tables + stoi_tw512_at(half));
    const int64_t Rs = p.r_off[nb], Fs = p.f_off[nb], Ts = p.tile_off[nb];
    double* d = static_cast<double*>(ctx->time_score.p);
    p.rs = d;
    p.cs = p.rs + 2 * Rs;
    p.energy = p.cs + 2 * Rs;
    p.tob = p.energy + Fs;
    p.partial = p.tob + 2 * STOI_BANDS * Fs;
    p.src = reinterpret_cast<int*>(p.partial + Ts);
    p.kept = p.src + Fs;
    p.out = out + (size_t)s * 2;
    e = launch_score_time(p, st);
    ctx->launches += Ts > 0 ? 8 : 7;
  }
  rc = mark_use(ctx, ctx->time_score.order, st);
  if (e != cudaSuccess) return fail(ctx, VF_ECUDA, "time score launch: %s", cudaGetErrorString(e));
  return rc;
}
VF_API int vf_score_time_varlen(vf_ctx* ctx, const float* est, const int64_t* est_offsets, const float* target,
                                const int64_t* target_offsets, int batch, double* out, void* stream) {
  return vf_score_time_varlen_ex(ctx, est, est_offsets, target, target_offsets, batch, out, 44100, stream);
}

// ------------------------------------------------------------------------------------------------------ SR degradations
VF_API int vf_sosfiltfilt_varlen(vf_ctx* ctx, const double* x, const int64_t* offsets, int batch, const double* sos,
                                 const double* zi, const int* n_sections, int n_filters, const int* row_filter, const int* row_f32,
                                 double* out, void* stream) {
  static const char* fn = "vf_sosfiltfilt_varlen";
  int rc = begin_call(ctx, fn, x && sos && zi && n_sections && row_filter && out && batch > 0 && n_filters > 0);
  if (!rc) rc = check_offsets(ctx, fn, "x", "row", offsets, batch, 1);
  if (rc) return rc;
  std::vector<int> edge(n_filters);
  for (int f = 0; f < n_filters; ++f) {
    const int ns = n_sections[f];
    if (ns < 1 || ns > IIR_MAX_SECTIONS) return fail(ctx, VF_EINVAL, "%s: filter %d has %d sections (need 1 .. %d)", fn, f, ns, IIR_MAX_SECTIONS);
    const double* s = sos + (size_t)f * 6 * IIR_MAX_SECTIONS;
    int zb = 0, za = 0;
    for (int k = 0; k < ns; ++k) {
      if (s[6 * k + 3] != 1.0) return fail(ctx, VF_EINVAL, "%s: filter %d: sos[%d, 3] is not 1", fn, f, k);
      zb += s[6 * k + 2] == 0.0;
      za += s[6 * k + 5] == 0.0;
    }
    edge[f] = 3 * (2 * ns + 1 - std::min(zb, za));        // sosfiltfilt's default padlen
  }
  std::vector<int64_t> ne(batch);
  for (int i = 0; i < batch; ++i) {
    const int f = row_filter[i];
    if (f < 0 || f >= n_filters) return fail(ctx, VF_EINVAL, "%s: row %d: filter %d of %d", fn, i, f, n_filters);
    const int64_t n = offsets[i + 1] - offsets[i];
    if (n <= edge[f]) return fail(ctx, VF_EINVAL, "%s: row %d has %ld samples, not more than its padlen %d", fn, i, (long)n, edge[f]);
    ne[i] = n + 2 * (int64_t)edge[f];
  }
  auto chunks = [](int64_t n) { return (n + IIR_CHUNK - 1) / IIR_CHUNK; };
  // sub-batches of at most IIR_MAX_ROWS rows and IIR_CAP_SAMPLES extended samples; the call's filter tables lead the scratch
  const std::vector<int> starts = split(batch, IIR_MAX_ROWS, IIR_CAP_SAMPLES, [&](int i) { return ne[i]; });
  const size_t table_doubles = (size_t)n_filters * IIR_TABLE;
  cudaStream_t st = (cudaStream_t)stream;
  rc = acquire_scratch(ctx, ctx->iir, table_doubles * sizeof(double) + max_bytes(starts, [&](int i) {
    return (size_t)(ne[i] + chunks(ne[i]) * IIR_MAX_STATES) * sizeof(double);   // the row's extended samples and chunk states
  }), st);
  if (rc) return rc;
  double* tables = static_cast<double*>(ctx->iir.p);
  cudaError_t e = cudaSuccess;
  for (int f0 = 0; f0 < n_filters && e == cudaSuccess; f0 += IIR_DESIGN_FILTERS) {   // sos and zi go as kernel parameters
    IirDesignParams d;
    memset(&d, 0, sizeof d);
    d.tables = tables + (size_t)f0 * IIR_TABLE;
    d.n = std::min(IIR_DESIGN_FILTERS, n_filters - f0);
    for (int i = 0; i < d.n; ++i) {
      const int f = f0 + i;
      d.n_sections[i] = n_sections[f];
      std::copy(sos + (size_t)f * 6 * IIR_MAX_SECTIONS, sos + (size_t)f * 6 * IIR_MAX_SECTIONS + 6 * n_sections[f], d.sos[i]);
      std::copy(zi + (size_t)f * 2 * IIR_MAX_SECTIONS, zi + (size_t)f * 2 * IIR_MAX_SECTIONS + 2 * n_sections[f], d.zi[i]);
    }
    e = launch_iir_design(d, st);
    ctx->launches += 1;
  }
  for (size_t k = 0; k + 1 < starts.size() && e == cudaSuccess; ++k) {
    const int s = starts[k], nb = starts[k + 1] - starts[k];
    SosParams p;
    memset(&p, 0, sizeof p);
    p.batch = nb;
    p.x = x + offsets[s];
    p.out = out + offsets[s];
    for (int i = 0; i < nb; ++i) {
      const int f = row_filter[s + i];
      p.off[i + 1] = offsets[s + i + 1] - offsets[s];
      p.ext_off[i + 1] = p.ext_off[i] + ne[s + i];
      p.chunk_off[i + 1] = p.chunk_off[i] + chunks(ne[s + i]);
      p.edge[i] = edge[f];
      p.ext_f32[i] = row_f32 ? row_f32[s + i] != 0 : 0;
      p.n_sections[i] = n_sections[f];
      p.table[i] = tables + (size_t)f * IIR_TABLE;
    }
    p.yf = tables + table_doubles;
    p.state = p.yf + p.ext_off[nb];
    e = launch_sosfiltfilt(p, st);
    ctx->launches += 6;
  }
  rc = mark_use(ctx, ctx->iir.order, st);
  if (e != cudaSuccess) return fail(ctx, VF_ECUDA, "sosfiltfilt launch: %s", cudaGetErrorString(e));
  return rc;
}

VF_API int vf_resample_poly_f64_varlen(vf_ctx* ctx, const double* x, const int64_t* in_offsets, int batch, const double* taps,
                                       const int64_t* tap_offsets, const int* up, const int* down, int n_filters,
                                       const int* row_filter, double* y, const int64_t* out_offsets, void* stream) {
  static const char* fn = "vf_resample_poly_f64_varlen";
  int rc = begin_call(ctx, fn, x && taps && tap_offsets && up && down && row_filter && y && batch > 0 && n_filters > 0);
  if (!rc) rc = check_offsets(ctx, fn, "x", "row", in_offsets, batch, 1);
  if (!rc) rc = check_offsets(ctx, fn, "y", "row", out_offsets, batch, 0);
  if (rc) return rc;
  if (tap_offsets[0] != 0) return fail(ctx, VF_EINVAL, "%s: tap offsets must start at 0", fn);
  for (int f = 0; f < n_filters; ++f) {
    const int64_t nt = tap_offsets[f + 1] - tap_offsets[f];
    if (nt < 1 || nt % 2 == 0 || nt > (int64_t(1) << 30))
      return fail(ctx, VF_EINVAL, "%s: filter %d has %ld taps (need an odd count)", fn, f, (long)nt);
    if (up[f] < 1 || down[f] < 1) return fail(ctx, VF_EINVAL, "%s: filter %d: up %d, down %d (need >= 1)", fn, f, up[f], down[f]);
  }
  for (int i = 0; i < batch; ++i)
    if (row_filter[i] < 0 || row_filter[i] >= n_filters)
      return fail(ctx, VF_EINVAL, "%s: row %d: filter %d of %d", fn, i, row_filter[i], n_filters);
  const std::vector<int> starts = split(batch, IIR_MAX_ROWS);
  cudaError_t e = cudaSuccess;
  for (size_t k = 0; k + 1 < starts.size() && e == cudaSuccess; ++k) {
    const int s = starts[k], nb = starts[k + 1] - starts[k];
    ResampleF64Params p;
    memset(&p, 0, sizeof p);
    p.batch = nb;
    p.x = x + in_offsets[s];
    p.y = y + out_offsets[s];
    p.taps = taps;
    for (int i = 0; i < nb; ++i) {
      const int f = row_filter[s + i];
      p.in_off[i + 1] = in_offsets[s + i + 1] - in_offsets[s];
      p.out_off[i + 1] = out_offsets[s + i + 1] - out_offsets[s];
      p.tap_at[i] = tap_offsets[f];
      p.half[i] = (int)((tap_offsets[f + 1] - tap_offsets[f] - 1) / 2);
      p.up[i] = up[f];
      p.down[i] = down[f];
    }
    e = launch_resample_f64(p, (cudaStream_t)stream);
    ctx->launches += 1;
  }
  if (e != cudaSuccess) return fail(ctx, VF_ECUDA, "resample launch: %s", cudaGetErrorString(e));
  return VF_OK;
}

// ------------------------------------------------------------------------------------------- librosa.load's resampling
VF_API int vf_resample_sinc_varlen(vf_ctx* ctx, const float* x, const int64_t* in_offsets, int batch, const double* tables,
                                   const int64_t* table_offsets, const double* sample_ratio, const int* num_table, int n_filters,
                                   const int* row_filter, float* y, const int64_t* out_offsets, void* stream) {
  static const char* fn = "vf_resample_sinc_varlen";
  int rc = begin_call(ctx, fn, x && tables && table_offsets && sample_ratio && num_table && row_filter && y && batch > 0 &&
                               n_filters > 0);
  if (!rc && reinterpret_cast<uintptr_t>(tables) % alignof(double2) != 0)
    rc = fail(ctx, VF_EINVAL, "%s: tables must be 16-byte aligned (interleaved double2)", fn);
  if (!rc) rc = check_offsets(ctx, fn, "x", "row", in_offsets, batch, 1);
  if (!rc) rc = check_offsets(ctx, fn, "y", "row", out_offsets, batch, 0);
  if (rc) return rc;
  if (table_offsets[0] != 0) return fail(ctx, VF_EINVAL, "%s: table offsets must start at 0", fn);
  for (int f = 0; f < n_filters; ++f) {
    const int64_t nwin = table_offsets[f + 1] - table_offsets[f];
    const double r = sample_ratio[f];
    if (!(r > 0.0) || !std::isfinite(r)) return fail(ctx, VF_EINVAL, "%s: filter %d: sample_ratio %g (need > 0)", fn, f, r);
    if (num_table[f] < 1) return fail(ctx, VF_EINVAL, "%s: filter %d: num_table %d (need >= 1)", fn, f, num_table[f]);
    if ((int64_t)(std::min(r, 1.0) * num_table[f]) < 1)
      return fail(ctx, VF_EINVAL, "%s: filter %d: index step int(%g * %d) is 0", fn, f, std::min(r, 1.0), num_table[f]);
    if (nwin <= num_table[f] || nwin > (int64_t(1) << 30))
      return fail(ctx, VF_EINVAL, "%s: filter %d has %ld entries (need more than num_table %d)", fn, f, (long)nwin, num_table[f]);
  }
  std::vector<int64_t> n_valid(batch);
  for (int i = 0; i < batch; ++i) {
    const int f = row_filter[i];
    if (f < 0 || f >= n_filters) return fail(ctx, VF_EINVAL, "%s: row %d: filter %d of %d", fn, i, f, n_filters);
    const int64_t n = in_offsets[i + 1] - in_offsets[i];
    n_valid[i] = (int64_t)((double)n * sample_ratio[f]);          // resampy's int(n * sample_ratio)
    if (n_valid[i] < 1) return fail(ctx, VF_EINVAL, "%s: row %d has %ld samples, too few to resample by %g", fn, i, (long)n, sample_ratio[f]);
  }
  const std::vector<int> starts = split(batch, SINC_MAX_ROWS);
  cudaError_t e = cudaSuccess;
  for (size_t k = 0; k + 1 < starts.size() && e == cudaSuccess; ++k) {
    const int s = starts[k], nb = starts[k + 1] - starts[k];
    SincParams p;
    memset(&p, 0, sizeof p);
    p.batch = nb;
    p.x = x + in_offsets[s];
    p.y = y + out_offsets[s];
    p.tables = reinterpret_cast<const double2*>(tables);
    for (int i = 0; i < nb; ++i) {
      const int f = row_filter[s + i];
      p.in_off[i + 1] = in_offsets[s + i + 1] - in_offsets[s];
      p.out_off[i + 1] = out_offsets[s + i + 1] - out_offsets[s];
      p.tab_at[i] = table_offsets[f];
      p.nwin[i] = table_offsets[f + 1] - table_offsets[f];
      p.n_valid[i] = n_valid[s + i];
      p.ratio[i] = sample_ratio[f];
      p.num_table[i] = num_table[f];
    }
    e = launch_sinc_resample(p, (cudaStream_t)stream);
    ctx->launches += 1;
  }
  if (e != cudaSuccess) return fail(ctx, VF_ECUDA, "sinc resample launch: %s", cudaGetErrorString(e));
  return VF_OK;
}

// ------------------------------------------------------------------------------------- the pip package's mode-1 pre-filter
VF_API int vf_remove_higher_frequency_varlen(vf_ctx* ctx, const float* x, const int64_t* in_offsets, int batch, double ratio,
                                             float* y, const int64_t* out_offsets, int* cutoff, void* stream) {
  static const char* fn = "vf_remove_higher_frequency_varlen";
  int rc = begin_call(ctx, fn, x && cutoff && batch > 0);
  if (!rc && !(ratio > 0.0 && ratio <= 1.0)) rc = fail(ctx, VF_EINVAL, "%s: ratio %g (need 0 < ratio <= 1)", fn, ratio);
  if (!rc) rc = check_offsets(ctx, fn, "x", "row", in_offsets, batch, 1, ITEM_MAX);
  if (!rc && (!out_offsets || out_offsets[0] != 0)) rc = fail(ctx, VF_EINVAL, "%s: y offsets must start at 0", fn);
  if (rc) return rc;
  std::vector<int64_t> T(batch);
  for (int i = 0; i < batch; ++i) {
    const int64_t n = in_offsets[i + 1] - in_offsets[i], m = out_offsets[i + 1] - out_offsets[i];
    if (m != 512 * (n / 512))
      return fail(ctx, VF_EINVAL, "%s: y row %d has %ld samples (need 512 * (%ld // 512) = %ld)", fn, i, (long)m, (long)n,
                  (long)(512 * (n / 512)));
    T[i] = 1 + n / 512;
  }
  if (!y && out_offsets[batch] > 0) return fail(ctx, VF_EINVAL, "%s: no output for %ld samples", fn, (long)out_offsets[batch]);
  cudaStream_t st = (cudaStream_t)stream;
  // sub-batches of at most PREFILTER_MAX_ROWS rows and PREFILTER_CAP_FRAMES frames; scratch per row: its frames' spectra
  const std::vector<int> starts = split(batch, PREFILTER_MAX_ROWS, PREFILTER_CAP_FRAMES, [&](int i) { return T[i]; });
  rc = acquire_scratch(ctx, ctx->prefilter, max_bytes(starts, [&](int i) { return (size_t)T[i] * 1025 * sizeof(double2); }), st);
  if (rc) return rc;
  cudaError_t e = cudaSuccess;
  for (size_t k = 0; k + 1 < starts.size() && e == cudaSuccess; ++k) {
    const int s = starts[k], nb = starts[k + 1] - starts[k];
    PrefilterParams p;
    memset(&p, 0, sizeof p);
    p.batch = nb;
    p.x = x + in_offsets[s];
    p.y = y ? y + out_offsets[s] : nullptr;
    p.spec = static_cast<double2*>(ctx->prefilter.p);
    p.window = ctx->d_window64; p.tw1024 = ctx->d_tw1024d; p.tw2048 = ctx->d_tw2048d;
    p.cutoff = cutoff + s;
    p.err = ctx->d_err;
    p.ratio = ratio;
    for (int i = 0; i < nb; ++i) {
      p.in_off[i + 1] = in_offsets[s + i + 1] - in_offsets[s];
      p.out_off[i + 1] = out_offsets[s + i + 1] - out_offsets[s];
      p.frame_off[i + 1] = p.frame_off[i] + T[s + i];
    }
    e = launch_prefilter(p, st);
    ctx->launches += p.out_off[nb] > 0 ? 4 : 3;
  }
  rc = mark_use(ctx, ctx->prefilter.order, st);
  if (e != cudaSuccess) return fail(ctx, VF_ECUDA, "prefilter launch: %s", cudaGetErrorString(e));
  return rc;
}

// ------------------------------------------------------------------------------------------------ librosa.load's decode
VF_API int vf_decode_pcm_varlen(vf_ctx* ctx, const void* bytes, int n_rows, const vf_pcm_row* rows, float* mono_out,
                                double* first_out, void* stream) {
  static const char* fn = "vf_decode_pcm_varlen";
  static const int width[] = {1, 2, 3, 4, 4, 8};   // bytes per sample of VF_PCM_U8 .. VF_PCM_F64
  const int rc = begin_call(ctx, fn, bytes && rows && mono_out && n_rows > 0);
  if (rc) return rc;
  const uint8_t* base = static_cast<const uint8_t*>(bytes);
  for (int i = 0; i < n_rows; ++i) {
    const vf_pcm_row& r = rows[i];
    if (r.format < VF_PCM_U8 || r.format > VF_PCM_F64) return fail(ctx, VF_EINVAL, "%s: row %d: format %d", fn, i, r.format);
    if (r.channels < 1 || r.channels > 64)
      return fail(ctx, VF_EINVAL, "%s: row %d: %d channels (need 1 .. 64)", fn, i, r.channels);
    if (r.frames < 0 || r.byte_offset < 0 || r.frames > (INT64_MAX / 512))
      return fail(ctx, VF_EINVAL, "%s: row %d: %ld frames at byte %ld", fn, i, (long)r.frames, (long)r.byte_offset);
    const int align = r.format == VF_PCM_S24 ? 1 : width[r.format];
    if (reinterpret_cast<uintptr_t>(base + r.byte_offset) % align != 0)
      return fail(ctx, VF_EINVAL, "%s: row %d: %d-byte samples at a misaligned address", fn, i, width[r.format]);
  }
  const std::vector<int> starts = split(n_rows, PCM_MAX_ROWS);
  cudaError_t e = cudaSuccess;
  int64_t out_at = 0;                    // the first output frame of the sub-batch
  for (size_t k = 0; k + 1 < starts.size() && e == cudaSuccess; ++k) {
    const int s = starts[k], nb = starts[k + 1] - starts[k];
    PcmParams p;
    memset(&p, 0, sizeof p);
    p.batch = nb;
    p.bytes = base;
    p.mono = mono_out + out_at;
    p.first = first_out ? first_out + out_at : nullptr;
    for (int i = 0; i < nb; ++i) {
      const vf_pcm_row& r = rows[s + i];
      p.out_off[i + 1] = p.out_off[i] + r.frames;
      p.byte_off[i] = r.byte_offset;
      p.channels[i] = r.channels;
      p.format[i] = r.format;
    }
    e = launch_decode_pcm(p, (cudaStream_t)stream);
    ctx->launches += p.out_off[nb] > 0 ? 1 : 0;
    out_at += p.out_off[nb];
  }
  if (e != cudaSuccess) return fail(ctx, VF_ECUDA, "decode launch: %s", cudaGetErrorString(e));
  return VF_OK;
}

// ------------------------------------------------------------------------------------------------- FLAC frames to PCM
constexpr int64_t FLAC_CAP_BYTES = int64_t(64) << 20;   // FLAC bytes per sub-batch; a larger file runs alone

VF_API int vf_decode_flac_varlen(vf_ctx* ctx, const void* bytes, int n_rows, const vf_flac_row* rows, void* pcm,
                                 unsigned long long* status, void* stream) {
  static const char* fn = "vf_decode_flac_varlen";
  int rc = begin_call(ctx, fn, bytes && rows && pcm && status && n_rows > 0);
  if (rc) return rc;
  const uint8_t* base = static_cast<const uint8_t*>(bytes);
  for (int i = 0; i < n_rows; ++i) {
    const vf_flac_row& r = rows[i];
    if (r.byte_offset < 0 || r.byte_offset % 8 || r.nbytes <= 0 || r.nbytes > (int64_t(1) << 40) ||
        reinterpret_cast<uintptr_t>(base + r.byte_offset) % 8)
      return fail(ctx, VF_EINVAL, "%s: row %d: %ld bytes at byte %ld (need > 0 bytes at a multiple of 8)", fn, i, (long)r.nbytes,
                  (long)r.byte_offset);
    if (r.channels < 1 || r.channels > 8) return fail(ctx, VF_EINVAL, "%s: row %d: %d channels (need 1 .. 8)", fn, i, r.channels);
    if (r.bits != 8 && r.bits != 16 && r.bits != 24) return fail(ctx, VF_EINVAL, "%s: row %d: %d bits (need 8, 16 or 24)", fn, i, r.bits);
    if (r.total_samples <= 0 || r.total_samples > (int64_t(1) << 36) || r.pcm_offset < 0 || r.rate <= 0)
      return fail(ctx, VF_EINVAL, "%s: row %d: %ld samples at %d Hz to byte %ld", fn, i, (long)r.total_samples, r.rate,
                  (long)r.pcm_offset);
    if (r.variable != 0 && r.variable != 1) return fail(ctx, VF_EINVAL, "%s: row %d: blocking strategy %d", fn, i, r.variable);
    if (r.first_block < 1 || r.first_block > 65535)
      return fail(ctx, VF_EINVAL, "%s: row %d: first block size %d (need 1 .. 65535)", fn, i, r.first_block);
  }
  cudaStream_t st = (cudaStream_t)stream;
  // scratch of a sub-batch: the per-row candidate counters, ends (int32 per FLAC byte), its working samples (int32), then
  // the candidate tables, each 16-byte aligned.  A sub-batch has (sum of nbytes) / 8 + 2 nb candidate slots, which
  // sum_i (nbytes_i / 8 + 3) bounds.
  auto al = [](size_t n) { return (n + 15) / 16 * 16; };
  auto cap_of = [&](int i) { return rows[i].nbytes / 8 + 3; };
  const std::vector<int> starts = split(n_rows, FLAC_MAX_ROWS, FLAC_CAP_BYTES, [&](int i) { return rows[i].nbytes; });
  rc = acquire_scratch(ctx, ctx->flac, al(4 * FLAC_MAX_ROWS) + max_bytes(starts, [&](int i) {
    return al(4 * rows[i].nbytes) + al(4 * rows[i].total_samples * rows[i].channels) + 13 * cap_of(i) + 48;
  }), st);
  if (rc) return rc;
  cudaError_t e = cudaMemsetAsync(status, 0xFF, sizeof(unsigned long long) * n_rows, st);
  for (size_t k = 0; k + 1 < starts.size() && e == cudaSuccess; ++k) {
    const int s = starts[k], nb = starts[k + 1] - starts[k];
    FlacParams p;
    memset(&p, 0, sizeof p);
    p.batch = nb;
    p.bytes = base;
    p.pcm = static_cast<uint8_t*>(pcm);
    p.status = status + s;
    int64_t smp = 0;
    for (int i = 0; i < nb; ++i) {
      const vf_flac_row& r = rows[s + i];
      p.scan_off[i + 1] = p.scan_off[i] + r.nbytes;
      p.byte_off[i] = r.byte_offset;
      p.total[i] = r.total_samples;
      p.pcm_off[i] = r.pcm_offset;
      p.smp_off[i] = smp;
      smp += r.total_samples * r.channels;
      p.channels[i] = r.channels;
      p.bits[i] = r.bits;
      p.rate[i] = r.rate;
      p.first_block[i] = r.first_block;
      p.variable[i] = (uint8_t)r.variable;
    }
    p.cap = (p.scan_off[nb] >> 3) + 2 * (int64_t)nb;      // row b's slots from (scan_off[b] >> 3) + 2 b (flac.cu)
    char* at = static_cast<char*>(ctx->flac.p);
    p.count = reinterpret_cast<int*>(at);
    at += al(4 * FLAC_MAX_ROWS);
    p.ends = reinterpret_cast<int32_t*>(at);
    at += al(4 * p.scan_off[nb]);
    p.smp = reinterpret_cast<int32_t*>(at);
    at += al(4 * smp);
    p.cand_at = reinterpret_cast<int64_t*>(at);
    at += al(8 * p.cap);
    p.cand_len = reinterpret_cast<int32_t*>(at);
    at += al(4 * p.cap);
    p.chained = reinterpret_cast<uint8_t*>(at);
    e = launch_decode_flac(p, st);
    ctx->launches += 4;
  }
  rc = mark_use(ctx, ctx->flac.order, st);
  if (e != cudaSuccess) return fail(ctx, VF_ECUDA, "FLAC decode launch: %s", cudaGetErrorString(e));
  return rc;
}

// ----------------------------------------------------------------------------------------- live streams' rate conversion
VF_API int vf_resample_rings(vf_ctx* ctx, const float* in_ring, int n_streams, int64_t in_len, const vf_resample_row* rows,
                             int n_rows, float* out, int n_out_streams, int64_t out_len, void* stream) {
  static const char* fn = "vf_resample_rings";
  const int rc = begin_call(ctx, fn, in_ring && rows && out && n_streams > 0 && in_len > 0 && n_rows > 0 && n_out_streams >= 0 &&
                                         out_len >= 0);
  if (rc) return rc;
  std::vector<RingRow> checked(n_rows);
  for (int i = 0; i < n_rows; ++i) {
    const char* why = ring_row(rows[i], n_streams, in_len, n_out_streams, out_len, &checked[i]);
    if (why) return fail(ctx, VF_EINVAL, "%s: row %d: %s", fn, i, why);
  }
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaSuccess;
  for (int family = VF_RESAMPLE_POLY; family <= VF_RESAMPLE_SINC && e == cudaSuccess; ++family) {
    std::vector<int> mine;
    for (int i = 0; i < n_rows; ++i)
      if (rows[i].family == family && rows[i].m1 > rows[i].m0) mine.push_back(i);
    for (size_t s = 0; s < mine.size() && e == cudaSuccess; s += RING_RESAMPLE_ROWS) {
      const int nb = (int)std::min<size_t>(RING_RESAMPLE_ROWS, mine.size() - s);
      auto fill = [&](RingResampleRows& q) {
        q.ring = in_ring; q.out = out; q.in_len = in_len; q.out_len = out_len; q.rows = nb;
        for (int k = 0; k < nb; ++k) {
          const vf_resample_row& w = rows[mine[s + k]];
          const RingRow& c = checked[mine[s + k]];
          q.off[k + 1] = q.off[k] + (w.m1 - w.m0);
          q.src[k] = (int64_t)w.stream * in_len;
          q.a0[k] = c.a0;
          q.a_ph[k] = c.a0 % in_len;
          q.m0[k] = w.m0;
          q.n[k] = w.n;
          q.dst[k] = w.out_stream >= 0 ? (int64_t)w.out_stream * out_len : w.out_offset;
          q.d_ph[k] = w.out_stream >= 0 ? w.m0 % out_len : -1;
        }
      };
      if (family == VF_RESAMPLE_POLY) {
        PolyRingParams p;
        memset(&p, 0, sizeof p);
        fill(p.r);
        for (int k = 0; k < nb; ++k) {
          const vf_resample_row& w = rows[mine[s + k]];
          p.taps[k] = w.taps; p.up[k] = w.up; p.down[k] = w.down;
        }
        e = launch_stream_resample(p, st);
      } else {
        SincRingParams p;
        memset(&p, 0, sizeof p);
        fill(p.r);
        for (int k = 0; k < nb; ++k) {
          const vf_resample_row& w = rows[mine[s + k]];
          p.tab[k] = reinterpret_cast<const double2*>(w.table);
          p.nwin[k] = w.nwin;
          p.n_valid[k] = checked[mine[s + k]].n_valid;
          p.ratio[k] = w.ratio;
          p.num_table[k] = w.num_table;
        }
        e = launch_stream_resample(p, st);
      }
      ctx->launches += 1;
    }
  }
  if (e != cudaSuccess) return fail(ctx, VF_ECUDA, "ring resample launch: %s", cudaGetErrorString(e));
  return VF_OK;
}

// ------------------------------------------------------------------------------------------- finalize and conversions
VF_API int vf_finalize(vf_ctx* ctx, const float* wav, int batch, int64_t len, int64_t n, float* wav_out, void* stream) {
  const int rc = begin_call(ctx, "vf_finalize", wav && wav_out && batch > 0 && len > 0 && n > 0);
  if (rc) return rc;
  const long d = (long)len - (long)n;
  // trim_center (tools/utils.py:57-70) for an estimate at least as long as the reference; d == 1 is the reference's
  // empty-slice case (est[..., 0:-0])
  if (d < 0 || d == 1) return fail(ctx, VF_EINVAL, "vf_finalize: estimate length %ld vs reference %ld is not a trim_center case the path produces", (long)len, (long)n);
  cudaStream_t st = (cudaStream_t)stream;
  unsigned int* peak = nullptr;
  CK(cudaMallocAsync((void**)&peak, (size_t)batch * 4, st));
  CK(cudaMemsetAsync(peak, 0, (size_t)batch * 4, st));
  cudaError_t e1 = launch_peak(wav, batch, (long)len, peak, st);
  FinalizeParams f;
  memset(&f, 0, sizeof f);
  f.wav = wav; f.peak_bits = peak; f.batch = batch; f.L = (long)len; f.n = (long)n; f.skip = d / 2;
  f.out = wav_out; f.out_ld = (long)n; f.out_off = 0;
  cudaError_t e2 = e1 == cudaSuccess ? launch_finalize(f, st) : e1;
  cudaFreeAsync(peak, st);
  if (e2 != cudaSuccess) return fail(ctx, VF_ECUDA, "finalize launch: %s", cudaGetErrorString(e2));
  ctx->launches += 2;
  return VF_OK;
}

VF_API int vf_to_log(vf_ctx* ctx, const float* in, float* out, int64_t n, void* stream) {
  const int rc = begin_call(ctx, "vf_to_log", in && out && n > 0);
  if (rc) return rc;
  CK(launch_to_log(in, out, (size_t)n, ctx->d_err + 1, (cudaStream_t)stream));
  ctx->launches++;
  return VF_OK;
}
VF_API int vf_from_log(vf_ctx* ctx, const float* in, float* out, int64_t n, void* stream) {
  const int rc = begin_call(ctx, "vf_from_log", in && out && n > 0);
  if (rc) return rc;
  CK(launch_from_log(in, out, (size_t)n, (cudaStream_t)stream));
  ctx->launches++;
  return VF_OK;
}

VF_API int vf_to_pcm16_ex(vf_ctx* ctx, const float* in, int16_t* out, int64_t n, int saturate, void* stream) {
  const int rc = begin_call(ctx, "vf_to_pcm16_ex", in && out && n > 0);
  if (rc) return rc;
  CK(launch_pcm16(in, out, (size_t)n, saturate ? 1 : 0, (cudaStream_t)stream));
  ctx->launches++;
  return VF_OK;
}
VF_API int vf_to_pcm16(vf_ctx* ctx, const float* in, int16_t* out, int64_t n, void* stream) {
  return vf_to_pcm16_ex(ctx, in, out, n, 0, stream);
}

}  // extern "C"
