// Parameter blocks and launchers of the non-GEMM kernels on the hot path, and the packed sets' row lookup.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vf {

struct FrontendParams {
  const float* wav;      // [batch, n]
  long n;
  int batch, T;          // T = 1 + n / 441
  const float* window;   // [2048] periodic hann
  const float2* tw1024;  // e^{-2 pi i j / 1024}
  const float2* tw2048;  // e^{-2 pi i k / 2048}, k = 0..1024
  const int* fb_f0;      // [128] first non-zero frequency bin of each mel filter
  const int* fb_len;     // [128]
  const int* fb_ofs;     // [128] offset into fb_val
  const float* fb_val;
  float* sp_out;         // [batch, T, 1025] or null
  float* cos_out;        // with sp_out, or null
  float* sin_out;
  float* mel_out;        // [batch, T, 128] linear mel or null
  float* logmel_out;     // [batch, T, 128] log10(clip(mel, 1e-8)) or null
  const int64_t* vl_off; // varlen: clip b = wav[vl_off[b] .. vl_off[b + 1]) (device), 1 + n_b / 441 frames at row stride T; or null
};
cudaError_t launch_frontend(const FrontendParams& p, cudaStream_t stream);

// Varlen plans (vf_restore_varlen, vf_ssr_restore_varlen): per clip lengths in a plan-owned device table, written on the
// call's stream by varlen_setup_kernel from the call's offsets (a kernel parameter: no host memory is read after the call
// returns), so a captured launch chain with fixed pointers serves any mix of lengths.  Rows of the table, VL_ROWS x batch ints:
enum {
  VL_T = 0,          // frames T = 1 + n / hop
  VL_TP = 1,         // UNet time extent Tp = 64 * ceil(T / 64)
  VL_UNET = 2,       // + l (l = 0..6): UNet rows of level l, (Tp >> l) * ((w0 >> l) + 1); w0 = 127 (mel UNet) or 1024 (unet_v2)
  VL_TV = 9,         // vocoder frames Tv = T + T % 2 + tail_base
  VL_VOC = 10,       // + s: samples of vocoder stage s, Tv * scales[0] * ... * scales[s]
  VL_ROWS = 18
};
constexpr int VL_MAX_CLIPS = 256;  // clips per launch chain: keeps the setup kernel's parameters within 4 KB
struct VarlenSetupParams {
  int64_t off[VL_MAX_CLIPS + 1];   // relative sample offsets of the chain's clips
  int batch, hop, tail_base, w0, n_stages;
  int scales[8];
  int64_t* d_off;                  // [batch + 1]
  int* d_rows;                     // [VL_ROWS][batch]
};
cudaError_t launch_varlen_setup(const VarlenSetupParams& p, cudaStream_t stream);

// The row of a packed set that holds element i (i < off[n]): the c with off[c] <= i < off[c + 1], off[0..n] increasing,
// the convention of the offsets tables below.
__device__ __forceinline__ int packed_row(const int64_t* off, int n, int64_t i) {
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (off[mid] <= i) lo = mid; else hi = mid;
  }
  return lo;
}

// The row copy (stream.cu) of every packed and streaming call: the mel gathers of vf_restore_varlen_mels and
// vf_ssr_restore_varlen_mels, vf_vocoder_varlen's scatter into d_mel and pack of d_voc_wav, and the streaming calls' gathers
// from the device rings and crops of the kept samples.  Row c writes dst[c][j] for j < off[c + 1] - off[c]: src[c][(phase[c]
// + j) mod ring] when lead[c] <= j < n_valid[c], else 0.  ring: the source's wrap length in floats, INT64_MAX for a flat
// source, phase 0.  A ring of R mel frames is a ring of 128 R floats, its phase, lead and n_valid scaled by 128.  Callers
// keep phase < ring and no row longer than ring, so one subtraction wraps.  The table is a kernel parameter, like the
// lengths table's offsets; it holds two rows per clip of a sub-batch, so the gather of both of a sub-batch's mel outputs is
// one launch.
constexpr int ROW_COPY_ROWS = 2 * VL_MAX_CLIPS;
struct RowCopyParams {
  int64_t ring;
  int rows;
  int64_t off[ROW_COPY_ROWS + 1];
  const float* src[ROW_COPY_ROWS];
  float* dst[ROW_COPY_ROWS];
  int64_t phase[ROW_COPY_ROWS], lead[ROW_COPY_ROWS], n_valid[ROW_COPY_ROWS];
};
static_assert(sizeof(RowCopyParams) <= 32764, "the row copy table must fit the kernel parameter space");
cudaError_t launch_row_copy(const RowCopyParams& p, cudaStream_t stream);

// vf_restore_windows' overlap-add of one sub-batch.  Its windows are grouped into runs, one per stream, each run's windows in
// ascending start.  Thread pos[r] + i handles output position t = lo[r] + i of run r: for every window w in first[r] ..
// first[r + 1] - 1 with start[w] <= t < end[w], in that order, acc[acc_row[r] + t mod acc_len] += fl(synth[t - start[w]] *
// restored[src[w] + t - start[w]]) (acc_row: the stream times acc_len; acc_phase: lo mod acc_len; end: min(start + W, the
// stream's valid); src: the window's packed offset).
struct WindowOlaParams {
  const float* restored;
  const float* synth;
  float* acc;
  int64_t acc_len;
  int W, runs;
  int64_t pos[VL_MAX_CLIPS + 1];
  int64_t lo[VL_MAX_CLIPS];
  int64_t acc_row[VL_MAX_CLIPS];
  int64_t acc_phase[VL_MAX_CLIPS];
  int first[VL_MAX_CLIPS + 1];
  int64_t start[VL_MAX_CLIPS];
  int64_t end[VL_MAX_CLIPS];
  int64_t src[VL_MAX_CLIPS];
};
cudaError_t launch_window_ola(const WindowOlaParams& p, cudaStream_t stream);
// vf_restore_windows' emission: packed sample off[e] + j (j < off[e + 1] - off[e]) is acc[row[e] + (phase[e] + j) mod
// acc_len], which is then zeroed (row: the stream times acc_len; phase: the range's start mod acc_len).
struct WindowEmitParams {
  float* acc;
  float* out;
  int64_t acc_len;
  int n;
  int64_t off[VL_MAX_CLIPS + 1];
  int64_t row[VL_MAX_CLIPS];
  int64_t phase[VL_MAX_CLIPS];
};
cudaError_t launch_window_emit(const WindowEmitParams& p, cudaStream_t stream);

struct PlanePtr {
  __half* hi;
  __half* lo;
};

// encoder_block1.conv_block1: BN(1ch) -> LeakyReLU -> Conv3x3 1->32, then bn2 -> LeakyReLU of the same
// block fused in (the only consumer), plus the 1->32 1x1 shortcut of the raw input (modules.py:263-271).
struct UnetFirstParams {
  const float* logmel;   // [batch, T, in_ld]; bins 0..W-1 feed the UNet (unet.py:78: log-mel, W = 127 of 128;
                         // unet_v2.py:108: linear magnitude, W = 1024 of 1025)
  int batch, T, Tp;      // Tp = T padded to a multiple of 64 with zero *input* rows (unet.py:75-77)
  int W, in_ld;          // valid bins per frame / input row stride; the planes use row pitch Wp = W + 1
  float bn1_scale, bn1_shift;
  const float* w1;       // [32][9]
  const float* bn2_scale;  // [32]
  const float* bn2_shift;
  const float* w_sc;     // [32] shortcut weight
  const float* b_sc;     // [32] shortcut bias
  float slope;
  PlanePtr a2;           // [batch, Tp*Wp, 32] act(bn2(conv1(...))), pad column zero
  float* sc_raw;         // [batch, Tp*Wp, 32] fp32 shortcut(x), pad column zero
  const int* vl_T;       // varlen: per clip T and Tp (rows t >= Tp_b are written as zeros), or null: T, Tp for every clip
  const int* vl_Tp;
  int* err;
};
cudaError_t launch_unet_first(const UnetFirstParams& p, cudaStream_t stream);

// avg_pool2d(2,2) (modules.py:183) + the consumer's BN/LeakyReLU + hi/lo split.
struct PoolParams {
  const float* in;       // [batch, H*Wp, C] fp32
  int batch, H, Wp, C;
  int Wpo;               // output row pitch = (Wp - 1) / 2 + 1 (floor pooling of the W = Wp - 1 valid columns + pad column)
  PlanePtr out_r;        // [batch, (H/2)*Wpo, C] pooled raw
  PlanePtr out_a;        // act(scale*pooled+shift)
  float* out_raw;        // fp32 pooled or null
  const float* a_scale;
  const float* a_shift;
  float slope;
  const int* row_valid;  // varlen: per clip valid output rows (of H/2 * Wpo), the rest written as zeros; or null
  int* err;
};
cudaError_t launch_pool(const PoolParams& p, cudaStream_t stream);

// gru_tc.cu: one bidirectional GRU layer of the bi_gru analysis module (hidden size GRU_HIDDEN), one launch for the whole
// sequence: clusters of GRU_CTAS CTAs, one per (direction, group of GRU_CLIPS clips); grid GRU_CTAS * gru_groups(batch) x 2.
constexpr int GRU_HIDDEN = 256, GRU_CTAS = 8, GRU_CLIPS = 4;
struct GruParams {
  const float* G;            // [batch, T, 6 * GRU_HIDDEN] x W_ih^T + b_ih + (b_hr, b_hz, 0): forward gates (r, z, n) in columns
                             // [0, 768), reverse in [768, 1536)
  const float* w_hh[2];      // per direction [3 * GRU_HIDDEN][GRU_HIDDEN] fp32
  const float* b_hn[2];      // per direction [GRU_HIDDEN]: applied inside r * (W_hn h + b_hn)
  PlanePtr out;              // [batch, T, 2 * GRU_HIDDEN] hi/lo planes: forward h at channels [0, 256), reverse at [256, 512)
  int batch, T;
  int relu;                  // 1: the planes hold relu(h) (the module's ReLU after the last layer); the recurrence keeps h
  const int* vl_T;           // varlen: clip b has vl_T[b] frames (the reverse direction starts at its own last frame, rows past
                             // it are written as zeros); or null: T for every clip
  int* err;                  // fp16 range flag: raised when an h of a clip's frames is not finite
};
int gru_groups(int batch);
cudaError_t launch_gru(const GruParams& p, cudaStream_t stream);
// hi/lo planes of scale * in + shift over [batch, T, C] fp32 (the first GEMM operand of bi_gru / dnn: BatchNorm2d(1) of
// the log-mel, or the log-mel itself); rows t >= vl_T[b] are zeros when vl_T is given
struct AffinePlanesParams {
  const float* in;
  int batch, T, C;
  float scale, shift;
  PlanePtr out;
  const int* vl_T;
  int* err;              // fp16 range flag: raised when a written value is NaN or above 65504 in magnitude
};
cudaError_t launch_affine_planes(const AffinePlanesParams& p, cudaStream_t stream);

// to_log / from_log (tools/pytorch/pytorch_util.py:157-163) for the stage-level API.
cudaError_t launch_to_log(const float* in, float* out, size_t n, int* neg_count, cudaStream_t stream);
cudaError_t launch_from_log(const float* in, float* out, size_t n, cudaStream_t stream);

// Vocoder prologue: mel / w -> dB -> normalise -> [T + tail, 128] planes with the constant tail.
struct VocCondParams {
  const float* mel;      // [batch, T, 128]; linear mel, or log10 mel when is_log (from_log fused)
  int is_log;
  int batch, T, Tv;
  const float* weight;       // [128] per-bin mel weight (divided out)
  float amp_floor, ref_db, min_db, tail_value;
  const float* band_sums;    // [batch][2] (target, estimate) low-band sums from launch_band_energy, or null:
                             // amp_to_original_f (tools/utils.py:50-55) scales the estimate by target/estimate
  PlanePtr out;          // [batch, Tv, 128]
  const int* vl_T;       // varlen: per clip T and Tv (rows tv >= Tv_b are written as zeros), or null
  const int* vl_Tv;
};
cudaError_t launch_voc_condition(const VocCondParams& p, cudaStream_t stream);

// amp_to_original_f, reduction half: per clip, sums over frames and mel bins [5, int(128*0.2)) of the noisy
// linear mel (target) and of from_log(restored log-mel) (estimate).  sums must be zeroed before the launch.
// vl_T (varlen, or null): clip b sums its first vl_T[b] frames of the [batch, T, 128] buffers, in the order of a T = vl_T[b] launch.
cudaError_t launch_band_energy(const float* mel_target_lin, const float* logmel_est, int batch, int T, float* sums,
                               cudaStream_t stream, const int* vl_T = nullptr);

// amp_to_original_f as a stand-alone op: out = est * (low-band mean of target / low-band mean of est), linear mels [batch, T, 128].
cudaError_t launch_amp_to_original(const float* est, const float* tgt, int batch, int T, float* out, cudaStream_t stream);

// nn.ReflectionPad1d(3): rows [3, L+3) of each image are already written; fill 3 + 3 mirrored rows.
// vl_L (varlen, or null): clip b is vl_L[b] rows long and mirrors at its own end (images keep their L + 6 row stride).
cudaError_t launch_reflect_fill(PlanePtr planes, int batch, int L, int C, int pad, cudaStream_t stream, const int* vl_L = nullptr);

// Tail: ReflectionPad(3) (pre-filled) + Conv1d(C -> 1, k7) + tanh, plus the per-clip peak |out|.
struct VocTailParams {
  PlanePtr in;           // [batch, L + 6, C]
  int batch, L, C, terms;
  int tanh_out;          // 1: tanh on the output (the generator's last op); 0: linear (test configurations that exceed |1|)
  const float* w;        // [7][C]
  float bias;
  float* wav;            // [batch, L]
  unsigned int* peak_bits;   // [batch] max |out| as float bits (non-negative floats order like uints)
  const int* vl_L;       // varlen: clip b writes (and peaks over) its first vl_L[b] samples; or null
};
cudaError_t launch_voc_tail(const VocTailParams& p, cudaStream_t stream);
// dynamic shared memory of one tail CTA: the [7][C] weights and the fp16 input tile (both planes when terms == 3)
size_t voc_tail_smem_bytes(int C, int terms);

// eval_gsr_voicefixer.py:68-72: out /= max|out| if it exceeds 1; trim_center (tools/utils.py:57-70).
struct FinalizeParams {
  const float* wav;      // [batch, L]
  const unsigned int* peak_bits;
  int batch;
  long L, n, skip;       // out[b, i] = wav[b, skip + i], i < n
  float* out;            // [batch, out_ld]
  long out_ld, out_off;
  // varlen (or null): clip b has n_b = vl_off[b + 1] - vl_off[b] samples and a vl_L[b]-sample vocoder output; it is
  // trimmed by skip_b = (vl_L[b] - n_b) / 2 and written to out[vl_off[b] ..]  (n then bounds every n_b)
  const int64_t* vl_off;
  const int* vl_L;
};
cudaError_t launch_finalize(const FinalizeParams& p, cudaStream_t stream);
cudaError_t launch_pcm16(const float* in, int16_t* out, size_t n, int saturate, cudaStream_t stream);

// max |wav| per clip as float bits (atomicMax), for the stand-alone peak normalise + trim entry point.
cudaError_t launch_peak(const float* wav, int batch, long L, unsigned int* peak_bits, cudaStream_t stream);
// vf_ssr_restore_varlen_mels: in place, clip b = wav[vl_off[b] .. vl_off[b + 1]) (device offsets, clips of at most n_max
// samples) is divided by its max |x| when that exceeds 1 (eval_gsr_unet.py:66-67).  Two kernels: the per-clip max as float
// bits into peak_bits[batch], which must be zeroed before the launch, then the scale.
cudaError_t launch_peak_normalise_varlen(float* wav, const int64_t* vl_off, int batch, long n_max, unsigned int* peak_bits,
                                         cudaStream_t stream);

// MelScale.forward (tools/pytorch/mel_scale.py:52-64) as a stand-alone op on any [..., freq, time] view:
// out[o, t, m] = sum_f in[o * so + f * sf + t * st] * fb[f, m] with the filterbank in its sparse form.  Two geometries:
// n_freq x n_mels = 1025 x 128 (44.1 kHz, the model's) and 372 x 80 (AudioMetrics' mel_16k); any other is
// cudaErrorInvalidValue.
struct MelParams {
  const float* in;
  long n_outer, T;
  long so, sf, st;       // input strides (elements) of the outer, frequency and time axes
  float* out;            // [n_outer, T, n_mels] contiguous
  const int* fb_f0;
  const int* fb_len;
  const int* fb_ofs;
  const float* fb_val;
};
cudaError_t launch_mel(const MelParams& p, cudaStream_t stream, int n_freq = 1025, int n_mels = 128);

// ISTFT (FDomainHelper.istft, fDomainHelper.py:30-32,127 -> torchlibrosa ISTFT: n_fft = win = 2048, hop 441, periodic
// hann, center): stage 1 writes the windowed inverse-DFT frames, stage 2 overlap-adds them in a fixed order and divides
// by the overlap-added squared window (clamped at 1e-11).  Stage 1 takes the spectrum either as (real, imag), or -
// unet_v2.py:96,136-139 fused - as a magnitude plus the waveform whose STFT phase it is to carry:
// real = mag * cos, imag = mag * sin with cos, sin = re/|X|, im/|X| of the input (fDomainHelper.py:62-64).
struct IstftFramesParams {
  const float* real;     // [batch, T, 1025] or null
  const float* imag;
  const float* mag;      // [batch, T, 1025] (with wav) or null
  const float* wav;      // [batch, n]
  long n;
  int batch, T;
  const float* window;   // [2048]
  const float2* tw1024;
  const float2* tw2048;
  float* frames;         // [batch, T, 2048]
  // varlen (with mag, or null): clip b = wav[vl_off[b] .. vl_off[b + 1]) (device), reflect padded at its own ends; only its
  // first vl_T[b] frames are computed (mag and frames keep the row stride T, the rows past vl_T[b] are not touched)
  const int64_t* vl_off;
  const int* vl_T;
  int* err;              // with mag: raised (ERR_NAN_PHASE) when a frame's phase is NaN - a NaN or infinite input sample
};
cudaError_t launch_istft_frames(const IstftFramesParams& p, cudaStream_t stream);
struct IstftOlaParams {
  const float* frames;   // [batch, T, 2048]
  int batch, T;
  long length;           // output samples per clip: y[n_fft/2 : n_fft/2 + length]
  const float* window;
  float* out;            // [batch, out_ld]
  long out_ld;
  // varlen (or null): clip b produces n_b = vl_off[b + 1] - vl_off[b] samples from its first vl_T[b] frames, in the
  // order of a one-clip launch, written to out[vl_off[b] ..]  (length then bounds every n_b)
  const int64_t* vl_off;
  const int* vl_T;
};
cudaError_t launch_istft_ola(const IstftOlaParams& p, cudaStream_t stream);

// edges.cu: polyphase resampling (load_wav) and the handler's mel metrics
cudaError_t launch_resample_poly(const float* x, int batch, long n, int up, int down, const float* h, int half, float* out, long n_out,
                                 cudaStream_t stream);
cudaError_t launch_lsd(const float* est, const float* tgt, int images, int T, int F, float* out, cudaStream_t stream);
cudaError_t launch_sispec(const float* est, const float* tgt, int batch, long n, int est_map, int tgt_map, float* out, cudaStream_t stream);

// Scoring (AudioMetrics.evaluation, evaluation_proc/metrics.py:53-81) over sets of images of different frame counts.  The
// images' extents are kernel parameters, so one launch serves a set of up to SCORE_MAX_IMAGES images.
constexpr int SCORE_MAX_IMAGES = 128;
struct ImageSet {
  int batch;
  int64_t frame_off[SCORE_MAX_IMAGES + 1];   // image b = rows [frame_off[b], frame_off[b + 1]) of a packed [rows, F] buffer
};
// edges.cu: lsd -> out[b * out_stride]; sispec non-log -> out[b * out_stride], to_log of both -> out[b * out_stride + 1]
cudaError_t launch_lsd_varlen(const float* est, const float* tgt, int F, const ImageSet& s, double* out, int out_stride, cudaStream_t stream);
cudaError_t launch_sispec_varlen(const float* est, const float* tgt, int F, const ImageSet& s, double* out, int out_stride, cudaStream_t stream);

// metrics.cu: |librosa.stft(wav, n_fft, hop_length)| (librosa 0.8: reflect padding by n_fft / 2, periodic hann, float64
// DFT stored as complex64) of up to two packed sources at once (blockIdx.y = source), one CTA per frame.  Two geometries:
// launch_metric_stft is n_fft 2048, hop 441 (44.1 kHz: radix FFT), launch_metric_dft743 is n_fft 743, hop 160 (16 kHz:
// 743 is prime, a direct DFT).
struct MetricStftParams {
  const float* wav[2];                       // packed samples; clip b of source z = wav[z][off[z][b] .. off[z][b + 1])
  float* sp[2];                              // [sum T_b, 1 + n_fft / 2]: clip b's frames at rows frame_off[b] ..
  const double* window;                      // [n_fft] periodic hann, float64
  const double2* tw1024;                     // e^{-2 pi i j / 1024}, float64
  const double2* tw2048;                     // e^{-2 pi i k / 2048}, k = 0..1024
  const double2* tw743;                      // e^{-2 pi i j / 743}, j = 0..742 (metric_dft743_kernel)
  int batch, sources;
  int64_t off[2][SCORE_MAX_IMAGES + 1];
  // T_b = 1 + (n_b - n_fft % 2) / hop: 1 + n_b / 441, or 1 + (n_b - 1) / 160 (the sources have equal frame counts)
  int64_t frame_off[SCORE_MAX_IMAGES + 1];
};
cudaError_t launch_metric_stft(const MetricStftParams& p, cudaStream_t stream);
cudaError_t launch_metric_dft743(const MetricStftParams& p, cudaStream_t stream);

// skimage.metrics.structural_similarity(x, y, win_size=7) of scikit-image <= 0.18 on float32 images (data_range 2, 7x7
// uniform filter, sample covariance, mean over the image cropped by 3), in float64.  Stage 1: one CTA per tile of
// SSIM_TILE_R x SSIM_TILE_C output pixels writes the tile's sum to partial[]; stage 2: one CTA per image sums its tiles in
// order and writes the mean to out[b * out_stride].
constexpr int SSIM_TILE_R = 8, SSIM_TILE_C = 64;
struct SsimParams {
  const float* x;                            // packed [rows, F] images (frame_off as in ImageSet)
  const float* y;
  int F, batch;
  double* partial;                           // [tile_off[batch]]
  int64_t frame_off[SCORE_MAX_IMAGES + 1];
  int tile_off[SCORE_MAX_IMAGES + 1];        // first tile of image b (ssim_tiles)
};
// Tiles of one T x F image (T, F >= 7)
inline int ssim_tiles(long T, int F) {
  return (int)((T - 6 + SSIM_TILE_R - 1) / SSIM_TILE_R) * ((F - 6 + SSIM_TILE_C - 1) / SSIM_TILE_C);
}
cudaError_t launch_ssim(const SsimParams& p, double* out, int out_stride, cudaStream_t stream);

// speech_metrics.cu: the time-domain keys of AudioMetrics.evaluation (metrics.py:58-64), speechmetrics' sisdr and stoi
// (pystoi 0.3.3, extended=False) for pairs of packed 44.1 kHz or 16 kHz clips, all in float64.  A pair is zero-padded at
// the end to its longer clip (N_b samples) by index math.  STOI's pipeline runs at 10 kHz: resample (up / down = 100 / 441
// with Octave's 31947-tap window, or 5 / 8 with its 581-tap window), the target's frame energies, the silent-frame mask and
// its kept-frame scan, the overlap-add of the kept frames into a compacted buffer, a 512-point STFT with the 15
// one-third-octave band values per frame, and the 30-frame segment correlations, summed per tile and then per pair in a
// fixed order.  The silence removal makes the frame count of a pair a device value (kept[b] - 1 STFT frames); the buffers
// and grids are sized by its host-known upper bound, and slots past it are skipped.  Every value depends on its own pair
// only, so a pair's bits do not depend on its batch.
constexpr int STOI_FRAME = 256, STOI_HOP = 128, STOI_BANDS = 15, STOI_SEG = 30;
// 10 kHz samples of a pair of padded length n resampled by up / down, and its frames before silence removal (starts
// range(0, n10 - 256, 128))
inline int64_t stoi_len10(int64_t n, int up, int down) { return (n * up + down - 1) / down; }
inline int64_t stoi_frames(int64_t n10) { return n10 > STOI_FRAME ? (n10 - STOI_FRAME + STOI_HOP - 1) / STOI_HOP : 0; }
// correlation tiles of 256 (segment, band) items for at most nF - 1 STFT frames (nF - 30 segments)
inline int64_t stoi_tiles(int64_t nF) { return nF > STOI_SEG ? ((nF - STOI_SEG) * STOI_BANDS + 255) / 256 : 0; }
struct TimeScoreParams {
  const float* est;                          // packed samples: pair b = est[e_off[b] .. e_off[b + 1]), target likewise
  const float* tgt;
  int batch;
  int64_t e_off[SCORE_MAX_IMAGES + 1], t_off[SCORE_MAX_IMAGES + 1];
  int64_t r_off[SCORE_MAX_IMAGES + 1];       // 10 kHz samples: stoi_len10(N_b, up, down)
  int64_t f_off[SCORE_MAX_IMAGES + 1];       // frame slots: stoi_frames
  int64_t tile_off[SCORE_MAX_IMAGES + 1];    // correlation tiles: stoi_tiles
  int band_lo[STOI_BANDS], band_hi[STOI_BANDS];   // band k = rfft bins [band_lo[k], band_hi[k])
  double clip;                               // 1 + 10^(15 / 20)
  int up, down, half;                        // the resampling ratio to 10 kHz and its filter's half length
  const double* taps;                        // [2 * half + 1] Octave's window / its sum * up
  const double* window;                      // [256] np.hanning(258)[1:-1]
  const double2* tw256;                      // e^{-2 pi i j / 256}
  const double2* tw512;                      // e^{-2 pi i k / 512}, k = 0..256
  double* rs;                                // [2][r_off[batch]] resampled target (0) and estimate (1)
  double* cs;                                // [2][r_off[batch]] their compacted signals ((kept + 1) * 128 <= n10 samples)
  double* energy;                            // [f_off[batch]] the target's frame energies, dB
  double* tob;                               // [2][f_off[batch]][15] band values of the STFT frames
  double* partial;                           // [tile_off[batch]] correlation tile sums
  int* src;                                  // [f_off[batch]] kept frame k of pair b -> its frame index
  int* kept;                                 // [batch] kept frames
  double* out;                               // [batch][2]: sisdr, stoi
};
cudaError_t launch_score_time(const TimeScoreParams& p, cudaStream_t stream);   // eight launches

// iir.cu: scipy.signal.sosfiltfilt(sos, x) (padtype "odd") of packed float64 rows, each with its own filter, as an exact
// chunked scan.  Row b's odd extension (edge[b] samples each side, index math) is cut into IIR_CHUNK-sample chunks.  Phase
// A runs every chunk but the last from zero state and stores its end state; phase B carries the true chunk-start states
// along the row, s_{k+1} = M s_k + e_k with M = the cascade's IIR_CHUNK-step zero-input transition (iir_design_kernel);
// phase C runs every chunk again from its true start state, in scipy's per-sample order (sections inner), and writes it.
// The forward pass writes yf; the backward pass reads yf reversed and writes the cropped output.  Its only error is fp64
// rounding: no warm-up truncation.
constexpr int IIR_MAX_SECTIONS = 10, IIR_MAX_STATES = 2 * IIR_MAX_SECTIONS;
constexpr int IIR_CHUNK = 1024;
constexpr int IIR_MAX_ROWS = 64;                       // rows per sub-batch
constexpr int64_t IIR_CAP_SAMPLES = int64_t(1) << 24;   // extended samples per sub-batch (a longer row runs alone)
// per-filter device table (doubles): sos [10][6] (rows past n_sections unused), zi [20], M [20][20] (zero past 2 n_sections)
constexpr int IIR_ZI_AT = 6 * IIR_MAX_SECTIONS, IIR_M_AT = IIR_ZI_AT + IIR_MAX_STATES,
              IIR_TABLE = IIR_M_AT + IIR_MAX_STATES * IIR_MAX_STATES;
struct SosParams {
  const double* x;                           // packed input rows: row b = x[off[b] .. off[b + 1])
  double* out;                               // packed output, same offsets
  int batch;
  int64_t off[IIR_MAX_ROWS + 1];
  int64_t ext_off[IIR_MAX_ROWS + 1];         // row b's extended samples (n + 2 edge) in yf
  int64_t chunk_off[IIR_MAX_ROWS + 1];       // row b's chunks (ceil((n + 2 edge) / IIR_CHUNK)) in state
  int edge[IIR_MAX_ROWS];
  int ext_f32[IIR_MAX_ROWS];                 // row b was float32: its odd extension is rounded to float32, as numpy makes it
  int n_sections[IIR_MAX_ROWS];
  const double* table[IIR_MAX_ROWS];         // row b's filter table (IIR_TABLE doubles)
  double* yf;                                // [ext_off[batch]] forward pass
  double* state;                             // [chunk_off[batch]][20] chunk end (phase A) / start (phase B) states
};
cudaError_t launch_sosfiltfilt(const SosParams& p, cudaStream_t stream);   // six launches
// The per-call tables of up to IIR_DESIGN_FILTERS filters (one launch; sos and zi travel in the parameters)
constexpr int IIR_DESIGN_FILTERS = 6;
struct IirDesignParams {
  double* tables;                            // [n][IIR_TABLE]
  int n;
  int n_sections[IIR_DESIGN_FILTERS];
  double sos[IIR_DESIGN_FILTERS][6 * IIR_MAX_SECTIONS];
  double zi[IIR_DESIGN_FILTERS][2 * IIR_MAX_SECTIONS];
};
cudaError_t launch_iir_design(const IirDesignParams& p, cudaStream_t stream);

// iir.cu: scipy.signal.resample_poly(x, up, down) of packed float64 rows with float64 taps (firwin x up, odd length 2 half
// + 1, designed by the caller), one thread per output sample: y[m] = sum_j x[j] h[m down + half - up j].  Row b writes
// out_off[b + 1] - out_off[b] samples: resample_poly's first ceil(n up / down), then zeros (align_length's pad).
struct ResampleF64Params {
  const double* x;
  double* y;
  const double* taps;
  int batch;
  int64_t in_off[IIR_MAX_ROWS + 1], out_off[IIR_MAX_ROWS + 1];
  int64_t tap_at[IIR_MAX_ROWS];              // row b's taps start in `taps`
  int half[IIR_MAX_ROWS], up[IIR_MAX_ROWS], down[IIR_MAX_ROWS];
};
cudaError_t launch_resample_f64(const ResampleF64Params& p, cudaStream_t stream);

// sinc.cu: resampy's resample (librosa 0.8 resample, res_type kaiser_best / kaiser_fast) of packed float32 rows, one thread
// per output sample.  Row b reads table tables[tab_at[b] ..][nwin[b]] of (win, delta) pairs, already scaled for its
// sample_ratio ratio[b]; it writes out_off[b + 1] - out_off[b] samples, resampy's first n_valid[b] = int(n ratio) and
// zeros past them (librosa's fix_length).  Everything travels in the parameters: no scratch, one launch per
// SINC_MAX_ROWS rows.
constexpr int SINC_MAX_ROWS = 512;                        // keeps SincParams under the 32 KiB kernel-parameter limit
struct SincParams {
  const float* x;
  float* y;
  const double2* tables;
  int batch;
  int64_t in_off[SINC_MAX_ROWS + 1], out_off[SINC_MAX_ROWS + 1];
  int64_t tab_at[SINC_MAX_ROWS], nwin[SINC_MAX_ROWS], n_valid[SINC_MAX_ROWS];
  double ratio[SINC_MAX_ROWS];
  int num_table[SINC_MAX_ROWS];
};
cudaError_t launch_sinc_resample(const SincParams& p, cudaStream_t stream);

// vf_resample_rings (stream.cu): the rows of one family of one launch, kernel parameters like the chunk gather's.  Thread
// off[r] + j (j < off[r + 1] - off[r]) computes output m = m0[r] + j of row r from the input ring row at ring + src[r]
// (absolute input i at (a_ph[r] + i - a0[r]) mod in_len, a0: the first input the row may read) for a signal of n[r] inputs
// (INT64_MAX while open), and writes it to out[dst[r] + (d_ph[r] + j) mod out_len] (a ring row: dst = its stream times
// out_len, d_ph = m0 mod out_len) or, with d_ph[r] < 0, to out[dst[r] + j] (packed).  Poly rows read their own taps, sinc
// rows their own (win, delta) table, with slots at or past n_valid[r] = int(n ratio) written as zeros.
constexpr int RING_RESAMPLE_ROWS = 256;                   // keeps either struct under the 32 KiB kernel-parameter limit
struct RingResampleRows {
  const float* ring;
  float* out;
  int64_t in_len, out_len;
  int rows;
  int64_t off[RING_RESAMPLE_ROWS + 1];
  int64_t src[RING_RESAMPLE_ROWS], a0[RING_RESAMPLE_ROWS], a_ph[RING_RESAMPLE_ROWS];
  int64_t m0[RING_RESAMPLE_ROWS], n[RING_RESAMPLE_ROWS];
  int64_t dst[RING_RESAMPLE_ROWS], d_ph[RING_RESAMPLE_ROWS];
};
struct PolyRingParams {
  RingResampleRows r;
  const float* taps[RING_RESAMPLE_ROWS];
  int up[RING_RESAMPLE_ROWS], down[RING_RESAMPLE_ROWS];
};
struct SincRingParams {
  RingResampleRows r;
  const double2* tab[RING_RESAMPLE_ROWS];
  int64_t nwin[RING_RESAMPLE_ROWS], n_valid[RING_RESAMPLE_ROWS];
  double ratio[RING_RESAMPLE_ROWS];
  int num_table[RING_RESAMPLE_ROWS];
};
cudaError_t launch_stream_resample(const PolyRingParams& p, cudaStream_t stream);
cudaError_t launch_stream_resample(const SincRingParams& p, cudaStream_t stream);

// prefilter.cu: the pip package's remove_higher_frequency (vf_remove_higher_frequency_varlen) of one sub-batch of packed
// float32 rows, four launches: STFT, per-row cutoff, masked inverse frames, overlap-add.  Row b has T_b = 1 + n_b / 512
// frames at frame_off[b] of the scratch `spec`, 1025 double2 per frame (the spectrum, then the frame's 2048 doubles).
constexpr int PREFILTER_MAX_ROWS = 256;                   // rows per sub-batch
constexpr int64_t PREFILTER_CAP_FRAMES = 16384;           // frames per sub-batch (16.4 KB of scratch each); a longer row runs alone
struct PrefilterParams {
  const float* x;                            // row b = x[in_off[b] .. in_off[b + 1])
  float* y;                                  // row b = y[out_off[b] .. out_off[b + 1]), 512 (n_b / 512) samples
  double2* spec;                             // [frame_off[batch]][1025]
  const double* window;                      // [2048] periodic hann, float64
  const double2* tw1024;                     // e^{-2 pi i j / 1024}
  const double2* tw2048;                     // e^{-2 pi i k / 2048}, k = 0..1024
  int* cutoff;                               // [batch] first removed bin (1025: none)
  int* err;                                  // raised (ERR_NONFINITE_INPUT) by a NaN or infinite sample
  double ratio;
  int batch;
  int64_t in_off[PREFILTER_MAX_ROWS + 1], out_off[PREFILTER_MAX_ROWS + 1], frame_off[PREFILTER_MAX_ROWS + 1];
};
cudaError_t launch_prefilter(const PrefilterParams& p, cudaStream_t stream);

// pcm.cu: vf_decode_pcm_varlen of one sub-batch of WAV data chunks, one thread per output frame.  Row b's frames start at
// bytes + byte_off[b], channels[b] interleaved samples of format[b] (VF_PCM_*) each; its outputs are frames
// out_off[b] .. out_off[b + 1] - 1 of mono (and of first, when not null).
constexpr int PCM_MAX_ROWS = 1024;                        // keeps PcmParams under the 32 KiB kernel-parameter limit
struct PcmParams {
  const uint8_t* bytes;
  float* mono;
  double* first;
  int batch;
  int64_t out_off[PCM_MAX_ROWS + 1];
  int64_t byte_off[PCM_MAX_ROWS];
  int channels[PCM_MAX_ROWS], format[PCM_MAX_ROWS];
};
static_assert(sizeof(PcmParams) <= 32764, "the decode table must fit the kernel parameter space");
cudaError_t launch_decode_pcm(const PcmParams& p, cudaStream_t stream);

// flac.cu: vf_decode_flac_varlen of one sub-batch of FLAC audio regions.  Row b's region is bytes + byte_off[b] (8-byte
// aligned), scan_off[b + 1] - scan_off[b] bytes long; byte j of it is scan element scan_off[b] + j.  Its PCM output starts
// at pcm + pcm_off[b]; its int32 working samples at smp + smp_off[b] (total[b] * channels[b] of them).  Scratch, per scan
// element: ends; per candidate slot (cap of them, row b's from (scan_off[b] >> 3) + 2b): cand_at (scan element of its sync
// code), cand_len (its length in bytes, or -FLAC_E*), chained (1 when the row's chain takes it); count[b]: row b's number of
// candidates.  status[b]: (byte << 8) | code of the row's first error (atomicMin), all ones when there is none.
constexpr int FLAC_MAX_ROWS = 512;                        // keeps FlacParams under the 32 KiB kernel-parameter limit
struct FlacParams {
  const uint8_t* bytes;
  uint8_t* pcm;
  unsigned long long* status;
  int32_t* ends;
  int32_t* smp;
  int64_t* cand_at;
  int32_t* cand_len;
  uint8_t* chained;
  int* count;
  int64_t cap;
  int batch;
  int64_t scan_off[FLAC_MAX_ROWS + 1];
  int64_t byte_off[FLAC_MAX_ROWS], total[FLAC_MAX_ROWS], pcm_off[FLAC_MAX_ROWS], smp_off[FLAC_MAX_ROWS];
  int32_t channels[FLAC_MAX_ROWS], bits[FLAC_MAX_ROWS], rate[FLAC_MAX_ROWS], first_block[FLAC_MAX_ROWS];
  uint8_t variable[FLAC_MAX_ROWS];
};
static_assert(sizeof(FlacParams) <= 32764, "the FLAC table must fit the kernel parameter space");
cudaError_t launch_decode_flac(const FlacParams& p, cudaStream_t stream);

}  // namespace vf
