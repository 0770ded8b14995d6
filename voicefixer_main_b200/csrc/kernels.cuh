// Parameter blocks and launchers of the non-GEMM kernels on the hot path.
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
// vf_restore_varlen_mels: rows t < T_b of clip b in a varlen plan's [batch, T, 128] mel buffers (row stride T = the bucket)
// -> rows [frame_off[b], frame_off[b + 1]) of packed caller buffers (either output may be null).  The frame offsets are a
// kernel parameter, as the lengths table's sample offsets are.
struct MelGatherParams {
  const float* mel;
  const float* logmel;
  float* mel_out;
  float* logmel_out;
  int batch, T;
  int64_t frame_off[VL_MAX_CLIPS + 1];
};
cudaError_t launch_gather_mels(const MelGatherParams& p, cudaStream_t stream);

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
// out[o, t, m] = sum_f in[o * so + f * sf + t * st] * fb[f, m] with the filterbank in its sparse form.
struct MelParams {
  const float* in;
  long n_outer, T;
  long so, sf, st;       // input strides (elements) of the outer, frequency and time axes
  float* out;            // [n_outer, T, 128] contiguous
  const int* fb_f0;
  const int* fb_len;
  const int* fb_ofs;
  const float* fb_val;
};
cudaError_t launch_mel(const MelParams& p, cudaStream_t stream);

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

// metrics.cu: |librosa.stft(wav, n_fft=2048, hop_length=441)| (librosa 0.8: reflect padding, periodic hann, float64 FFT
// stored as complex64) of up to two packed sources at once (blockIdx.y = source), one CTA per frame.
struct MetricStftParams {
  const float* wav[2];                       // packed samples; clip b of source z = wav[z][off[z][b] .. off[z][b + 1])
  float* sp[2];                              // [sum T_b, 1025]: clip b's frames at rows frame_off[b] ..
  const double* window;                      // [2048] periodic hann, float64
  const double2* tw1024;                     // e^{-2 pi i j / 1024}, float64
  const double2* tw2048;                     // e^{-2 pi i k / 2048}, k = 0..1024
  int batch, sources;
  int64_t off[2][SCORE_MAX_IMAGES + 1];
  int64_t frame_off[SCORE_MAX_IMAGES + 1];   // T_b = 1 + n_b / 441 (the sources have equal frame counts)
};
cudaError_t launch_metric_stft(const MetricStftParams& p, cudaStream_t stream);

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

}  // namespace vf
