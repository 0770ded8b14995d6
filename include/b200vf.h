/* b200vf.h - C ABI of libb200vf.so: the H100-native (sm_90a) VoiceFixer inference hot path.
 *
 * The reference (haoheliu/voicefixer_main) has no FFI for this path; its boundary is the Python object
 * protocol that eval_gsr_voicefixer.py:handler() consumes (SURVEY.md 8(b)).  Each entry point below
 * replaces one reference interface and is what a ctypes / cgo / JNI binding of that interface would bind:
 *
 *   vf_create / vf_load_weights   Model(hp, ...).load_from_checkpoint(ckpt); model.eval(); model.to(device)
 *                                 eval_gsr_voicefixer.py:31-35,40; config keys config/vctk_base_voicefixer_unet.json:68-78
 *   vf_frontend                   VoiceFixer.pre  models/gsr_voicefixer.py:178-181
 *                                 = FDomainHelper.wav_to_spectrogram_phase tools/pytorch/modules/fDomainHelper.py:67-89
 *                                 + MelScale.forward tools/pytorch/mel_scale.py:52-64
 *   vf_unet_mel                   VoiceFixer.forward models/gsr_voicefixer.py:183-193 -> Generator.forward :86-91
 *                                 -> UNetResComplex_100Mb.forward models/components/unet.py:60-103
 *   vf_vocoder                    model.vocoder(mel) eval_gsr_voicefixer.py:66 (third-party voicefixer.Vocoder)
 *   vf_restore / vf_restore_host  one iteration of the segment loop of handler(), eval_gsr_voicefixer.py:49-74:
 *                                 pre -> model -> from_log -> vocoder -> peak normalise -> trim_center
 *   vf_restore_varlen             the same for clips of different lengths in one call (handler() run over a test set)
 *   vf_restore_varlen_mels        + each clip's stage A / B mels, the inputs of handler()'s metrics (handler_batch)
 *   vf_to_log / vf_from_log       tools/pytorch/pytorch_util.py:157-163
 *   vf_to_pcm16                   the int16 conversion of save_wave, tools/file/wav.py:22-24 (SURVEY.md 8(f) row 3)
 *   vf_mel                        MelScale.forward on any spectrogram, tools/pytorch/mel_scale.py:52-64
 *   vf_finalize                   peak normalise + trim_center, eval_gsr_voicefixer.py:68-72, tools/utils.py:57-70
 *   vf_ssr_forward / vf_ssr_restore(_host) / vf_ssr_unet
 *                                 SSR_UNet / GSR_UNet inference (BASELINE config 3): models/ssr_unet.py:140-155 ->
 *                                 Generator.forward :51-54 -> unet_v2 UNetResComplex_100Mb.forward
 *                                 models/components/unet_v2.py:86-148 (magnitude net, input phase, ISTFT)
 *   vf_ssr_restore_varlen         the same for clips of different lengths in one call (eval_ssr_unet.py:handler()'s test set)
 *   vf_ssr_restore_varlen_mels    + each clip's output mel and peak normalise, the rest of eval_gsr_unet.py:handler()'s
 *                                 segment loop (handler_unet.handler_batch)
 *   vf_istft                      FDomainHelper.istft tools/pytorch/modules/fDomainHelper.py:30-32,127 (torchlibrosa ISTFT)
 *   vf_resample_poly              load_wav's rate conversion, tools/utils.py:46-48
 *   vf_lsd / vf_sispec            AudioMetrics.lsd / .sispec evaluation_proc/metrics.py:83-95 (handler's mel metrics,
 *                                 eval_gsr_voicefixer.py:56-64)
 *   vf_metric_spectrogram         AudioMetrics.wav_to_spectrogram metrics.py:37-51 (librosa STFT magnitude + mel) at 44.1 kHz
 *   vf_ssim                       AudioMetrics.ssim metrics.py:97-106 (scikit-image structural_similarity, win_size 7)
 *   vf_score_varlen               the spectral part of AudioMetrics.evaluation metrics.py:53-81 for a set of file pairs
 *
 * Conventions: every function returns 0 on success or a negative VF_E* code and never throws; the message is
 * available from vf_last_error().  All tensor arguments are contiguous fp32.  Unless a name ends in `_host`,
 * pointers are DEVICE pointers owned by the caller (e.g. PyTorch tensors); the library never frees or retains
 * them.  `stream` is a cudaStream_t passed as void* (torch.cuda.current_stream().cuda_stream); calls are
 * asynchronous with respect to the host and contain no hidden synchronisation, except where stated.  One
 * context per device; calls on one context must be serialised by the caller.  There is no CPU fallback: without
 * a CUDA device every call fails with VF_ENODEVICE.
 */
#ifndef B200VF_H_
#define B200VF_H_

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define VF_API __attribute__((visibility("default")))
#else
#define VF_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define VF_OK 0
#define VF_EINVAL (-1)     /* bad argument / unsupported shape */
#define VF_ENODEVICE (-2)  /* no usable CUDA device */
#define VF_ECUDA (-3)      /* CUDA runtime / driver error */
#define VF_ESTATE (-4)     /* weights not loaded, missing tensor, ... */
#define VF_EDEVICE (-5)    /* sticky device-side error flag (fp16 range overflow, pipeline time-out) */
#define VF_EASSERT (-6)    /* reference assertion would have fired (to_log on negative input) */

typedef struct vf_ctx vf_ctx;

/* Geometry of the front end (reference config "model"/"data" keys) and of the vocoder restatement. */
typedef struct vf_config {
  int sample_rate;        /* 44100 */
  int n_fft;              /* 2048  (window_size) */
  int hop;                /* 441   (hop_size) */
  int n_mels;             /* 128   (mel_freq_bins) */
  /* vocoder generator (voicefixer_main_b200/arch.py:VocoderConfig) */
  int voc_cond_channels;  /* 512 */
  int voc_cond_layers;    /* 5 */
  int voc_channels;       /* 1024 */
  int voc_num_stages;     /* 4 */
  int voc_scales[8];      /* 7,7,3,3 */
  int voc_depth[8];       /* 8,8,8,8 */
  float voc_stage_slope;  /* 0.2 */
  float voc_res_slope;    /* 0.01 */
  float voc_min_db;       /* -115 */
  float voc_ref_db;       /* 20 */
  float voc_amp_floor;    /* 1e-5 */
  float voc_tail_value;   /* -4 */
  int voc_tail_base;      /* 4 */
  double voc_mel_weight_a;
  double voc_mel_weight_b;
  int voc_tail_tanh;      /* 1 (the generator ends in tanh); 0 leaves the tail linear - test configurations only */
} vf_config;

/* Fills *cfg with the reference defaults listed above. */
VF_API void vf_default_config(vf_config* cfg);

typedef struct vf_tensor_desc {
  const char* name;      /* reference state-dict key, e.g. "generator.analysis_module.encoder_block1.conv_block1.bn1.weight",
                            "mel.fb", or "vocoder.<key>" (arch.py:vocoder_keys) */
  const void* data;      /* fp32, contiguous */
  int ndim;
  int64_t shape[4];
  int on_device;         /* 0: host pointer, 1: device pointer */
} vf_tensor_desc;

VF_API int vf_create(vf_ctx** out, int device, const vf_config* cfg);
VF_API void vf_destroy(vf_ctx* ctx);
VF_API const char* vf_last_error(vf_ctx* ctx);   /* ctx may be NULL: error of the last failed vf_create */

/* Copies and packs the tensors (BN folded to per-channel affine, conv weights to K-major fp16 hi/lo
 * matrices, mel filterbank to its sparse form).  Synchronous.  "mel.fb" is required; of the three networks -
 * "generator.analysis_module.*" (VoiceFixer's mel UNet; unet.py and unet_small.py share its keys), "vocoder.*",
 * "generator.unet.*" (unet_v2 of SSR_UNet / GSR_UNet) - whichever are present are loaded, and a network that is
 * present must be complete (missing key -> VF_ESTATE).  Entry points that need an absent network fail with VF_ESTATE; "mel.fb"
 * alone is enough for the front end and for scoring (vf_metric_spectrogram, vf_score_varlen). */
VF_API int vf_load_weights(vf_ctx* ctx, const vf_tensor_desc* descs, int n);

/* wav [B,N] -> mel_out [B,T,128] linear mel (T = 1 + N/hop); optional sp/cos/sin [B,T,1025] (NULL to skip). */
VF_API int vf_frontend(vf_ctx* ctx, const float* wav, int batch, int64_t n_samples, float* mel_out, float* sp_out,
                float* cos_out, float* sin_out, void* stream);

/* mel_lin [B,T,128] (non-negative) -> logmel_out [B,T,128] = unet(log10 mel) + log10 mel.
 * Negative inputs are counted on the device; vf_check_errors() then reports VF_EASSERT (to_log's assert). */
VF_API int vf_unet_mel(vf_ctx* ctx, const float* mel_lin, int batch, int frames, float* logmel_out, void* stream);

/* mel_lin [B,T,128] -> wav_out [B,L], L = vf_vocoder_out_len(ctx, T). */
VF_API int vf_vocoder(vf_ctx* ctx, const float* mel_lin, int batch, int frames, float* wav_out, void* stream);
VF_API int64_t vf_vocoder_out_len(vf_ctx* ctx, int frames);

/* Fused stages A -> B -> C + peak normalise + centre trim: wav [B,N] -> wav_out [B,N] (device pointers). */
VF_API int vf_restore(vf_ctx* ctx, const float* wav, int batch, int64_t n_samples, float* wav_out, void* stream);
/* vf_restore with per-call behaviour flags (re-entrant: nothing is stored in the context). */
#define VF_RESTORE_UNIFY_ENERGY 1u   /* amp_to_original_f (tools/utils.py:50-55) as handler() applies it when
                                        meta["unify_energy"] is set, eval_gsr_voicefixer.py:54-55 */
VF_API int vf_restore_ex(vf_ctx* ctx, const float* wav, int batch, int64_t n_samples, float* wav_out, unsigned flags,
                         void* stream);
/* Clips of different lengths in one call.  wav: packed device buffer, clip i = wav[offsets[i] .. offsets[i+1]);
 * offsets: HOST array of batch + 1 increasing int64, offsets[0] = 0 (read during the call only); wav_out: packed the same
 * way.  flags as vf_restore_ex.  Clip i's output is bit-identical to vf_restore_ex on that clip alone (batch 1, same flags,
 * same options).  Every clip needs more than 1024 samples and a length trim_center accepts (as vf_restore_ex); a bad
 * argument fails before any work is queued.  Plans are cached per (batch, bucket), bucket = the longest clip's frames
 * rounded up to a multiple of 64, so any mix of lengths under one bucket reuses one plan and its CUDA graph; the clips'
 * lengths reach the device through a kernel parameter on `stream`.  Large calls run as consecutive sub-batches of at most
 * 256 clips (fewer under the plan budget), each with its own bucket; clips keep their order. */
VF_API int vf_restore_varlen(vf_ctx* ctx, const float* wav, const int64_t* offsets, int batch, float* wav_out,
                             unsigned flags, void* stream);
/* vf_restore_varlen, and in addition: clip i's linear mel (stage A) and restored log10 mel (stage B), T_i = 1 + n_i / hop
 * frames of 128 bins, written at frame offset F_i = sum_{j<i} T_j of mel_out / log_mel_out ([sum T_i, 128], device,
 * either may be NULL).  Bit-identical to what vf_restore_stages returns after vf_restore_ex on that clip alone.  Each
 * sub-batch adds one copy kernel on `stream` (none when both are NULL: the call is then vf_restore_varlen). */
VF_API int vf_restore_varlen_mels(vf_ctx* ctx, const float* wav, const int64_t* offsets, int batch, float* wav_out,
                                  unsigned flags, float* mel_out, float* log_mel_out, void* stream);
/* The same for the SSR_UNet / GSR_UNet path: clips of different lengths, packed and with HOST offsets as in
 * vf_restore_varlen, no flags.  Clip i's output is bit-identical to vf_ssr_restore on that clip alone (batch 1, same
 * options).  Every clip needs more than 1024 samples and at most 2^30 (no trim_center constraint: there is no vocoder); a
 * bad argument fails with VF_EINVAL before any work is queued, and a context without the unet_v2 weights
 * (generator.unet.*) with VF_ESTATE.  Plans, buckets, sub-batches and the lengths' path to the device as in
 * vf_restore_varlen. */
VF_API int vf_ssr_restore_varlen(vf_ctx* ctx, const float* wav, const int64_t* offsets, int batch, float* wav_out,
                                 void* stream);
/* vf_ssr_restore_varlen plus the rest of one iteration of the SSR / GSR-UNet handler's segment loop (eval_gsr_unet.py:54-67,
 * eval_ssr_unet.py:116-136):
 * - mel_out ([sum T_i, 128], device, or NULL): the linear mel of clip i's restored, un-normalised output,
 *   mel(wav_to_spectrogram_phase(out)[0]), T_i = 1 + n_i / hop frames at frame offset F_i = sum_{j<i} T_j.  Bit-identical
 *   to vf_frontend's mel_out on vf_ssr_restore's output for that clip alone.
 * - flags & VF_SSR_PEAK_NORMALISE: after the mel is taken, clip i of wav_out is divided by its own max |x| when that
 *   exceeds 1.  Bit-identical to vf_finalize(len = n_i, n_samples = n_i) on vf_ssr_restore's output for that clip alone.
 * Per sub-batch, on `stream` after the ISTFT: with mel_out one front-end launch and one copy kernel, with the flag one
 * memset and two kernels.  Unknown flag bits fail with VF_EINVAL before any work is queued.  With mel_out NULL and flags 0
 * the call is vf_ssr_restore_varlen. */
#define VF_SSR_PEAK_NORMALISE 1u
VF_API int vf_ssr_restore_varlen_mels(vf_ctx* ctx, const float* wav, const int64_t* offsets, int batch, float* wav_out,
                                      unsigned flags, float* mel_out, void* stream);
/* Same through HOST buffers (pinned for true asynchrony).  The copies and the compute run on library-owned streams with
 * two staging buffer pairs, so back-to-back calls overlap (the H2D of call i+1 and the D2H of call i-1 run under the
 * compute of call i); `stream` only receives a wait on this call's D2H.  Contract: wav_host holds its data when the
 * call is made (host-written; it is not ordered after work queued on `stream`), and the caller synchronises `stream`
 * before reading out_host or reusing wav_host.  Option "host_pipeline" = 0 restores the single-stream behaviour. */
VF_API int vf_restore_host(vf_ctx* ctx, const float* wav_host, int batch, int64_t n_samples, float* out_host, void* stream);
/* Copies the intermediate results of the last vf_restore of this (batch, n_samples) into caller buffers
 * [B,T,128] (either may be NULL): the linear mel of stage A and the restored log10 mel of stage B. */
VF_API int vf_restore_stages(vf_ctx* ctx, int batch, int64_t n_samples, float* mel_lin_out, float* log_mel_out,
                             void* stream);

/* ---- SSR_UNet / GSR_UNet (unet_v2) path.  vf_ssr_forward = model(sp, wav)['wav'] of models/ssr_unet.py:145-155:
 * sp [B,T,1025] is the network input (NULL: the STFT magnitude of wav itself, i.e. pre() fused in), wav [B,N] supplies
 * the phase (unet_v2.py:96) and the output length; wav_out [B,N].  vf_ssr_restore(wav) == vf_ssr_forward(NULL, wav). */
VF_API int vf_ssr_forward(vf_ctx* ctx, const float* sp, const float* wav, int batch, int64_t n_samples, float* wav_out,
                          void* stream);
VF_API int vf_ssr_restore(vf_ctx* ctx, const float* wav, int batch, int64_t n_samples, float* wav_out, void* stream);
VF_API int vf_ssr_restore_host(vf_ctx* ctx, const float* wav_host, int batch, int64_t n_samples, float* out_host,
                               void* stream);
/* The magnitude branch alone (unet_v2.py:99-132): sp [B,T,1025] -> out_mag [B,T,1025] (last bin 0, F.pad :128). */
VF_API int vf_ssr_unet(vf_ctx* ctx, const float* sp, int batch, int frames, float* mag_out, void* stream);
/* Intermediates of the last vf_ssr_* call of this shape: input magnitude and predicted magnitude [B,T,1025]. */
VF_API int vf_ssr_stages(vf_ctx* ctx, int batch, int64_t n_samples, float* sp_out, float* mag_out, void* stream);
/* FDomainHelper.istft(real, imag, length): real, imag [B,T,1025] -> wav_out [B,length]. */
VF_API int vf_istft(vf_ctx* ctx, const float* real, const float* imag, int batch, int frames, int64_t length,
                    float* wav_out, void* stream);

/* MelScale.forward on an arbitrary spectrogram view: mel_out[o, t, m] = sum_f specgram[o*stride_outer + f*stride_freq +
 * t*stride_time] * fb[f, m]; strides in elements, mel_out [n_outer, frames, 128] contiguous (n_outer <= 65535). */
VF_API int vf_mel(vf_ctx* ctx, const float* specgram, int64_t n_outer, int64_t frames, int64_t stride_outer,
                  int64_t stride_freq, int64_t stride_time, float* mel_out, void* stream);
/* eval_gsr_voicefixer.py:68-72 as one op: wav [B,len] -> per clip `if max|x| > 1: x /= max|x|`, then trim_center to n
 * samples -> wav_out [B,n].  (handler() sees batch 1, so "per clip" is its semantics.) */
VF_API int vf_finalize(vf_ctx* ctx, const float* wav, int batch, int64_t len, int64_t n_samples, float* wav_out,
                       void* stream);

/* ---- I/O edges of handler() (SURVEY.md 8(f) rows 3-4).
 * Polyphase resampling by up/down (load_wav -> librosa.load(sr=44100), tools/utils.py:46-48, with the arithmetic of
 * scipy.signal.resample_poly as the reference uses it in tools/dsp/lowpass.py:138-141): out[b,m] = sum_i taps[m*down -
 * i*up + n_taps/2] * wav[b,i]; taps = the caller's symmetric FIR (odd n_taps, device pointer), n_out = ceil(n*up/down). */
VF_API int vf_resample_poly(vf_ctx* ctx, const float* wav, int batch, int64_t n_samples, int up, int down, const float* taps,
                            int n_taps, float* out, int64_t n_out, void* stream);
/* amp_to_original_f (tools/utils.py:50-55; handler() applies it when meta["unify_energy"], eval_gsr_voicefixer.py:54-55) on
 * linear mels [B,T,128]: mel_out = mel_est * (mean of mel_target over bins 5..24 / mean of mel_est over bins 5..24), per clip.
 * vf_restore_ex fuses the same step into the restore chain (VF_RESTORE_UNIFY_ENERGY). */
VF_API int vf_amp_to_original_f(vf_ctx* ctx, const float* mel_est, const float* mel_target, int batch, int frames, float* mel_out,
                                void* stream);
/* AudioMetrics.lsd (evaluation_proc/metrics.py:83-87): est, target [images, frames, bins] (non-log) -> out [images]. */
VF_API int vf_lsd(vf_ctx* ctx, const float* est, const float* target, int images, int frames, int bins, float* out, void* stream);
/* AudioMetrics.sispec (metrics.py:89-95) per batch item over n values -> out [batch] (the reference then averages over
 * the batch).  est_map / target_map: 0 none, 1 to_log, 2 from_log applied on the fly (eval_gsr_voicefixer.py:60-62). */
VF_API int vf_sispec(vf_ctx* ctx, const float* est, const float* target, int batch, int64_t n, int est_map, int target_map,
                     float* out, void* stream);

/* ---- Scoring a restored file against its target (AudioMetrics.evaluation, evaluation_proc/metrics.py:53-81).
 * Versions: the STFT is librosa 0.8's default (reflect padding; librosa >= 0.10 pads with zeros, not built), and SSIM is
 * scikit-image <= 0.18's float64 structural_similarity with data_range 2 (the dtype range of float32; >= 0.19 computes in
 * float32 and refuses float input without data_range, not built).
 *
 * np.abs(librosa.stft(wav, n_fft=2048, hop_length=441)) per clip, transposed: wav and offsets packed as in vf_restore_varlen
 * (HOST offsets, batch + 1, offsets[0] = 0, every clip 1025 .. 2^30 samples); clip i's T_i = 1 + n_i / 441 frames land at
 * row F_i = sum_{j<i} T_j of sp_out [sum T_i, 1025].  Float64 window and FFT, the spectrum rounded to complex64, |.| of that;
 * no clamp (digital silence gives exact zeros).  mel_out [sum T_i, 128] (or NULL): MelScale(n_mels=128, sample_rate=44100,
 * n_stft=1025) of those rows, the arithmetic of vf_mel; it needs "mel.fb" loaded (VF_ESTATE otherwise). */
VF_API int vf_metric_spectrogram(vf_ctx* ctx, const float* wav, const int64_t* offsets, int batch, float* sp_out, float* mel_out,
                                 void* stream);
/* SSIM of each [frames, bins] image pair of est / target ([images, frames, bins] fp32, frames and bins >= 7) -> out[images].
 * The result is float64, as scikit-image's is: the one exception to the fp32 convention above.  Computed in float64 with a
 * fixed reduction order (deterministic); identical images give exactly 1.0. */
VF_API int vf_ssim(vf_ctx* ctx, const float* est, const float* target, int images, int frames, int bins, double* out, void* stream);
/* The spectral part of AudioMetrics.evaluation for `batch` (est, target) pairs at 44.1 kHz: est and target packed with their
 * own HOST offsets (as in vf_metric_spectrogram).  out [batch, 8] float64 in the reference's key order: lsd, non_log_sispec,
 * sispec, ssim on the spectrogram, then final_mel_lsd, final_non_log_mel_sispec, final_mel_sispec, final_mel_ssim on its
 * mel.  lsd and sispec are the fp32 values of vf_lsd / vf_sispec on each pair alone, widened; sispec is on to_log of both
 * spectrograms.  (sisdr, stoi and pesq come from the third-party speechmetrics package and are not computed.)  Every pair
 * is checked before any work is queued: equal frame counts and at least 7 frames, else VF_EINVAL naming the pair.  The
 * scratch (two spectrograms, two mels, SSIM tile sums) is owned by the context and freed by vf_destroy; it is allocated
 * stream-ordered, so there is no host synchronisation.  Pairs run in consecutive sub-batches of at most 16384 frames
 * (about 164 s of audio per side) and 128 pairs; a single longer pair gets a sub-batch, and scratch, of its own.  Ten
 * launches per sub-batch.  Needs "mel.fb" loaded (no network). */
VF_API int vf_score_varlen(vf_ctx* ctx, const float* est, const int64_t* est_offsets, const float* target,
                           const int64_t* target_offsets, int batch, double* out, void* stream);

VF_API int vf_to_log(vf_ctx* ctx, const float* in, float* out, int64_t n, void* stream);
VF_API int vf_from_log(vf_ctx* ctx, const float* in, float* out, int64_t n, void* stream);
/* fp32 samples -> 16-bit PCM exactly as save_wave does it: x * 2^15, truncation toward zero through a 32-bit integer,
 * low 16 bits kept (so +1.0 wraps to -32768 like numpy's astype(np.short) on the reference's hosts).  `out` is a
 * device buffer of n int16. */
VF_API int vf_to_pcm16(vf_ctx* ctx, const float* in, int16_t* out, int64_t n, void* stream);
/* saturate != 0: clamp to [-32768, 32767] first, so a peak-normalised +1.0 becomes 32767 instead of wrapping to -32768 (an
 * audible click the reference's cast produces; not bit-compatible with save_wave, hence opt-in). */
VF_API int vf_to_pcm16_ex(vf_ctx* ctx, const float* in, int16_t* out, int64_t n, int saturate, void* stream);

/* Device memory the plan for (batch, n_samples) holds (activations + packed weights). */
VF_API int vf_workspace_bytes(vf_ctx* ctx, int batch, int64_t n_samples, size_t* bytes);

/* Synchronises `stream`, reads and clears the sticky device flags.  VF_OK, VF_EDEVICE or VF_EASSERT. */
VF_API int vf_check_errors(vf_ctx* ctx, void* stream);

/* Options: "vocoder_terms" (1 or 3 fp16 split terms; "unet_terms" accepts only 3), "unify_energy" (default flag of
 * vf_restore / vf_restore_host; prefer vf_restore_ex's per-call flag), "plan_cache_mb" (cap on the device memory
 * held by cached per-shape plans, least recently used evicted first; 0 = half of the free device memory),
 * "graphs" (default 1: the fixed-pointer launch chain of a plan is captured on its second use and replayed as one CUDA graph from then on),
 * "host_pipeline" (default 1, see vf_restore_host),
 * "validate_simt" (1: run every GEMM on the SIMT validation kernel instead of the wgmma kernel - tests only). */
VF_API int vf_set_option(vf_ctx* ctx, const char* key, int value);
/* Plans are cached per (path, batch, frames) - vf_restore_varlen and vf_ssr_restore_varlen: (path, batch, bucket) - ; the cache is bounded (see "plan_cache_mb").  A batch whose plan would not fit
 * the budget is processed in sub-batches through a smaller plan (same results: rows are independent); the *_stages accessors
 * then only see the last sub-batch. */
VF_API int vf_plan_cache_info(vf_ctx* ctx, int* n_plans, size_t* bytes, size_t* budget, int64_t* evicted);
/* Number of kernels this context has launched since creation. */
VF_API int64_t vf_launch_count(vf_ctx* ctx);

/* Stage timing: wraps the stages of subsequent vf_restore calls in CUDA events on the call's stream.
 * vf_stage_times synchronises and returns milliseconds of the last vf_restore: [frontend, unet, vocoder, tail]. */
VF_API int vf_enable_stage_timing(vf_ctx* ctx, int enable);
VF_API int vf_stage_times(vf_ctx* ctx, float ms[4]);

/* Per-launch profile: with op timing enabled, the next vf_restore records a CUDA event before every kernel of
 * the UNet and vocoder launch chains.  vf_op_info(i) synchronises and returns the device time of launch i
 * together with its ALGORITHMIC flops / minimum HBM bytes (the reference op's own counts), the flops the tensor
 * cores actually executed for it (3 MMAs per product in 3-term mode, tile / phase padding, identity taps), the tensor-core tile
 * (bn, bk, fp16 split terms; 0 for non-GEMM kernels) and a label such as "enc3.b2.conv1".  For roofline reporting only. */
VF_API int vf_enable_op_timing(vf_ctx* ctx, int enable);
VF_API int vf_op_count(vf_ctx* ctx);
VF_API int vf_op_info(vf_ctx* ctx, int i, float* ms, double* flops, double* bytes, int* bn, int* bk, int* terms,
                      char* label, int label_cap, double* exec_flops /* nullable: tensor-core flops actually issued */);

/* TEST ONLY.  One conv layer built the way the plans build it (the product's weight packers and tap lists, the plan
 * builder's GEMM / fused-pair set-up), run once and copied back.  Synchronous; every pointer is a host pointer.
 * Activation operands are fp16 bit patterns in the kernels' layout: [plane (hi, lo)][n_img][img_rows][C], rows of a 2-D
 * layer flattened (h, w) with one pad column (row pitch W + 1).  Output buffers are read AND written: they are uploaded
 * before the launch, so what the layer must not touch comes back unchanged. */
enum { VF_LAYER_CONV2D = 0, VF_LAYER_CONVT2D = 1, VF_LAYER_CONV1D = 2, VF_LAYER_CONVT1D = 3, VF_LAYER_PAIR = 4 };
enum { VF_LAYER_PRODUCT = 0, VF_LAYER_SIMT = 1 };
enum { VF_RESID_NONE = 0, VF_RESID_FP32 = 1, VF_RESID_PLANES = 2, VF_RESID_AR = 3, VF_RESID_IDENTITY = 4 };
typedef struct vf_layer_case {
  int kind, impl, terms;    /* VF_LAYER_*, VF_LAYER_PRODUCT / SIMT (no (a, r) support: VF_EINVAL), 1 or 3 */
  int n_img;
  int H, W;                 /* CONV2D / CONVT2D input pixels; GEMM rows per image H * (W + 1) */
  int L;                    /* CONV1D / CONVT1D / PAIR input rows per image */
  int cin, cout, sc_cin;    /* sc_cin: CONV2D 1x1 shortcut source channels, 0 = none */
  int k, dilation, centered;   /* CONV1D */
  int stride;               /* CONVT1D: stride s, padding s / 2 + s % 2 */
  int both;                 /* CONVT2D: 1 = prune time and frequency (output pitch 2 (W + 1) - 1), 0 = time only */
  /* PyTorch layouts, fp32: w [cout][cin][3][3] / [cin][cout][3][3] / [cout][cin][k] / [cin][cout][2 s]; PAIR: w, b = conv_a, w2, b2 = conv_b */
  const float* w;
  const float* b;           /* [cout] or NULL */
  const float* sc_w;        /* [cout][sc_cin] */
  const float* sc_b;        /* [cout] */
  const float* w2;
  const float* b2;
  const uint16_t* x;        /* [2][n_img][x_img_rows][cin]; rows [x_row0, x_img_rows) of each image are the layer's input
                               (PAIR: the (a, r) planes of x) */
  int x_img_rows, x_row0;
  const uint16_t* sc_x;     /* [2][n_img][rows][sc_cin] */
  int resid_kind;           /* VF_RESID_*: FP32 [n_img][rows][cout] floats; PLANES / AR / IDENTITY [2][n_img][rows][cout] fp16 */
  const void* resid;
  float ar_slope;           /* AR (input and output streams): the LeakyReLU slope whose fp16 inverse the stream uses */
  float* out_raw;           /* [n_img][out_img_rows][raw_ld] or NULL */
  int raw_ld;
  uint16_t* out_r;          /* [2][n_img][out_img_rows][r_ld] or NULL */
  int r_ld, r_c_off;
  uint16_t* out_a;          /* [2][n_img][out_img_rows][a_ld] or NULL: act(scale * v + shift) */
  int a_ld, a_c_off;
  int out_ar;               /* out_a is written as the (a, r) pair of x itself (1-term, LeakyReLU ar_slope, no affine) */
  const float* a_scale;     /* [cout] or NULL */
  const float* a_shift;
  int act;                  /* 0 none, 1 LeakyReLU (slope), 2 ELU */
  float slope;
  int out_row0, out_img_rows;
  const float* head_w;      /* [32]: fused 1x1 head of a 32-channel CONV2D, or NULL */
  float head_b;
  const float* head_in;     /* [n_img][head_T][W + 1] or NULL */
  float* head_out;          /* [n_img][head_T][W + 1] */
  int head_T;
  const int* row_valid;     /* [n_img] or NULL */
  const int* head_valid;    /* [n_img] or NULL */
  float pair_slope_h, pair_slope_out;   /* PAIR: activation of h, and of x_new (the stage slope after the last pair) */
  int pair_last;            /* PAIR: no correction plane out (last pair of a stack) */
  /* reported: the launch configuration the builder chose */
  int bn, bk, stages, resid_tma, tma_out, grid;
  int64_t tiles;
  int div_fallback;         /* a tile decode divides (its multiply-high magic would not be exact) */
} vf_layer_case;
VF_API int vf_selftest_layer(vf_ctx* ctx, vf_layer_case* lc);

/* TEST ONLY.  One non-GEMM op of the launch chains, set up by the same helpers the plan builders and restore paths use and
 * launched as they launch it (run_ops or the same launch_* call), then copied back.  Synchronous; every pointer is a host
 * pointer, and output buffers are read AND written as in vf_selftest_layer.  fp16 planes are bit patterns [2][batch][rows][C].
 * Fields a kind does not use are zero.  The mel-weight table, window and twiddles are the context's own. */
enum { VF_OP_FIRST = 0, VF_OP_POOL = 1, VF_OP_COND = 2, VF_OP_REFLECT = 3, VF_OP_TAIL = 4, VF_OP_FINALIZE = 5, VF_OP_ISTFT = 6,
       VF_OP_PEAK_NORM = 7 };
typedef struct vf_op_case {
  int kind, batch;
  /* Clips of different lengths (any kind; PEAK_NORM needs them): host sample offsets [batch + 1], clip b = [off[b], off[b + 1]).
   * The hook writes a lengths table with the product's setup kernel (unet_w0: 127 or 1024, the UNet's valid bins) and hands
   * the kernel the rows its plan would: FIRST T / Tp, POOL the UNet rows of level + 1, COND T / Tv, REFLECT / TAIL the last
   * vocoder stage's samples (REFLECT with cond_pad: Tv), FINALIZE and ISTFT the offsets and the last stage / T.  The table
   * comes back in vl_rows [18][batch] when that is not NULL. */
  const int64_t* clip_off;
  int unet_w0;
  int* vl_rows;
  /* FIRST: x [batch][T][W + 1], w1 [32][9], bn2 / shortcut [32]; out a2 planes [batch][Tp (W + 1)][32], sc_raw floats */
  int T, W;
  float bn1_scale, bn1_shift;
  const float* x;
  const float* w1;
  const float* bn2_scale;
  const float* bn2_shift;
  const float* w_sc;
  const float* b_sc;
  uint16_t* a2;
  float* sc_raw;
  /* POOL (H, W, C, level): pin [batch][H (W + 1)][C] floats, the next block's bn1 [C]; out_r / out_a planes and out_raw floats
   * [batch][(H / 2) Wpo][C] (any of them NULL) */
  int H, C, level;
  const float* pin;
  const float* a_scale;
  const float* a_shift;
  uint16_t* out_r;
  uint16_t* out_a;
  float* out_raw;
  /* COND (T): mel [batch][T][128], log10 when is_log; unify: mel_target [batch][T][128] linear, the band sums come back in
   * band_sums [batch][2]; out cond planes [batch][Tv][128] */
  int is_log, unify;
  const float* mel;
  const float* mel_target;
  float* band_sums;
  uint16_t* cond;
  /* REFLECT (C, L, cond_pad): planes [batch][L + 6][C] in place.  TAIL (C, L, terms, tanh_out): tail_in [batch][L + 6][C]
   * planes (already reflect padded), tail_w [1][C][7] (PyTorch layout), out wav [batch][L] and peak_bits [batch] */
  int64_t L;
  int cond_pad, terms, tanh_out;
  uint16_t* planes;
  const uint16_t* tail_in;
  const float* tail_w;
  float tail_b;
  float* wav;
  uint32_t* peak_bits;
  /* FINALIZE (L, n): wav [batch][L] and peak_bits [batch] in; out [batch][n] (varlen: packed by clip_off).
   * ISTFT (T, n): mag [batch][T][1025], wav [batch][n] (varlen: packed by clip_off); frames [batch][T][2048], out as FINALIZE.
   * PEAK_NORM (n = the longest clip): wav packed by clip_off, normalised in place; the per-clip peaks come back in peak_bits */
  int64_t n;
  const float* in_wav;
  const float* mag;
  float* frames;
  float* out;
  /* reported: what the set-up derived */
  int Tp, Wpo, Tv;
  int64_t skip;
  int64_t tail_smem;
} vf_op_case;
VF_API int vf_selftest_op(vf_ctx* ctx, vf_op_case* oc);

#ifdef __cplusplus
}
#endif
#endif /* B200VF_H_ */
