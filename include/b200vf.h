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
 *   vf_vocoder_varlen             the stand-alone vocoder (pip voicefixer's Vocoder.forward) on mels of different lengths
 *                                 in one call; needs only the vocoder's weights and mel.fb
 *   vf_resynth / vf_resynth_varlen  vocoder resynthesis: handler()'s segment step without the analysis module,
 *                                 pre -> vocoder on the linear mel -> peak normalise -> trim_center (vocoder weights only)
 *   vf_restore / vf_restore_host  one iteration of the segment loop of handler(), eval_gsr_voicefixer.py:49-74:
 *                                 pre -> model -> from_log -> vocoder -> peak normalise -> trim_center
 *   vf_restore_varlen             the same for clips of different lengths in one call (handler() run over a test set)
 *   vf_restore_varlen_mels        + each clip's stage A / B mels, the inputs of handler()'s metrics (handler_batch)
 *   vf_restore_chunks             the chunks of many live streams, gathered from device rings and cropped on the device:
 *                                 LambdaOverlapAdd (tools/dsp/overlapadd_boxcar.py:338-534) run incrementally
 *   vf_vocoder_chunks             the chunks of many live mel streams (a TTS or voice-conversion model's output),
 *                                 gathered from device frame rings, vocoded and cropped on the device
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
 *   vf_ssr_restore_chunks         vf_restore_chunks for SSR_UNet / GSR_UNet: live streams of the denoising, declipping,
 *                                 dereverberation and super-resolution models
 *   vf_restore_windows            the windows of many live streams, gathered from device rings, weighted by a synthesis
 *                                 window and overlap-added into caller-owned accumulators on the device: the windowed
 *                                 LambdaOverlapAdd (tools/dsp/overlapadd.py:338-484) run incrementally
 *   vf_ssr_restore_windows        vf_restore_windows for SSR_UNet / GSR_UNet
 *   vf_istft                      FDomainHelper.istft tools/pytorch/modules/fDomainHelper.py:30-32,127 (torchlibrosa ISTFT)
 *   vf_resample_poly              load_wav's rate conversion, tools/utils.py:46-48
 *   vf_lsd / vf_sispec            AudioMetrics.lsd / .sispec evaluation_proc/metrics.py:83-95 (handler's mel metrics,
 *                                 eval_gsr_voicefixer.py:56-64)
 *   vf_metric_spectrogram         AudioMetrics.wav_to_spectrogram metrics.py:37-51 (librosa STFT magnitude + mel) at 44.1 kHz;
 *                                 the _ex forms of it and the two calls below take the rate (44.1 or 16 kHz)
 *   vf_ssim                       AudioMetrics.ssim metrics.py:97-106 (scikit-image structural_similarity, win_size 7)
 *   vf_score_varlen               the spectral part of AudioMetrics.evaluation metrics.py:53-81 for a set of file pairs
 *   vf_score_time_varlen          its sisdr and stoi keys (speechmetrics, metrics.py:58-64) for a set of file pairs
 *   vf_sosfiltfilt_varlen         the IIR types of tools/dsp/lowpass.py lowpass() / bandpass() (scipy sosfiltfilt)
 *   vf_resample_poly_f64_varlen   its "stft" type (resample_poly down and up), collate_fn_val's SR inputs
 *                                 dataloaders/data_module.py:130-150
 *   vf_resample_sinc_varlen       librosa.load(sr=...)'s resampling as librosa 0.8 does it (resampy kaiser_best /
 *                                 kaiser_fast), tools/utils.py:46-48 and metrics.py:33-34; opt-in (res_type)
 *   vf_resample_rings             either resampler on live streams, incrementally from device rings: the input
 *                                 conversion of load_wav for audio that arrives while it is restored
 *   vf_remove_higher_frequency_varlen  the pip package's mode-1 pre-filter, remove_higher_frequency, before a restore
 *   vf_decode_pcm_varlen          the decode and downmix of librosa.load(path, mono=True) (tools/utils.py:46-48,
 *                                 metrics.py:33-34) for 8-, 16-, 24-, 32-bit and float WAV data of any channel count
 *   vf_decode_flac_varlen         the same files as FLAC (8-, 16- and 24-bit, 1 .. 8 channels), decoded into the bytes of
 *                                 a WAV data chunk holding the same samples, which vf_decode_pcm_varlen then converts
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
 * alone is enough for the front end and for scoring (vf_metric_spectrogram, vf_score_varlen).  The optional
 * "metrics.mel_16k.fb" [372, 80] (MelScale(n_mels=80, sample_rate=16000, n_stft=372)) enables 16 kHz scoring (the _ex
 * scoring calls with rate 16000). */
VF_API int vf_load_weights(vf_ctx* ctx, const vf_tensor_desc* descs, int n);

/* wav [B,N] -> mel_out [B,T,128] linear mel (T = 1 + N/hop); optional sp/cos/sin [B,T,1025] (NULL to skip).
 * B <= 65535 (one launch: the clips are the grid's y dimension). */
VF_API int vf_frontend(vf_ctx* ctx, const float* wav, int batch, int64_t n_samples, float* mel_out, float* sp_out,
                float* cos_out, float* sin_out, void* stream);

/* mel_lin [B,T,128] (non-negative) -> logmel_out [B,T,128] = module(log10 mel) + log10 mel, where module is the loaded
 * analysis module (generator.analysis_module.*: the ResUNet of unet / unet_small, bi_gru or dnn).
 * Negative inputs are counted on the device; vf_check_errors() then reports VF_EASSERT (to_log's assert). */
VF_API int vf_unet_mel(vf_ctx* ctx, const float* mel_lin, int batch, int frames, float* logmel_out, void* stream);

/* mel_lin [B,T,128] -> wav_out [B,L], L = vf_vocoder_out_len(ctx, T). */
VF_API int vf_vocoder(vf_ctx* ctx, const float* mel_lin, int batch, int frames, float* wav_out, void* stream);
VF_API int64_t vf_vocoder_out_len(vf_ctx* ctx, int frames);
/* The vocoder on linear mels of different lengths in one call, on a context that holds the vocoder's weights ("vocoder.*"
 * and "mel.fb"; an analysis module may be loaded or not).  mel: packed device buffer [sum T_i, 128], clip i = rows
 * frame_offsets[i] .. frame_offsets[i+1]; frame_offsets: HOST array of batch + 1 increasing int64, frame_offsets[0] = 0
 * (read during the call only).  wav_out (device) receives each clip's full vocoder output, L_i = vf_vocoder_out_len(ctx,
 * T_i) samples at sum_{j<i} L_j: no peak normalise and no trim, as vf_vocoder.  Clip i is bit-identical to vf_vocoder on
 * that clip alone (batch 1, same options).  A clip may have any T_i >= 1 up to 2^30 / hop + 1 frames; an empty or
 * decreasing range fails with VF_EINVAL and a context without the vocoder with VF_ESTATE, before any work is queued.
 * Sub-batches, plans per (batch, bucket) and their CUDA graphs as vf_restore_varlen; the plans hold the vocoder's
 * buffers only.  Each sub-batch adds one scatter of its mels into the plan and one pack of its outputs on `stream`. */
VF_API int vf_vocoder_varlen(vf_ctx* ctx, const float* mel, const int64_t* frame_offsets, int batch, float* wav_out, void* stream);
/* Vocoder resynthesis, wav [B,N] -> wav_out [B,N]: vf_frontend's linear mel -> the vocoder -> peak normalise ->
 * trim_center, needing only the vocoder's weights.  Bit-identical to vf_frontend -> vf_vocoder -> vf_finalize.  Length
 * rules as vf_restore_ex. */
VF_API int vf_resynth(vf_ctx* ctx, const float* wav, int batch, int64_t n_samples, float* wav_out, void* stream);
/* vf_resynth for clips of different lengths, packed with HOST offsets as vf_restore_varlen (no flags).  Clip i is
 * bit-identical to vf_resynth on that clip alone (batch 1). */
VF_API int vf_resynth_varlen(vf_ctx* ctx, const float* wav, const int64_t* offsets, int batch, float* wav_out, void* stream);

/* Fused stages A -> B -> C + peak normalise + centre trim: wav [B,N] -> wav_out [B,N] (device pointers). */
VF_API int vf_restore(vf_ctx* ctx, const float* wav, int batch, int64_t n_samples, float* wav_out, void* stream);
/* vf_restore with per-call behaviour flags (re-entrant: nothing is stored in the context).  Every clip needs more than 1024
 * samples and a length trim_center accepts; a bad argument fails before any work is queued, and a context without the
 * analysis module or the vocoder with VF_ESTATE. */
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
/* Chunks of live audio streams, restored in one call (chunked boxcar-margin streaming, voicefixer_main_b200/streaming.py).
 * ring [n_streams, ring_len] (device) holds each stream's recent samples: absolute position p of stream s is at
 * ring[s * ring_len + p mod ring_len].  chunks: HOST table of n_chunks entries (read during the call only).  Chunk c reads
 * positions start .. start + length - 1 of stream `stream`; a position >= valid reads as 0 (valid = the stream's length once
 * it has ended, INT64_MAX while it is open: BoxcarOverlapAdd's zero padding).  Its restored samples [crop_left, length -
 * crop_right) are written to kept_out (device), chunk after chunk.  Chunk c's kept samples are bit-identical to vf_restore_ex
 * (batch 1, same flags) on its zero-filled samples, cropped.  Every argument is checked before any work is queued (VF_EINVAL:
 * a stream out of range, length > ring_len, a length vf_restore_ex rejects - 1024 samples or fewer, over 2^30, or one
 * trim_center refuses -, crops that leave nothing, start < 0); the context stays usable.  One gather launch, the
 * vf_restore_varlen chain and one crop launch per sub-batch; each sub-batch runs on the plan for the next power of two of its
 * chunk count (the extra rows repeat its first chunk and are discarded), and holds at most the largest power of two P <= 256
 * whose batch shapes 1, 2, .., P fit the plan budget together, so a session whose chunk count changes every step reuses a
 * few cached plans.  The packed input and output scratch is owned by the context, grown on
 * demand stream-ordered and freed by vf_destroy. */
typedef struct vf_chunk {
  int32_t stream;
  int32_t length;
  int32_t crop_left;
  int32_t crop_right;
  int64_t start;
  int64_t valid;
} vf_chunk;
VF_API int vf_restore_chunks(vf_ctx* ctx, const float* ring, int n_streams, int64_t ring_len, const vf_chunk* chunks, int n_chunks,
                             float* kept_out, unsigned flags, void* stream);
/* Chunks of live mel streams, vocoded in one call (voicefixer_main_b200/streaming.py StreamingVocoder), on a context that
 * holds the vocoder's weights (as vf_vocoder_varlen).  ring [n_streams, ring_frames, 128] (device) holds each stream's recent
 * linear mel frames: absolute frame p of stream s is row s * ring_frames + p mod ring_frames.  chunks: HOST table of
 * n_chunks vf_chunk entries (read during the call only), as in vf_restore_chunks except that start, length and valid
 * count frames and crop_left / crop_right count samples of the chunk's vf_vocoder_out_len(length) output: chunk c vocodes
 * frames start .. start + length - 1 of stream `stream`, a frame >= valid reading as zeros, and its output samples
 * [crop_left, vf_vocoder_out_len(length) - crop_right) are written to kept_out (device), chunk after chunk.  Chunk c's kept
 * samples are bit-identical to vf_vocoder_varlen on its (zero-filled) frames alone, cropped.  Every argument is checked
 * before any work is queued (VF_EINVAL: a stream out of range, length < 1, > ring_frames or over vf_vocoder_varlen's 2^30 /
 * hop + 1 frames, crops that leave nothing, start < 0; VF_ESTATE: a context without "vocoder.*"); the context stays usable.
 * Per sub-batch, on its PLAN_VOC_VARLEN plan: the lengths table, one gather launch of the chunks' frames from the rings
 * straight into the plan's mel rows, the vocoder chain (replayed as a CUDA graph) and one crop launch straight out of the
 * plan's output rows.  Sub-batches and plan shapes as vf_restore_chunks (next power of two of the chunk count, the extra
 * rows repeating the first chunk; the largest sub-batch follows the vocoder-only plan size per frame).  No scratch. */
VF_API int vf_vocoder_chunks(vf_ctx* ctx, const float* ring, int n_streams, int64_t ring_frames, const vf_chunk* chunks,
                             int n_chunks, float* kept_out, void* stream);
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
/* vf_restore_chunks for the SSR_UNet / GSR_UNet path: the same ring, vf_chunk table, `valid` zero fill and crops, no flags.
 * Chunk c's kept samples are bit-identical to vf_ssr_restore (batch 1, same options) on its zero-filled samples, cropped.
 * Every argument is checked before any work is queued (VF_EINVAL: a stream out of range, length > ring_len, 1024 samples or
 * fewer, over 2^30, crops that leave nothing, start < 0; there is no trim_center constraint, so a length vf_restore_chunks
 * refuses only for trim_center is accepted), and a context without the unet_v2 weights (generator.unet.*) fails with
 * VF_ESTATE; the context stays usable.  One gather launch, the vf_ssr_restore_varlen chain and one crop launch per
 * sub-batch, with vf_restore_chunks' power-of-two plan shapes and repeated first chunk; the largest sub-batch follows the SSR
 * plan size per frame, larger than VoiceFixer's.  No peak normalisation: divide a stream by its peak, if at all, after it
 * has ended.  The scratch is the one vf_restore_chunks uses. */
VF_API int vf_ssr_restore_chunks(vf_ctx* ctx, const float* ring, int n_streams, int64_t ring_len, const vf_chunk* chunks,
                                 int n_chunks, float* kept_out, void* stream);
/* Windows of live audio streams, restored, weighted and overlap-added in one call (windowed streaming,
 * voicefixer_main_b200/streaming.py WindowedStreamingRestorer).  ring / ring_len / n_streams as in vf_restore_chunks.
 * windows: HOST table of n_windows entries (read during the call only); window w reads positions start .. start + W - 1 of
 * stream `stream` (W = window_len), where positions below 0 and at or past `valid` read as 0 (start may be as low as -W: the
 * W zeros F.unfold(padding=W) puts before the signal).  synthesis: [W] device fp32 (the synthesis window, or W times
 * 1 / (W / hop) for the unweighted average).  acc [n_streams, acc_len] (device, caller-owned, zero where nothing is pending):
 * output position t of stream s accumulates at acc[s * acc_len + t mod acc_len].  For every window, in table order, each
 * position t in [max(0, start), min(valid, start + W)) gets acc += fl(synthesis[t - start] * restored[t - start]) (the product
 * rounded, then the add), restored being vf_restore_ex (batch 1, same flags) of the window's zero-filled samples: with one
 * stream's windows in ascending start, each position sums its windows in ascending order from 0, as F.fold does on CUDA.
 * Then emits: HOST table of n_emits ranges, at most one per stream; range e copies positions start .. start + count - 1 of
 * its stream out of acc to `out` (device; may be NULL when no range holds samples), range after range, and zeroes their
 * slots.  A stream's pending span is
 * [start, start + acc_len) of its emission range; every window needs one for its stream.  Every argument is checked before
 * any work is queued (VF_EINVAL: a stream out of range; W > ring_len; a W vf_restore_ex refuses; no synthesis table; a
 * window start below -W; windows of one stream not in strictly ascending start; a window with no emission range for its
 * stream, or writing outside the stream's pending span; a second range for a stream, start < 0, count < 0 or count >
 * acc_len); the context stays usable.  One gather launch, the vf_restore_varlen chain and one overlap-add launch per
 * sub-batch (sub-batches, plan shapes and scratch as in vf_restore_chunks), then one emission launch per 256 ranges that
 * hold samples.  The library keeps no stream state: the rings and accumulators are the caller's. */
typedef struct vf_window {
  int32_t stream;
  int64_t start;
  int64_t valid;
} vf_window;
typedef struct vf_emit {
  int32_t stream;
  int64_t start;
  int64_t count;
} vf_emit;
VF_API int vf_restore_windows(vf_ctx* ctx, const float* ring, int n_streams, int64_t ring_len, const vf_window* windows,
                              int n_windows, int window_len, const float* synthesis, float* acc, int64_t acc_len,
                              const vf_emit* emits, int n_emits, float* out, unsigned flags, void* stream);
/* vf_restore_windows for the SSR_UNet / GSR_UNet path: no flags, the window's restored samples are vf_ssr_restore's (batch
 * 1), no trim_center constraint on W, and a context without the unet_v2 weights fails with VF_ESTATE. */
VF_API int vf_ssr_restore_windows(vf_ctx* ctx, const float* ring, int n_streams, int64_t ring_len, const vf_window* windows,
                                  int n_windows, int window_len, const float* synthesis, float* acc, int64_t acc_len,
                                  const vf_emit* emits, int n_emits, float* out, void* stream);
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
/* FDomainHelper.istft(real, imag, length): real, imag [B,T,1025] -> wav_out [B,length], B <= 65535, length + n_fft/2 <=
 * (T - 1) * hop + n_fft. */
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
 * spectrograms.  (sisdr and stoi: vf_score_time_varlen; pesq is not computed.)  Every pair
 * is checked before any work is queued: equal frame counts and at least 7 frames, else VF_EINVAL naming the pair.  The
 * scratch (two spectrograms, two mels, SSIM tile sums) is owned by the context and freed by vf_destroy; it is allocated
 * stream-ordered, so there is no host synchronisation.  Pairs run in consecutive sub-batches of at most 16384 frames
 * (about 164 s of audio per side) and 128 pairs; a single longer pair gets a sub-batch, and scratch, of its own.  Ten
 * launches per sub-batch.  Needs "mel.fb" loaded (no network). */
VF_API int vf_score_varlen(vf_ctx* ctx, const float* est, const int64_t* est_offsets, const float* target,
                           const int64_t* target_offsets, int batch, double* out, void* stream);
/* The time-domain keys of AudioMetrics.evaluation for `batch` (est, target) pairs of 44.1 kHz samples, packed with their
 * own HOST offsets: out [batch, 2] float64 = sisdr, stoi, as speechmetrics computes them with window np.inf (restated in
 * oracle/speech_metrics.py): the shorter clip of a pair is zero-padded at the end to the longer one; sisdr is the
 * scale-invariant SDR without mean removal, stoi is pystoi 0.3.3's stoi(target, est, 44100, extended=False) - Octave-window
 * resampling to 10 kHz, removal of the frames 40 dB below the target's loudest, 512-point STFT, 15 one-third-octave bands,
 * 30-frame segment correlations; fewer than 30 frames left give 1e-5, as pystoi returns with a warning.  All arithmetic
 * is float64 with fixed reduction orders: a pair's result does not depend on its batch or position.  Every pair is checked
 * before any work is queued: each clip 1 .. 2^30 samples, and the padded pair more than 256 samples at 10 kHz (one STOI
 * frame; pystoi fails on fewer), else VF_EINVAL naming the pair.  The tables (31947 resampling taps and the rest, designed
 * in float64 on the host on first use) and the scratch are owned by the context and freed by vf_destroy; the scratch is
 * allocated stream-ordered.  Sub-batches as in vf_score_varlen (at most 128 pairs and 16384 * 441 padded samples; a
 * longer pair runs alone); eight launches per sub-batch.  Needs no weights.  PESQ is not computed. */
VF_API int vf_score_time_varlen(vf_ctx* ctx, const float* est, const int64_t* est_offsets, const float* target,
                                const int64_t* target_offsets, int batch, double* out, void* stream);

/* The three scoring calls above at the rate of a test set: `rate` 44100 is exactly the call without _ex; 16000 is
 * AudioMetrics' 16 kHz branch (metrics.py:43-46); any other rate is VF_EINVAL.  At 16 kHz:
 * - the spectrogram is np.abs(librosa.stft(wav, n_fft=743, hop_length=160)): reflect padding by 371, the float64 periodic
 *   hann of length 743, a direct float64 DFT of the prime length 743 (372 bins) rounded to complex64, |.| of that.  Clip i
 *   has T_i = 1 + (n_i - 1) / 160 frames and needs at least 372 samples (one reflection of the padding).  The mel is
 *   MelScale(n_mels=80, sample_rate=16000, n_stft=372), [sum T_i, 80]; it needs "metrics.mel_16k.fb" [372, 80] loaded
 *   (VF_ESTATE otherwise).
 * - vf_score_varlen_ex computes the same eight keys on the [T, 372] spectrogram and its [T, 80] mel; every pair needs equal
 *   frame counts and at least 7 frames (961 samples).
 * - vf_score_time_varlen_ex runs stoi(target, est, 16000): resample_oct(x, 10000, 16000) is resample_poly by 5 / 8 with
 *   Octave's 581-tap window (ceil(5 n / 8) samples); the rest is unchanged.  Sub-batches hold at most 16384 * 160 padded
 *   samples, the same 10 kHz scratch as at 44.1 kHz. */
VF_API int vf_metric_spectrogram_ex(vf_ctx* ctx, const float* wav, const int64_t* offsets, int batch, float* sp_out,
                                    float* mel_out, int rate, void* stream);
VF_API int vf_score_varlen_ex(vf_ctx* ctx, const float* est, const int64_t* est_offsets, const float* target,
                              const int64_t* target_offsets, int batch, double* out, int rate, void* stream);
VF_API int vf_score_time_varlen_ex(vf_ctx* ctx, const float* est, const int64_t* est_offsets, const float* target,
                                   const int64_t* target_offsets, int batch, double* out, int rate, void* stream);

/* scipy.signal.sosfiltfilt(sos, x) (padtype "odd", default padlen) of `batch` packed FLOAT64 rows, each with its own filter:
 * x and out are device float64, packed with HOST offsets [batch + 1]; row i uses filter row_filter[i] (host) of
 * `n_filters` second-order-section filters given on the HOST as sos [n_filters][10][6] and sosfilt_zi(sos)
 * [n_filters][10][2], filter f using its first n_sections[f] (1 .. 10) rows.  row_f32 (host, or NULL for none) marks rows
 * whose samples came from float32 input: numpy builds sosfiltfilt's odd extension in the input's dtype, so theirs is
 * rounded to float32 (the filtering itself is float64 either way, as in scipy).  Filter f's padlen is 3 * (2 n_sections + 1 -
 * min(#(sos[:, 2] == 0), #(sos[:, 5] == 0))); every row must be longer than its padlen, and sos[:, 3] must be 1, else
 * VF_EINVAL naming the row or filter before any work is queued.  float64 throughout: the odd extension is index math, each
 * pass (forward from zi * x_ext[0], backward from zi * y[-1]) is an exact chunked scan whose only error is fp64 rounding, in
 * scipy's per-sample section order.  A row's bits do not depend on its batch or position.  Each filter's table (sos, zi and
 * its 1024-step transition matrix) is designed on the device by one more launch per 6 filters, in the call's scratch: no
 * host synchronisation and nothing kept between calls.  The scratch is owned by the context and allocated stream-ordered.
 * Rows run in sub-batches of at most 64 rows and 2^24 extended samples (a longer row runs alone); six launches per
 * sub-batch. */
VF_API int vf_sosfiltfilt_varlen(vf_ctx* ctx, const double* x, const int64_t* offsets, int batch, const double* sos,
                                 const double* zi, const int* n_sections, int n_filters, const int* row_filter, const int* row_f32,
                                 double* out, void* stream);
/* scipy.signal.resample_poly(x, up, down) of `batch` packed FLOAT64 rows in float64: x packed with HOST in_offsets, y with HOST
 * out_offsets.  Row i uses filter row_filter[i] (host) of `n_filters`: up[f], down[f] >= 1 (already reduced by their gcd)
 * and the odd-length float64 taps taps[tap_offsets[f] .. tap_offsets[f + 1]) (device; host tap_offsets), firwin x up as
 * resample_poly designs them.  Row i writes out_offsets[i + 1] - out_offsets[i] samples: resample_poly's first
 * ceil(n up / down) and zeros past them, so an output length other than ceil(n up / down) is align_length's pad or cut.
 * No scratch; one launch per 64 rows. */
VF_API int vf_resample_poly_f64_varlen(vf_ctx* ctx, const double* x, const int64_t* in_offsets, int batch, const double* taps,
                                       const int64_t* tap_offsets, const int* up, const int* down, int n_filters,
                                       const int* row_filter, double* y, const int64_t* out_offsets, void* stream);
/* librosa 0.8 resample(x, orig_sr, target_sr, res_type, fix=True) for res_type kaiser_best / kaiser_fast (resampy's sinc
 * interpolation) of `batch` packed float32 rows: x packed with HOST in_offsets (every row at least 1 sample), y with HOST
 * out_offsets.  Row i uses filter row_filter[i] (host) of `n_filters`: its table is tables[2 table_offsets[f] .. 2
 * table_offsets[f + 1]) (device, 16-byte aligned; host table_offsets, in entries), nwin interleaved (win, delta) float64
 * pairs as resampy hands them to its loop (win already multiplied by sample_ratio when it is below 1, delta = diff(win)
 * with a last entry 0), for sample_ratio[f] = target_sr / orig_sr (host) and num_table[f] = 2^precision table entries per
 * zero crossing (host).  Row i writes out_offsets[i + 1] - out_offsets[i] samples: resampy's first int(n sample_ratio) (a
 * float64 product) and zeros past them, librosa's fix_length pad (a shorter output cuts).  The arithmetic is resampy's:
 * float64 time register t / sample_ratio, float64 weights and products without FMA contraction, the output rounded to
 * float32 after every tap.  A row's bits do not depend on its batch or position.  Every argument is checked before any work
 * is queued (VF_EINVAL): a sample_ratio that is not positive, num_table < 1, an index step int(min(1, ratio) num_table) of
 * 0, a table of at most num_table entries, a row filter out of range, a row whose int(n sample_ratio) is 0.  No scratch, no
 * host synchronisation; one launch per 512 rows. */
VF_API int vf_resample_sinc_varlen(vf_ctx* ctx, const float* x, const int64_t* in_offsets, int batch, const double* tables,
                                   const int64_t* table_offsets, const double* sample_ratio, const int* num_table, int n_filters,
                                   const int* row_filter, float* y, const int64_t* out_offsets, void* stream);
/* The VoiceFixer pip package's pre-filter, remove_higher_frequency(wav, ratio) (restore_inmem's mode 1), of `batch` packed
 * float32 rows: x packed with HOST in_offsets (every row 1 .. 2^30 samples), y with HOST out_offsets, row i holding 512 (n_i
 * // 512) samples (librosa 0.8's istft with length None; a row under 512 samples gives an empty output).  cutoff (device,
 * int32 [batch]) receives each row's first removed bin.  Per row, in float64: librosa 0.8's stft (n_fft 2048, hop 512,
 * periodic hann, reflect padding as np.pad makes it for any length), per-bin energies sum over frames of max(log10(|X| +
 * 1e-8), 0), the package's sequential scan for the first bin whose running sum reaches ratio times their total, the bins
 * below it scaled by |X| / (|X| + 1e-8) and the others zeroed, librosa's istft (overlap-add divided by the window sum of
 * squares where that exceeds float32 tiny); the output is rounded to float32 once.  Only bins with |X| >= 1 carry energy: a
 * quiet row has cutoff 0 and an all-zero output.  Where rounding makes the last running sum miss the threshold (the
 * package would raise IndexError) every bin is kept, cutoff 1025.  A row's bits do not depend on its batch, its position
 * or the sub-batching.  Every argument is checked before any work is queued (VF_EINVAL, naming the row): 0 < ratio <= 1,
 * the row lengths, out_offsets matching them.  A NaN or infinite sample raises the device flag (VF_EDEVICE at
 * vf_check_errors).  Sub-batches of at most 256 rows and 16384 frames (a longer row runs alone), four launches each, on a
 * context-owned scratch of 16.4 KB per frame, allocated stream-ordered; no host synchronisation, no weights needed.  The
 * scratch holds every frame of the largest sub-batch and is kept until vf_destroy: at most 269 MB for rows of up to 16384
 * frames (190 s), but a longer row runs alone with all its frames resident, about 5.1 GB per hour of audio (34 GB for a
 * 2^30-sample row); a call whose scratch cannot be allocated fails with VF_ECUDA before any kernel is queued.
 * Split long recordings into segments, as the package's 30 s segmentation does. */
VF_API int vf_remove_higher_frequency_varlen(vf_ctx* ctx, const float* x, const int64_t* in_offsets, int batch, double ratio,
                                             float* y, const int64_t* out_offsets, int* cutoff, void* stream);

/* librosa.load(path, sr=None, mono=True)'s samples of `n_rows` WAV data chunks (soundfile's float read, then librosa 0.8's
 * to_mono), decoded on the device.  bytes: one device buffer holding every row's data chunk.  rows: HOST table (read during
 * the call only); row i holds `frames` interleaved frames of `channels` (1 .. 64) samples of `format` from bytes +
 * byte_offset; the caller keeps every row inside the buffer.  byte_offset is a multiple of the sample width for u8, s16,
 * s32, f32 and f64 data (those are read with aligned loads); s24 frames may sit at any byte (byte loads).  Samples convert
 * as libsndfile's float read does: u8 (b - 128) / 128, s16 v 2^-15, s24 v 2^-23 (sign-extended), s32 float32(v) 2^-31
 * (rounded to nearest), f32 unchanged (NaN and Inf included), f64 rounded to float32.  mono_out (device, float32) receives
 * the rows packed back to back, row i at sum_{j<i} frames_j: the channel itself for one channel (librosa leaves a 1-D
 * signal alone), else numpy's float32 x.mean(axis=1) of the row's [frames, channels] samples, bit for bit: numpy's
 * add.reduce order over the frame's channels (sequential below 8, its eight running sums from 8 on, added to the
 * identity 0) and one float32 division by the channel count.  first_out (device, float64, packed the same; may be NULL)
 * receives channel 0 as soundfile reads it in float64, speechmetrics' input: the exact quotient for the integer formats,
 * the value itself for the float formats.  A row's bits do not depend on its batch, position or sub-batch.  Every
 * argument is checked before any work is queued (VF_EINVAL, naming the row).  One thread per output frame, one launch per
 * 1024 rows; no scratch, no host synchronisation. */
#define VF_PCM_U8 0
#define VF_PCM_S16 1
#define VF_PCM_S24 2
#define VF_PCM_S32 3
#define VF_PCM_F32 4
#define VF_PCM_F64 5
typedef struct vf_pcm_row {
  int64_t byte_offset;      /* of the row's first frame in `bytes` */
  int64_t frames;           /* >= 0 */
  int32_t channels;         /* 1 .. 64 */
  int32_t format;           /* VF_PCM_* */
} vf_pcm_row;
VF_API int vf_decode_pcm_varlen(vf_ctx* ctx, const void* bytes, int n_rows, const vf_pcm_row* rows, float* mono_out,
                                double* first_out, void* stream);

/* The FLAC audio (RFC 9639) of `n_rows` files, decoded as libsndfile's read of a FLAC file returns it, into the bytes of
 * a WAV data chunk holding the same samples: interleaved little-endian u8 (stored as v + 128), s16 or s24.  Those bytes
 * are what vf_decode_pcm_varlen converts, so a FLAC file's samples are the WAV path's bit for bit.  bytes: one device
 * buffer; rows: HOST table (read during the call only).  Row i's audio region (its frames, from the first frame's sync code
 * to the end of the file, as voicefixer_main_b200/flacfile.py finds it) is `nbytes` bytes at bytes + byte_offset, which is
 * a multiple of 8; the bytes up to the next multiple of 8 after the region must be readable.  Its STREAMINFO facts:
 * total_samples (> 0) per channel, channels (1 .. 8), bits (8, 16, 24), rate, the blocking strategy (`variable`: 0 fixed,
 * 1 variable) and first_block, the first frame's block size (the frame-number multiplier under fixed blocking).  Its
 * total_samples x channels x bits / 8 output bytes go to pcm + pcm_offset.  Every subframe type, wasted bits, the four
 * channel assignments, both Rice codings with escapes and partition orders 0 .. 15 are decoded.  status (device,
 * n_rows): all ones for a row that decoded, else (byte << 8) | VF_FLAC_E* of its first bad frame, `byte` counted from
 * the start of its region; the output of a row whose status is not all ones, and of the whole call, must not be used.
 * Every argument is checked before any work is queued (VF_EINVAL, naming the row).  Sub-batches of at most 512 rows and
 * 64 MiB of FLAC data (a larger file runs alone); per sub-batch, four kernel launches and a context-owned scratch of 4 bytes
 * per FLAC byte, 13 bytes per 8 FLAC bytes (frame candidates, each row with its own share) and 4 bytes per decoded sample.  One thread per FLAC byte
 * finds candidate frames (sync code, header, CRC-8, agreement with STREAMINFO), one per candidate walks its subframes to
 * its end and checks CRC-16, one per row chains the frames from the first (a header-shaped pattern inside a frame never
 * changes the result), then one per chained frame decodes it.  No host synchronisation. */
#define VF_FLAC_ENOSYNC 1      /* no frame sync code where a frame must start */
#define VF_FLAC_ERESERVED 2    /* a reserved or forbidden code in a frame header */
#define VF_FLAC_EMISMATCH 3    /* a frame header disagrees with STREAMINFO (channels, bit depth, rate, blocking) */
#define VF_FLAC_ECRC8 4        /* frame header CRC-8 mismatch */
#define VF_FLAC_ESUBFRAME 5    /* a reserved or forbidden subframe code (type, LPC precision, negative shift, coding) */
#define VF_FLAC_EPARTITION 6   /* invalid residual partitioning */
#define VF_FLAC_ETRUNCATED 7   /* a frame runs past the end of the data */
#define VF_FLAC_ECRC16 8       /* frame CRC-16 mismatch */
#define VF_FLAC_ERANGE 9       /* a decoded sample (or residual) outside its bit depth's range */
#define VF_FLAC_ESEQUENCE 10   /* a frame or sample number out of sequence, or a short fixed-blocking frame before the last */
#define VF_FLAC_ELENGTH 11     /* the frames' sample counts do not add up to STREAMINFO's total */
#define VF_FLAC_ECANDIDATES 12 /* more candidate frames in a row than one per 8 of its bytes */
typedef struct vf_flac_row {
  int64_t byte_offset;      /* of the row's first frame in `bytes`, a multiple of 8 */
  int64_t nbytes;           /* of its audio region, > 0 */
  int64_t total_samples;    /* per channel, > 0 */
  int64_t pcm_offset;       /* of its first output byte in `pcm` */
  int32_t channels;         /* 1 .. 8 */
  int32_t bits;             /* 8, 16, 24 */
  int32_t rate;             /* > 0 */
  int32_t variable;         /* 0: fixed blocking, 1: variable blocking */
  int32_t first_block;      /* 1 .. 65535 */
  int32_t pad_;
} vf_flac_row;
VF_API int vf_decode_flac_varlen(vf_ctx* ctx, const void* bytes, int n_rows, const vf_flac_row* rows, void* pcm,
                                 unsigned long long* status, void* stream);

/* Live streams resampled from device rings in one call (voicefixer_main_b200/streaming.py StreamingResampler, and the
 * restorers' streams at other rates).  in_ring [n_streams, in_len] (device) holds each stream's recent float32 samples at
 * its own rate: absolute input i of stream s is at in_ring[s * in_len + i mod in_len].  rows: HOST table of n_rows entries
 * (read during the call only).  Row r computes outputs m0 .. m1 - 1 of its stream's signal of n inputs (n =
 * VF_RESAMPLE_OPEN while the stream is open: no output is clamped to its end) with the arithmetic of a whole-signal call, so
 * each output is bit-identical to that output of vf_resample_poly (family VF_RESAMPLE_POLY: up, down and taps = the
 * 20 max(up, down) + 1 float32 taps of resample_poly's FIR, device) or of vf_resample_sinc_varlen (VF_RESAMPLE_SINC:
 * table = nwin (win, delta) float64 pairs, device, 16-byte aligned, for sample_ratio `ratio` and num_table entries per zero
 * crossing) on the whole signal; a closed sinc row's slots at or past int(n ratio) are zeros (librosa's fix_length).  Only
 * inputs below `avail` have been written, and the ring holds those from avail - in_len on.  The outputs go to row
 * out_stream of `out` as a ring of out_len positions (output m at out[out_stream * out_len + m mod out_len], n_out_streams
 * rows), or with out_stream = -1 to out[out_offset + m - m0] (packed).  Every argument is checked before any work is
 * queued (VF_EINVAL, naming the row): a stream or out_stream out of range, m0 < 0 or m1 < m0, an input window that reaches
 * past avail or below what the ring holds (a sinc row may read from max(0, int(m0 / ratio) - K + 1) on, K = nwin / step,
 * step = int(min(1, ratio) num_table)), a closed row's range past ceil(n up / down) or ceil(n ratio) outputs or with
 * int(n ratio) = 0, more outputs than out_len, an unknown family or a filter that does not match it (a poly row with no
 * taps or a table, a sinc row with no table, taps, a ratio that is not positive, num_table < 1, a step of 0 or a table of at
 * most num_table entries); the context stays usable.  Empty rows (m0 = m1) are checked and launch nothing.  One launch per
 * family present, per 256 rows of it, whatever the number of streams; no scratch, no host synchronisation. */
#define VF_RESAMPLE_POLY 0
#define VF_RESAMPLE_SINC 1
#define VF_RESAMPLE_OPEN INT64_MAX
typedef struct vf_resample_row {
  int32_t stream;           /* row of in_ring */
  int32_t family;           /* VF_RESAMPLE_POLY or VF_RESAMPLE_SINC */
  int64_t m0, m1;           /* absolute output range [m0, m1) */
  int64_t n;                /* the stream's input count once closed, VF_RESAMPLE_OPEN while open */
  int64_t avail;            /* inputs written to the ring so far (at most n) */
  int32_t up, down;         /* poly */
  const float* taps;        /* poly: device, NULL for sinc */
  const double* table;      /* sinc: device, NULL for poly */
  int64_t nwin;             /* sinc: table entries */
  double ratio;             /* sinc: target_sr / orig_sr */
  int32_t num_table;        /* sinc */
  int32_t out_stream;       /* row of the output ring, or -1: packed */
  int64_t out_offset;       /* packed: where output m0 goes */
} vf_resample_row;
VF_API int vf_resample_rings(vf_ctx* ctx, const float* in_ring, int n_streams, int64_t in_len, const vf_resample_row* rows,
                             int n_rows, float* out, int n_out_streams, int64_t out_len, void* stream);

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

/* Options: "vocoder_terms" (1 or 3 fp16 split terms), "unify_energy" (default flag of
 * vf_restore / vf_restore_host; prefer vf_restore_ex's per-call flag), "plan_cache_mb" (cap on the device memory
 * held by cached per-shape plans, least recently used evicted first; 0 = half of the free device memory),
 * "graphs" (default 1: the fixed-pointer launch chain of a plan is captured on its second use and replayed as one CUDA graph from then on),
 * "host_pipeline" (default 1, see vf_restore_host). */
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
 * cores actually executed for it (3 MMAs per product in 3-term mode, tile / phase padding), the tensor-core tile
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
enum { VF_LAYER_CONV2D = 0, VF_LAYER_CONVT2D = 1, VF_LAYER_CONV1D = 2, VF_LAYER_CONVT1D = 3, VF_LAYER_PAIR = 4,
       VF_LAYER_LINEAR = 5 };
enum { VF_RESID_NONE = 0, VF_RESID_FP32 = 1, VF_RESID_PLANES = 2, VF_RESID_AR = 3 };
typedef struct vf_layer_case {
  int kind, terms;          /* VF_LAYER_*, 1 or 3 */
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
  int resid_kind;           /* VF_RESID_*: FP32 [n_img][rows][cout] floats; PLANES / AR [2][n_img][rows][cout] fp16 */
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
  /* LINEAR: one nn.Linear of the bi_gru / dnn modules on L rows per image (x_row0 = 0, x_img_rows = L), packed and set up as
   * the loader and the plan builder do it: w [cout][cin], b [cout]; in_bn (or NULL) = (weight, bias, running_mean,
   * running_var) of a BatchNorm2d(1) applied to the input, folded into w and b.  With b_hh the layer is a GRU input
   * projection: w = W_ih [2][768][cin] and b = b_ih, b_hh [2][768] of both directions (cout = 1536, no in_bn). */
  const float* in_bn;
  const float* b_hh;
  /* reported: the launch configuration the builder chose */
  int bn, bk, stages, resid_tma, tma_out, grid;
  int64_t tiles;
  int div_fallback;         /* a tile decode divides (its multiply-high magic would not be exact) */
  char sig[160];            /* PRODUCT: the configuration signature of the launch (the one vf_selftest_plan_gemms reports) */
} vf_layer_case;
VF_API int vf_selftest_layer(vf_ctx* ctx, vf_layer_case* lc);

/* TEST ONLY.  Builds a plan of `plan_kind` (0 GSR, 1 SSR, 2 GSR varlen, 3 SSR varlen, 4 vocoder-only, 5 vocoder-only
 * varlen) for (batch, frames) with the loaded
 * weights and the context's options, launches nothing, and reports each GEMM and fused-pair launch: its label, the
 * configuration signature vf_selftest_layer reports for a layer, and the size of its persistent tile loop (tiles and grid,
 * as vf_selftest_layer reports them, and the column tiles among which a CTA's consecutive tiles move).  Records past `cap`
 * are dropped; *count = all of them. */
typedef struct vf_plan_gemm {
  char label[48];
  char sig[160];
  int64_t tiles;            /* output tiles of the launch */
  int grid;                 /* persistent CTAs: min(tiles, SMs) */
  int col_tiles;            /* column (N) tiles per row block: tiles of a CTA change column block unless it divides grid */
} vf_plan_gemm;
VF_API int vf_selftest_plan_gemms(vf_ctx* ctx, int plan_kind, int batch, int frames, vf_plan_gemm* records, int cap, int* count);
/* TEST ONLY.  The sub-batch a call of `batch` clips on plans of `plan_kind` (as vf_selftest_plan_gemms) with `frames` frames
 * would run in under the plan budget, as the context stands (cached plans refine the per-frame size); builds nothing. */
VF_API int vf_selftest_sub_batch(vf_ctx* ctx, int plan_kind, int batch, int frames);

/* TEST ONLY.  One non-GEMM op of the launch chains, set up by the same helpers the plan builders and restore paths use and
 * launched as they launch it (run_ops or the same launch_* call), then copied back.  Synchronous; every pointer is a host
 * pointer, and output buffers are read AND written as in vf_selftest_layer.  fp16 planes are bit patterns [2][batch][rows][C].
 * Fields a kind does not use are zero.  The mel-weight table, window and twiddles are the context's own. */
enum { VF_OP_FIRST = 0, VF_OP_POOL = 1, VF_OP_COND = 2, VF_OP_REFLECT = 3, VF_OP_TAIL = 4, VF_OP_FINALIZE = 5, VF_OP_ISTFT = 6,
       VF_OP_PEAK_NORM = 7, VF_OP_FRONTEND = 8, VF_OP_PLANES = 9 };
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
  /* FRONTEND (n; the mel filterbank must be loaded): the front end as every restore runs it, on in_wav [batch][n] with the
   * outputs that are not NULL: mel_out / logmel_out [batch][T][128], sp_out / cos_out / sin_out [batch][T][1025] (cos and
   * sin together, and only with sp).  Uniform: T = 1 + n / hop is reported back.  With clip_off: in_wav packed, n = the
   * longest clip, T = the caller's rows per clip (the varlen plans' bucket; a clip with more frames, or with 1024 samples
   * or fewer, fails with VF_EINVAL); rows t >= T_b of clip b are not written. */
  float* mel_out;
  float* logmel_out;
  float* sp_out;
  float* cos_out;
  float* sin_out;
  /* PLANES (T): the bi_gru / dnn input planes of x [batch][T][128] floats, fma(x, bn1_scale, bn1_shift) split hi/lo into planes
   * [2][batch][T][128]; with clip_off, rows t >= the clip's frames are zeros */
} vf_op_case;
VF_API int vf_selftest_op(vf_ctx* ctx, vf_op_case* oc);

/* Test hook (tests only): one bidirectional GRU layer of the bi_gru analysis module (hidden size 256), launched as the plans
 * launch it, synchronously.  All buffers are host memory.  G [batch, T, 1536] fp32 is x W_ih^T + b_ih + (b_hr, b_hz, 0) of
 * both directions (forward gates r, z, n in columns 0..767, reverse in 768..1535); w_hh [2][768][256] and b_hn [2][256] are
 * per direction.  lengths [batch] (or null: T each) are the clips' frames, each in 1..T: the reverse direction of clip b
 * starts at its frame lengths[b] - 1.  out [2][batch][T][512] fp16 bits is in/out: the hi plane, then the lo plane, of
 * relu ? relu(h) : h with the forward direction at channels 0..255 and the reverse at 256..511, zeros at frames past a
 * clip's end; the device copy starts as the caller's buffer. */
typedef struct vf_gru_case {
  int batch, T;
  const float* G;
  const float* w_hh;
  const float* b_hn;
  const int* lengths;
  int relu;
  uint16_t* out;
} vf_gru_case;
VF_API int vf_selftest_gru(vf_ctx* ctx, vf_gru_case* gc);

/* TEST ONLY.  One restore on a plan of `plan_kind` (0 GSR, 1 SSR, 2 GSR varlen, 3 SSR varlen, 4 / 5 vocoder-only as
 * vf_resynth / vf_resynth_varlen) built for this call with the
 * loaded weights and the context's options, run as the restore entry points run it (front end, lengths table, the UNet's
 * launches, the band sums of VF_RESTORE_UNIFY_ENERGY, the vocoder's, then the finalize or the ISTFT) but eagerly, one
 * launch at a time, synchronising around each traced step.  The traced steps are the launches of the UNet and vocoder
 * lists and the finalize; with VF_TRACE_DIRECT_STEPS also the launches the restore makes itself (list 3: the front end,
 * the band sums, the ISTFT), so that only the lengths table of a varlen plan is written untraced, ahead of the first
 * step.  wav and wav_out are device buffers as vf_restore (offsets NULL: batch clips of n samples) or vf_restore_varlen
 * (offsets [batch + 1], host; n is ignored) take them; flags are vf_restore_ex's (GSR plans only) and
 * VF_TRACE_DIRECT_STEPS (any plan).  Synchronous; the plan is freed on return and the plan cache is not touched.
 *
 * fn(user, after, op) runs before (after = 0) and after (after = 1) each traced step; a nonzero return stops the run
 * (VF_EINVAL).  op describes the step as the builder set it up, with DEVICE pointers: a GEMM or a fused pair (kind 0 / 8)
 * in vf_layer_case's terms (layer; x / sc_x / resid / out_* / head_* / a_scale / a_shift point at the plan's buffers, fp16
 * planes [2][n_img][img_rows][C] with the lo plane right after the hi plane; sig: the signature vf_selftest_plan_gemms
 * reports), a GRU layer in vf_trace_gru's (gru), the other kinds in vf_op_case's (op).
 * row_valid / head_valid / gru.lengths and vl_rows are HOST pointers into a copy of the plan's lengths table [18][batch]
 * (NULL: uniform).  out_ptr / out_bytes are the byte ranges the step may write (the ISTFT's and the finalize's output is
 * the caller's wav_out, outside the plan); allocs are every device buffer of the plan.  launches (valid when after = 1) is
 * what the step added to vf_launch_count. */
enum { VF_TRACE_GEMM = 0, VF_TRACE_FIRST = 1, VF_TRACE_POOL = 2, VF_TRACE_COND = 3, VF_TRACE_REFLECT = 4, VF_TRACE_TAIL = 5,
       VF_TRACE_FINALIZE = 6, VF_TRACE_MEMSET = 7, VF_TRACE_PAIR = 8, VF_TRACE_PLANES = 9, VF_TRACE_GRU = 10,
       VF_TRACE_FRONTEND = 11, VF_TRACE_BAND = 12, VF_TRACE_ISTFT = 13 };
/* One bidirectional GRU layer of a bi_gru plan, as vf_gru_case describes it, with each direction's weights where the loader
 * put them: G [batch][T][1536] fp32; w_hh[d] [768][256] and b_hn[d] [256] fp32; out planes [2][batch][T][512] */
typedef struct vf_trace_gru {
  int batch, T, relu;
  const float* G;
  const float* w_hh[2];
  const float* b_hn[2];
  const int* lengths;       /* host: the lengths table's frames row, or NULL (T each) */
  uint16_t* out;
} vf_trace_gru;
typedef struct vf_trace_op {
  int list, index, kind;    /* list 0: the analysis module's launches, 1: the vocoder's, 2: the finalize, 3: the steps the
                               restore launches itself (front end, band sums, ISTFT); kind: VF_TRACE_* */
  char label[48];
  vf_layer_case layer;      /* GEMM / PAIR (the pair: x = the (a, r) planes it reads, out_a = the planes it writes) */
  vf_op_case op;            /* FIRST, POOL, COND (mel_target, band_sums: the unify inputs and sums, else NULL), REFLECT,
                               TAIL, FINALIZE; MEMSET: planes = the cleared buffer, n = its bytes; PLANES (x, planes, T,
                               bn1_scale / bn1_shift); FRONTEND (in_wav, n, T, the outputs it writes; clip_off: the host
                               offsets of a varlen call); BAND: the memset and band_energy of unify_energy, in COND's unify
                               fields (mel: the restored log-mel, mel_target, band_sums, T); ISTFT: the frames and
                               overlap-add launches (mag, in_wav, frames, out, n, T, clip_off) */
  const int* vl_rows;       /* [18][batch] host, or NULL */
  int n_out;
  uint64_t out_ptr[4], out_bytes[4];
  int n_allocs;
  const uint64_t* alloc_ptr;
  const uint64_t* alloc_bytes;
  vf_trace_gru gru;         /* GRU */
  int launches;
} vf_trace_op;
typedef int (*vf_trace_fn)(void* user, int after, const vf_trace_op* op);
#define VF_TRACE_DIRECT_STEPS 0x100u   /* vf_selftest_plan_trace: trace the front end, band sums and ISTFT as list 3 */
VF_API int vf_selftest_plan_trace(vf_ctx* ctx, int plan_kind, const float* wav, const int64_t* offsets, int batch, int64_t n,
                                  unsigned flags, float* wav_out, vf_trace_fn fn, void* user);

#ifdef __cplusplus
}
#endif
#endif /* B200VF_H_ */
