"""ctypes binding of libb200vf.so (C ABI in include/b200vf.h).

There is no fallback: if the shared library has not been built (python __graft_entry__.py build, or
make -C voicefixer_main_b200/csrc) importing the engine raises, and without a CUDA device vf_create fails
with VF_ENODEVICE.  Nothing here computes on the data path; it only marshals pointers.
"""
import ctypes
import os
from ctypes import (POINTER, Structure, byref, c_char, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_size_t, c_uint, c_uint64, c_void_p)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200vf.so")

VF_OK, VF_EINVAL, VF_ENODEVICE, VF_ECUDA, VF_ESTATE, VF_EDEVICE, VF_EASSERT = 0, -1, -2, -3, -4, -5, -6

EXPORTS = [
    "vf_default_config", "vf_create", "vf_destroy", "vf_last_error", "vf_load_weights", "vf_frontend",
    "vf_unet_mel", "vf_vocoder", "vf_vocoder_out_len", "vf_restore", "vf_restore_host", "vf_restore_stages",
    "vf_to_log", "vf_from_log", "vf_to_pcm16", "vf_workspace_bytes", "vf_check_errors", "vf_set_option", "vf_launch_count",
    "vf_enable_stage_timing", "vf_stage_times", "vf_selftest_layer", "vf_enable_op_timing", "vf_op_count", "vf_op_info",
    "vf_restore_ex", "vf_ssr_forward", "vf_ssr_restore", "vf_ssr_restore_host", "vf_ssr_unet", "vf_ssr_stages", "vf_istft",
    "vf_mel", "vf_finalize", "vf_plan_cache_info", "vf_resample_poly", "vf_lsd", "vf_sispec", "vf_to_pcm16_ex", "vf_amp_to_original_f",
    "vf_restore_varlen", "vf_ssr_restore_varlen", "vf_restore_varlen_mels", "vf_metric_spectrogram", "vf_ssim", "vf_score_varlen",
    "vf_ssr_restore_varlen_mels", "vf_selftest_op", "vf_selftest_gru", "vf_score_time_varlen",
    "vf_sosfiltfilt_varlen", "vf_resample_poly_f64_varlen", "vf_metric_spectrogram_ex", "vf_score_varlen_ex",
    "vf_score_time_varlen_ex", "vf_restore_chunks", "vf_ssr_restore_chunks", "vf_restore_windows", "vf_ssr_restore_windows",
    "vf_selftest_plan_gemms", "vf_resample_sinc_varlen", "vf_selftest_plan_trace", "vf_vocoder_varlen", "vf_resynth",
    "vf_resynth_varlen", "vf_selftest_sub_batch", "vf_vocoder_chunks", "vf_resample_rings",
    "vf_remove_higher_frequency_varlen", "vf_decode_pcm_varlen", "vf_decode_flac_varlen",
]
VF_RESTORE_UNIFY_ENERGY = 1
VF_TRACE_DIRECT_STEPS = 0x100
VF_SSR_PEAK_NORMALISE = 1
VF_RESAMPLE_POLY, VF_RESAMPLE_SINC = 0, 1
VF_RESAMPLE_OPEN = (1 << 63) - 1


class VfConfig(Structure):
    _fields_ = [("sample_rate", c_int), ("n_fft", c_int), ("hop", c_int), ("n_mels", c_int),
                ("voc_cond_channels", c_int), ("voc_cond_layers", c_int), ("voc_channels", c_int),
                ("voc_num_stages", c_int), ("voc_scales", c_int * 8), ("voc_depth", c_int * 8),
                ("voc_stage_slope", c_float), ("voc_res_slope", c_float), ("voc_min_db", c_float),
                ("voc_ref_db", c_float), ("voc_amp_floor", c_float), ("voc_tail_value", c_float),
                ("voc_tail_base", c_int), ("voc_mel_weight_a", c_double), ("voc_mel_weight_b", c_double),
                ("voc_tail_tanh", c_int)]


class VfTensorDesc(Structure):
    _fields_ = [("name", c_char_p), ("data", c_void_p), ("ndim", c_int), ("shape", c_int64 * 4),
                ("on_device", c_int)]


class VfLayerCase(Structure):
    """vf_layer_case (include/b200vf.h): one conv layer for vf_selftest_layer (tests only)."""
    _fields_ = [(f, c_int) for f in ("kind", "terms", "n_img", "H", "W", "L", "cin", "cout", "sc_cin", "k", "dilation",
                                      "centered", "stride", "both")] + \
               [(f, c_void_p) for f in ("w", "b", "sc_w", "sc_b", "w2", "b2", "x")] + \
               [("x_img_rows", c_int), ("x_row0", c_int), ("sc_x", c_void_p), ("resid_kind", c_int), ("resid", c_void_p),
                ("ar_slope", c_float), ("out_raw", c_void_p), ("raw_ld", c_int), ("out_r", c_void_p), ("r_ld", c_int),
                ("r_c_off", c_int), ("out_a", c_void_p), ("a_ld", c_int), ("a_c_off", c_int), ("out_ar", c_int),
                ("a_scale", c_void_p), ("a_shift", c_void_p), ("act", c_int), ("slope", c_float), ("out_row0", c_int),
                ("out_img_rows", c_int), ("head_w", c_void_p), ("head_b", c_float), ("head_in", c_void_p),
                ("head_out", c_void_p), ("head_T", c_int), ("row_valid", c_void_p), ("head_valid", c_void_p),
                ("pair_slope_h", c_float), ("pair_slope_out", c_float), ("pair_last", c_int), ("in_bn", c_void_p),
                ("b_hh", c_void_p)] + \
               [(f, c_int) for f in ("bn", "bk", "stages", "resid_tma", "tma_out", "grid")] + \
               [("tiles", c_int64), ("div_fallback", c_int), ("sig", c_char * 160)]


class VfOpCase(Structure):
    """vf_op_case (include/b200vf.h): one non-GEMM op for vf_selftest_op (tests only)."""
    _fields_ = [("kind", c_int), ("batch", c_int), ("clip_off", c_void_p), ("unet_w0", c_int), ("vl_rows", c_void_p),
                ("T", c_int), ("W", c_int), ("bn1_scale", c_float), ("bn1_shift", c_float)] + \
               [(f, c_void_p) for f in ("x", "w1", "bn2_scale", "bn2_shift", "w_sc", "b_sc", "a2", "sc_raw")] + \
               [("H", c_int), ("C", c_int), ("level", c_int)] + \
               [(f, c_void_p) for f in ("pin", "a_scale", "a_shift", "out_r", "out_a", "out_raw")] + \
               [("is_log", c_int), ("unify", c_int)] + \
               [(f, c_void_p) for f in ("mel", "mel_target", "band_sums", "cond")] + \
               [("L", c_int64), ("cond_pad", c_int), ("terms", c_int), ("tanh_out", c_int), ("planes", c_void_p),
                ("tail_in", c_void_p), ("tail_w", c_void_p), ("tail_b", c_float), ("wav", c_void_p), ("peak_bits", c_void_p),
                ("n", c_int64)] + \
               [(f, c_void_p) for f in ("in_wav", "mag", "frames", "out")] + \
               [("Tp", c_int), ("Wpo", c_int), ("Tv", c_int), ("skip", c_int64), ("tail_smem", c_int64)] + \
               [(f, c_void_p) for f in ("mel_out", "logmel_out", "sp_out", "cos_out", "sin_out")]     # VF_OP_FRONTEND


class VfPlanGemm(Structure):
    """vf_plan_gemm (include/b200vf.h): one GEMM / fused-pair launch of a plan for vf_selftest_plan_gemms (tests only)."""
    _fields_ = [("label", c_char * 48), ("sig", c_char * 160), ("tiles", c_int64), ("grid", c_int), ("col_tiles", c_int)]


class VfTraceGru(Structure):
    """vf_trace_gru (include/b200vf.h): one GRU layer of a traced bi_gru plan (tests only)."""
    _fields_ = [("batch", c_int), ("T", c_int), ("relu", c_int), ("G", c_void_p), ("w_hh", c_void_p * 2),
                ("b_hn", c_void_p * 2), ("lengths", c_void_p), ("out", c_void_p)]


class VfTraceOp(Structure):
    """vf_trace_op (include/b200vf.h): one step of a plan as vf_selftest_plan_trace describes it (tests only)."""
    _fields_ = [("list", c_int), ("index", c_int), ("kind", c_int), ("label", c_char * 48), ("layer", VfLayerCase),
                ("op", VfOpCase), ("vl_rows", c_void_p), ("n_out", c_int), ("out_ptr", c_uint64 * 4),
                ("out_bytes", c_uint64 * 4), ("n_allocs", c_int), ("alloc_ptr", POINTER(c_uint64)),
                ("alloc_bytes", POINTER(c_uint64)), ("gru", VfTraceGru), ("launches", c_int)]


VF_TRACE_FN = ctypes.CFUNCTYPE(c_int, c_void_p, c_int, POINTER(VfTraceOp))


class VfGruCase(Structure):
    """vf_gru_case (include/b200vf.h): one bidirectional GRU layer for vf_selftest_gru (tests only)."""
    _fields_ = [("batch", c_int), ("T", c_int), ("G", c_void_p), ("w_hh", c_void_p), ("b_hn", c_void_p), ("lengths", c_void_p),
                ("relu", c_int), ("out", c_void_p)]


class VfChunk(Structure):
    """vf_chunk (include/b200vf.h): one chunk of a vf_restore_chunks call (of a vf_vocoder_chunks call: start, length and
    valid in frames, the crops in output samples)."""
    _fields_ = [("stream", c_int32), ("length", c_int32), ("crop_left", c_int32), ("crop_right", c_int32),
                ("start", c_int64), ("valid", c_int64)]


class VfWindow(Structure):
    """vf_window (include/b200vf.h): one window of a vf_restore_windows call."""
    _fields_ = [("stream", c_int32), ("start", c_int64), ("valid", c_int64)]


class VfEmit(Structure):
    """vf_emit (include/b200vf.h): one stream's emission range of a vf_restore_windows call."""
    _fields_ = [("stream", c_int32), ("start", c_int64), ("count", c_int64)]


class VfResampleRow(Structure):
    """vf_resample_row (include/b200vf.h): one stream's output range of a vf_resample_rings call."""
    _fields_ = [("stream", c_int32), ("family", c_int32), ("m0", c_int64), ("m1", c_int64), ("n", c_int64), ("avail", c_int64),
                ("up", c_int32), ("down", c_int32), ("taps", c_void_p), ("table", c_void_p), ("nwin", c_int64),
                ("ratio", c_double), ("num_table", c_int32), ("out_stream", c_int32), ("out_offset", c_int64)]


class VfPcmRow(Structure):
    """vf_pcm_row (include/b200vf.h): one WAV data chunk of a vf_decode_pcm_varlen call."""
    _fields_ = [("byte_offset", c_int64), ("frames", c_int64), ("channels", c_int32), ("format", c_int32)]


class VfFlacRow(Structure):
    """vf_flac_row (include/b200vf.h): one FLAC file's audio region of a vf_decode_flac_varlen call."""
    _fields_ = [("byte_offset", c_int64), ("nbytes", c_int64), ("total_samples", c_int64), ("pcm_offset", c_int64),
                ("channels", c_int32), ("bits", c_int32), ("rate", c_int32), ("variable", c_int32), ("first_block", c_int32),
                ("pad_", c_int32)]


class EngineError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libb200vf error {code}: {msg}")
        self.code = code


_lib = None


def load_library():
    """Load libb200vf.so or raise: the product has no CPU / PyTorch fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build the CUDA extension first "
            "(python -c 'import __graft_entry__ as g; g.build()' or make -C voicefixer_main_b200/csrc). "
            "voicefixer_main_b200 has no CPU fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    P = c_void_p
    lib.vf_default_config.argtypes = [POINTER(VfConfig)]
    lib.vf_default_config.restype = None
    lib.vf_create.argtypes = [POINTER(P), c_int, POINTER(VfConfig)]
    lib.vf_destroy.argtypes = [P]
    lib.vf_destroy.restype = None
    lib.vf_last_error.argtypes = [P]
    lib.vf_last_error.restype = c_char_p
    lib.vf_load_weights.argtypes = [P, POINTER(VfTensorDesc), c_int]
    lib.vf_frontend.argtypes = [P, P, c_int, c_int64, P, P, P, P, P]
    lib.vf_unet_mel.argtypes = [P, P, c_int, c_int, P, P]
    lib.vf_vocoder.argtypes = [P, P, c_int, c_int, P, P]
    lib.vf_vocoder_out_len.argtypes = [P, c_int]
    lib.vf_vocoder_out_len.restype = c_int64
    lib.vf_vocoder_varlen.argtypes = [P, P, POINTER(c_int64), c_int, P, P]
    lib.vf_resynth.argtypes = [P, P, c_int, c_int64, P, P]
    lib.vf_resynth_varlen.argtypes = [P, P, POINTER(c_int64), c_int, P, P]
    lib.vf_selftest_sub_batch.argtypes = [P, c_int, c_int, c_int]
    lib.vf_restore.argtypes = [P, P, c_int, c_int64, P, P]
    lib.vf_restore_host.argtypes = [P, P, c_int, c_int64, P, P]
    lib.vf_restore_stages.argtypes = [P, c_int, c_int64, P, P, P]
    lib.vf_to_log.argtypes = [P, P, P, c_int64, P]
    lib.vf_from_log.argtypes = [P, P, P, c_int64, P]
    lib.vf_to_pcm16.argtypes = [P, P, P, c_int64, P]
    lib.vf_workspace_bytes.argtypes = [P, c_int, c_int64, POINTER(c_size_t)]
    lib.vf_check_errors.argtypes = [P, P]
    lib.vf_set_option.argtypes = [P, c_char_p, c_int]
    lib.vf_launch_count.argtypes = [P]
    lib.vf_launch_count.restype = c_int64
    lib.vf_enable_stage_timing.argtypes = [P, c_int]
    lib.vf_stage_times.argtypes = [P, POINTER(c_float * 4)]
    lib.vf_selftest_layer.argtypes = [P, POINTER(VfLayerCase)]
    lib.vf_selftest_op.argtypes = [P, POINTER(VfOpCase)]
    lib.vf_selftest_gru.argtypes = [P, POINTER(VfGruCase)]
    lib.vf_selftest_plan_gemms.argtypes = [P, c_int, c_int, c_int, POINTER(VfPlanGemm), c_int, POINTER(c_int)]
    lib.vf_selftest_plan_trace.argtypes = [P, c_int, P, POINTER(c_int64), c_int, c_int64, c_uint, P, VF_TRACE_FN, P]
    lib.vf_enable_op_timing.argtypes = [P, c_int]
    lib.vf_op_count.argtypes = [P]
    lib.vf_op_info.argtypes = [P, c_int, POINTER(c_float), POINTER(c_double), POINTER(c_double), POINTER(c_int),
                               POINTER(c_int), POINTER(c_int), c_char_p, c_int, POINTER(c_double)]
    lib.vf_restore_ex.argtypes = [P, P, c_int, c_int64, P, c_uint, P]
    lib.vf_restore_varlen.argtypes = [P, P, POINTER(c_int64), c_int, P, c_uint, P]
    lib.vf_restore_chunks.argtypes = [P, P, c_int, c_int64, POINTER(VfChunk), c_int, P, c_uint, P]
    lib.vf_vocoder_chunks.argtypes = [P, P, c_int, c_int64, POINTER(VfChunk), c_int, P, P]
    lib.vf_restore_varlen_mels.argtypes = [P, P, POINTER(c_int64), c_int, P, c_uint, P, P, P]
    lib.vf_ssr_forward.argtypes = [P, P, P, c_int, c_int64, P, P]
    lib.vf_ssr_restore.argtypes = [P, P, c_int, c_int64, P, P]
    lib.vf_ssr_restore_host.argtypes = [P, P, c_int, c_int64, P, P]
    lib.vf_ssr_restore_varlen.argtypes = [P, P, POINTER(c_int64), c_int, P, P]
    lib.vf_ssr_restore_varlen_mels.argtypes = [P, P, POINTER(c_int64), c_int, P, c_uint, P, P]
    lib.vf_ssr_restore_chunks.argtypes = [P, P, c_int, c_int64, POINTER(VfChunk), c_int, P, P]
    lib.vf_restore_windows.argtypes = [P, P, c_int, c_int64, POINTER(VfWindow), c_int, c_int, P, P, c_int64, POINTER(VfEmit),
                                       c_int, P, c_uint, P]
    lib.vf_ssr_restore_windows.argtypes = [P, P, c_int, c_int64, POINTER(VfWindow), c_int, c_int, P, P, c_int64,
                                           POINTER(VfEmit), c_int, P, P]
    lib.vf_ssr_unet.argtypes = [P, P, c_int, c_int, P, P]
    lib.vf_ssr_stages.argtypes = [P, c_int, c_int64, P, P, P]
    lib.vf_istft.argtypes = [P, P, P, c_int, c_int, c_int64, P, P]
    lib.vf_mel.argtypes = [P, P, c_int64, c_int64, c_int64, c_int64, c_int64, P, P]
    lib.vf_finalize.argtypes = [P, P, c_int, c_int64, c_int64, P, P]
    lib.vf_plan_cache_info.argtypes = [P, POINTER(c_int), POINTER(c_size_t), POINTER(c_size_t), POINTER(c_int64)]
    lib.vf_resample_poly.argtypes = [P, P, c_int, c_int64, c_int, c_int, P, c_int, P, c_int64, P]
    lib.vf_to_pcm16_ex.argtypes = [P, P, P, c_int64, c_int, P]
    lib.vf_amp_to_original_f.argtypes = [P, P, P, c_int, c_int, P, P]
    lib.vf_lsd.argtypes = [P, P, P, c_int, c_int, c_int, P, P]
    lib.vf_sispec.argtypes = [P, P, P, c_int, c_int64, c_int, c_int, P, P]
    lib.vf_metric_spectrogram.argtypes = [P, P, POINTER(c_int64), c_int, P, P, P]
    lib.vf_ssim.argtypes = [P, P, P, c_int, c_int, c_int, P, P]
    lib.vf_score_varlen.argtypes = [P, P, POINTER(c_int64), P, POINTER(c_int64), c_int, P, P]
    lib.vf_score_time_varlen.argtypes = [P, P, POINTER(c_int64), P, POINTER(c_int64), c_int, P, P]
    lib.vf_metric_spectrogram_ex.argtypes = [P, P, POINTER(c_int64), c_int, P, P, c_int, P]
    lib.vf_score_varlen_ex.argtypes = [P, P, POINTER(c_int64), P, POINTER(c_int64), c_int, P, c_int, P]
    lib.vf_score_time_varlen_ex.argtypes = [P, P, POINTER(c_int64), P, POINTER(c_int64), c_int, P, c_int, P]
    lib.vf_sosfiltfilt_varlen.argtypes = [P, P, POINTER(c_int64), c_int, POINTER(c_double), POINTER(c_double), POINTER(c_int),
                                          c_int, POINTER(c_int), POINTER(c_int), P, P]
    lib.vf_resample_poly_f64_varlen.argtypes = [P, P, POINTER(c_int64), c_int, P, POINTER(c_int64), POINTER(c_int),
                                                POINTER(c_int), c_int, POINTER(c_int), P, POINTER(c_int64), P]
    lib.vf_resample_sinc_varlen.argtypes = [P, P, POINTER(c_int64), c_int, P, POINTER(c_int64), POINTER(c_double),
                                            POINTER(c_int), c_int, POINTER(c_int), P, POINTER(c_int64), P]
    lib.vf_resample_rings.argtypes = [P, P, c_int, c_int64, POINTER(VfResampleRow), c_int, P, c_int, c_int64, P]
    lib.vf_remove_higher_frequency_varlen.argtypes = [P, P, POINTER(c_int64), c_int, c_double, P, POINTER(c_int64), P, P]
    lib.vf_decode_pcm_varlen.argtypes = [P, P, c_int, POINTER(VfPcmRow), P, P, P]
    lib.vf_decode_flac_varlen.argtypes = [P, P, c_int, POINTER(VfFlacRow), P, P, P]
    _lib = lib
    return lib


def check(lib, ctx, rc):
    if rc != VF_OK:
        msg = lib.vf_last_error(ctx)
        raise EngineError(rc, msg.decode() if msg else "")
    return rc
