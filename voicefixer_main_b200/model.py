"""Host-side mirror of the reference's model objects for the inference hot path.

Same names, arguments and error behaviour as the objects eval_gsr_voicefixer.py:handler() uses
(SURVEY.md 8(b)), backed entirely by libb200vf.so:

    VoiceFixer(hp, channels, type_target)       models/gsr_voicefixer.py:94
      .load_from_checkpoint(ckpt) / .load_state_dict(sd) / .eval() / .to(device)
      .pre(wav[B,1,N]) -> (sp, mel_orig)         models/gsr_voicefixer.py:178-181
      .forward(mel_orig) -> {'mel': log10 mel}   models/gsr_voicefixer.py:183-193
      .f_helper.wav_to_spectrogram_phase(x)      tools/pytorch/modules/fDomainHelper.py:67-89
      .mel(specgram[..., freq, time])            tools/pytorch/mel_scale.py:52-64
      .vocoder(mel[B,1,T,128]) -> wav[B,1,L]     eval_gsr_voicefixer.py:66
    plus the batched fused entry points the reference lacks:
      .restore(wav[B,N]) -> wav[B,N]             one launch chain for stages A -> B -> C + normalise + trim
      .restore_host(pinned_in, pinned_out)
      .restore_batch([wav_i]) -> [out_i]         clips of different lengths in one launch chain
    SSR_UNet / GSR_UNet (models/ssr_unet.py) have .restore(wav[B,N]), .restore_host and .restore_batch([wav_i]) the same way.

PyTorch is used only to own device memory and streams; every tensor handed back is written by a
hand-written sm_90a kernel.  Tensors must be fp32 CUDA tensors on the model's device.
"""
import ctypes
import itertools
import json
import math
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib as L
from .arch import (SSR_PREFIX, UNET_PREFIX, VocoderConfig, bigru_keys, dnn_keys, frames_for, metric_frames, unet_keys,
                   vocoder_keys, vocoder_out_len)


class HParams(dict):
    """Nested config mapping with attribute access.  Any mapping subscriptable by the reference's string keys works as
    `hp` (the reference's own tools/utils.py HParams included); this is only the default container."""

    def __init__(self, **kw):
        super().__init__({k: HParams(**v) if isinstance(v, dict) else v for k, v in kw.items()})

    __getattr__ = dict.__getitem__


def get_hparams_from_file(config_path) -> HParams:
    """tools/utils.py:114-120."""
    with open(config_path, "r") as f:
        return HParams(**json.loads(f.read()))


def default_hparams() -> HParams:
    """The hot-path-relevant keys of config/vctk_base_voicefixer_unet.json."""
    return HParams(**{
        "task": {"gsr": {"gsr_model": {"voicefixer": {"unet": True, "unet_small": False, "bi_gru": False, "dnn": False}}}},
        "data": {"sampling_rate": 44100},
        "model": {"mel_freq_bins": 128, "window_size": 2048, "hop_size": 441, "pad_mode": "reflect",
                  "window": "hann", "channels_in": 1},
    })


def melscale_fbanks(n_freqs=1025, f_min=0.0, f_max=22050.0, n_mels=128, sample_rate=44100):
    """HTK triangular filterbank, same fp32 op order as tools/pytorch/mel_scale.py:131-221 (norm=None)."""
    all_freqs = torch.linspace(0, sample_rate // 2, n_freqs)
    m_min = 2595.0 * math.log10(1.0 + (f_min / 700.0))
    m_max = 2595.0 * math.log10(1.0 + (f_max / 700.0))
    m_pts = torch.linspace(m_min, m_max, n_mels + 2)
    f_pts = 700.0 * (10.0 ** (m_pts / 2595.0) - 1.0)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts.unsqueeze(0) - all_freqs.unsqueeze(1)
    down_slopes = (-1.0 * slopes[:, :-2]) / f_diff[:-1]
    up_slopes = slopes[:, 2:] / f_diff[1:]
    return torch.max(torch.zeros(1), torch.min(down_slopes, up_slopes))


def mel16k_fbanks():
    """AudioMetrics' mel_16k filterbank: MelScale(n_mels=80, sample_rate=16000, n_stft=372).fb, [372, 80]."""
    return melscale_fbanks(372, 0.0, 8000.0, 80, 16000)


def _ptr(t: Optional[torch.Tensor]):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _offsets(lengths):
    """Host int64 offsets of a packed set: 0, then the running sum of `lengths`."""
    return (ctypes.c_int64 * (len(lengths) + 1))(0, *itertools.accumulate(lengths))


def _check_in(t: torch.Tensor, device, what: str):
    if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or not t.is_cuda or t.device != device:
        raise TypeError(f"{what} must be a float32 CUDA tensor on {device}")
    return t.contiguous()


class Engine:
    """One vf_ctx on one device."""

    def __init__(self, device, cfg: Optional[VocoderConfig] = None):
        self.lib = L.load_library()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("voicefixer_main_b200 runs on CUDA devices only (no CPU fallback)")
        self.index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.device = torch.device("cuda", self.index)
        self.voc_cfg = cfg or VocoderConfig()
        c = L.VfConfig()
        self.lib.vf_default_config(ctypes.byref(c))
        v = self.voc_cfg
        c.voc_cond_channels, c.voc_cond_layers, c.voc_channels = v.cond_channels, v.cond_layers, v.channels
        c.voc_num_stages = len(v.upsample_scales)
        for i, (s, d) in enumerate(zip(v.upsample_scales, v.resstack_depth)):
            c.voc_scales[i], c.voc_depth[i] = s, d
        c.voc_stage_slope, c.voc_res_slope, c.voc_min_db, c.voc_ref_db = v.stage_slope, v.res_slope, v.min_db, v.ref_db
        c.voc_amp_floor, c.voc_tail_value, c.voc_tail_base = v.amp_floor, v.tail_pad_value, v.tail_pad_base
        c.voc_mel_weight_a, c.voc_mel_weight_b = v.mel_weight_a, v.mel_weight_b
        c.voc_tail_tanh = int(getattr(v, "tail_tanh", True))
        self.ctx = ctypes.c_void_p()
        rc = self.lib.vf_create(ctypes.byref(self.ctx), self.index, ctypes.byref(c))
        if rc != L.VF_OK:
            msg = self.lib.vf_last_error(None)
            raise L.EngineError(rc, msg.decode() if msg else "")
        self.loaded = False

    def close(self):
        if getattr(self, "ctx", None) is not None and self.ctx.value:
            self.lib.vf_destroy(self.ctx)
            self.ctx = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        return L.check(self.lib, self.ctx, rc)

    def load_state(self, state: Dict[str, torch.Tensor], need=("unet", "vocoder")):
        """Hands the tensors of the networks in `need` to vf_load_weights: "unet" / "bi_gru" / "dnn" =
        generator.analysis_module.* (VoiceFixer's analysis module: the mel UNet, arch.bigru_keys or arch.dnn_keys),
        "vocoder" = vocoder.* (the restated generator, arch.vocoder_keys), "ssr" = generator.unet.* (unet_v2 of SSR_UNet /
        GSR_UNet).  A missing key raises KeyError naming its source."""
        groups = {
            "unet": [UNET_PREFIX + k for k, s in unet_keys() if not k.endswith("num_batches_tracked")],
            "bi_gru": [UNET_PREFIX + k for k, s in bigru_keys() if not k.endswith("num_batches_tracked")],
            "dnn": [UNET_PREFIX + k for k, s in dnn_keys() if not k.endswith("num_batches_tracked")],
            "ssr": [SSR_PREFIX + k for k, s in unet_keys() if not k.endswith("num_batches_tracked")],
            "vocoder": ["vocoder." + k for k, _ in vocoder_keys(self.voc_cfg)],
        }
        needed = []
        for g in need:
            missing = [k for k in groups[g] if k not in state]
            if missing:
                hint = ""
                if g == "bi_gru":
                    gru = [k for k in missing if ".gru." in k]
                    hint = f" - missing GRU tensors: {gru}" if gru else ""
                if g == "vocoder":
                    hint = (" - the vocoder of a reference checkpoint is the pip `voicefixer` package's own module with its "
                            "own key names and a separately downloaded weight file; convert it to arch.vocoder_keys "
                            "(weight norm folded) and pass it as vocoder_state")
                raise KeyError(f"state dict is missing {len(missing)} '{g}' tensors, e.g. {missing[:3]}{hint}")
            needed += groups[g]
        fb = state["mel.fb"] if "mel.fb" in state else melscale_fbanks()
        # AudioMetrics' mel_16k (metrics.py:30), so that any engine also scores 16 kHz test sets
        items = [("mel.fb", fb), ("metrics.mel_16k.fb", mel16k_fbanks())] + [(k, state[k]) for k in needed]
        descs = (L.VfTensorDesc * len(items))()
        keep = []
        for d, (k, t) in zip(descs, items):
            t = t.detach().to(dtype=torch.float32).contiguous()
            keep.append(t)
            d.name = k.encode()
            d.data = t.data_ptr()
            d.ndim = t.dim()
            for i, s in enumerate(t.shape):
                d.shape[i] = s
            d.on_device = 1 if t.is_cuda else 0
        self._ck(self.lib.vf_load_weights(self.ctx, descs, len(items)))
        self.loaded = True

    # ---- stage entry points (device tensors in, device tensors out)
    def frontend(self, wav: torch.Tensor, want_sp: bool = False, want_phase: bool = False, want_mel: bool = True):
        wav = _check_in(wav, self.device, "wav")
        b, n = wav.shape
        t = frames_for(n)
        mel = torch.empty(b, t, 128, device=self.device) if want_mel else None
        sp = torch.empty(b, t, 1025, device=self.device) if (want_sp or want_phase) else None
        cos = torch.empty_like(sp) if want_phase else None
        sin = torch.empty_like(sp) if want_phase else None
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_frontend(self.ctx, _ptr(wav), b, n, _ptr(mel), _ptr(sp), _ptr(cos), _ptr(sin), _stream()))
        return mel, sp, cos, sin

    def unet_mel(self, mel_lin: torch.Tensor) -> torch.Tensor:
        mel_lin = _check_in(mel_lin, self.device, "mel")
        b, t, m = mel_lin.shape
        assert m == 128
        out = torch.empty_like(mel_lin)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_unet_mel(self.ctx, _ptr(mel_lin), b, t, _ptr(out), _stream()))
        return out

    def vocoder(self, mel_lin: torch.Tensor) -> torch.Tensor:
        mel_lin = _check_in(mel_lin, self.device, "mel")
        b, t, m = mel_lin.shape
        assert m == 128
        out = torch.empty(b, self.lib.vf_vocoder_out_len(self.ctx, t), device=self.device)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_vocoder(self.ctx, _ptr(mel_lin), b, t, _ptr(out), _stream()))
        return out

    def vocoder_varlen(self, mel_packed: torch.Tensor, frames, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The vocoder on linear mels of different lengths in one call (vf_vocoder_varlen): mel_packed [sum(frames), 128]
        holds the clips' frames back to back; returns each clip's full vocoder output, arch.vocoder_out_len(T_i) samples,
        packed in clip order (no peak normalise, no trim).  Clip i is bit-identical to vocoder(mel_i[None])[0].  Needs only
        the vocoder's weights."""
        if not isinstance(mel_packed, torch.Tensor) or mel_packed.dtype != torch.float32 or mel_packed.device != self.device:
            raise TypeError(f"mel_packed must be a float32 CUDA tensor on {self.device}")
        frames = [int(t) for t in frames]
        if mel_packed.dim() != 2 or mel_packed.shape[1] != 128 or not frames or sum(frames) != mel_packed.shape[0]:
            raise ValueError("mel_packed must be [sum(frames), 128] and hold the frames of at least one clip")
        offsets = _offsets(frames)
        n_out = sum(vocoder_out_len(t, self.voc_cfg) for t in frames) if min(frames) > 0 else 0
        out = torch.empty(n_out, device=self.device) if out is None else out
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_vocoder_varlen(self.ctx, _ptr(mel_packed.contiguous()), offsets, len(frames), _ptr(out),
                                                _stream()))
        return out

    def resynth(self, wav: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Vocoder resynthesis (vf_resynth): wav [B,N] -> the vocoder on its linear mel, peak normalised and trimmed to [B,N]
        (restore() without the analysis module).  Needs only the vocoder's weights."""
        wav = _check_in(wav, self.device, "wav")
        b, n = wav.shape
        out = torch.empty_like(wav) if out is None else out
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_resynth(self.ctx, _ptr(wav), b, n, _ptr(out), _stream()))
        return out

    def resynth_varlen(self, wav_packed: torch.Tensor, lengths, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """resynth for clips of different lengths in one call (vf_resynth_varlen), packed as restore_varlen: clip i of the
        result is bit-identical to resynth(clip_i[None])[0]."""
        wav_packed, offsets = self._varlen_args(wav_packed, lengths)
        out = torch.empty_like(wav_packed) if out is None else out
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_resynth_varlen(self.ctx, _ptr(wav_packed), offsets, len(offsets) - 1, _ptr(out), _stream()))
        return out

    def restore(self, wav: torch.Tensor, out: Optional[torch.Tensor] = None, unify_energy: bool = False) -> torch.Tensor:
        wav = _check_in(wav, self.device, "wav")
        b, n = wav.shape
        out = torch.empty_like(wav) if out is None else out
        flags = L.VF_RESTORE_UNIFY_ENERGY if unify_energy else 0
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_restore_ex(self.ctx, _ptr(wav), b, n, _ptr(out), flags, _stream()))
        return out

    def restore_varlen(self, wav_packed: torch.Tensor, lengths, out: Optional[torch.Tensor] = None,
                       unify_energy: bool = False, mel_out: Optional[torch.Tensor] = None,
                       log_mel_out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Clips of different lengths in one call (vf_restore_varlen): wav_packed [sum(lengths)] holds the clips back to back;
        the result is packed the same way, and clip i is bit-identical to restore(clip_i[None])[0].
        mel_out / log_mel_out (vf_restore_varlen_mels), each [sum(frames_for(n_i)), 128] or None: clip i's linear mel and
        restored log10 mel land in rows sum_{j<i} frames_for(n_j) onwards, the bits restore_stages(1, n_i) gives after
        restore(clip_i[None])."""
        wav_packed, offsets = self._varlen_args(wav_packed, lengths)
        out = torch.empty_like(wav_packed) if out is None else out
        self._packed_rows(offsets, mel_out=mel_out, log_mel_out=log_mel_out)
        flags = L.VF_RESTORE_UNIFY_ENERGY if unify_energy else 0
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_restore_varlen_mels(self.ctx, _ptr(wav_packed), offsets, len(offsets) - 1, _ptr(out), flags,
                                                     _ptr(mel_out), _ptr(log_mel_out), _stream()))
        return out

    def restore_chunks(self, ring: torch.Tensor, table, unify_energy: bool = False) -> torch.Tensor:
        """Chunks of live streams in one call (vf_restore_chunks): ring [n_streams, ring_len] float32 on the device holds
        stream s's absolute sample p at ring[s, p % ring_len]; table is a sequence of (stream, length, crop_left, crop_right,
        start, valid) tuples.  Returns the kept samples out_c[crop_left : length - crop_right] of every chunk, packed in table
        order, where out_c is restore() of positions start .. start + length - 1 with those >= valid read as 0."""
        ring, rows, out = self._chunks_args(ring, table)
        flags = L.VF_RESTORE_UNIFY_ENERGY if unify_energy else 0
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_restore_chunks(self.ctx, _ptr(ring), ring.shape[0], ring.shape[1], rows, len(table), _ptr(out),
                                                flags, _stream()))
        return out

    def vocoder_chunks(self, ring: torch.Tensor, table) -> torch.Tensor:
        """Chunks of live mel streams vocoded in one call (vf_vocoder_chunks): ring [n_streams, ring_frames, 128] float32 on
        the device holds stream s's absolute frame p at ring[s, p % ring_frames]; table is a sequence of (stream, length,
        crop_left, crop_right, start, valid) tuples, start / length / valid in frames and the crops in output samples.
        Returns the kept samples out_c[crop_left : vocoder_out_len(length) - crop_right] of every chunk, packed in table
        order, where out_c is vocoder_varlen of frames start .. start + length - 1 with those >= valid read as zeros.  Needs
        only the vocoder's weights."""
        ring, rows, out = self._chunks_args(ring, table, lambda n: vocoder_out_len(n, self.voc_cfg) if n > 0 else 0)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_vocoder_chunks(self.ctx, _ptr(ring), ring.shape[0], ring.shape[1], rows, len(table), _ptr(out),
                                                _stream()))
        return out

    def ssr_restore_chunks(self, ring: torch.Tensor, table) -> torch.Tensor:
        """restore_chunks for the SSR / GSR-UNet path (vf_ssr_restore_chunks): the same ring and table, and out_c is
        ssr_forward(None, chunk[None])[0] of the zero-filled chunk."""
        ring, rows, out = self._chunks_args(ring, table)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_ssr_restore_chunks(self.ctx, _ptr(ring), ring.shape[0], ring.shape[1], rows, len(table),
                                                    _ptr(out), _stream()))
        return out

    def restore_windows(self, ring: torch.Tensor, windows, window_len: int, synthesis: torch.Tensor, acc: torch.Tensor,
                        emits, unify_energy: bool = False) -> torch.Tensor:
        """Windows of live streams restored, weighted and overlap-added in one call (vf_restore_windows).  ring as in
        restore_chunks; windows is a sequence of (stream, start, valid): positions start .. start + window_len - 1, those below
        0 or >= valid read as 0.  Each window's restore() output times `synthesis` ([window_len] float32) is added, rounded
        product by product, into acc [n_streams, acc_len] (stream s's position t at acc[s, t % acc_len]) over positions
        [max(0, start), min(valid, start + window_len)).  Then emits, a sequence of (stream, start, count), copies each
        stream's finished positions out of acc and zeroes them.  Returns the emitted samples, packed in emits order."""
        ring, acc, synthesis, rows, ems, out = self._windows_args(ring, windows, window_len, synthesis, acc, emits)
        flags = L.VF_RESTORE_UNIFY_ENERGY if unify_energy else 0
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_restore_windows(self.ctx, _ptr(ring), ring.shape[0], ring.shape[1], rows, len(windows),
                                                 int(window_len), _ptr(synthesis), _ptr(acc), acc.shape[1], ems, len(emits),
                                                 _ptr(out), flags, _stream()))
        return out

    def ssr_restore_windows(self, ring: torch.Tensor, windows, window_len: int, synthesis: torch.Tensor, acc: torch.Tensor,
                            emits) -> torch.Tensor:
        """restore_windows for the SSR / GSR-UNet path (vf_ssr_restore_windows): each window's output is
        ssr_forward(None, window[None])[0] of the zero-filled window."""
        ring, acc, synthesis, rows, ems, out = self._windows_args(ring, windows, window_len, synthesis, acc, emits)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_ssr_restore_windows(self.ctx, _ptr(ring), ring.shape[0], ring.shape[1], rows, len(windows),
                                                     int(window_len), _ptr(synthesis), _ptr(acc), acc.shape[1], ems,
                                                     len(emits), _ptr(out), _stream()))
        return out

    def _windows_args(self, ring, windows, window_len, synthesis, acc, emits):
        """Checked ring, accumulators and synthesis table, the host vf_window / vf_emit tables and the packed output of a
        windows call."""
        ring = _check_in(ring, self.device, "ring")
        _check_in(acc, self.device, "acc")
        if not acc.is_contiguous():
            raise ValueError("acc must be contiguous: the call updates it in place")
        if ring.dim() != 2 or acc.dim() != 2 or acc.shape[0] != ring.shape[0]:
            raise ValueError("ring must be [n_streams, ring_len] and acc [n_streams, acc_len]")
        if synthesis is not None:
            synthesis = _check_in(synthesis, self.device, "synthesis")
            if synthesis.dim() != 1 or synthesis.numel() != int(window_len):
                raise ValueError("synthesis must be [window_len]")
        rows = (L.VfWindow * max(1, len(windows)))(*[L.VfWindow(*map(int, t)) for t in windows])
        ems = (L.VfEmit * max(1, len(emits)))(*[L.VfEmit(*map(int, t)) for t in emits])
        return ring, acc, synthesis, rows, ems, torch.empty(sum(max(0, int(t[2])) for t in emits), device=self.device)

    def _chunks_args(self, ring: torch.Tensor, table, out_len=None):
        """Checked ring, the host vf_chunk table and the packed output of a chunks call.  out_len: the output samples of a
        chunk of `length` positions, for a ring of mel frames ([n_streams, ring_frames, 128]); None: a ring of samples."""
        ring = _check_in(ring, self.device, "ring")
        if out_len is None and ring.dim() != 2:
            raise ValueError("ring must be [n_streams, ring_len]")
        if out_len is not None and (ring.dim() != 3 or ring.shape[2] != 128):
            raise ValueError("ring must be [n_streams, ring_frames, 128]")
        out_len = out_len or (lambda n: n)
        rows = (L.VfChunk * max(1, len(table)))(*[L.VfChunk(*map(int, t)) for t in table])
        kept = sum(max(0, out_len(int(t[1])) - int(t[2]) - int(t[3])) for t in table)
        return ring, rows, torch.empty(kept, device=self.device)

    def _varlen_args(self, packed: torch.Tensor, lengths, dtype=torch.float32):
        """Checked packed `dtype` input and the host offsets array of a varlen call."""
        if not isinstance(packed, torch.Tensor) or packed.dtype != dtype or packed.device != self.device:
            raise TypeError(f"the packed input must be a {str(dtype)[6:]} CUDA tensor on {self.device}")
        lengths = [int(n) for n in lengths]
        if packed.dim() != 1 or not lengths or sum(lengths) != packed.numel():
            raise ValueError("the packed input must be 1-D and hold exactly sum(lengths) samples of at least one item")
        return packed.contiguous(), _offsets(lengths)

    def _packed_rows(self, offsets, **outs) -> int:
        """Rows sum_i frames_for(n_i) of a varlen call's packed per-frame outputs (clip i from row sum_{j<i} frames_for(n_j));
        checks that each output of `outs` (name -> tensor or None) is a contiguous [rows, 128] float32 tensor on the device."""
        rows = sum(frames_for(offsets[i + 1] - offsets[i]) for i in range(len(offsets) - 1))
        for name, t in outs.items():
            if t is not None:
                _check_in(t, self.device, name)
                if not t.is_contiguous() or tuple(t.shape) != (rows, 128):
                    raise ValueError(f"{name} must be a contiguous [{rows}, 128] tensor (the clips' frames, packed)")
        return rows

    def mel(self, specgram: torch.Tensor) -> torch.Tensor:
        """MelScale.forward: specgram [..., 1025, time] (any strides) -> [..., 128, time]."""
        if not isinstance(specgram, torch.Tensor) or specgram.dtype != torch.float32 or specgram.device != self.device:
            raise TypeError(f"specgram must be a float32 CUDA tensor on {self.device}")
        assert specgram.dim() >= 2 and specgram.shape[-2] == 1025, "specgram: (..., freq = n_stft, time)"
        lead, t = specgram.shape[:-2], specgram.shape[-1]
        x = specgram.reshape(-1, 1025, t)               # a view whenever the leading dims are mergeable (else one copy)
        out = torch.empty(x.shape[0], t, 128, device=self.device)
        with torch.cuda.device(self.device):
            for o0 in range(0, x.shape[0], 65535):
                xs = x[o0:o0 + 65535]
                self._ck(self.lib.vf_mel(self.ctx, _ptr(xs), xs.shape[0], t, xs.stride(0), xs.stride(1), xs.stride(2),
                                         ctypes.c_void_p(out[o0:].data_ptr()), _stream()))
        return out.view(*lead, t, 128).transpose(-1, -2)     # same memory layout as the reference's matmul result

    def metric_spectrogram(self, wav_packed: torch.Tensor, lengths, want_mel: bool = True, rate: int = 44100):
        """vf_metric_spectrogram: |librosa.stft(n_fft=2048, hop_length=441)| of each clip of wav_packed (clips back to back,
        `lengths` samples each) -> (sp [sum T_i, 1025], mel [sum T_i, 128] or None), clip i at rows sum_{j<i} T_i.
        rate=16000 (vf_metric_spectrogram_ex): n_fft 743, hop 160 -> sp [sum T_i, 372], mel [sum T_i, 80] with
        T_i = arch.metric_frames(n_i, 16000)."""
        wav_packed, offsets = self._varlen_args(wav_packed, lengths)
        if rate == 44100:
            rows, bins, mels = self._packed_rows(offsets), 1025, 128
        else:
            rows, bins, mels = sum(metric_frames(offsets[i + 1] - offsets[i], 16000) for i in range(len(offsets) - 1)), 372, 80
        sp = torch.empty(rows, bins, device=self.device)
        mel = torch.empty(rows, mels, device=self.device) if want_mel else None
        with torch.cuda.device(self.device):
            if rate == 44100:
                rc = self.lib.vf_metric_spectrogram(self.ctx, _ptr(wav_packed), offsets, len(offsets) - 1, _ptr(sp), _ptr(mel),
                                                    _stream())
            else:
                rc = self.lib.vf_metric_spectrogram_ex(self.ctx, _ptr(wav_packed), offsets, len(offsets) - 1, _ptr(sp), _ptr(mel),
                                                       int(rate), _stream())
            self._ck(rc)
        return sp, mel

    def ssim(self, est: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        """vf_ssim: est, target [images, frames, bins] float32 -> float64 [images]."""
        est, target = _check_in(est, self.device, "est"), _check_in(target, self.device, "target")
        if est.dim() != 3 or est.shape != target.shape:
            raise ValueError("ssim: est and target must be [images, frames, bins] tensors of one shape")
        n, t, f = est.shape
        out = torch.empty(n, dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_ssim(self.ctx, _ptr(est), _ptr(target), n, t, f, _ptr(out), _stream()))
        return out

    def score_varlen(self, est_packed: torch.Tensor, est_lengths, target_packed: torch.Tensor, target_lengths,
                     rate: int = 44100) -> torch.Tensor:
        """vf_score_varlen: the spectral metrics of each (est, target) pair of two packed sets -> float64 [pairs, 8], columns
        in the order of edges.SCORE_KEYS.  rate=16000 scores with the 16 kHz geometry (vf_score_varlen_ex)."""
        est_packed, est_off = self._varlen_args(est_packed, est_lengths)
        target_packed, target_off = self._varlen_args(target_packed, target_lengths)
        if len(est_off) != len(target_off):
            raise ValueError("score_varlen: est and target must hold the same number of clips")
        out = torch.empty(len(est_off) - 1, 8, dtype=torch.float64, device=self.device)
        args = (self.ctx, _ptr(est_packed), est_off, _ptr(target_packed), target_off, len(est_off) - 1, _ptr(out))
        with torch.cuda.device(self.device):
            if rate == 44100:
                self._ck(self.lib.vf_score_varlen(*args, _stream()))
            else:
                self._ck(self.lib.vf_score_varlen_ex(*args, int(rate), _stream()))
        return out

    def score_time_varlen(self, est_packed: torch.Tensor, est_lengths, target_packed: torch.Tensor, target_lengths,
                          rate: int = 44100) -> torch.Tensor:
        """vf_score_time_varlen: speechmetrics' sisdr and stoi of each (est, target) pair of two packed sets at `rate`
        (44100, or 16000 through vf_score_time_varlen_ex) -> float64 [pairs, 2], columns sisdr, stoi.  The clips of a pair
        may differ in length (the shorter is zero-padded)."""
        est_packed, est_off = self._varlen_args(est_packed, est_lengths)
        target_packed, target_off = self._varlen_args(target_packed, target_lengths)
        if len(est_off) != len(target_off):
            raise ValueError("score_time_varlen: est and target must hold the same number of clips")
        out = torch.empty(len(est_off) - 1, 2, dtype=torch.float64, device=self.device)
        args = (self.ctx, _ptr(est_packed), est_off, _ptr(target_packed), target_off, len(est_off) - 1, _ptr(out))
        with torch.cuda.device(self.device):
            if rate == 44100:
                self._ck(self.lib.vf_score_time_varlen(*args, _stream()))
            else:
                self._ck(self.lib.vf_score_time_varlen_ex(*args, int(rate), _stream()))
        return out

    def sosfiltfilt_varlen(self, x_packed: torch.Tensor, lengths, sos, zi, row_filter, row_f32=None) -> torch.Tensor:
        """vf_sosfiltfilt_varlen: scipy.signal.sosfiltfilt(sos[f], row) of each float64 row of x_packed (rows back to back,
        `lengths` samples each), row i with filter f = row_filter[i]; sos[f] is an [n_sections <= 10, 6] float64 array and
        zi[f] its sosfilt_zi.  row_f32[i] true: row i holds float32 input, whose odd extension scipy rounds to float32.
        -> float64, packed like x_packed."""
        x_packed, off = self._varlen_args(x_packed, lengths, torch.float64)
        nf = len(sos)
        sos_t = (ctypes.c_double * (nf * 60))()
        zi_t = (ctypes.c_double * (nf * 20))()
        ns = (ctypes.c_int * nf)()
        for f, (s, z) in enumerate(zip(sos, zi)):
            s, z = np.asarray(s, dtype=np.float64), np.asarray(z, dtype=np.float64)
            ns[f] = s.shape[0]
            for k, v in enumerate(s[:10].reshape(-1).tolist()):
                sos_t[f * 60 + k] = v
            for k, v in enumerate(z[:10].reshape(-1).tolist()):
                zi_t[f * 20 + k] = v
        rows = (ctypes.c_int * len(row_filter))(*[int(f) for f in row_filter])
        f32 = (ctypes.c_int * len(row_filter))(*[int(bool(v)) for v in row_f32]) if row_f32 is not None else None
        out = torch.empty_like(x_packed)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_sosfiltfilt_varlen(self.ctx, _ptr(x_packed), off, len(off) - 1, sos_t, zi_t, ns, nf, rows,
                                                    f32, _ptr(out), _stream()))
        return out

    def resample_poly_f64_varlen(self, x_packed: torch.Tensor, lengths, filters, row_filter, out_lengths) -> torch.Tensor:
        """vf_resample_poly_f64_varlen: scipy.signal.resample_poly of each float64 row of x_packed, row i with filter
        filters[row_filter[i]] = (up, down, taps: float64 device tensor of odd length) -> float64 rows of out_lengths[i]
        samples packed back to back (ceil(n up / down) is resample_poly's length; more pads zeros, fewer cuts)."""
        x_packed, off = self._varlen_args(x_packed, lengths, torch.float64)
        out_lengths = [int(n) for n in out_lengths]
        out_off = _offsets(out_lengths)
        taps = torch.cat([t.to(self.device, torch.float64).reshape(-1) for _, _, t in filters]).contiguous()
        tap_off = _offsets([t.numel() for _, _, t in filters])
        up = (ctypes.c_int * len(filters))(*[int(u) for u, _, _ in filters])
        down = (ctypes.c_int * len(filters))(*[int(d) for _, d, _ in filters])
        rows = (ctypes.c_int * len(row_filter))(*[int(f) for f in row_filter])
        out = torch.empty(sum(out_lengths), dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_resample_poly_f64_varlen(self.ctx, _ptr(x_packed), off, len(off) - 1, _ptr(taps), tap_off, up,
                                                          down, len(filters), rows, _ptr(out), out_off, _stream()))
        return out

    def resample_sinc_varlen(self, x_packed: torch.Tensor, lengths, filters, row_filter, out_lengths) -> torch.Tensor:
        """vf_resample_sinc_varlen: resampy's sinc resampling (librosa 0.8 resample, res_type kaiser_best / kaiser_fast) of
        each float32 row of x_packed, row i with filter filters[row_filter[i]] = (table: float64 [nwin, 2] (win, delta) pairs
        as edges.sinc_table designs them, sample_ratio, num_table) -> float32 rows of out_lengths[i] samples packed back to
        back (resampy's int(n * sample_ratio), then zeros)."""
        x_packed, off = self._varlen_args(x_packed, lengths)
        out_lengths = [int(n) for n in out_lengths]
        out_off = _offsets(out_lengths)
        tables = torch.cat([t.to(self.device, torch.float64).reshape(-1, 2) for t, _, _ in filters]).contiguous()
        table_off = _offsets([t.numel() // 2 for t, _, _ in filters])
        ratio = (ctypes.c_double * len(filters))(*[float(r) for _, r, _ in filters])
        num_table = (ctypes.c_int * len(filters))(*[int(k) for _, _, k in filters])
        rows = (ctypes.c_int * len(row_filter))(*[int(f) for f in row_filter])
        out = torch.empty(sum(out_lengths), device=self.device)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_resample_sinc_varlen(self.ctx, _ptr(x_packed), off, len(off) - 1, _ptr(tables), table_off,
                                                      ratio, num_table, len(filters), rows, _ptr(out), out_off, _stream()))
        return out

    def remove_higher_frequency_varlen(self, x_packed: torch.Tensor, lengths, ratio: float = 0.95):
        """vf_remove_higher_frequency_varlen: the pip package's pre-filter remove_higher_frequency(wav, ratio) of each float32
        row of x_packed (rows back to back, `lengths` samples each, 1 .. 2^30) -> (packed float32 output, its row lengths
        512 * (n // 512), int32 device tensor of each row's first removed bin).  A quiet row (no bin with |X| >= 1) has cutoff
        0 and zeros; a row under 512 samples an empty output.  A NaN or infinite sample raises VF_EDEVICE at check_errors.
        Device scratch: 16.4 KB per frame (1 + n // 512) of the call's largest sub-batch, kept by the engine; a row longer than
        16384 frames (190 s) runs alone with all its frames resident, about 5.1 GB per hour of audio."""
        x_packed, off = self._varlen_args(x_packed, lengths)
        out_lengths = [512 * ((off[i + 1] - off[i]) // 512) for i in range(len(off) - 1)]
        out = torch.empty(sum(out_lengths), device=self.device)
        cutoff = torch.empty(len(off) - 1, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_remove_higher_frequency_varlen(self.ctx, _ptr(x_packed), off, len(off) - 1, float(ratio),
                                                                _ptr(out) if out.numel() else None, _offsets(out_lengths),
                                                                _ptr(cutoff), _stream()))
        return out, out_lengths, cutoff

    def _stage(self, buffers, align: int = 16):
        """The byte buffers `buffers` in one pinned staging buffer, each at an `align`-byte aligned offset, sent to the
        device in one copy -> (device uint8 tensor, offsets)."""
        at, end = [], 0
        for b in buffers:
            at.append(end)
            end += (len(b) + align - 1) // align * align
        staging = torch.empty(end + align, dtype=torch.uint8, pin_memory=True)
        host = staging.numpy()
        for b, a in zip(buffers, at):
            host[a:a + len(b)] = np.frombuffer(b, dtype=np.uint8)
        return staging.to(self.device, non_blocking=True), at

    def _decode_pcm_rows(self, dev, rows, first: bool):
        """vf_decode_pcm_varlen of the (byte offset, frames, channels, format) rows of the device bytes `dev`."""
        table = (L.VfPcmRow * max(1, len(rows)))(*[L.VfPcmRow(*r) for r in rows])
        n = sum(r[1] for r in rows)
        mono = torch.empty(n, device=self.device)
        ch0 = torch.empty(n, dtype=torch.float64, device=self.device) if first else None
        if rows:
            with torch.cuda.device(self.device):
                self._ck(self.lib.vf_decode_pcm_varlen(self.ctx, _ptr(dev), len(rows), table, _ptr(mono), _ptr(ch0), _stream()))
        return mono, ch0

    def decode_pcm_varlen(self, files, first: bool = False):
        """vf_decode_pcm_varlen: librosa.load(path, sr=None, mono=True)'s samples of every wavfile.WavInfo of `files` ->
        (mono float32 [sum frames], channel 0 float64 [sum frames] or None), file i at rows sum_{j<i} frames_j.  The data
        chunks go to one pinned staging buffer, each at a 16-byte aligned offset, and to the device in one copy."""
        files = list(files)
        dev, at = self._stage([w.data for w in files])
        return self._decode_pcm_rows(dev, [(a, w.frames, w.channels, w.format) for w, a in zip(files, at)], first)

    def flac_pcm(self, files):
        """vf_decode_flac_varlen: the samples of every flacfile.FlacInfo of `files` as the bytes of a WAV data chunk
        (interleaved little-endian u8 as v + 128, s16 or s24) -> (device uint8 buffer, byte offset of each file's bytes).
        The audio regions go to the device in one copy.  A file the decoder rejects raises ValueError naming it, the reason
        and the file offset of the first bad frame; this reads the per-file status back, the call's one synchronisation."""
        from .flacfile import ERRORS
        files = list(files)
        if not files:
            return torch.empty(0, dtype=torch.uint8, device=self.device), []
        dev, at = self._stage([w.audio for w in files])
        out, end = [], 0
        for w in files:
            out.append(end)
            end += (w.total * w.channels * (w.bits // 8) + 15) // 16 * 16
        pcm = torch.empty(max(end, 16), dtype=torch.uint8, device=self.device)
        status = torch.empty(len(files), dtype=torch.int64, device=self.device)
        rows = (L.VfFlacRow * len(files))(*[L.VfFlacRow(a, len(w.audio), w.total, o, w.channels, w.bits, w.rate, w.variable,
                                                        w.first_block, 0) for w, a, o in zip(files, at, out)])
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_decode_flac_varlen(self.ctx, _ptr(dev), len(files), rows, _ptr(pcm), _ptr(status), _stream()))
        for w, st in zip(files, status.cpu().tolist()):
            if st != -1:
                byte, code = (st & (1 << 64) - 1) >> 8, st & 0xFF
                raise ValueError(f"{w.path}: {ERRORS.get(code, f'FLAC error {code}')} (frame at byte {w.audio_start + byte})")
        return pcm, out

    def decode_flac_varlen(self, files, first: bool = False):
        """librosa.load(path, sr=None, mono=True)'s samples of every flacfile.FlacInfo of `files`, as decode_pcm_varlen
        returns them: the FLAC frames decode to WAV data bytes on the device (flac_pcm), which vf_decode_pcm_varlen then
        converts and downmixes, so the result is the WAV path's for the same samples, bit for bit."""
        files = list(files)
        pcm, out = self.flac_pcm(files)
        fmt = {8: 0, 16: 1, 24: 2}                         # VF_PCM_U8, VF_PCM_S16, VF_PCM_S24
        return self._decode_pcm_rows(pcm, [(o, w.total, w.channels, fmt[w.bits]) for w, o in zip(files, out)], first)

    def decode_flac_pcm(self, files) -> list:
        """The WAV data bytes of every flacfile.FlacInfo of `files` (flac_pcm), as host numpy uint8 arrays."""
        files = list(files)
        pcm, out = self.flac_pcm(files)
        host = pcm.cpu().numpy()
        return [host[o:o + w.total * w.channels * (w.bits // 8)] for w, o in zip(files, out)]

    def resample_rings(self, in_ring: torch.Tensor, rows, out: torch.Tensor) -> torch.Tensor:
        """Live streams resampled from a device ring in one call (vf_resample_rings).  in_ring [n_streams, in_len] float32
        holds stream s's absolute input i at in_ring[s, i % in_len].  rows is a sequence of (stream, filter, m0, m1, n, avail,
        out_stream, out_offset): outputs m0 .. m1 - 1 of the stream's signal of n inputs (_lib.VF_RESAMPLE_OPEN while it is
        open), of which the first `avail` have been pushed, with `filter` an edges.StreamFilter; each output has the bits of
        that output of the whole-signal resample.  out is the output ring [n_out_streams, out_len] (output m of a row to
        out[out_stream, m % out_len]) or a 1-D packed tensor (out_stream -1: output m to out[out_offset + m - m0]).
        Returns out."""
        in_ring = _check_in(in_ring, self.device, "in_ring")
        if in_ring.dim() != 2 or not isinstance(out, torch.Tensor) or out.dtype != torch.float32 or out.device != self.device \
                or not out.is_contiguous() or out.dim() not in (1, 2):
            raise TypeError("resample_rings: in_ring [n_streams, in_len] and out [n_out_streams, out_len] or [n] float32 "
                            f"contiguous tensors on {self.device}")
        table = (L.VfResampleRow * len(rows))()
        for t, (s, f, m0, m1, n, avail, os_, oo) in zip(table, rows):
            t.stream, t.m0, t.m1, t.n, t.avail, t.out_stream, t.out_offset = s, m0, m1, n, avail, os_, oo
            t.family = f.family
            if f.family == L.VF_RESAMPLE_POLY:
                t.up, t.down, t.taps = f.up, f.down, f.taps.data_ptr()
            else:
                t.table, t.nwin, t.ratio, t.num_table = f.table.data_ptr(), f.table.shape[0], f.ratio, f.num_table
        n_out, out_len = (out.shape[0], out.shape[1]) if out.dim() == 2 else (0, 0)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_resample_rings(self.ctx, _ptr(in_ring), in_ring.shape[0], in_ring.shape[1], table, len(rows),
                                                _ptr(out), n_out, out_len, _stream()))
        return out

    def amp_to_original_f(self, mel_est: torch.Tensor, mel_target: torch.Tensor) -> torch.Tensor:
        """tools/utils.py:50-55 on linear mels [B,T,128]: the estimate scaled to the target's low-band energy."""
        mel_est, mel_target = _check_in(mel_est, self.device, "mel_est"), _check_in(mel_target, self.device, "mel_target")
        b, t, m = mel_est.shape
        assert m == 128 and mel_target.shape == mel_est.shape
        out = torch.empty_like(mel_est)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_amp_to_original_f(self.ctx, _ptr(mel_est), _ptr(mel_target), b, t, _ptr(out), _stream()))
        return out

    def finalize(self, wav: torch.Tensor, n: int) -> torch.Tensor:
        """eval_gsr_voicefixer.py:68-72: per-clip peak normalise (if max|x| > 1) + trim_center to n samples."""
        wav = _check_in(wav, self.device, "wav")
        b, length = wav.shape
        out = torch.empty(b, n, device=self.device)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_finalize(self.ctx, _ptr(wav), b, length, n, _ptr(out), _stream()))
        return out

    # ---- SSR / GSR-UNet path (unet_v2 + ISTFT)
    def ssr_forward(self, sp: Optional[torch.Tensor], wav: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        wav = _check_in(wav, self.device, "wav")
        b, n = wav.shape
        if sp is not None:
            sp = _check_in(sp, self.device, "sp")
            assert tuple(sp.shape) == (b, frames_for(n), 1025)
        out = torch.empty_like(wav) if out is None else out
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_ssr_forward(self.ctx, _ptr(sp), _ptr(wav), b, n, _ptr(out), _stream()))
        return out

    def ssr_restore_varlen(self, wav_packed: torch.Tensor, lengths, out: Optional[torch.Tensor] = None,
                           mel_out: Optional[torch.Tensor] = None, peak_normalise: bool = False) -> torch.Tensor:
        """restore_varlen for the SSR / GSR-UNet path (vf_ssr_restore_varlen): clip i of the packed result is bit-identical
        to ssr_forward(None, clip_i[None])[0].
        mel_out ([sum(frames_for(n_i)), 128] or None) and peak_normalise (vf_ssr_restore_varlen_mels): clip i's linear mel
        of that output lands in rows sum_{j<i} frames_for(n_j) onwards, the bits frontend() gives on it; then, with
        peak_normalise, clip i is divided by its max |x| when that exceeds 1, the bits of finalize(out_i[None], n_i)."""
        wav_packed, offsets = self._varlen_args(wav_packed, lengths)
        out = torch.empty_like(wav_packed) if out is None else out
        self._packed_rows(offsets, mel_out=mel_out)
        flags = L.VF_SSR_PEAK_NORMALISE if peak_normalise else 0
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_ssr_restore_varlen_mels(self.ctx, _ptr(wav_packed), offsets, len(offsets) - 1, _ptr(out),
                                                         flags, _ptr(mel_out), _stream()))
        return out

    def ssr_restore_host(self, wav_host: torch.Tensor, out_host: torch.Tensor):
        assert wav_host.dtype == torch.float32 and out_host.dtype == torch.float32
        assert not wav_host.is_cuda and not out_host.is_cuda and wav_host.is_contiguous() and out_host.is_contiguous()
        b, n = wav_host.shape
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_ssr_restore_host(self.ctx, _ptr(wav_host), b, n, _ptr(out_host), _stream()))

    def ssr_unet(self, sp: torch.Tensor) -> torch.Tensor:
        sp = _check_in(sp, self.device, "sp")
        b, t, f = sp.shape
        assert f == 1025
        out = torch.empty_like(sp)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_ssr_unet(self.ctx, _ptr(sp), b, t, _ptr(out), _stream()))
        return out

    def ssr_stages(self, batch: int, n: int):
        t = frames_for(n)
        sp = torch.empty(batch, t, 1025, device=self.device)
        mag = torch.empty(batch, t, 1025, device=self.device)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_ssr_stages(self.ctx, batch, n, _ptr(sp), _ptr(mag), _stream()))
        return sp, mag

    def istft(self, real: torch.Tensor, imag: torch.Tensor, length: int) -> torch.Tensor:
        real, imag = _check_in(real, self.device, "real"), _check_in(imag, self.device, "imag")
        b, t, f = real.shape
        assert f == 1025 and imag.shape == real.shape
        out = torch.empty(b, length, device=self.device)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_istft(self.ctx, _ptr(real), _ptr(imag), b, t, length, _ptr(out), _stream()))
        return out

    def plan_cache_info(self):
        n, by, bu, ev = ctypes.c_int(), ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_int64()
        self._ck(self.lib.vf_plan_cache_info(self.ctx, ctypes.byref(n), ctypes.byref(by), ctypes.byref(bu), ctypes.byref(ev)))
        return {"plans": n.value, "bytes": by.value, "budget": bu.value, "evicted": ev.value}

    def restore_host(self, wav_host: torch.Tensor, out_host: torch.Tensor):
        """Pinned host tensors [B,N] in/out; asynchronous on the current stream."""
        assert wav_host.dtype == torch.float32 and out_host.dtype == torch.float32
        assert not wav_host.is_cuda and not out_host.is_cuda and wav_host.is_contiguous() and out_host.is_contiguous()
        b, n = wav_host.shape
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_restore_host(self.ctx, _ptr(wav_host), b, n, _ptr(out_host), _stream()))

    def restore_stages(self, batch: int, n: int):
        """(linear mel, restored log10 mel), each [B,T,128], of the last restore() of this shape."""
        t = frames_for(n)
        mel = torch.empty(batch, t, 128, device=self.device)
        log_mel = torch.empty(batch, t, 128, device=self.device)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_restore_stages(self.ctx, batch, n, _ptr(mel), _ptr(log_mel), _stream()))
        return mel, log_mel

    def to_log(self, x):
        x = _check_in(x, self.device, "input")
        out = torch.empty_like(x)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_to_log(self.ctx, _ptr(x), _ptr(out), x.numel(), _stream()))
        return out

    def from_log(self, x):
        x = _check_in(x, self.device, "input")
        out = torch.empty_like(x)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_from_log(self.ctx, _ptr(x), _ptr(out), x.numel(), _stream()))
        return out

    def to_pcm16(self, x, saturate: bool = False):
        """fp32 samples -> int16 PCM exactly as save_wave (tools/file/wav.py:22-24) converts them; saturate=True clamps
        instead of wrapping +1.0 to -32768 (not bit-compatible with the reference, see INTEGRATION.md)."""
        x = _check_in(x, self.device, "input")
        out = torch.empty(x.shape, dtype=torch.int16, device=x.device)
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_to_pcm16_ex(self.ctx, _ptr(x), _ptr(out), x.numel(), int(saturate), _stream()))
        return out

    def check_errors(self):
        """Synchronises the current stream and raises on sticky device errors (AssertionError for the
        to_log negative-input assertion, as tools/pytorch/pytorch_util.py:158 does)."""
        with torch.cuda.device(self.device):
            rc = self.lib.vf_check_errors(self.ctx, _stream())
        if rc == L.VF_EASSERT:
            raise AssertionError(self.lib.vf_last_error(self.ctx).decode())
        self._ck(rc)

    def set_option(self, key: str, value: int):
        self._ck(self.lib.vf_set_option(self.ctx, key.encode(), int(value)))

    def launch_count(self) -> int:
        return int(self.lib.vf_launch_count(self.ctx))

    def workspace_bytes(self, batch: int, n: int) -> int:
        v = ctypes.c_size_t()
        self._ck(self.lib.vf_workspace_bytes(self.ctx, batch, n, ctypes.byref(v)))
        return int(v.value)

    def enable_stage_timing(self, on: bool = True):
        self._ck(self.lib.vf_enable_stage_timing(self.ctx, int(on)))

    def stage_times(self):
        arr = (ctypes.c_float * 4)()
        self._ck(self.lib.vf_stage_times(self.ctx, ctypes.byref(arr)))
        return dict(zip(("frontend_ms", "unet_ms", "vocoder_ms", "tail_ms"), [float(x) for x in arr]))

    def enable_op_timing(self, on: bool = True):
        self._ck(self.lib.vf_enable_op_timing(self.ctx, int(on)))

    def op_profile(self):
        """Per-launch records of the last restore() run with op timing enabled."""
        recs = []
        buf = ctypes.create_string_buffer(64)
        for i in range(self.lib.vf_op_count(self.ctx)):
            ms, fl, by, ex = ctypes.c_float(), ctypes.c_double(), ctypes.c_double(), ctypes.c_double()
            bn, bk, tm = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
            self._ck(self.lib.vf_op_info(self.ctx, i, ctypes.byref(ms), ctypes.byref(fl), ctypes.byref(by),
                                         ctypes.byref(bn), ctypes.byref(bk), ctypes.byref(tm), buf, 64, ctypes.byref(ex)))
            recs.append({"label": buf.value.decode(), "ms": ms.value, "flops": fl.value, "bytes": by.value,
                         "exec_flops": ex.value, "bn": bn.value, "bk": bk.value, "terms": tm.value})
        return recs

    def selftest_layer(self, case: "L.VfLayerCase"):
        """Runs one conv layer as the plans build it (vf_selftest_layer; tests only).  Synchronous."""
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_selftest_layer(self.ctx, ctypes.byref(case)))

    def selftest_gru(self, case: "L.VfGruCase"):
        """Runs one bidirectional GRU layer of the bi_gru analysis module as the plans launch it (vf_selftest_gru; tests
        only).  Synchronous."""
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_selftest_gru(self.ctx, ctypes.byref(case)))

    def selftest_op(self, case: "L.VfOpCase"):
        """Runs one non-GEMM op of the launch chains as the plans set it up (vf_selftest_op; tests only).  Synchronous."""
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_selftest_op(self.ctx, ctypes.byref(case)))

    def selftest_plan_gemms(self, plan_kind: int, batch: int, frames: int, tile_loop: bool = False):
        """[(label, signature)] of every GEMM / fused-pair launch of a plan of plan_kind (0 GSR, 1 SSR, 2 GSR varlen, 3 SSR
        varlen, 4 vocoder-only, 5 vocoder-only varlen) built with the loaded weights and the current options; nothing is launched (vf_selftest_plan_gemms; tests
        only).  With tile_loop, [(label, signature, tiles, grid, col_tiles)]: each launch's persistent tile loop as well."""
        cap, n = 2048, ctypes.c_int()
        recs = (L.VfPlanGemm * cap)()
        with torch.cuda.device(self.device):
            self._ck(self.lib.vf_selftest_plan_gemms(self.ctx, plan_kind, batch, frames, recs, cap, ctypes.byref(n)))
        assert n.value <= cap, n.value
        if tile_loop:
            return [(r.label.decode(), r.sig.decode(), r.tiles, r.grid, r.col_tiles) for r in recs[:n.value]]
        return [(r.label.decode(), r.sig.decode()) for r in recs[:n.value]]

    def selftest_sub_batch(self, plan_kind: int, batch: int, frames: int) -> int:
        """The sub-batch a call of `batch` clips of `frames` frames on plans of plan_kind runs in under the plan budget
        (vf_selftest_sub_batch; tests only)."""
        rc = self.lib.vf_selftest_sub_batch(self.ctx, plan_kind, batch, frames)
        if rc < 0:
            self._ck(rc)
        return rc

    def selftest_plan_trace(self, plan_kind: int, wav: torch.Tensor, lengths=None, on_op=None, unify_energy: bool = False,
                            direct_steps: bool = False):
        """One restore on a fresh plan of plan_kind (0 GSR, 1 SSR, 4 vocoder-only resynthesis: wav [B, n]; 2 GSR varlen,
        3 SSR varlen, 5 vocoder-only varlen: wav packed, lengths per clip), one launch at a time: on_op(after, op) runs before (after = False) and after (True) each launch
        with its L.VfTraceOp (vf_selftest_plan_trace; tests only).  An exception in on_op stops the run and is raised here.
        direct_steps: also trace the launches the restore makes itself (front end, band sums, ISTFT) as list 3.
        Returns the restored output, shaped as the matching restore call returns it."""
        wav = _check_in(wav, self.device, "wav")
        out = torch.empty_like(wav)
        caught = []

        def cb(_user, after, op):
            try:
                on_op(bool(after), op.contents)
                return 0
            except BaseException as e:          # noqa: BLE001 - handed back to the caller below
                caught.append(e)
                return 1

        fn = L.VF_TRACE_FN(cb)
        if lengths is not None:
            batch, n, offp = len(lengths), 0, _offsets(lengths)
        else:
            batch, n, offp = wav.shape[0], wav.shape[1], None
        flags = (L.VF_RESTORE_UNIFY_ENERGY if unify_energy else 0) | (L.VF_TRACE_DIRECT_STEPS if direct_steps else 0)
        with torch.cuda.device(self.device):
            torch.cuda.synchronize()            # the hook runs on the legacy default stream
            rc = self.lib.vf_selftest_plan_trace(self.ctx, plan_kind, _ptr(wav), offp, batch, n, flags, _ptr(out), fn, None)
        if caught:
            raise caught[0]
        self._ck(rc)
        return out


# --------------------------------------------------------------------------------------------------------------
class FDomainHelper:
    """tools/pytorch/modules/fDomainHelper.py:12-152 without the sub-band (PQMF) variants: STFT analysis and ISTFT
    synthesis, window 2048 / hop 441 / hann / reflect."""

    def __init__(self, owner, window_size=2048, hop_size=441, center=True, pad_mode="reflect", window="hann",
                 freeze_parameters=True, subband=None):
        if (window_size, hop_size, center, pad_mode, window, subband) != (2048, 441, True, "reflect", "hann", None):
            raise NotImplementedError("libb200vf implements the reference geometry only (2048/441/hann/reflect)")
        self._owner = owner

    def _run(self, input, phase):
        eng = self._owner._engine()
        assert input.dim() == 3, "input: (batch_size, channels_num, segment_samples)"
        b, c, n = input.shape
        _, sp, cos, sin = eng.frontend(input.reshape(b * c, n), want_sp=True, want_phase=phase, want_mel=False)
        t = sp.shape[1]
        sp = sp.view(b, c, t, 1025)
        if phase:
            return sp, cos.view(b, c, t, 1025), sin.view(b, c, t, 1025)
        return sp

    def wav_to_spectrogram_phase(self, input, eps=1e-8):
        assert eps == 1e-8
        return self._run(input, True)

    def wav_to_spectrogram(self, input, eps=1e-8):
        assert eps == 1e-8
        return self._run(input, False)

    def istft(self, real, imag, length):
        """fDomainHelper.py:127 (torchlibrosa ISTFT.forward): real, imag [B,1,T,1025] -> [B,length]."""
        assert real.dim() == 4 and real.shape[1] == 1 and imag.shape == real.shape
        return self._owner._engine().istft(real[:, 0], imag[:, 0], int(length))

    def spectrogram_phase_to_wav(self, sps, coss, sins, length):
        """fDomainHelper.py:91-97: per channel istft(sp * cos, sp * sin) -> [B,C,length]."""
        eng = self._owner._engine()
        outs = [eng.istft((sps[:, c] * coss[:, c]).contiguous(), (sps[:, c] * sins[:, c]).contiguous(), int(length))
                for c in range(sps.size()[1])]
        return torch.stack(outs, dim=1)


class MelScale:
    """tools/pytorch/mel_scale.py:8-64.  forward(specgram[..., freq, time]) -> [..., n_mels, time] for ANY float32
    spectrogram on the model's device (a sparse-filterbank kernel reading the view's own strides)."""

    def __init__(self, owner, n_mels=128, sample_rate=44100, n_stft=1025):
        if (n_mels, sample_rate, n_stft) != (128, 44100, 1025):
            raise NotImplementedError("libb200vf implements the reference geometry only (128 mels, 44.1 kHz, 1025 bins)")
        self.n_mels, self.sample_rate = n_mels, sample_rate
        self.f_min, self.f_max = 0.0, float(sample_rate // 2)
        self.fb = melscale_fbanks(n_stft, self.f_min, self.f_max, n_mels, sample_rate)
        self._owner = owner

    def __call__(self, specgram):
        return self.forward(specgram)

    def forward(self, specgram):
        return self._owner._engine().mel(specgram)


class Vocoder:
    """Stand-in for voicefixer.Vocoder(sample_rate): __call__(mel [B,1,T,128]) -> wav [B,1,L]."""

    def __init__(self, owner, sample_rate=44100):
        assert sample_rate == 44100
        self.rate = sample_rate
        self._owner = owner

    def __call__(self, mel, cuda=False):
        return self.forward(mel)

    def forward(self, mel, cuda=False):
        assert mel.size()[-1] == 128
        assert mel.dim() == 4 and mel.shape[1] == 1
        out = self._owner._engine().vocoder(mel[:, 0])
        return out[:, None, :]


class Generator:
    """models/gsr_voicefixer.py:44-91 with any of the four analysis modules: mel_orig -> {'mel': log10 mel}.
    Generator.forward is not sync-free - to_log's assert is a device->host round trip in the reference too
    (pytorch_util.py:158); VoiceFixer.restore() is the entry point without host synchronisation."""

    def __init__(self, owner):
        self._owner = owner

    def __call__(self, mel_orig):
        return self.forward(mel_orig)

    def forward(self, mel_orig):
        assert mel_orig.dim() == 4 and mel_orig.shape[1] == 1 and mel_orig.shape[-1] == 128
        eng = self._owner._engine()
        out = eng.unet_mel(mel_orig[:, 0])
        eng.check_errors()          # to_log's assert (pytorch_util.py:158)
        return {"mel": out[:, None]}


class _EngineModel:
    """nn.Module / Lightning surface the reference handlers use (load_from_checkpoint, eval, to, cuda), over one Engine."""
    _NEED = ("unet", "vocoder")

    def _init_common(self, hp, vocoder_config):
        self.hp = hp
        self.sampling_rate = hp["data"]["sampling_rate"]
        if hp["model"]["channels_in"] != 1:
            raise NotImplementedError("channels_in must be 1")
        self.voc_cfg = vocoder_config or VocoderConfig()
        self.f_helper = FDomainHelper(self, window_size=hp["model"]["window_size"], hop_size=hp["model"]["hop_size"],
                                      center=True, pad_mode=hp["model"]["pad_mode"], window=hp["model"]["window"])
        self.mel_freq_bins = hp["model"]["mel_freq_bins"]
        self.mel = MelScale(self, n_mels=self.mel_freq_bins, sample_rate=self.sampling_rate,
                            n_stft=hp["model"]["window_size"] // 2 + 1)
        self.vocoder = Vocoder(self, sample_rate=44100)
        self.downsample_ratio = 2 ** 6
        self.device = None
        self._eng: Optional[Engine] = None
        self._state: Optional[Dict[str, torch.Tensor]] = None
        self.training = False

    def _engine(self) -> Engine:
        if self._eng is None:
            raise RuntimeError("model is not on a CUDA device yet: call .to(device) (there is no CPU path)")
        if not self._eng.loaded:
            raise RuntimeError("no weights loaded: call load_state_dict / load_from_checkpoint first")
        return self._eng

    def _need(self):
        return self._NEED

    def _batch_engine(self, wavs):
        """The engine and the clip lengths for restore_batch(wavs), after checking the clips before anything is launched: a
        non-empty list of 1-D float32 tensors on the model's device, each longer than 1024 samples."""
        eng = self._engine()
        if not isinstance(wavs, (list, tuple)) or not wavs:
            raise ValueError("restore_batch: expected a non-empty list of 1-D tensors")
        for i, w in enumerate(wavs):
            if not isinstance(w, torch.Tensor) or w.dim() != 1:
                raise ValueError(f"restore_batch: clip {i} must be a 1-D tensor")
            if w.dtype != torch.float32 or w.device != eng.device:
                raise TypeError(f"restore_batch: clip {i} must be float32 on {eng.device} (got {w.dtype} on {w.device})")
            if w.numel() <= 1024:
                raise ValueError(f"restore_batch: clip {i} has {w.numel()} samples; reflect padding needs more than 1024")
        return eng, [w.numel() for w in wavs]

    def load_state_dict(self, state_dict, strict=True, vocoder_state=None):
        """state_dict: reference names for the analysis network (generator.analysis_module.* / generator.unet.*).
        The vocoder is NOT part of what a reference Lightning checkpoint can provide in loadable form (see
        Engine.load_state): pass its tensors, converted to arch.vocoder_keys names, as `vocoder_state`, or include
        them as `vocoder.<key>` entries.  strict=True (the default) raises KeyError on missing tensors; strict=False
        is not supported - a partial network cannot run."""
        if not strict:
            raise NotImplementedError("strict=False: libb200vf cannot run a partially loaded network")
        st = {k: v for k, v in state_dict.items() if isinstance(v, torch.Tensor)}
        if vocoder_state is not None:
            st.update({(k if k.startswith("vocoder.") else "vocoder." + k): v for k, v in vocoder_state.items()})
        self._state = st
        if self._eng is not None:
            self._eng.load_state(self._state, need=self._need())
        return self

    def load_from_checkpoint(self, ckpt, map_location="cpu", vocoder_state=None):
        """Lightning-style: returns the loaded model (eval_gsr_voicefixer.py:33 discards the receiver).  `ckpt` is a
        torch.save'd dict (optionally under "state_dict"); vocoder tensors as in load_state_dict."""
        blob = torch.load(ckpt, map_location=map_location, weights_only=False)
        sd = blob["state_dict"] if isinstance(blob, dict) and "state_dict" in blob else blob
        self.load_state_dict(sd, vocoder_state=vocoder_state)
        return self

    def state_dict(self):
        return dict(self._state or {})

    def eval(self):
        self.training = False
        return self

    def train(self, mode=True):
        if mode:
            raise NotImplementedError("inference-only engine: BatchNorm is folded in eval mode")
        return self

    def to(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("voicefixer_main_b200 has no CPU path; move the model to a CUDA device")
        if self._eng is not None and self._eng.device == torch.device("cuda", device.index if device.index is not None else torch.cuda.current_device()):
            return self
        if self._eng is not None:
            self._eng.close()
        self._eng = Engine(device, self.voc_cfg)
        self.device = self._eng.device
        if self._state is not None:
            self._eng.load_state(self._state, need=self._need())
        return self

    def cuda(self, device=None):
        return self.to(torch.device("cuda", device if device is not None else torch.cuda.current_device()))

    def get_vocoder(self):
        return self.vocoder

    def get_f_helper(self):
        return self.f_helper

    def pre(self, input):
        """gsr_voicefixer.py:178-181 / ssr_unet.py:140-143: input [B,1,N] -> (sp [B,1,T,1025], mel_orig [B,1,T,128]);
        one fused front-end launch produces both."""
        assert input.dim() == 3 and input.shape[1] == 1
        mel, sp, _, _ = self._engine().frontend(input[:, 0], want_sp=True)
        return sp[:, None], mel[:, None]


class VoiceFixer(_EngineModel):
    """Drop-in for models.gsr_voicefixer.VoiceFixer on the inference path (eval mode only)."""

    def __init__(self, hp=None, channels=2, type_target="vocals", vocoder_config: Optional[VocoderConfig] = None):
        hp = hp if hp is not None else default_hparams()
        self.channels, self.type_target = channels, type_target
        sel = hp["task"]["gsr"]["gsr_model"]["voicefixer"]
        # gsr_voicefixer.py:48-85: `unet` wins over `unet_small`, which wins over `bi_gru`, which wins over `dnn`.  The two
        # UNets (models/components/unet.py and unet_small.py, whose *Res1B blocks hold four ConvBlockRes like *Res4B,
        # modules.py:112-165) have the same layers and state-dict keys, so they share one plan
        for name in ("unet", "unet_small", "bi_gru", "dnn"):
            if sel[name]:
                self.analysis_module_name = name
                break
        else:
            raise NotImplementedError("no analysis module selected: task.gsr.gsr_model.voicefixer must enable one of "
                                      "unet, unet_small, bi_gru, dnn")
        self._init_common(hp, vocoder_config)
        self.generator = Generator(self)

    def _need(self):
        m = self.analysis_module_name
        return ("unet" if m in ("unet", "unet_small") else m, "vocoder")

    def forward(self, mel_orig):
        return self.generator(mel_orig)

    def __call__(self, mel_orig):
        return self.forward(mel_orig)

    # ---- batched fused path
    def restore(self, wav, out=None, unify_energy: bool = False, **pip_kwargs):
        """wav [B,N] fp32 on device -> restored [B,N]; one 60 s-or-shorter segment per row.
        unify_energy: apply amp_to_original_f (tools/utils.py:50-55) as handler() does for the SSR test sets
        (a per-call flag of vf_restore_ex: no context state is touched).

        Called with file paths - `restore(input="in.wav", output="out.wav", cuda=True, mode=0, your_vocoder_func=None)` -
        it is the pip package's file entry point (SURVEY.md 8(b); handler.restore_file)."""
        if isinstance(wav, (str, bytes)) or hasattr(wav, "__fspath__"):
            from .handler import restore_file
            return restore_file(self, wav, out if out is not None else pip_kwargs.pop("output"), **pip_kwargs)
        if pip_kwargs:
            raise TypeError(f"restore(tensor): unexpected arguments {sorted(pip_kwargs)}")
        return self._engine().restore(wav, out, unify_energy=unify_energy)

    def restore_batch(self, wavs: Sequence[torch.Tensor], unify_energy: bool = False) -> List[torch.Tensor]:
        """Clips of different lengths - a test set, a request queue - restored in one packed call: wavs is a list of 1-D fp32
        tensors on the model's device, each longer than 1024 samples; returns one view per clip into a packed output.
        Every clip gets exactly the bits restore(clip[None]) would give it (no zero-padding to a common length)."""
        eng, lengths = self._batch_engine(wavs)
        out = eng.restore_varlen(torch.cat(wavs), lengths, unify_energy=unify_energy)
        return list(torch.split(out, lengths))

    def remove_higher_frequency(self, wav, ratio=0.95) -> np.ndarray:
        """The pip package's pre-filter (VoiceFixer.remove_higher_frequency, the first step of restore_inmem's mode 1) of one
        1-D clip: bins from the first one where the running sum of per-bin energies sum_t max(log10(|X| + 1e-8), 0) reaches
        ratio times their total are removed, the rest scaled by |X| / (|X| + 1e-8), in librosa 0.8's stft / istft (n_fft 2048,
        hop 512).  -> 1-D float32 numpy of 512 * (len(wav) // 512) samples (istft with length None); a quiet clip, with no
        bin of |X| >= 1, comes back as zeros.  One remove_higher_frequency_batch call."""
        outs, _ = self.remove_higher_frequency_batch([wav], ratio)
        return outs[0].cpu().numpy()

    def remove_higher_frequency_batch(self, wavs, ratio=0.95):
        """remove_higher_frequency of every 1-D clip of `wavs` (numpy arrays or tensors, on the host or the device, any
        lengths from 1 to 2^30 samples) in one vf_remove_higher_frequency_varlen call -> (list of float32 tensors on the
        model's device, 512 * (n // 512) samples each: empty under 512; int32 device tensor of each clip's first removed bin,
        0 for a quiet clip, which comes back as zeros).  Each clip gets the bits it gets alone.  A ratio outside (0, 1], an
        empty list, or a clip that is not 1-D or is empty raises ValueError before any GPU work; a NaN or infinite sample
        raises VF_EDEVICE at the engine's check_errors."""
        if not isinstance(ratio, (int, float, np.floating, np.integer)) or not 0 < float(ratio) <= 1:
            raise ValueError(f"remove_higher_frequency: ratio {ratio!r} (need 0 < ratio <= 1)")
        if not isinstance(wavs, (list, tuple)) or not wavs:
            raise ValueError("remove_higher_frequency_batch: expected a non-empty list of 1-D clips")
        for i, w in enumerate(wavs):
            if np.ndim(w) != 1 or not 1 <= np.shape(w)[0] <= 1 << 30:
                raise ValueError(f"remove_higher_frequency_batch: clip {i} must be 1-D with 1 .. 2^30 samples "
                                 f"(got shape {tuple(np.shape(w))})")
        eng = self._engine()
        xs = [torch.as_tensor(w).to(eng.device, torch.float32) for w in wavs]
        out, lengths, cutoff = eng.remove_higher_frequency_varlen(torch.cat(xs), [x.numel() for x in xs], float(ratio))
        return list(torch.split(out, lengths)), cutoff

    def restore_inmem(self, wav_10k, cuda=True, mode=0, your_vocoder_func=None):
        """The pip package's in-memory entry point: 44.1 kHz samples -> restored [1, N] numpy (handler.restore_inmem)."""
        from .handler import restore_inmem
        return restore_inmem(self, wav_10k, cuda=cuda, mode=mode, your_vocoder_func=your_vocoder_func)

    def restore_host(self, wav_host: torch.Tensor, out_host: torch.Tensor):
        self._engine().restore_host(wav_host, out_host)

    def restore_pcm16(self, wav: torch.Tensor, unify_energy: bool = False) -> torch.Tensor:
        """restore() followed by the on-GPU int16 conversion of save_wave (tools/file/wav.py:22-24): [B,N] int16,
        half the device-to-host bytes of the fp32 result."""
        return self._engine().to_pcm16(self.restore(wav, unify_energy=unify_energy))

    def finalize(self, out: torch.Tensor, n_samples: int) -> torch.Tensor:
        """eval_gsr_voicefixer.py:68-72 on the vocoder output [B,1,L]: peak normalise (per clip) + trim_center -> [B,1,N]."""
        assert out.dim() == 3 and out.shape[1] == 1
        return self._engine().finalize(out[:, 0].contiguous(), n_samples)[:, None]


class SSRGenerator:
    """models/ssr_unet.py:44-54: forward(sp, noisy_wav) -> {'wav': unet(sp, wav)['wav'], 'clean': sp}."""

    def __init__(self, owner):
        self._owner = owner

    def __call__(self, sp, noisy_wav):
        return self.forward(sp, noisy_wav)

    def forward(self, sp, noisy_wav):
        assert sp.dim() == 4 and sp.shape[1] == 1 and sp.shape[-1] == 1025
        assert noisy_wav.dim() == 3 and noisy_wav.shape[1] == 1
        out = self._owner._engine().ssr_forward(sp[:, 0], noisy_wav[:, 0])
        return {"wav": out[:, None, :], "clean": sp}


class SSR_UNet(_EngineModel):
    """Drop-in for models.ssr_unet.SSR_UNet on the inference path (BASELINE config 3): pre(wav) -> (sp, mel);
    model(sp, wav)['wav'] = ISTFT(unet_v2(sp) * phase(wav)) (models/ssr_unet.py:140-155, unet_v2.py:86-148)."""
    _NEED = ("ssr",)

    def __init__(self, hp=None, channels=1, type_target="vocals", vocoder_config: Optional[VocoderConfig] = None):
        hp = hp if hp is not None else default_hparams()
        self.channels, self.type_target = channels, type_target
        self._init_common(hp, vocoder_config)
        self.generator = SSRGenerator(self)

    def forward(self, sp, noisy_wav):
        return self.generator(sp, noisy_wav)

    def __call__(self, sp, noisy_wav):
        return self.forward(sp, noisy_wav)

    def restore(self, wav: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """pre + forward fused: wav [B,N] -> denoised [B,N] (the magnitude never leaves the device plan)."""
        return self._engine().ssr_forward(None, wav, out)

    def restore_batch(self, wavs: Sequence[torch.Tensor]) -> List[torch.Tensor]:
        """Clips of different lengths - eval_ssr_unet.py:handler()'s test set, a request queue - in one packed call: wavs is a
        list of 1-D fp32 tensors on the model's device, each longer than 1024 samples; returns one view per clip into a packed
        output.  Every clip gets exactly the bits restore(clip[None]) would give it (no zero-padding to a common length)."""
        eng, lengths = self._batch_engine(wavs)
        out = eng.ssr_restore_varlen(torch.cat(wavs), lengths)
        return list(torch.split(out, lengths))

    def restore_host(self, wav_host: torch.Tensor, out_host: torch.Tensor):
        self._engine().ssr_restore_host(wav_host, out_host)


class GSR_UNet(SSR_UNet):
    """models/gsr_unet.py: same network and forward as SSR_UNet (they differ in training targets only)."""
