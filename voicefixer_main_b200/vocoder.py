"""The stand-alone vocoder the pip `voicefixer` package exports (`from voicefixer import Vocoder`), over the CUDA engine:

    Vocoder(sample_rate=44100, vocoder_config=None)
      .load_state_dict(state)                       arch.vocoder_keys names, with or without the "vocoder." prefix
      .to(device) / .cuda() / .eval()
      .forward(mel [B,1,T,128], cuda=False) -> wav [B,1,L]   (and __call__), L = arch.vocoder_out_len(T)
      .forward_batch([mel_i [T_i,128]]) -> [wav_i [L_i]]     mels of different lengths in packed calls
      .resynth_batch([wav_i]) -> [out_i]                     vocoder resynthesis of clips of different lengths
      .oracle(fpath, out_path, cuda=True) / .oracle_batch([(fpath, out_path)])

Live mel streams (a TTS or voice-conversion model's frames, a few at a time) are vocoded chunk by chunk by
streaming.StreamingVocoder; chunk_plan holds its geometry and vocode_chunked the composition its outputs equal.

Its engine holds the vocoder and the built-in mel filterbank (model.melscale_fbanks) only: no restorer checkpoint and no
analysis network is needed, and the plans hold the vocoder's buffers only (vf_vocoder_varlen, vf_resynth_varlen).
model.Vocoder, the restorer's own `model.vocoder`, is a view onto a VoiceFixer's engine and stays as it is.

`cuda` follows the package: forward's cuda=True moves a host mel to the vocoder's device; a mel already there runs as it
is.  A host mel with cuda=False, and oracle(cuda=False), raise: there is no CPU path.

`oracle` is handler() without the analysis module, a choice of this library and not the package's own oracle (which,
with the mel it computes, is not reproduced): the file is read by handler.load_wav (44.1 kHz, other rates converted on
the GPU), cut into handler()'s 60 s segments, and each segment is resynthesised (its linear mel -> the vocoder -> peak
normalise -> trim_center) and written as 16-bit PCM by save_wave.  It is the usual upper bound when scoring a restorer:
what is left of a clean file after the vocoder alone.
"""
from typing import List, Sequence, Tuple

import numpy as np
import torch

from .arch import VocoderConfig, frames_for, padded_frames, vocoder_keys, vocoder_out_len
from .model import _EngineModel


def packing(frames: Sequence[int], cfg: VocoderConfig = None):
    """(frame offsets, sample offsets) of a packed vocoder call on clips of `frames` frames: clip i's mel is rows
    F_i .. F_{i+1} of the packed input and its output samples S_i .. S_{i+1}, S_{i+1} - S_i = arch.vocoder_out_len(T_i)."""
    cfg = cfg or VocoderConfig()
    f, s = [0], [0]
    for t in frames:
        f.append(f[-1] + int(t))
        s.append(s[-1] + vocoder_out_len(int(t), cfg))
    return f, s


def length_groups(frames: Sequence[int]) -> List[List[int]]:
    """The clips of a batch call, by index, grouped for packed calls: longest first, each group the clips whose 64-frame
    bucket exceeds half the bucket of the group's longest clip.  A packed call runs every clip of a sub-batch on the bucket
    of its longest clip, so a 60 s clip among 1 s clips would make each of them cost 60 s of vocoder work (on an H100 that
    made one call over 1-10 s clips and a 60 s one twice as slow as a call per clip); within a group no clip is padded to
    more than twice its own bucket.  A clip's bits do not depend on its group."""
    groups: List[List[int]] = []
    for i in sorted(range(len(frames)), key=lambda k: -frames[k]):
        if groups and 2 * padded_frames(frames[i]) > padded_frames(frames[groups[-1][0]]):
            groups[-1].append(i)
        else:
            groups.append([i])
    return groups


def check_chunking(window_frames: int, margin_frames: int):
    """The chunk geometry's argument check: W >= 2 and M >= 0, both even (so every chunk's length has the parity of the
    whole mel, and the chunks' outputs add up to its output length)."""
    W, M = int(window_frames), int(margin_frames)
    if W < 2 or W % 2:
        raise ValueError(f"window_frames must be even and at least 2 (got {W})")
    if M < 0 or M % 2:
        raise ValueError(f"margin_frames must be even and at least 0 (got {M})")
    return W, M


def chunk_plan(T: int, window_frames: int, margin_frames: int, cfg: VocoderConfig = None) -> List[Tuple[int, int, int, int]]:
    """The chunks that vocode a mel of T frames with W = window_frames frames kept per chunk and M = margin_frames frames of
    context on each side: (start, length, crop_left, crop_right) per chunk, start and length in frames, the crops in samples
    of the chunk's vocoder_out_len(length) output.  Chunk i (i < ceil(T / W)) reads frames [s, e), s = max(0, i W - M), e =
    min(T, (i + 1) W + M), and keeps its samples [(i W - s) hop, (min(T, (i + 1) W) - s) hop); the last chunk keeps everything
    from (i W - s) hop to the end of its output, the vocoder's tail padding included.  The kept samples add up to
    vocoder_out_len(T), forward's length.  T = 0 has no chunks."""
    cfg = cfg or VocoderConfig()
    W, M = check_chunking(window_frames, margin_frames)
    n = -(-int(T) // W)
    out = []
    for i in range(n):
        s, e = max(0, i * W - M), min(T, (i + 1) * W + M)
        right = 0 if i == n - 1 else vocoder_out_len(e - s, cfg) - ((i + 1) * W - s) * cfg.hop
        out.append((s, e - s, (i * W - s) * cfg.hop, right))
    return out


def vocode_chunked(vocoder, mel: torch.Tensor, window_frames: int, margin_frames: int) -> torch.Tensor:
    """The reference composition of a chunked stream: chunk_plan(T, W, M)'s chunks of mel [T, 128], each through
    vocoder.forward on its torch slice alone, cropped and concatenated.  A StreamingVocoder stream's outputs are these bits."""
    cfg = getattr(vocoder, "voc_cfg", None) or VocoderConfig()
    kept = []
    for s, length, left, right in chunk_plan(int(mel.shape[0]), window_frames, margin_frames, cfg):
        out = vocoder.forward(mel[s:s + length][None, None])[0, 0]
        kept.append(out[left:out.numel() - right])
    return torch.cat(kept) if kept else mel.new_zeros(0)


def _grouped(frames, items, call, out_len):
    """call(packed items of a group, their lengths) per length_groups group -> one view per item, in the items' order"""
    out = [None] * len(items)
    for g in length_groups(frames):
        res = call(torch.cat([items[i] for i in g]), [int(items[i].shape[0]) for i in g])
        for i, v in zip(g, torch.split(res, [out_len(frames[i], items[i]) for i in g])):
            out[i] = v
    return out


def check_mels(mels, device) -> List[int]:
    """forward_batch's argument check, before anything is launched: a non-empty list of float32 [T_i, 128] tensors
    (T_i >= 1) on `device`.  Returns the frame counts."""
    if not isinstance(mels, (list, tuple)) or not mels:
        raise ValueError("forward_batch: expected a non-empty list of [T, 128] mels")
    for i, m in enumerate(mels):
        if not isinstance(m, torch.Tensor) or m.dim() != 2 or m.shape[-1] != 128 or m.shape[0] < 1:
            raise ValueError(f"forward_batch: mel {i} must be a [T, 128] tensor with T >= 1")
        if m.dtype != torch.float32 or m.device != device:
            raise TypeError(f"forward_batch: mel {i} must be float32 on {device} (got {m.dtype} on {m.device})")
    return [int(m.shape[0]) for m in mels]


class Vocoder(_EngineModel):
    """The pip package's stand-alone Vocoder (see the module docstring)."""
    _NEED = ("vocoder",)

    def __init__(self, sample_rate=44100, vocoder_config: VocoderConfig = None):
        if sample_rate != 44100:
            raise NotImplementedError("the vocoder is built for 44.1 kHz only")
        self.rate = sample_rate
        self.voc_cfg = vocoder_config or VocoderConfig()
        self.device = None
        self._eng = None
        self._state = None
        self.training = False

    def load_state_dict(self, state_dict, strict=True):
        """The vocoder's tensors under arch.vocoder_keys names, each with or without the "vocoder." prefix (other keys, e.g.
        a restorer's generator.*, are left out).  A missing tensor raises KeyError; strict=False is not supported."""
        names = {k for k, _ in vocoder_keys(self.voc_cfg)}
        st = {}
        for k, v in state_dict.items():
            if isinstance(v, torch.Tensor) and (k.startswith("vocoder.") or k in names):
                st[k if k.startswith("vocoder.") else "vocoder." + k] = v
        return super().load_state_dict(st, strict=strict)

    def _mel(self, mel, cuda):
        """forward's argument check: a float32 [B, 1, T, 128] tensor on the vocoder's device (with cuda=True also on the host,
        then moved there).  Every refusal comes before anything is launched."""
        if not isinstance(mel, torch.Tensor) or mel.dtype != torch.float32:
            raise TypeError("mel must be a float32 tensor")
        if mel.dim() != 4 or mel.shape[1] != 1 or mel.shape[-1] != 128 or mel.shape[0] < 1 or mel.shape[2] < 1:
            raise ValueError(f"mel must be [B, 1, T, 128] with B, T >= 1 (got {tuple(mel.shape)})")
        eng = self._engine()
        if mel.device != eng.device:
            if not cuda:
                raise RuntimeError(f"mel is on {mel.device}: pass cuda=True to move it to {eng.device} (there is no CPU path)")
            mel = mel.to(eng.device)
        return eng, mel

    def forward(self, mel, cuda=False):
        """mel [B, 1, T, 128] linear -> wav [B, 1, L], L = arch.vocoder_out_len(T): the clips through vf_vocoder_varlen, each
        the bits vf_vocoder gives it alone."""
        eng, mel = self._mel(mel, cuda)
        b, _, t, _ = mel.shape
        out = eng.vocoder_varlen(mel.reshape(b * t, 128), [t] * b)
        return out.view(b, 1, -1)

    def __call__(self, mel, cuda=False):
        return self.forward(mel, cuda=cuda)

    def forward_batch(self, mels: Sequence[torch.Tensor]) -> List[torch.Tensor]:
        """Mels of different lengths - a TTS batch, a test set - in packed calls, one per group of similar lengths
        (length_groups): mels is a list of float32 [T_i, 128] tensors on the vocoder's device; returns one view per clip
        into the packed outputs, [L_i] samples each, the bits forward(mel_i[None, None])[0, 0] gives."""
        eng = self._engine()
        frames = check_mels(mels, eng.device)
        return _grouped(frames, list(mels), eng.vocoder_varlen, lambda t, m: vocoder_out_len(t, self.voc_cfg))

    def resynth_batch(self, wavs: Sequence[torch.Tensor]) -> List[torch.Tensor]:
        """Vocoder resynthesis of clips of different lengths in packed calls (vf_resynth_varlen), one per group of similar
        lengths (length_groups): wavs is a list of 1-D float32 tensors on the vocoder's device, each longer than 1024
        samples; returns one view per clip, each its linear mel through the vocoder, peak normalised and trimmed back to the
        clip's length: the bits resynth_batch([wav_i]) gives."""
        eng, lengths = self._batch_engine(wavs)
        return _grouped([frames_for(n) for n in lengths], list(wavs), eng.resynth_varlen, lambda t, w: int(w.shape[0]))

    def oracle(self, fpath, out_path, cuda=True):
        """A wav file through handler() without the analysis module (module docstring): load_wav, 60 s segments,
        resynth_batch on them, save_wave to out_path."""
        from .handler import _check_file, load_wav, save_wave, segment_bounds
        if not cuda:
            raise RuntimeError("oracle: cuda=False is not available (there is no CPU path)")
        eng = self._engine()
        wav = load_wav(fpath, sample_rate=44100, engine=eng)
        _check_file(fpath, len(wav))
        segs = [torch.from_numpy(np.ascontiguousarray(wav[s:e])).to(eng.device) for s, e in segment_bounds(len(wav))]
        out = torch.cat(self.resynth_batch(segs))
        save_wave(out.cpu().numpy(), fname=out_path, sample_rate=44100)

    def oracle_batch(self, items, cuda=True):
        """oracle(fpath, out_path) for every (fpath, out_path) of `items`, with the segments of all files in one packed call
        per group (full 60 s segments, then the others, as handler_batch groups them).  Every file is decoded and checked
        before any GPU work, and files are written last; each output file has the bytes oracle writes for it."""
        from .handler import restore_test_set
        if not cuda:
            raise RuntimeError("oracle_batch: cuda=False is not available (there is no CPU path)")
        eng = self._engine()
        restore_test_set(self, [(i, o, None) for i, o in items], 0, False, False, eng.resynth_varlen, None)
