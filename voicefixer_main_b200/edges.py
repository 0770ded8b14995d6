"""I/O edges of handler() on the GPU (SURVEY.md 8(f) rows 3-4): resampling to the model rate and the mel metrics.

* `resample_poly` / `resample_to`: zero-phase polyphase FIR rate conversion with the arithmetic of
  scipy.signal.resample_poly (Kaiser beta = 5 low-pass of 20 * max(up, down) + 1 taps), which is what the reference
  itself uses to change rates (tools/dsp/lowpass.py:138-141).  The reference's `load_wav` (tools/utils.py:46-48) calls
  librosa.load(sr=44100), whose resampler depends on the installed librosa (soxr_hq / kaiser_best) and is not available
  offline; the FIR here is of the same class (windowed-sinc, > 60 dB stop band) and is checked against scipy.
* `AudioMetrics.lsd` / `.sispec` / `.ssim`: evaluation_proc/metrics.py:83-106 for [B, C, T, F] tensors on the device, the
  metrics handler() logs per segment when a target is given (eval_gsr_voicefixer.py:56-64).
* `AudioMetrics.wav_to_spectrogram` / `.evaluation` / `.evaluation_batch`: scoring a restored file against its clean target
  (metrics.py:37-81), the second half of evaluation_proc/eval.py's evaluation().  The spectrogram is librosa 0.8's STFT
  (reflect padding; librosa >= 0.10 pads with zeros, not built) and SSIM is scikit-image <= 0.18's float64
  structural_similarity with data_range 2 (>= 0.19 computes float32 and needs data_range, not built).  sisdr, stoi and pesq
  come from the third-party speechmetrics package (CPU) and are not produced.

The filter design is host arithmetic (numpy); every sample / reduction is computed by libb200vf kernels (edges.cu).
"""
import ctypes
from fractions import Fraction

import numpy as np
import torch

from . import _lib as L
from .model import Engine, _check_in, _ptr, _stream


def design_filter(up: int, down: int) -> np.ndarray:
    """scipy.signal.resample_poly's default FIR: firwin(2 * half + 1, 1 / max(up, down), window=('kaiser', 5.0)) * up with
    half = 10 * max(up, down) (scipy/signal/_signaltools.py), restated with numpy: ideal low-pass sinc x Kaiser window,
    unity DC gain.  float64 taps, returned as float32."""
    max_rate = max(up, down)
    half = 10 * max_rate
    n = np.arange(-half, half + 1, dtype=np.float64)
    fc = 1.0 / max_rate                                    # cutoff as a fraction of Nyquist
    h = fc * np.sinc(fc * n) * np.kaiser(2 * half + 1, 5.0)
    h /= h.sum()
    return (h * up).astype(np.float32)


def resample_poly(eng: Engine, x: torch.Tensor, up: int, down: int) -> torch.Tensor:
    """x [B, N] float32 on the engine's device -> [B, ceil(N * up / down)]."""
    x = _check_in(x, eng.device, "x")
    g = np.gcd(int(up), int(down))
    up, down = int(up) // g, int(down) // g
    if up == down == 1:
        return x.clone()
    b, n = x.shape
    n_out = (n * up + down - 1) // down
    taps = torch.from_numpy(design_filter(up, down)).to(eng.device)
    out = torch.empty(b, n_out, device=eng.device)
    with torch.cuda.device(eng.device):
        eng._ck(eng.lib.vf_resample_poly(eng.ctx, _ptr(x), b, n, up, down, _ptr(taps), taps.numel(), _ptr(out), n_out, _stream()))
    return out


def resample_to(eng: Engine, x: torch.Tensor, rate_in: int, rate_out: int = 44100) -> torch.Tensor:
    """load_wav's rate conversion (tools/utils.py:46-48: librosa.load(path, sr=44100)) for a decoded signal."""
    fr = Fraction(int(rate_out), int(rate_in))
    return resample_poly(eng, x, fr.numerator, fr.denominator)


# AudioMetrics.evaluation's keys (metrics.py:70-78) in the column order of Engine.score_varlen
SCORE_KEYS = ("lsd", "non_log_sispec", "sispec", "ssim", "final_mel_lsd", "final_non_log_mel_sispec", "final_mel_sispec",
              "final_mel_ssim")


def check_rate(rate: int, what) -> None:
    """wav_to_spectrogram's rate branch (metrics.py:38-47): 44100 is built, 16000 (n_fft 743, hop 160, 80 mels) is not."""
    if rate == 16000:
        raise NotImplementedError(f"{what}: the 16 kHz metrics (n_fft 743, hop 160, 80 mels) are not built")
    if rate != 44100:
        raise ValueError(f"Bad Samplerate: {what} is {rate} Hz")


class AudioMetrics:
    """evaluation_proc/metrics.py:25-106 on the GPU: lsd, sispec and ssim of device tensors, the spectrogram and mel of a
    signal, and evaluation() of restored files against their targets."""

    def __init__(self, owner, rate: int = 44100):
        self.rate = rate
        self._owner = owner

    def _eng(self) -> Engine:
        return self._owner._engine() if hasattr(self._owner, "_engine") else self._owner

    def lsd(self, est: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        """metrics.py:83-87 (non-log inputs [B, C, T, F]) -> [B, C, 1, 1]."""
        eng = self._eng()
        est, target = _check_in(est, eng.device, "est"), _check_in(target, eng.device, "target")
        assert est.dim() == 4 and est.shape == target.shape
        b, c, t, f = est.shape
        out = torch.empty(b * c, device=eng.device)
        with torch.cuda.device(eng.device):
            eng._ck(eng.lib.vf_lsd(eng.ctx, _ptr(est), _ptr(target), b * c, t, f, _ptr(out), _stream()))
        return out.view(b, c, 1, 1)

    def sispec(self, est: torch.Tensor, target: torch.Tensor, est_map: int = 0, target_map: int = 0) -> torch.Tensor:
        """metrics.py:89-95: scalar = sum_b sp_loss[b] / B.  est_map / target_map fuse to_log (1) / from_log (2) of the
        operands (handler() passes to_log(target_mel) and from_log(out_model['mel']), eval_gsr_voicefixer.py:60-62).
        energy_unify's pow_norm sums per (batch, channel) and pow_p_norm per batch item (utils.py:81-101): identical for
        the single-channel tensors of this path, which is what is built."""
        eng = self._eng()
        est, target = _check_in(est, eng.device, "est"), _check_in(target, eng.device, "target")
        assert est.dim() == 4 and est.shape == target.shape and est.shape[1] == 1, "sispec: [B, 1, T, F] tensors"
        b = est.shape[0]
        n = est[0].numel()
        out = torch.empty(b, device=eng.device)
        with torch.cuda.device(eng.device):
            eng._ck(eng.lib.vf_sispec(eng.ctx, _ptr(est), _ptr(target), b, n, int(est_map), int(target_map), _ptr(out), _stream()))
        return torch.sum(out) / b

    def ssim(self, est: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        """metrics.py:97-106: structural_similarity(est[b, c], target[b, c], win_size=7) of [B, C, T, F] tensors ->
        float64 [B, C, 1, 1].  T or F below 7 raises ValueError, as scikit-image does."""
        eng = self._eng()
        if est.dim() != 4 or est.shape != target.shape:
            raise ValueError("ssim: est and target must be [B, C, T, F] tensors of one shape")
        b, c, t, f = est.shape
        if t < 7 or f < 7:
            raise ValueError(f"ssim: win_size 7 exceeds the {t} x {f} image")
        return eng.ssim(est.reshape(b * c, t, f), target.reshape(b * c, t, f)).view(b, c, 1, 1)

    def wav_to_spectrogram(self, wav, rate: int = 44100):
        """metrics.py:37-51 for one signal (numpy or tensor, 1-D): (sp [1, 1, T, 1025], mel [1, 1, T, 128]) on the device."""
        check_rate(rate, "wav")
        eng = self._eng()
        x = torch.as_tensor(np.ascontiguousarray(wav, dtype=np.float32) if not isinstance(wav, torch.Tensor) else wav)
        x = x.to(eng.device, torch.float32).reshape(-1).contiguous()
        sp, mel = eng.metric_spectrogram(x, [x.numel()])
        return sp[None, None], mel[None, None]

    def evaluation(self, est, target) -> dict:
        """metrics.py:53-81 for one (est, target) pair of wav paths: the 8 spectral keys; {} when target is None."""
        return self.evaluation_batch([(est, target)])[0]

    def evaluation_batch(self, pairs) -> list:
        """evaluation(est, target) of every pair, in order, in one vf_score_varlen call: each dict is float-identical to
        evaluation() of that pair.  Every file is decoded and checked before any GPU work; a bad pair fails the whole call,
        naming the file: a target at 16 kHz (NotImplementedError) or at another rate than 44.1 kHz (ValueError), an est
        whose frame count differs from its target's or a pair of fewer than 7 frames (ValueError)."""
        from .arch import frames_for
        from .handler import _rate_len, _to_rate, read_pcm16
        eng = self._eng()
        decoded = []
        for est, target in pairs:
            if target is None:
                decoded.append(None)
                continue
            t, rate = read_pcm16(target)
            check_rate(rate, target)
            e, e_rate = read_pcm16(est)
            te, tt = frames_for(_rate_len(len(e), e_rate, rate)), frames_for(len(t))
            if te != tt:
                raise ValueError(f"{est} has {te} frames at {rate} Hz, its target {target} {tt}")
            if tt < 7:
                raise ValueError(f"{est} / {target}: {tt} frames, fewer than SSIM's 7x7 window")
            decoded.append((est, e, e_rate, t))
        live = [d for d in decoded if d is not None]
        results = [{} for _ in decoded]
        if not live:
            return results
        ests = [_to_rate(path, e, e_rate, 44100, eng) for path, e, e_rate, _ in live]
        tgts = [t for _, _, _, t in live]
        scores = eng.score_varlen(torch.from_numpy(np.concatenate(ests)).to(eng.device), [len(e) for e in ests],
                                  torch.from_numpy(np.concatenate(tgts)).to(eng.device), [len(t) for t in tgts]).cpu()
        rows = iter(scores.tolist())
        for i, d in enumerate(decoded):
            if d is not None:
                results[i] = dict(zip(SCORE_KEYS, next(rows)))
        return results
