"""I/O edges of handler() on the GPU (SURVEY.md 8(f) rows 3-4): resampling to the model rate and the mel metrics.

* `resample_poly` / `resample_to`: zero-phase polyphase FIR rate conversion with the arithmetic of
  scipy.signal.resample_poly (Kaiser beta = 5 low-pass of 20 * max(up, down) + 1 taps), which is what the reference
  itself uses to change rates (tools/dsp/lowpass.py:138-141).  This is the default (res_type=None) everywhere.
* `resample` / `resample_to(..., res_type=...)`: what the reference's `load_wav` (tools/utils.py:46-48) and
  AudioMetrics.read (metrics.py:33-34) actually do, librosa.load(sr=...) with librosa 0.8, whose default resampler is
  resampy's "kaiser_best" sinc interpolation ("kaiser_fast" is its other filter).  Opt-in by res_type, named after
  librosa's argument; vf_resample_sinc_varlen computes it.  Parity status: restated, unpinned (oracle/resampy.py lists
  every choice; neither librosa nor resampy was available to check it against).  librosa >= 0.10's soxr_hq is not built.
* `AudioMetrics.lsd` / `.sispec` / `.ssim`: evaluation_proc/metrics.py:83-106 for [B, C, T, F] tensors on the device, the
  metrics handler() logs per segment when a target is given (eval_gsr_voicefixer.py:56-64).
* `AudioMetrics.wav_to_spectrogram` / `.evaluation` / `.evaluation_batch`: scoring a restored file against its clean target
  (metrics.py:37-81), the second half of evaluation_proc/eval.py's evaluation().  The spectrogram is librosa 0.8's STFT
  (reflect padding; librosa >= 0.10 pads with zeros, not built) and SSIM is scikit-image <= 0.18's float64
  structural_similarity with data_range 2 (>= 0.19 computes float32 and needs data_range, not built).  Both of the
  reference's geometries are built: 44.1 kHz (n_fft 2048, hop 441, 128 mels) and 16 kHz (n_fft 743, hop 160, 80 mels);
  an instance scores targets at its own rate, as aggregate_score builds one per test set (eval.py:43-45).
* `evaluation(..., time_domain=True)` / `evaluation_batch(..., time_domain=True)` add the sisdr and stoi keys, which the
  reference gets from the third-party speechmetrics package on the CPU (metrics.py:58-64): SI-SDR as speechmetrics
  computes it and pystoi 0.3.3's STOI, restated in oracle/speech_metrics.py and computed in float64 by
  vf_score_time_varlen.  pesq (ITU-T P.862, a large reference C program under its own licence) and bsseval are not
  produced.

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


def design_filter_f64(up: int, down: int) -> np.ndarray:
    """resample_poly's own float64 FIR for (up, down) already reduced by their gcd: scipy.signal.firwin(2 * half + 1,
    1 / max(up, down), window=('kaiser', 5.0)) * up with half = 10 * max(up, down), the taps of
    Engine.resample_poly_f64_varlen."""
    from scipy.signal import firwin
    max_rate = max(up, down)
    return firwin(2 * 10 * max_rate + 1, 1.0 / max_rate, window=("kaiser", 5.0)) * up


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


def resample_to(eng: Engine, x: torch.Tensor, rate_in: int, rate_out: int = 44100, res_type: str = None) -> torch.Tensor:
    """load_wav's rate conversion (tools/utils.py:46-48: librosa.load(path, sr=44100)) for decoded signals x [B, N]:
    resample_poly (res_type=None), or librosa 0.8's resample with `res_type` (see resample)."""
    if res_type is not None:
        return torch.stack(resample(eng, list(x), rate_in, rate_out, res_type))
    fr = Fraction(int(rate_out), int(rate_in))
    return resample_poly(eng, x, fr.numerator, fr.denominator)


# resampy's filters (resampy.filters.sinc_window parameters): res_type -> (num_zeros, precision, rolloff, Kaiser beta)
RES_TYPES = {
    "kaiser_best": (64, 9, 0.9475937167399596, 14.769656459379492),
    "kaiser_fast": (16, 7, 0.85, 8.555504641634386),
}


def check_res_type(res_type) -> None:
    """None (resample_poly) or one of RES_TYPES, else ValueError naming it."""
    if res_type is not None and res_type not in RES_TYPES:
        raise ValueError(f"unknown res_type {res_type!r}: need None, {' or '.join(map(repr, RES_TYPES))}")


def sinc_lengths(n: int, orig_sr: int, target_sr: int):
    """(resampy's int(n * ratio), librosa 0.8 resample's fix_length int(ceil(n * ratio))) for n samples, with the float64
    ratio = target_sr / orig_sr.  ValueError, as resampy raises it, when the first is 0."""
    ratio = float(target_sr) / orig_sr
    n_valid = int(n * ratio)
    if n_valid < 1:
        raise ValueError(f"Input signal length={n} is too small to resample from {orig_sr}->{target_sr}")
    return n_valid, int(np.ceil(n * ratio))


def sinc_table(res_type: str, sample_ratio: float) -> np.ndarray:
    """The float64 [nwin, 2] (win, delta) table resampy's loop reads for `res_type` at `sample_ratio`: resampy.filters'
    sinc_window(num_zeros, precision, rolloff, window=kaiser(beta)) = kaiser(2 n + 1)[n:] * (rolloff * sinc(rolloff *
    linspace(0, num_zeros, n + 1))) with n = 2^precision num_zeros, times sample_ratio when it is below 1; delta =
    diff(win) with a last entry 0."""
    from scipy.signal.windows import kaiser
    num_zeros, precision, rolloff, beta = RES_TYPES[res_type]
    n = 2 ** precision * num_zeros
    win = kaiser(2 * n + 1, beta)[n:] * (rolloff * np.sinc(rolloff * np.linspace(0, num_zeros, num=n + 1, endpoint=True)))
    if sample_ratio < 1:
        win = win * sample_ratio
    delta = np.zeros_like(win)
    delta[:-1] = np.diff(win)
    return np.stack([win, delta], axis=1)


def _sinc_filter(eng: Engine, res_type: str, orig_sr: int, target_sr: int):
    """(device table, sample_ratio, num_table) of Engine.resample_sinc_varlen, cached on the engine per (res_type, ratio)."""
    ratio = float(target_sr) / orig_sr
    cache = eng.__dict__.setdefault("_sinc_tables", {})
    if (res_type, ratio) not in cache:
        cache[res_type, ratio] = torch.from_numpy(sinc_table(res_type, ratio)).to(eng.device)
    return cache[res_type, ratio], ratio, 2 ** RES_TYPES[res_type][1]


class StreamFilter:
    """The filter of vf_resample_rings for one (rate_in, rate_out, res_type): family VF_RESAMPLE_POLY with up, down
    (reduced by their gcd) and taps (design_filter's float32 taps on the device), or VF_RESAMPLE_SINC with table (the
    float64 [nwin, 2] sinc_table on the device), ratio and num_table."""
    __slots__ = ("family", "up", "down", "taps", "table", "ratio", "num_table")


def stream_filter(eng: Engine, rate_in: int, rate_out: int, res_type: str = None) -> StreamFilter:
    """The StreamFilter converting rate_in to rate_out with res_type (None: resample_poly), cached on the engine per
    (rate_in, rate_out, res_type)."""
    check_res_type(res_type)
    cache = eng.__dict__.setdefault("_stream_filters", {})
    key = (int(rate_in), int(rate_out), res_type)
    if key not in cache:
        f = StreamFilter()
        if res_type is None:
            fr = Fraction(int(rate_out), int(rate_in))
            f.family, f.up, f.down = L.VF_RESAMPLE_POLY, fr.numerator, fr.denominator
            f.taps = torch.from_numpy(design_filter(f.up, f.down)).to(eng.device)
        else:
            f.family = L.VF_RESAMPLE_SINC
            f.table, f.ratio, f.num_table = _sinc_filter(eng, res_type, int(rate_in), int(rate_out))
        cache[key] = f
    return cache[key]


def resample(eng: Engine, ys, orig_sr, target_sr: int, res_type: str = "kaiser_best") -> list:
    """librosa 0.8 resample(y, orig_sr, target_sr, res_type, fix=True) of every 1-D float32 signal of `ys` (numpy arrays or
    tensors), all in one vf_resample_sinc_varlen call: orig_sr is one rate for all, or one per signal.  -> list of float32
    tensors on the engine's device; a signal already at target_sr comes back unchanged (on the device), as librosa returns
    it.  resampy's int(n * ratio) samples, then zeros up to int(ceil(n * ratio)).  An unknown res_type, or a signal too short
    for int(n * ratio) >= 1, raises ValueError before any GPU work."""
    if res_type is None:
        raise ValueError("resample: res_type None is resample_poly: call resample_to")
    check_res_type(res_type)
    rates = [int(orig_sr)] * len(ys) if np.ndim(orig_sr) == 0 else [int(r) for r in orig_sr]
    if len(rates) != len(ys):
        raise ValueError(f"resample: {len(rates)} rates for {len(ys)} signals")
    todo = [i for i, r in enumerate(rates) if r != target_sr]
    out_lengths = [sinc_lengths(int(np.prod(np.shape(ys[i]))), rates[i], target_sr)[1] for i in todo]
    xs = [torch.as_tensor(y).to(eng.device, torch.float32).reshape(-1) for y in ys]
    if not todo:
        return xs
    filters, keys, rows = [], {}, []
    for i in todo:
        if rates[i] not in keys:
            keys[rates[i]] = len(filters)
            filters.append(_sinc_filter(eng, res_type, rates[i], target_sr))
        rows.append(keys[rates[i]])
    y = eng.resample_sinc_varlen(torch.cat([xs[i] for i in todo]), [xs[i].numel() for i in todo], filters, rows, out_lengths)
    for i, part in zip(todo, torch.split(y, out_lengths)):
        xs[i] = part
    return xs


# AudioMetrics.evaluation's keys (metrics.py:70-78) in the column order of Engine.score_varlen
SCORE_KEYS = ("lsd", "non_log_sispec", "sispec", "ssim", "final_mel_lsd", "final_non_log_mel_sispec", "final_mel_sispec",
              "final_mel_ssim")
# its time-domain keys (metrics.py:58-64, without pesq) in the column order of Engine.score_time_varlen
TIME_KEYS = ("sisdr", "stoi")


RATES = (44100, 16000)      # wav_to_spectrogram's two branches (metrics.py:38-47)


def check_rate(rate: int, what, built: int = 44100) -> None:
    """wav_to_spectrogram's rate branch (metrics.py:38-47) for an AudioMetrics instance that scores at `built` Hz: a file at
    the other rate of RATES raises NotImplementedError naming the `rate=` it needs (aggregate_score builds one AudioMetrics
    per test set, evaluation_proc/eval.py:43-45), any other rate ValueError("Bad Samplerate ...")."""
    if rate == built:
        return
    if rate in RATES:
        raise NotImplementedError(f"{what} is at {rate} Hz: score it with AudioMetrics(..., rate={rate}), this instance "
                                  f"scores {built} Hz targets")
    raise ValueError(f"Bad Samplerate: {what} is {rate} Hz")


class AudioMetrics:
    """evaluation_proc/metrics.py:25-106 on the GPU: lsd, sispec and ssim of device tensors, the spectrogram and mel of a
    signal, and evaluation() of restored files against their targets."""

    def __init__(self, owner, rate: int = 44100, res_type: str = None):
        check_res_type(res_type)
        self.rate = rate
        self.res_type = res_type
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
        """metrics.py:37-51 for one signal (numpy or tensor, 1-D): (sp [1, 1, T, 1025], mel [1, 1, T, 128]) on the device, or
        at rate=16000 (sp [1, 1, T, 372], mel [1, 1, T, 80]); any instance computes both, as the reference's does."""
        if rate not in RATES:
            raise ValueError(f"Bad Samplerate: {rate} Hz")
        eng = self._eng()
        x = torch.as_tensor(np.ascontiguousarray(wav, dtype=np.float32) if not isinstance(wav, torch.Tensor) else wav)
        x = x.to(eng.device, torch.float32).reshape(-1).contiguous()
        sp, mel = eng.metric_spectrogram(x, [x.numel()]) if rate == 44100 else eng.metric_spectrogram(x, [x.numel()], rate=rate)
        return sp[None, None], mel[None, None]

    def evaluation(self, est, target, time_domain: bool = False) -> dict:
        """metrics.py:53-81 for one (est, target) pair of wav paths: the 8 spectral keys; {} when target is None.  With
        time_domain, also sisdr and stoi (see evaluation_batch)."""
        return self.evaluation_batch([(est, target)], time_domain=time_domain)[0]

    def evaluation_batch(self, pairs, time_domain: bool = False) -> list:
        """evaluation(est, target) of every pair, in order, in one vf_score_varlen call: each dict is float-identical to
        evaluation() of that pair.  The instance scores targets at its own rate, 44.1 kHz or 16 kHz (AudioMetrics(owner,
        rate=16000): n_fft 743, hop 160, 80 mels); an est at another rate is resampled to it on the GPU first, as
        librosa.load(sr=rate) does.  Every file is decoded (files other than 16-bit PCM in one vf_decode_pcm_varlen call,
        see handler.decode_wavs) and checked before any scoring; a bad pair fails the whole call, naming the file: a target at the other of the two rates (NotImplementedError naming the rate= it needs) or at any
        other rate (ValueError), an est whose frame count differs from its target's or a pair of fewer than 7 frames
        (ValueError).  The instance's res_type (None: resample_poly) picks how an est at another rate is resampled; with
        one, every such est goes through one edges.resample call, and the frame check uses librosa's resampled length.

        time_domain=True adds speechmetrics' sisdr and stoi (one more call, vf_score_time_varlen, on each file's first
        channel as speechmetrics reads it), and each dict is {"sisdr", "stoi", <the 8 spectral keys>} in metrics.py's
        order, without pesq.  The spectral values are those of time_domain=False.  The est must then be at its target's
        rate (ValueError naming it): speechmetrics would compare samples at two rates, which is not reproduced."""
        from .arch import metric_frames
        from .handler import _rate_len, _to_rate, decode_wavs
        rate = self.rate
        pairs = list(pairs)                  # read twice below: any iterable of pairs
        live_pairs = [(est, target) for est, target in pairs if target is not None]
        files = iter(decode_wavs([p for pair in live_pairs for p in pair], self._eng() if live_pairs else None,
                                 first=time_domain))
        decoded, channels = [], []
        for est, target in pairs:
            if target is None:
                decoded.append(None)
                continue
            e, e_rate, *e0 = next(files)
            t, t_rate, *t0 = next(files)
            check_rate(t_rate, target, rate)
            if time_domain and e_rate != rate:
                raise ValueError(f"{est} is at {e_rate} Hz: sisdr / stoi need it at its target's {rate} Hz")
            te, tt = metric_frames(_rate_len(len(e), e_rate, rate, self.res_type), rate), metric_frames(len(t), rate)
            if te != tt:
                raise ValueError(f"{est} has {te} frames at {rate} Hz, its target {target} {tt}")
            if tt < 7:
                raise ValueError(f"{est} / {target}: {tt} frames, fewer than SSIM's 7x7 window")
            decoded.append((est, e, e_rate, t))
            if time_domain:       # 7 frames are more than STOI's one frame at 10 kHz: no check of its own
                channels.append((e0[0], t0[0]))
        live = [d for d in decoded if d is not None]
        results = [{} for _ in decoded]
        if not live:
            return results
        eng = self._eng()
        at = {} if rate == 44100 else {"rate": rate}     # the 44.1 kHz calls are the entry points without a rate
        if self.res_type is None:
            ests = [_to_rate(path, e, e_rate, rate, eng) for path, e, e_rate, _ in live]
            est_packed = torch.from_numpy(np.concatenate(ests)).to(eng.device)
        else:
            ests = resample(eng, [e for _, e, _, _ in live], [e_rate for _, _, e_rate, _ in live], rate, self.res_type)
            est_packed = torch.cat(ests)
        tgts = [t for _, _, _, t in live]
        scores = eng.score_varlen(est_packed, [len(e) for e in ests],
                                  torch.from_numpy(np.concatenate(tgts)).to(eng.device), [len(t) for t in tgts], **at).cpu()
        rows = iter(scores.tolist())
        if time_domain:
            ests, tgts = [e for e, _ in channels], [t for _, t in channels]
            td = eng.score_time_varlen(torch.from_numpy(np.concatenate(ests)).to(eng.device), [len(e) for e in ests],
                                       torch.from_numpy(np.concatenate(tgts)).to(eng.device), [len(t) for t in tgts], **at)
            time_rows = iter(td.cpu().tolist())
        for i, d in enumerate(decoded):
            if d is not None:
                spectral = dict(zip(SCORE_KEYS, next(rows)))
                results[i] = dict(zip(TIME_KEYS, next(time_rows)), **spectral) if time_domain else spectral
        return results
