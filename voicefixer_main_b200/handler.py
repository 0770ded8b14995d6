"""Mirror of eval_gsr_voicefixer.py (pre :19-25, refresh_model :31-35, handler :37-77) over the CUDA engine.

Same signature and contract as the reference handler that evaluation_proc/eval.py:128-132 calls:
    handler(input, output, target, ckpt, device, needrefresh=False, meta={}) -> dict of metrics
It writes a 16-bit wav at `output`.  Differences, all outside the hot path: audio decoding uses the stdlib `wave`
module (librosa / soundfile are not in this image): PCM16 wav of ANY sample rate, converted to 44.1 kHz on the GPU by
the polyphase resampler (edges.py; load_wav -> librosa.load(sr=44100), tools/utils.py:46-48).  With a `target` the
per-segment mel metrics of eval_gsr_voicefixer.py:56-64 are computed on the GPU (lsd, sispec, non-log sispec, and with
meta["mel_ssim"] the reference's `mel-ssim`, evaluation_proc/metrics.py:97-106).
The segment loop, from_log, peak normalisation, trim_center, concat and the int16 conversion of
tools/file/wav.py:22-24 are reproduced exactly; the per-segment stages run as one fused launch chain.
handler_batch(items, ...) is handler() over a whole list of files, with the same files and dicts, as batched restores.
"""
import wave
from fractions import Fraction

import numpy as np
import torch

from ._lib import VF_EINVAL, EngineError
from .arch import frames_for
from .model import VoiceFixer, default_hparams

model = None
hp = None
SEG_LENGTH = 44100 * 60          # eval_gsr_voicefixer.py:47


def read_pcm16(path):
    """(mono float32 samples in [-1, 1), sample rate) of a 16-bit PCM wav."""
    with wave.open(path, "rb") as w:
        if w.getsampwidth() != 2:
            raise ValueError(f"{path}: need 16-bit PCM (got {8 * w.getsampwidth()} bit)")
        rate = w.getframerate()
        data = np.frombuffer(w.readframes(w.getnframes()), dtype=np.int16).reshape(-1, w.getnchannels())
    return (data.astype(np.float32) / 32768.0).mean(axis=1).astype(np.float32), rate


def load_wav(path, sample_rate=44100, engine=None):
    """tools/utils.py:46-48 (librosa.load(path, sr=sample_rate)): decode + convert to `sample_rate`.  Rate conversion
    runs on the GPU (`engine`, edges.resample_to); a file already at the target rate needs no engine."""
    return _to_rate(path, *read_pcm16(path), sample_rate, engine)


def _to_rate(path, wav, rate, sample_rate, engine):
    """load_wav's conversion of decoded samples `wav` at `rate` to `sample_rate`."""
    if rate == sample_rate:
        return wav
    if engine is None:
        raise ValueError(f"{path}: {rate} Hz input needs an engine for the GPU resampler (pass engine=model._engine())")
    from .edges import resample_to
    return resample_to(engine, torch.from_numpy(wav)[None].to(engine.device), rate, sample_rate)[0].cpu().numpy()


def _rate_len(n, rate, sample_rate=44100):
    """Length of what load_wav returns for n samples at `rate`: resample_poly's ceil(n * up / down)."""
    if rate == sample_rate:
        return n
    fr = Fraction(sample_rate, rate)
    return (n * fr.numerator + fr.denominator - 1) // fr.denominator


def save_wave(frames: np.ndarray, fname, sample_rate=44100):
    """tools/file/wav.py:10-27: scale by 2^15 when max <= 1 and truncate toward zero to int16."""
    frames = np.array(frames, dtype=np.float32, copy=True).reshape(-1)
    if np.max(frames) <= 1:
        frames *= 2 ** 15
    pcm = frames.astype(np.short)
    with wave.open(fname, "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(sample_rate)
        w.writeframes(pcm.tobytes())


def save_pcm16(pcm: np.ndarray, fname, sample_rate=44100):
    """Write already-converted int16 samples (VoiceFixer.restore_pcm16 / Engine.to_pcm16)."""
    with wave.open(fname, "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(sample_rate)
        w.writeframes(np.ascontiguousarray(pcm, dtype=np.int16).reshape(-1).tobytes())


def refresh_model(ckpt):
    global model
    model = VoiceFixer(hp if hp is not None else default_hparams(), channels=2, type_target="vocals").load_from_checkpoint(ckpt)
    model.eval()


def restore_array(mdl: VoiceFixer, wav_10k: np.ndarray, device, unify_energy: bool = False, target: np.ndarray = None,
                  metrics: dict = None, mel_ssim: bool = False) -> torch.Tensor:
    """The segment loop of handler() for one in-memory file: returns [1, N] on `device`.  With `target` (the clean
    signal, same rate) the mel metrics of the LAST segment land in `metrics`, as the reference's loop leaves them
    (eval_gsr_voicefixer.py:56-64 overwrites the dict every segment)."""
    res = []
    for s, e in segment_bounds(wav_10k.shape[0]):
        seg = torch.from_numpy(np.ascontiguousarray(wav_10k[s:e]))[None, :].to(device)
        res.append(mdl.restore(seg, unify_energy=unify_energy))
        if target is not None and metrics is not None:
            tseg = torch.from_numpy(np.ascontiguousarray(target[s:s + SEG_LENGTH]))[None, None, :].to(device)
            mel_noisy, log_mel = mdl._engine().restore_stages(1, seg.shape[1])
            metrics.update(_mel_metrics(mdl, tseg, mel_noisy[:, None], log_mel[:, None], unify_energy, mel_ssim))
    return torch.cat(res, -1)


def _mel_metrics(mdl: VoiceFixer, tseg, mel_noisy, log_mel, unify_energy: bool, mel_ssim: bool = False) -> dict:
    """eval_gsr_voicefixer.py:56-64 for one segment: tseg [1, 1, n] the clean target on the device, mel_noisy / log_mel
    [1, 1, T, 128] the restore's linear mel (stage A) and restored log10 mel (stage B).  mel_ssim adds "mel-ssim" (:63), the
    SSIM of the same mels as "mel-lsd"; a segment of fewer than 7 frames then raises ValueError, as skimage does."""
    from .edges import AudioMetrics
    am = AudioMetrics(mdl)
    eng = mdl._engine()
    _, target_mel = mdl.pre(tseg)
    denoised = eng.from_log(log_mel)
    if unify_energy:                     # eval_gsr_voicefixer.py:54-55 (tools/utils.py:50-55) before the lsd
        denoised = eng.amp_to_original_f(denoised[:, 0].contiguous(), mel_noisy[:, 0].contiguous())[:, None]
    res = {
        "mel-lsd": float(am.lsd(denoised.contiguous(), target_mel.contiguous())),
        "mel-sispec": float(am.sispec(log_mel, target_mel.contiguous(), target_map=1)),             # in log scale
        "mel-non-log-sispec": float(am.sispec(log_mel, target_mel.contiguous(), est_map=2)),
    }
    if mel_ssim:
        res["mel-ssim"] = float(am.ssim(denoised.contiguous(), target_mel.contiguous()))
    return res


def segment_bounds(n):
    """(start, end) of the segments of a file of n samples, as the reference's break_point loop cuts them
    (eval_gsr_voicefixer.py:47-74): SEG_LENGTH each, the last one ragged.  A segment's target slice is [start, start + SEG_LENGTH)."""
    return [(bp - SEG_LENGTH, min(bp, n)) for bp in range(SEG_LENGTH, n + SEG_LENGTH, SEG_LENGTH)]


def _check_file(path, n, n_target=None, mel_ssim=False):
    """Raises what handler() would raise on a file of n samples (at 44.1 kHz) with a target of n_target samples (None: no
    target), without touching the GPU: nothing to concatenate (RuntimeError); a segment, or the target slice of one, of at
    most 1024 samples, which the front end's reflect padding rejects (EngineError); a target slice with another frame count
    than its segment, which the metrics' shape check rejects (AssertionError); with mel_ssim, a segment with a target and
    fewer than 7 frames, which SSIM's 7x7 window rejects (ValueError).  Segments are checked in handler()'s order."""
    bounds = segment_bounds(n)
    if not bounds:
        raise RuntimeError(f"{path}: no samples to restore")
    for s, e in bounds:
        if e - s <= 1024:
            raise EngineError(VF_EINVAL, f"{path}: segment [{s}, {e}) has {e - s} samples; reflect padding needs more than 1024")
        if n_target is None:
            continue
        t = max(0, min(s + SEG_LENGTH, n_target) - s)
        if t <= 1024:
            raise EngineError(VF_EINVAL, f"{path}: the target slice of segment [{s}, {e}) has {t} samples; reflect padding "
                                         f"needs more than 1024")
        if frames_for(t) != frames_for(e - s):
            raise AssertionError(f"{path}: the target slice of segment [{s}, {e}) has {frames_for(t)} frames, the segment "
                                 f"{frames_for(e - s)}")
        if mel_ssim and frames_for(e - s) < 7:
            raise ValueError(f"{path}: segment [{s}, {e}) has {frames_for(e - s)} frames; mel-ssim's 7x7 window needs 7")


def handler(input, output, target, ckpt, device, needrefresh=False, meta={}):
    if needrefresh:
        refresh_model(ckpt)
    global model
    model = model.to(device)
    metrics = {}
    wav_10k = load_wav(input, sample_rate=44100, engine=model._engine())
    tgt = load_wav(target, sample_rate=44100, engine=model._engine()) if target is not None else None
    out = restore_array(model, wav_10k, model.device, unify_energy=bool(meta.get("unify_energy", False)), target=tgt, metrics=metrics,
                        mel_ssim=bool(meta.get("mel_ssim", False)))
    # save_wave's float -> int16 conversion runs on the GPU (its `max <= 1` condition always holds after the
    # per-segment peak normalisation), so only 2 bytes per sample cross PCIe.  meta["saturate"] (not in the reference)
    # clamps instead of reproducing numpy's +1.0 -> -32768 wrap, see INTEGRATION.md
    pcm = model._engine().to_pcm16(out[0], saturate=bool(meta.get("saturate", False)))
    save_pcm16(pcm.cpu().numpy(), fname=output, sample_rate=44100)
    return metrics


def handler_batch(items, ckpt, device, needrefresh=False, meta={}):
    """handler(input, output, target, ckpt, device, needrefresh, meta) for every (input, output, target) of `items`, in
    order, as one batched restore: returns the list of metrics dicts, and every output file and dict is exactly what
    handler() gives that item.  The segments of all files go through vf_restore_varlen_mels, longest first so that each
    sub-batch's bucket fits its clips: one call for the full 60 s segments and one for the others, instead of one restore
    (and one plan per distinct length) per segment.  Every file is decoded and checked before any GPU work: an item
    handler() would reject fails the whole call with handler()'s exception class, naming the file, and no file is written.
    needrefresh reloads the model once.  All segments and their mels are held on the device at once: split a test set too
    large for that into several calls."""
    if needrefresh:
        refresh_model(ckpt)
    global model
    model = model.to(device)
    eng = model._engine()
    unify, mel_ssim = bool(meta.get("unify_energy", False)), bool(meta.get("mel_ssim", False))
    return restore_test_set(
        model, items, 2, mel_ssim, bool(meta.get("saturate", False)),
        lambda x, lengths, mel, log_mel: eng.restore_varlen(x, lengths, unify_energy=unify, mel_out=mel, log_mel_out=log_mel),
        lambda tseg, mel, log_mel: _mel_metrics(model, tseg, mel, log_mel, unify, mel_ssim))


def restore_test_set(mdl, items, n_mels, mel_ssim, saturate, restore, score):
    """The body of handler_batch and handler_unet.handler_batch, which differ only in `restore` and `score`: the list of
    handler()'s dicts for `items`, and handler()'s output files, from batched restores.  Every item is decoded and checked
    (_check_file, with `mel_ssim`) before any GPU work.  Segments go longest first through
    restore(packed, lengths, *mel_bufs) -> the packed restored samples, where mel_bufs are `n_mels` packed [rows, 128]
    outputs when some item has a target and Nones otherwise.  score(tseg, *mels) -> dict scores a file's last segment: tseg
    [1, 1, n] its target slice on the device, mels its [1, 1, T, 128] rows of each buffer.  Files are written last."""
    eng = mdl._engine()
    items = [tuple(it) for it in items]
    if not items:
        return []
    decoded = []
    for inp, _, tgt in items:
        x = read_pcm16(inp)
        t = read_pcm16(tgt) if tgt is not None else None
        _check_file(inp, _rate_len(len(x[0]), x[1]), None if t is None else _rate_len(len(t[0]), t[1]), mel_ssim=mel_ssim)
        decoded.append((x, t))
    sigs = [_to_rate(inp, *x, 44100, eng) for (inp, _, _), (x, _) in zip(items, decoded)]
    tgts = [None if t is None else _to_rate(tgt, *t, 44100, eng) for (_, _, tgt), (_, t) in zip(items, decoded)]
    segs = [(f, s, e) for f, x in enumerate(sigs) for s, e in segment_bounds(len(x))]    # (file, start, end), file order
    want_mels = any(t is not None for t in tgts)
    pcm, mels = [None] * len(segs), [None] * len(segs)   # per segment: int16 samples; its [1, 1, T, 128] mel views
    # Full 60 s segments get a call of their own.  A call's longest clip sizes all of its sub-batches (plan budget), and a
    # 60 s segment needs the plan memory of about six 10 s clips: next to short clips it would cap every sub-batch at a few
    # clips, each sub-batch a plan of its own shape.
    full = [k for k, (_, s, e) in enumerate(segs) if e - s == SEG_LENGTH]
    rest = [k for k, (_, s, e) in enumerate(segs) if e - s < SEG_LENGTH]
    for group in (full, rest):
        if not group:
            continue
        order = sorted(group, key=lambda k: segs[k][1] - segs[k][2])                    # longest first, stable
        lengths = [segs[k][2] - segs[k][1] for k in order]
        off = np.concatenate([[0], np.cumsum(lengths)])
        f_off = np.concatenate([[0], np.cumsum([frames_for(n) for n in lengths])])
        packed = torch.from_numpy(np.concatenate([sigs[f][s:e] for f, s, e in (segs[k] for k in order)])).to(mdl.device)
        bufs = [torch.empty(int(f_off[-1]), 128, device=mdl.device) if want_mels else None for _ in range(n_mels)]
        out = restore(packed, lengths, *bufs)
        # to_pcm16 is elementwise: one conversion of the packed output gives every file the bytes of its own conversion
        out16 = eng.to_pcm16(out, saturate=saturate).cpu().numpy()
        for p, k in enumerate(order):
            pcm[k] = out16[off[p]:off[p + 1]]
            if want_mels:
                mels[k] = [b[int(f_off[p]):int(f_off[p + 1])][None, None] for b in bufs]
    file_segs = [[] for _ in items]
    for k, (f, _, _) in enumerate(segs):
        file_segs[f].append(k)
    results = []
    for f, tgt in enumerate(tgts):                 # handler() leaves the metrics of a file's last segment
        if tgt is None:
            results.append({})
            continue
        k = file_segs[f][-1]
        s = segs[k][1]
        tseg = torch.from_numpy(np.ascontiguousarray(tgt[s:s + SEG_LENGTH]))[None, None, :].to(mdl.device)
        results.append(score(tseg, *mels[k]))
    for (_, output, _), ks in zip(items, file_segs):
        save_pcm16(np.concatenate([pcm[k] for k in ks]), fname=output, sample_rate=44100)
    return results


# ---- the pip package's entry points (SURVEY.md 8(b): `VoiceFixer.restore(input, output, cuda, mode, your_vocoder_func)` /
# `restore_inmem(wav_10k, cuda, mode, your_vocoder_func)`; the package is not in /root/reference - the signatures and the
# 30 s segmentation follow the survey's description of it, mode 0 is the parity target)
PIP_SEG_LENGTH = 44100 * 30


def restore_inmem(mdl: VoiceFixer, wav_10k, cuda=True, mode=0, your_vocoder_func=None, unify_energy=True) -> np.ndarray:
    """One in-memory 44.1 kHz file -> restored samples [1, N] (numpy), 30 s segments, each
    pre -> analysis module -> from_log -> amp_to_original_f -> vocoder -> trim, concatenated.

    All whole segments of the file go through ONE batched restore call (the segments are independent), the ragged last
    one through a second.  cuda=False raises (there is no CPU path); mode 1 (pre low-pass) and mode 2 (train-mode
    BatchNorm) are not built.  `your_vocoder_func(mel [B,1,T,128] linear) -> wav [B,1,L]` replaces stage C; the stages
    then run one by one through the object protocol."""
    if not cuda:
        raise RuntimeError("restore_inmem: cuda=False is not available (there is no CPU path)")
    if mode != 0:
        raise NotImplementedError(f"restore_inmem: mode {mode} is not built (mode 0 only)")
    if mdl.device is None:
        raise RuntimeError("model is not on a CUDA device yet: call .to(device)")
    wav = torch.as_tensor(np.ascontiguousarray(wav_10k, dtype=np.float32)).reshape(-1)
    n = wav.shape[0]
    if n == 0:
        return np.zeros((1, 0), np.float32)
    n_full = n // PIP_SEG_LENGTH
    dev = wav.to(mdl.device)
    res = []

    def run(x):                                  # x [B, n_seg] on the device
        if your_vocoder_func is None:
            return mdl.restore(x, unify_energy=unify_energy)
        eng = mdl._engine()
        _, mel_noisy = mdl.pre(x[:, None])
        denoised = eng.from_log(mdl(mel_noisy)["mel"])
        if unify_energy:
            denoised = eng.amp_to_original_f(denoised[:, 0].contiguous(), mel_noisy[:, 0].contiguous())[:, None]
        out = your_vocoder_func(denoised)
        return mdl.finalize(out.to(mdl.device, torch.float32).contiguous(), x.shape[1])[:, 0]

    if n_full:
        res.append(run(dev[:n_full * PIP_SEG_LENGTH].view(n_full, PIP_SEG_LENGTH)).reshape(1, -1))
    if n > n_full * PIP_SEG_LENGTH:
        res.append(run(dev[None, n_full * PIP_SEG_LENGTH:].contiguous()))
    return torch.cat(res, -1).cpu().numpy()


def restore_file(mdl: VoiceFixer, input, output, cuda=True, mode=0, your_vocoder_func=None):
    """The package's `restore(input, output, cuda, mode, your_vocoder_func)`: wav file in, 16-bit 44.1 kHz wav out."""
    if not cuda:
        raise RuntimeError("restore: cuda=False is not available (there is no CPU path)")
    if mdl.device is None:
        raise RuntimeError("model is not on a CUDA device yet: call .to(device)")
    wav_10k = load_wav(input, sample_rate=44100, engine=mdl._engine())
    out = restore_inmem(mdl, wav_10k, cuda=cuda, mode=mode, your_vocoder_func=your_vocoder_func)
    save_wave(out, fname=output, sample_rate=44100)
