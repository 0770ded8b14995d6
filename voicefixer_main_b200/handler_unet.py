"""Mirror of eval_gsr_unet.py (refresh_model :31-35, handler :37-75) and of eval_ssr_unet.py's handler (:95-143, the same
loop body) for the SSR / GSR-UNet models (unet_v2 on linear magnitudes + ISTFT) over the CUDA engine.

Both reference scripts fail as shipped: eval_gsr_unet.py builds the VoiceFixer class and then calls it as model(sp, segment),
and eval_ssr_unet.py imports modules that do not exist.  This module is the working form of their handler, with the contract
evaluation_proc/eval.py:128-132 calls:
    handler(input, output, target, ckpt, device, needrefresh=False, meta={}) -> dict of metrics
Per 60 s segment: restore; the linear mel of the restored output; with a target, the dict is replaced by the four mel metrics
of that output against the target's mel (so the last segment's values come back); peak normalise when max|out| > 1.  The
segments are concatenated and written as 16-bit PCM.  There is no unify_energy and no vocoder on this path; of `meta` only
"saturate" is read (as handler.handler does).  Decoding, resampling and the file writes are handler.py's.
handler_batch(items, ...) is handler() over a whole list of files, with the same files and dicts, as batched restores.
"""
import numpy as np
import torch

from .arch import frames_for
from .edges import AudioMetrics
from .handler import SEG_LENGTH, _check_file, _rate_len, _to_rate, load_wav, read_pcm16, save_pcm16, segment_bounds
from .model import GSR_UNet, SSR_UNet, default_hparams

model = None
hp = None


def _ssr_selected(h) -> bool:
    """hp["task"]["ssr"]["ssr_model"]["unet"] (config/vctk_base_ssr_unet_*.json); absent counts as false."""
    try:
        return bool(h["task"]["ssr"]["ssr_model"]["unet"])
    except KeyError:
        return False


def refresh_model(ckpt):
    global model
    h = hp if hp is not None else default_hparams()
    model = (SSR_UNet if _ssr_selected(h) else GSR_UNet)(h).load_from_checkpoint(ckpt)
    model.eval()


def _mel_metrics(mdl, mel_out, tseg) -> dict:
    """eval_gsr_unet.py:57-64 for one segment: mel_out [1, 1, T, 128] the linear mel of the restored output, tseg [1, 1, n] the
    clean target on the device.  Keys in the reference's order."""
    am = AudioMetrics(mdl)
    _, target_mel = mdl.pre(tseg)
    mel_out, target_mel = mel_out.contiguous(), target_mel.contiguous()
    return {
        "mel-lsd": float(am.lsd(mel_out, target_mel)),
        "mel-sispec": float(am.sispec(mel_out, target_mel, est_map=1, target_map=1)),     # to_log of both
        "mel-non-log-sispec": float(am.sispec(mel_out, target_mel)),
        "mel-ssim": float(am.ssim(mel_out, target_mel)),
    }


def handler(input, output, target, ckpt, device, needrefresh=False, meta={}):
    if needrefresh:
        refresh_model(ckpt)
    global model
    model = model.to(device)
    eng = model._engine()
    metrics = {}
    wav_10k = load_wav(input, sample_rate=44100, engine=eng)
    tgt = load_wav(target, sample_rate=44100, engine=eng) if target is not None else None
    res = []
    break_point = SEG_LENGTH
    while break_point < wav_10k.shape[0] + SEG_LENGTH:
        segment = wav_10k[break_point - SEG_LENGTH:break_point]
        seg = torch.from_numpy(np.ascontiguousarray(segment))[None, :].to(model.device)
        out = model.restore(seg)                                     # model(pre(segment)[0], segment)['wav']
        _, mel_out = model.pre(out[:, None])                         # mel(wav_to_spectrogram_phase(out)[0])
        if tgt is not None:
            tseg = torch.from_numpy(np.ascontiguousarray(tgt[break_point - SEG_LENGTH:break_point]))[None, None, :]
            metrics = _mel_metrics(model, mel_out, tseg.to(model.device))
        res.append(eng.finalize(out, out.shape[1]))                  # peak normalise; trim_center keeps equal lengths
        break_point += SEG_LENGTH
    if not res:          # torch.cat of nothing: RuntimeError in the reference's torch (ValueError in newer ones)
        raise RuntimeError(f"{input}: no samples to restore")
    out = torch.cat(res, -1)
    # save_wave's `max <= 1` branch always holds after the peak normalise: its int16 conversion runs on the GPU
    pcm = eng.to_pcm16(out[0], saturate=bool(meta.get("saturate", False)))
    save_pcm16(pcm.cpu().numpy(), fname=output, sample_rate=44100)
    return metrics


def handler_batch(items, ckpt, device, needrefresh=False, meta={}):
    """handler(input, output, target, ckpt, device, needrefresh, meta) for every (input, output, target) of `items`, in
    order, as batched restores: returns the list of metrics dicts, and every output file and dict is exactly what handler()
    gives that item.  The segments of all files go through vf_ssr_restore_varlen_mels with the peak normalise, longest
    first: one call for the full 60 s segments and one for the others (as handler.handler_batch does, for the same reason).
    The mel of every restored segment comes from that call when some item has a target.  Every file is decoded and checked
    before any GPU work: an item handler() would reject fails the whole call with handler()'s exception class, naming the
    file, and no file is written.  needrefresh reloads the model once.  All segments and their mels are held on the device
    at once: split a test set too large for that into several calls."""
    if needrefresh:
        refresh_model(ckpt)
    global model
    model = model.to(device)
    eng = model._engine()
    items = [tuple(it) for it in items]
    if not items:
        return []
    decoded = []
    for inp, _, tgt in items:
        x = read_pcm16(inp)
        t = read_pcm16(tgt) if tgt is not None else None
        # mel-ssim is always computed here: a segment with a target needs SSIM's 7 frames
        _check_file(inp, _rate_len(len(x[0]), x[1]), None if t is None else _rate_len(len(t[0]), t[1]), mel_ssim=True)
        decoded.append((x, t))
    sigs = [_to_rate(inp, *x, 44100, eng) for (inp, _, _), (x, _) in zip(items, decoded)]
    tgts = [None if t is None else _to_rate(tgt, *t, 44100, eng) for (_, _, tgt), (_, t) in zip(items, decoded)]
    segs = [(f, s, e) for f, x in enumerate(sigs) for s, e in segment_bounds(len(x))]    # (file, start, end), file order
    want_mels = any(t is not None for t in tgts)
    pcm, mels = [None] * len(segs), [None] * len(segs)   # per segment: int16 samples; mel [1, 1, T, 128] view
    full = [k for k, (_, s, e) in enumerate(segs) if e - s == SEG_LENGTH]
    rest = [k for k, (_, s, e) in enumerate(segs) if e - s < SEG_LENGTH]
    for group in (full, rest):
        if not group:
            continue
        order = sorted(group, key=lambda k: segs[k][1] - segs[k][2])                    # longest first, stable
        lengths = [segs[k][2] - segs[k][1] for k in order]
        off = np.concatenate([[0], np.cumsum(lengths)])
        f_off = np.concatenate([[0], np.cumsum([frames_for(n) for n in lengths])])
        packed = torch.from_numpy(np.concatenate([sigs[f][s:e] for f, s, e in (segs[k] for k in order)])).to(model.device)
        mel = torch.empty(int(f_off[-1]), 128, device=model.device) if want_mels else None
        out = eng.ssr_restore_varlen(packed, lengths, mel_out=mel, peak_normalise=True)
        # to_pcm16 is elementwise: one conversion of the packed output gives every file the bytes of its own conversion
        out16 = eng.to_pcm16(out, saturate=bool(meta.get("saturate", False))).cpu().numpy()
        for p, k in enumerate(order):
            pcm[k] = out16[off[p]:off[p + 1]]
            if want_mels:
                mels[k] = mel[int(f_off[p]):int(f_off[p + 1])][None, None]
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
        tseg = torch.from_numpy(np.ascontiguousarray(tgt[s:s + SEG_LENGTH]))[None, None, :].to(model.device)
        results.append(_mel_metrics(model, mels[k], tseg))
    for (_, output, _), ks in zip(items, file_segs):
        save_pcm16(np.concatenate([pcm[k] for k in ks]), fname=output, sample_rate=44100)
    return results
