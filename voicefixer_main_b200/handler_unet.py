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

from .edges import AudioMetrics
from .handler import SEG_LENGTH, load_wav, restore_test_set, save_pcm16, segment_bounds
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
    for s, e in segment_bounds(wav_10k.shape[0]):
        seg = torch.from_numpy(np.ascontiguousarray(wav_10k[s:e]))[None, :].to(model.device)
        out = model.restore(seg)                                     # model(pre(segment)[0], segment)['wav']
        _, mel_out = model.pre(out[:, None])                         # mel(wav_to_spectrogram_phase(out)[0])
        if tgt is not None:
            tseg = torch.from_numpy(np.ascontiguousarray(tgt[s:s + SEG_LENGTH]))[None, None, :]
            metrics = _mel_metrics(model, mel_out, tseg.to(model.device))
        res.append(eng.finalize(out, out.shape[1]))                  # peak normalise; trim_center keeps equal lengths
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
    first: one call for the full 60 s segments and one for the others (handler.restore_test_set, handler.handler_batch's driver).
    The mel of every restored segment comes from that call when some item has a target.  Every file is decoded and checked
    before any GPU work: an item handler() would reject fails the whole call with handler()'s exception class, naming the
    file, and no file is written.  needrefresh reloads the model once.  All segments and their mels are held on the device
    at once: split a test set too large for that into several calls."""
    if needrefresh:
        refresh_model(ckpt)
    global model
    model = model.to(device)
    eng = model._engine()
    # mel-ssim is always computed here: a segment with a target needs SSIM's 7 frames
    return restore_test_set(
        model, items, 1, True, bool(meta.get("saturate", False)),
        lambda x, lengths, mel: eng.ssr_restore_varlen(x, lengths, mel_out=mel, peak_normalise=True),
        lambda tseg, mel: _mel_metrics(model, mel, tseg))
