"""tools/dsp/lowpass.py on the GPU: the degradations of the speech super-resolution test sets.

The reference makes its SR validation inputs in dataloaders/data_module.py:130-150 (collate_fn_val): for each cutoff c in
{1000, 2000, 4000, 8000, 12000}, lowpass(x, c, 44100, order=8, _type="butter") and then lowpass(..., _type="stft").  This
module restates lowpass.py with the engine (or a model) as the first argument, so a test set can go clean -> degraded ->
restored -> scored without leaving the device.  Every function takes a 1-D numpy array or tensor and returns a tensor on the
engine's device.

* The IIR types (butter, cheby1, cheby2, ellip, bessel) design their second-order sections on the host with scipy.signal,
  as the reference does, and filter with vf_sosfiltfilt_varlen: scipy.signal.sosfiltfilt (padtype "odd") in float64, whose
  only error is fp64 rounding.  They return float64, as sosfiltfilt does.  Like numpy, the odd extension of a float32
  input is computed in float32 (the filtering is float64 either way).
* "stft" is stft_hard_lowpass: resample_poly down to int(ratio * 44100) and back up, vf_resample_poly_f64_varlen with
  resample_poly's own float64 taps, computed in float64 and returned as float64.  scipy 1.18 casts the FIR to the input's
  dtype, so on float32 input scipy itself computes in float32; on float64 input (what collate_fn_val hands it: the butter
  stage's output) every scipy version computes in float64, and that is the case this path reproduces.
* "stft_hard" is stft_hard_lowpass_v0: the front end's spectrogram (FDomainHelper 2048 / 441), the bins from
  int(1025 * ratio) up zeroed, and the ISTFT; float32, as the reference returns.

Dispatch copies the reference's quirks: the type is matched by substring test in the reference's order (`_type in
"butter"`, so "", "b" and "e" select butter), cheby2 is reachable only through lowpass_filter / bandpass_filter, the
order is clamped by limit(order, 10, 2), the IIR cutoffs are int()-ed, and "stft" takes lowpass_ratio = highcut /
int(fs / 2) with the original rate fixed at 44100 whatever fs is.  Every rejection (a 2-D input, an unknown type, a
cutoff outside (0, 1) of Nyquist, a signal not longer than sosfiltfilt's padlen, a zero down-sampled rate) raises the
reference's or scipy's exception before any GPU work.

lowpass_batch runs clips of different lengths in one launch chain, sr_validation_inputs is collate_fn_val's recipe, and
make_sr_testset writes such inputs as files and pair lists for handler_batch / evaluation_batch.
"""
import math
import os

import numpy as np
import torch
from scipy import signal

from .edges import design_filter_f64

SR_CUTOFFS = (1000, 2000, 4000, 8000, 12000)     # collate_fn_val's cutoffs (data_module.py:134)
_FS_ORI = 44100                                  # stft_hard_lowpass's fs_ori as lowpass() calls it


def _eng(owner):
    return owner._engine() if hasattr(owner, "_engine") else owner


def limit(integer, high, low):
    """lowpass.py:148-151."""
    if integer > high:
        return high
    elif integer < low:
        return low
    else:
        return int(integer)


def align_length(x, y):
    """lowpass.py:34-54: y padded with zeros at the end, or cut, to len(x)."""
    lx, ly = len(x), len(y)
    if lx == ly:
        return y
    if lx > ly:
        if isinstance(y, torch.Tensor):
            return torch.cat([y, y.new_zeros(lx - ly)])
        return np.pad(y, (0, lx - ly), mode="constant")
    return y[:lx]


def _design(ftype, order, wn, btype, kind):
    """The sos of lowpass_filter / bandpass_filter (lowpass.py:75-87, 115-126), by equality of ftype."""
    if ftype == "butter":
        return signal.butter(order, wn, btype=btype, output="sos")
    if ftype == "cheby1":
        return signal.cheby1(order, 0.1, wn, btype=btype, output="sos")
    if ftype == "cheby2":
        return signal.cheby2(order, 60, wn, btype=btype, output="sos")
    if ftype == "ellip":
        return signal.ellip(order, 0.1, 60, wn, btype=btype, output="sos")
    if ftype == "bessel":
        return signal.bessel(order, wn, btype=btype, output="sos")
    raise Exception(f"The {kind} filter {ftype} is not supported!")


def padlen(sos) -> int:
    """sosfiltfilt's default padlen: 3 * (2 n_sections + 1 - min(#(b2 == 0), #(a2 == 0)))."""
    sos = np.asarray(sos)
    ntaps = 2 * sos.shape[0] + 1 - min(int((sos[:, 2] == 0).sum()), int((sos[:, 5] == 0).sum()))
    return 3 * ntaps


def _iir(n, sos):
    edge = padlen(sos)
    if n <= edge:
        raise ValueError(f"The length of the input vector x must be greater than padlen, which is {edge}.")
    return ("iir", sos)


def _lowpass_spec(n, highcut, fs, order, ftype):
    """lowpass_filter's design and checks (lowpass.py:96-133) for a signal of n samples."""
    return _iir(n, _design(ftype, order, highcut / (0.5 * fs), "low", "lowpass"))


def _bandpass_spec(n, lowcut, highcut, fs, order, ftype):
    """bandpass_filter's (lowpass.py:57-94)."""
    nyq = 0.5 * fs
    return _iir(n, _design(ftype, order, [lowcut / nyq, highcut / nyq], "band", "bandpass"))


def _stft_spec(lowpass_ratio, fs_ori=_FS_ORI):
    """stft_hard_lowpass's two resample_poly calls (lowpass.py:135-145) as gcd-reduced (up, down) pairs."""
    fs_down = int(lowpass_ratio * fs_ori)
    if fs_down < 1:
        raise ValueError("up and down must be >= 1")
    g = math.gcd(fs_down, fs_ori)
    return ("stft", (fs_down // g, fs_ori // g))


def _check_1d(data):
    if len(list(data.shape)) != 1:
        raise ValueError("Error (chebyshev_lowpass_filter): Data " + str(data.shape) +
                         " should be type 1d time array, (samples,) , can not be (samples, 1)")


def _lowpass_row(data, highcut, fs, order, _type):
    """lowpass()'s dispatch (lowpass.py:153-187) -> the row's spec, every check done."""
    _check_1d(data)
    n = data.shape[0]
    for ftype in ("butter", "cheby1", "ellip", "bessel"):
        if _type in ftype:
            return _lowpass_spec(n, int(highcut), fs, limit(order, high=10, low=2), ftype)
    if _type in "stft":
        return _stft_spec(highcut / int(fs / 2))
    if _type in "stft_hard":
        return ("stft_hard", highcut / int(fs / 2))
    raise ValueError("Error: Unexpected filter type " + _type)


def _to_device(eng, data, dtype):
    if isinstance(data, torch.Tensor):
        return data.to(eng.device, dtype).reshape(-1).contiguous()
    return torch.from_numpy(np.ascontiguousarray(data, dtype=np.float64)).to(eng.device, dtype)


def _is_f32(data) -> bool:
    return data.dtype in (torch.float32, np.float32)


def _run_iir(eng, xs, soss, f32):
    """sosfiltfilt of each float64 device row with its sos, one vf_sosfiltfilt_varlen call (equal filters shared); f32[i]:
    row i came from float32 input."""
    index, filters, rows = {}, [], []
    for sos in soss:
        key = (sos.shape, sos.tobytes())
        if key not in index:
            index[key] = len(filters)
            filters.append(sos)
        rows.append(index[key])
    lengths = [x.numel() for x in xs]
    y = eng.sosfiltfilt_varlen(torch.cat(xs), lengths, filters, [signal.sosfilt_zi(s) for s in filters], rows, f32)
    return list(torch.split(y, lengths))


def _taps(eng, up, down):
    """resample_poly's float64 taps for (up, down) on the device, designed once per engine."""
    cache = eng.__dict__.setdefault("_resample_f64_taps", {})
    if (up, down) not in cache:
        cache[(up, down)] = torch.from_numpy(design_filter_f64(up, down)).to(eng.device)
    return cache[(up, down)]


def _resample_rows(eng, xs, rates, out_lengths):
    """resample_poly(x, up, down) of each float64 device row, align_length-ed to out_lengths, in one call."""
    index, filters, rows = {}, [], []
    for up, down in rates:
        if (up, down) not in index:
            index[(up, down)] = len(filters)
            filters.append((up, down, _taps(eng, up, down)))
        rows.append(index[(up, down)])
    y = eng.resample_poly_f64_varlen(torch.cat(xs), [x.numel() for x in xs], filters, rows, out_lengths)
    return list(torch.split(y, out_lengths))


def _run_stft(eng, xs, rates, f32=None):
    """stft_hard_lowpass of each row: down to fs_down, back up, align_length to the input (copies where up == down)."""
    outs = [x.clone() if r == (1, 1) else None for x, r in zip(xs, rates)]
    live = [i for i, r in enumerate(rates) if r != (1, 1)]
    if live:
        xl = [xs[i] for i in live]
        rl = [rates[i] for i in live]
        mid = _resample_rows(eng, xl, rl, [-(-x.numel() * u // d) for x, (u, d) in zip(xl, rl)])
        back = _resample_rows(eng, mid, [(d, u) for u, d in rl], [x.numel() for x in xl])
        for i, y in zip(live, back):
            outs[i] = y
    return outs


def stft_hard_lowpass_v0(eng, data, lowpass_ratio):
    """lowpass.py:21-32: zero the spectrogram bins from int(1025 * lowpass_ratio) up and resynthesise with the input phase
    (the front end's STFT, vf_istft) -> float32."""
    eng = _eng(eng)
    x = _to_device(eng, data, torch.float32)
    _, sp, cos, sin = eng.frontend(x[None], want_sp=True, want_phase=True, want_mel=False)
    cut = int(sp.size()[-1] * lowpass_ratio)
    sp[..., cut:] = 0
    return eng.istft((sp * cos).contiguous(), (sp * sin).contiguous(), x.numel())[0]


def stft_hard_lowpass(eng, data, lowpass_ratio, fs_ori=44100):
    """lowpass.py:135-145, in float64 (see the module docstring for float32 input)."""
    eng = _eng(eng)
    _, rate = _stft_spec(lowpass_ratio, fs_ori)
    return _run_stft(eng, [_to_device(eng, data, torch.float64)], [rate])[0]


def lowpass_filter(eng, x, highcut, fs, order, ftype):
    """lowpass.py:96-133 (cheby2 included) -> float64."""
    eng = _eng(eng)
    _check_1d(x)
    _, sos = _lowpass_spec(x.shape[0], highcut, fs, order, ftype)
    return _run_iir(eng, [_to_device(eng, x, torch.float64)], [sos], [_is_f32(x)])[0]


def bandpass_filter(eng, x, lowcut, highcut, fs, order, ftype):
    """lowpass.py:57-94 (cheby2 included) -> float64."""
    eng = _eng(eng)
    _check_1d(x)
    _, sos = _bandpass_spec(x.shape[0], lowcut, highcut, fs, order, ftype)
    return _run_iir(eng, [_to_device(eng, x, torch.float64)], [sos], [_is_f32(x)])[0]


def lowpass(eng, data, highcut, fs, order=5, _type="butter"):
    """lowpass.py:153-187: float64 for the IIR types and "stft", float32 for "stft_hard"."""
    return lowpass_batch(eng, [data], [highcut], [order], [_type], fs)[0]


def bandpass(eng, data, lowcut, highcut, fs, order=5, _type="butter"):
    """lowpass.py:189-216 -> float64."""
    eng = _eng(eng)
    _check_1d(data)
    for ftype in ("butter", "cheby1", "ellip", "bessel"):
        if _type in ftype:
            _, sos = _bandpass_spec(data.shape[0], int(lowcut), int(highcut), fs, limit(order, high=10, low=2), ftype)
            return _run_iir(eng, [_to_device(eng, data, torch.float64)], [sos], [_is_f32(data)])[0]
    raise ValueError("Error: Unexpected filter type " + _type)


def lowpass_batch(eng, wavs, highcuts, orders, types, fs=44100):
    """lowpass(eng, wavs[i], highcuts[i], fs, orders[i], types[i]) of every clip, clips of different lengths, in one
    vf_sosfiltfilt_varlen call for the IIR rows and two vf_resample_poly_f64_varlen calls for the "stft" rows.  Each
    result is bit-identical to that clip's own lowpass().  Every clip is checked before any GPU work."""
    eng = _eng(eng)
    if not (len(wavs) == len(highcuts) == len(orders) == len(types)):
        raise ValueError("lowpass_batch: wavs, highcuts, orders and types must have one entry per clip")
    specs = [_lowpass_row(w, h, fs, o, t) for w, h, o, t in zip(wavs, highcuts, orders, types)]
    outs = [None] * len(wavs)
    for kind, run in (("iir", _run_iir), ("stft", _run_stft)):
        idx = [i for i, s in enumerate(specs) if s[0] == kind]
        if idx:
            ys = run(eng, [_to_device(eng, wavs[i], torch.float64) for i in idx], [specs[i][1] for i in idx],
                     [_is_f32(wavs[i]) for i in idx])
            for i, y in zip(idx, ys):
                outs[i] = y
    for i, s in enumerate(specs):
        if s[0] == "stft_hard":
            outs[i] = stft_hard_lowpass_v0(eng, wavs[i], s[1])
    return outs


def sr_validation_inputs(eng, wavs, cutoffs=SR_CUTOFFS):
    """collate_fn_val's SR inputs (data_module.py:130-150) of each clip (1-D, 44.1 kHz): for each cutoff c, lowpass(x, c,
    44100, order=8, "butter") then lowpass(..., "stft") in float64, rounded once to float32 as stack_convert does ->
    {c: [float32 device tensor per clip]}, ready for restore_batch."""
    eng = _eng(eng)
    rows = [(c, w) for c in cutoffs for w in wavs]
    cs = [c for c, _ in rows]
    butter = lowpass_batch(eng, [w for _, w in rows], cs, [8] * len(rows), ["butter"] * len(rows), 44100)
    stft = lowpass_batch(eng, butter, cs, [8] * len(rows), ["stft"] * len(rows), 44100)
    out = {c: [] for c in cutoffs}
    for (c, _), y in zip(rows, stft):
        out[c].append(y.float())
    return out


def make_sr_testset(eng, clean_paths, out_dir, cutoffs=SR_CUTOFFS, list_type="cheby1"):
    """Write sr_validation_inputs of 44.1 kHz clean WAV files (any format, decoded in one handler.decode_wavs call) as
    out_dir/<list_type>/<c>/<file name> (16-bit PCM as save_wave converts it) and, per cutoff, the pair list
    out_dir/<list_type>/pair_<list_type>_<c>.lst of "degraded clean" lines in evaluation_proc/config.py's format, which
    handler_batch and evaluation_batch items can be read from.  Returns {c: list path}.

    list_type only names the files where config.py's SSR_DATA looks for them (SSR_ROOT/cheby1/pair_cheby1_<c>.lst).  The
    recipe of the downloaded vctk_cheby1_* test files is not in the reference tree; this writes collate_fn_val's
    validation recipe (butter order 8 + resample) and makes no claim to reproduce those files.

    Every file is checked before any GPU work or write: a path with white space, two clean files of one name (their
    degraded copies would overwrite each other) or a file not at 44.1 kHz raises ValueError naming it."""
    from .handler import decode_wavs, save_pcm16
    eng = _eng(eng)
    clean_paths = list(clean_paths)          # read three times below: any iterable of paths
    names = {}
    for path in clean_paths:
        if any(ch.isspace() for ch in str(path)) or any(ch.isspace() for ch in str(out_dir)):
            raise ValueError(f"{path}: the pair-list format cannot hold paths with white space")
        name = os.path.basename(path)
        if name in names:
            raise ValueError(f"{path} and {names[name]} share the file name {name}: their degraded copies would collide")
        names[name] = path
    clean = []
    for path, (x, rate) in zip(clean_paths, decode_wavs(clean_paths, eng)):
        if rate != 44100:
            raise ValueError(f"{path} is at {rate} Hz: the SR recipe needs 44.1 kHz input")
        clean.append(x)
    inputs = sr_validation_inputs(eng, clean, cutoffs)
    lists = {}
    for c in cutoffs:
        d = os.path.join(out_dir, list_type, str(c))
        os.makedirs(d, exist_ok=True)
        lines = []
        for path, y in zip(clean_paths, inputs[c]):
            dst = os.path.join(d, os.path.basename(path))
            save_pcm16(eng.to_pcm16(y).cpu().numpy(), dst)
            lines.append(f"{os.path.abspath(dst)} {os.path.abspath(path)}\n")
        lists[c] = os.path.join(out_dir, list_type, f"pair_{list_type}_{c}.lst")
        with open(lists[c], "w") as f:
            f.writelines(lines)
    return lists
