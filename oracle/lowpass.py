"""tools/dsp/lowpass.py and collate_fn_val (dataloaders/data_module.py:130-150) restated with numpy / scipy in float64, and a
numpy restatement of vf_sosfiltfilt_varlen's chunked scan (voicefixer_main_b200/csrc/iir.cu).

The restatement calls the same scipy.signal functions as the reference, so with the same scipy it equals the reference's
outputs bit for bit (tests/golden/ref_lowpass.npz, written by oracle/make_golden_lowpass.py from the reference's own
module).  stft_hard_lowpass_v0 goes through oracle.vf_oracle's STFT / ISTFT, the stand-ins the reference's FDomainHelper
runs on under oracle/ref_import's shims.

The error bar of the GPU's IIR output is IIR_BAR * max|x| (see iir_bar): the scan's only error is fp64 rounding, about
eps = 1.1e-16 per operation.  A rounding error made in a state or output enters the rest of the row through the
cascade's impulse response, so the a priori bound is of order eps * (2 n_sections + 1) * gain, where gain is the l1 norm
of the cascade's impulse response (rounding_gain) - below 1e3 for every filter the tests use (ellip order 10 at 1 kHz is
the largest) - for each of the two passes, a few 1e-12 * max|x| at most.  1e-9 leaves two and a half orders of magnitude
above that and still lands a carry that is off by one chunk, or a float32 state, far outside it.
"""
import numpy as np
import torch
from scipy import signal

IIR_CHUNK = 1024          # iir.cu's chunk (kernels.cuh IIR_CHUNK)
IIR_BAR = 1e-9
SR_CUTOFFS = (1000, 2000, 4000, 8000, 12000)


def iir_bar(x) -> float:
    return IIR_BAR * float(np.max(np.abs(np.asarray(x, dtype=np.float64)))) if len(x) else 0.0


def rounding_gain(sos, n: int = 1 << 16) -> float:
    """l1 norm of the cascade's impulse response over n samples: how much one rounding error can grow."""
    imp = np.zeros(n)
    imp[0] = 1.0
    return float(np.abs(signal.sosfilt(sos, imp)).sum())


# ---- the reference's module (lowpass.py), restated


def limit(integer, high, low):
    if integer > high:
        return high
    elif integer < low:
        return low
    else:
        return int(integer)


def align_length(x, y):
    lx, ly = len(x), len(y)
    if lx == ly:
        return y
    if lx > ly:
        return np.pad(y, (0, lx - ly), mode="constant")
    return y[:lx]


def design(ftype, order, wn, btype):
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
    raise Exception(f"The {'bandpass' if btype == 'band' else 'lowpass'} filter {ftype} is not supported!")


def lowpass_filter(x, highcut, fs, order, ftype):
    return align_length(x, signal.sosfiltfilt(design(ftype, order, highcut / (0.5 * fs), "low"), x))


def bandpass_filter(x, lowcut, highcut, fs, order, ftype):
    nyq = 0.5 * fs
    return align_length(x, signal.sosfiltfilt(design(ftype, order, [lowcut / nyq, highcut / nyq], "band"), x))


def stft_hard_lowpass(data, lowpass_ratio, fs_ori=44100):
    fs_down = int(lowpass_ratio * fs_ori)
    y = signal.resample_poly(data, fs_down, fs_ori)
    y = signal.resample_poly(y, fs_ori, fs_down)
    return align_length(data, y)


def stft_hard_lowpass_v0(data, lowpass_ratio):
    from oracle import vf_oracle as O
    x = torch.tensor(np.asarray(data), dtype=torch.float32)
    sps, coss, sins = O.wav_to_spectrogram_phase(x[None, None])
    cut = int(sps.size()[-1] * lowpass_ratio)
    sps[..., cut:] = torch.zeros_like(sps[..., cut:])
    return O.istft(sps * coss, sps * sins, x.shape[0])[0].numpy()


def _check_1d(data):
    if len(list(data.shape)) != 1:
        raise ValueError("Error (chebyshev_lowpass_filter): Data " + str(data.shape) +
                         " should be type 1d time array, (samples,) , can not be (samples, 1)")


def lowpass(data, highcut, fs, order=5, _type="butter"):
    _check_1d(data)
    for ftype in ("butter", "cheby1", "ellip", "bessel"):
        if _type in ftype:
            return lowpass_filter(data, int(highcut), fs, limit(order, high=10, low=2), ftype)
    if _type in "stft":
        return stft_hard_lowpass(data, lowpass_ratio=highcut / int(fs / 2))
    if _type in "stft_hard":
        return stft_hard_lowpass_v0(data, lowpass_ratio=highcut / int(fs / 2))
    raise ValueError("Error: Unexpected filter type " + _type)


def bandpass(data, lowcut, highcut, fs, order=5, _type="butter"):
    _check_1d(data)
    for ftype in ("butter", "cheby1", "ellip", "bessel"):
        if _type in ftype:
            return bandpass_filter(data, int(lowcut), int(highcut), fs, limit(order, high=10, low=2), ftype)
    raise ValueError("Error: Unexpected filter type " + _type)


def collate_val(wavs, cutoffs=SR_CUTOFFS):
    """collate_fn_val's SR inputs of 1-D clips: {c: [float32 array per clip]} (each clip its own row, as batch_size 1
    gives it; stack_convert rounds the float64 result to float32)."""
    out = {}
    for c in cutoffs:
        out[c] = []
        for x in wavs:
            data = lowpass(x, highcut=c, fs=44100, order=8, _type="butter")
            out[c].append(lowpass(data, highcut=c, fs=44100, order=8, _type="stft").astype(np.float32))
    return out


# ---- vf_sosfiltfilt_varlen's chunked scan


def transition(sos, chunk=IIR_CHUNK, dtype=np.float64):
    """M: the state after `chunk` zero samples from each unit state (scipy's zi layout, flattened)."""
    ns = sos.shape[0]
    m = np.zeros((2 * ns, 2 * ns), dtype=dtype)
    for j in range(2 * ns):
        z = np.zeros((ns, 2), dtype=dtype)
        z.reshape(-1)[j] = 1.0
        _, zf = signal.sosfilt(sos, np.zeros(chunk, dtype=dtype), zi=z)
        m[:, j] = zf.reshape(-1)
    return m


def _scan(sos, x, s0, chunk, break_):
    """One pass: phase A (zero-state end states), phase B (s_{k+1} = M s_k + e_k), phase C (each chunk from its true state)."""
    dt = np.float32 if break_ == "float32_state" else np.float64
    m = transition(sos, chunk, dt)
    nc = -(-len(x) // chunk)
    chunks = [x[k * chunk:(k + 1) * chunk] for k in range(nc)]
    ends = [signal.sosfilt(sos, c, zi=np.zeros((sos.shape[0], 2)))[1].reshape(-1) for c in chunks[:-1]]
    starts, s = [], s0.reshape(-1).astype(dt)
    for k in range(nc):
        starts.append(s)
        if k < nc - 1:
            e = ends[k].astype(dt)
            s = e if (break_ == "skip_carry" and k == nc // 2) else (m @ s + e).astype(dt)
    return np.concatenate([signal.sosfilt(sos, c, zi=st.astype(np.float64).reshape(-1, 2))[0] for c, st in zip(chunks, starts)])


def chunked_sosfiltfilt(sos, x, chunk=IIR_CHUNK, break_=None):
    """sosfiltfilt(sos, x) as iir.cu computes it.  break_ selects one deliberately broken variant (tests only):
    "zi_unscaled", "even_ext", "edge+1", "edge-1", "float32_state", "skip_carry" (one chunk carry dropped), "drop_section"."""
    sos = np.asarray(sos, dtype=np.float64)
    x = np.asarray(x, dtype=np.float64)
    zb, za = int((sos[:, 2] == 0).sum()), int((sos[:, 5] == 0).sum())
    edge = 3 * (2 * sos.shape[0] + 1 - min(zb, za)) + {"edge+1": 1, "edge-1": -1}.get(break_, 0)
    zi = signal.sosfilt_zi(sos)
    if break_ == "drop_section":
        sos, zi = sos[:-1], zi[:-1]
    n = len(x)
    i = np.arange(n + 2 * edge)
    left, right = i < edge, i >= edge + n
    mid = np.clip(i - edge, 0, n - 1)
    ext = x[mid].copy()
    if break_ == "even_ext":
        ext[left] = x[edge - i[left]]
        ext[right] = x[n - 2 - (i[right] - edge - n)]
    else:
        ext[left] = 2 * x[0] - x[edge - i[left]]
        ext[right] = 2 * x[n - 1] - x[n - 2 - (i[right] - edge - n)]
    scale = (lambda v: 1.0) if break_ == "zi_unscaled" else (lambda v: v)
    y = _scan(sos, ext, zi * scale(ext[0]), chunk, break_)
    y = _scan(sos, y[::-1].copy(), zi * scale(y[-1]), chunk, break_)[::-1]
    return y[edge:-edge]
