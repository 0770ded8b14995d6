"""CPU restatement of the VoiceFixer pip package's pre-filter, `VoiceFixer.remove_higher_frequency(wav, ratio=0.95)`
(voicefixer/base.py), which `restore_inmem(..., mode=1)` applies to each 30 s segment before restoring it.  TEST
INFRASTRUCTURE.

The package is not in the reference tree and librosa is not in this image, so the method is restated from recollection.
Parity status: restated, unpinned.  What it does, with librosa 0.8's stft / istft defaults:

    stft = librosa.stft(wav)                 # n_fft 2048, hop 512, periodic hann, center, reflect pad
    mag = |stft|; cos, sin = re / (mag + EPS), im / (mag + EPS);  spec = |stft|
    feature = log10(spec + EPS); feature[feature < 0] = 0
    energy_level = sum(feature, axis=1)      # per bin, over frames
    threshold = sum(energy_level) * ratio
    i = first bin whose running sum energy_level[0] + ... + energy_level[i] is >= threshold
    spec[i:] = 0
    return librosa.istft(spec * cos + 1j * spec * sin)      # window-sum normalised, length None

Consequences: the output has 512 * (n // 512) samples; only bins with |X| >= 1 count, so a quiet clip has all energies 0,
cutoff 0 and an all-zero output; the kept bins are scaled by |X| / (|X| + EPS).  When rounding makes the running sum
miss the threshold at the last bin (reachable only with ratio near 1), the package would raise IndexError; both
functions here, like the kernels, keep every bin then (cutoff 1025).

`remove_higher_frequency` is the float64 reference of vf_remove_higher_frequency_varlen, summed in the kernels' orders:
per-bin energies over frames in ascending order, the total over bins in ascending order (so the scan's running sums are
its prefix sums), overlap-add over frames in ascending order.  `remove_higher_frequency_pkg` keeps the package's dtypes
(a complex64 spectrum, float32 magnitudes, log10 and sums, numpy's pairwise total, the float64 threshold of numpy 1.x
promotion, a float32 overlap-add); it measures what the float64 choice moves.
"""
import numpy as np
import scipy.signal

EPS = 1e-8
N_FFT, HOP = 2048, 512
BINS = N_FFT // 2 + 1


def _window():
    return scipy.signal.get_window("hann", N_FFT)          # periodic, float64


def _frames(x):
    """[T, 2048] float64 frames of the reflect-padded clip (np.pad reflects repeatedly when n <= 1024), T = 1 + n // 512."""
    x = np.asarray(x)
    n = x.shape[0]
    pad = np.pad(x.astype(np.float64), N_FFT // 2, mode="reflect")
    T = 1 + n // HOP
    idx = np.arange(T)[:, None] * HOP + np.arange(N_FFT)[None, :]
    return pad[idx]


def _ola(frames, n, dtype):
    """librosa 0.8 istft's overlap-add of windowed frames [T, 2048] and its window_sumsquare division (where the sum is
    above float32 tiny), trimmed to 512 * (n // 512) samples.  Frames are added in ascending order into `dtype`."""
    T = frames.shape[0]
    w2 = _window() ** 2
    L = N_FFT + HOP * (T - 1)
    y = np.zeros(L, dtype)
    ws = np.zeros(L, dtype)
    for t in range(T):
        y[t * HOP:t * HOP + N_FFT] += frames[t]
        ws[t * HOP:t * HOP + N_FFT] += w2
    keep = ws > np.finfo(np.float32).tiny
    y[keep] /= ws[keep]
    return y[N_FFT // 2:N_FFT // 2 + HOP * (n // HOP)]


def _scan(energy, threshold, dtype):
    """The package's while loop: the first bin i whose running sum reaches the threshold (1025 when none does)."""
    cur, i = energy[0], 0
    while i < BINS and cur < threshold:
        if i + 1 == BINS:
            return BINS
        cur = dtype(cur + energy[i + 1])
        i += 1
    return i


def _check(x, ratio):
    x = np.asarray(x)
    if x.ndim != 1 or x.shape[0] < 1:
        raise ValueError("remove_higher_frequency: need a 1-D clip of at least one sample")
    if not 0 < ratio <= 1:
        raise ValueError(f"remove_higher_frequency: ratio {ratio} (need 0 < ratio <= 1)")
    return x


def remove_higher_frequency(x, ratio=0.95, eps=EPS, cutoff=None):
    """float64 pre-filter of the float32 clip x -> (output float64 [512 * (n // 512)], cutoff, margin), margin =
    min(|cum(i - 1) - threshold|, |cum(i) - threshold|) of the chosen bin i (inf where a side does not exist).  A given
    `cutoff` replaces the scan's (the margin is then that of the scan); eps=0 with cutoff=1025 removes nothing and makes
    the pair a plain stft -> istft round trip."""
    x = _check(x, ratio)
    w = _window()
    X = np.fft.rfft(_frames(x) * w, axis=1)                 # [T, 1025] complex128
    re, im = X.real, X.imag
    mag = np.hypot(re, im)
    feature = np.maximum(np.log10(mag + eps), 0.0)
    energy = np.zeros(BINS)
    for t in range(feature.shape[0]):                       # ascending frames, one running sum per bin
        energy += feature[t]
    threshold = float(np.cumsum(energy)[-1]) * ratio        # ascending bins: the scan's own running sums
    found = _scan(energy, threshold, np.float64)
    cum_all = np.cumsum(energy)
    lo = abs(cum_all[found - 1] - threshold) if found > 0 else np.inf
    hi = abs(cum_all[found] - threshold) if found < BINS else np.inf
    cutoff = found if cutoff is None else cutoff
    keep = np.arange(BINS) < cutoff
    Y = np.where(keep, mag * (re / (mag + eps)), 0.0) + 1j * np.where(keep, mag * (im / (mag + eps)), 0.0)
    frames = np.fft.irfft(Y, n=N_FFT, axis=1) * w
    return _ola(frames, x.shape[0], np.float64), cutoff, min(lo, hi)


def remove_higher_frequency_pkg(x, ratio=0.95):
    """The package's dtypes: float32 clip -> (float32 output [512 * (n // 512)], cutoff)."""
    x = _check(x, ratio)
    w = _window()
    X = np.fft.rfft(_frames(np.asarray(x, np.float32)) * w, axis=1).astype(np.complex64)   # librosa's complex64 matrix
    re, im = X.real, X.imag
    mag = np.sqrt(re ** 2 + im ** 2)
    cos, sin = re / (mag + np.float32(EPS)), im / (mag + np.float32(EPS))
    spec = np.abs(X)
    feature = np.log10(spec + np.float32(EPS))
    feature[feature < 0] = 0
    energy = np.zeros(BINS, np.float32)
    for t in range(feature.shape[0]):                       # [1025, T] Fortran-ordered: sequential over frames
        energy += feature[t]
    threshold = np.float64(np.sum(energy)) * ratio          # float32 pairwise total, float64 product (numpy 1.x)
    cutoff = _scan(energy, threshold, np.float32)
    spec[:, cutoff:] = 0
    Y = (spec * cos + 1j * spec * sin).astype(np.complex64)
    frames = np.fft.irfft(Y, n=N_FFT, axis=1) * w             # float64 irfft of the complex64 matrix
    return _ola(frames, x.shape[0], np.float32), cutoff
