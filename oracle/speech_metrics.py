"""CPU restatement of the time-domain keys of AudioMetrics.evaluation (evaluation_proc/metrics.py:58-64).  TEST INFRASTRUCTURE.

The reference gets sisdr and stoi from the third-party speechmetrics package, which calls pystoi; neither is in this
image nor in the reference tree.  Their arithmetic is restated here in float64 with numpy / scipy.  Parity status:
restated, unpinned by the reference.  The choices below follow the published packages as recalled; they have NOT been
checked against those packages' source.

speechmetrics (2020-2021 master), as the reference calls it: sm.load(['sisdr', 'stoi', 'pesq', 'bsseval'], np.inf), then
metrics(est_path, target_path, rate=rate):
* each file is read with soundfile as float64 (int16 / 32768 for PCM16) and its first channel is used;
* the shorter signal is zero-padded at the end to the longer one; window np.inf makes the whole signal one window;
* sisdr, with r = target and e = estimate: eps = np.finfo(np.float64).eps, a = (eps + r.e) / (r.r + eps),
  Sss = sum (a r)^2, Snn = sum (e - a r)^2 (a second pass, no expansion), sisdr = 10 log10((eps + Sss) / (eps + Snn));
  there is no mean removal;
* stoi = pystoi.stoi(x=target, y=estimate, fs_sig=rate, extended=False).
pystoi 0.3.3:
1. resample_oct(., 10000, 44100): scipy.signal.resample_poly(x, 100, 441, window=h / h.sum()), h Octave's resample window:
   L = ceil((60 - 8) / (28.714 * (1 / 882) / 10)) = 15973, h = kaiser(2L + 1, 0.1102 * (60 - 8.7)) * 2 * 100 * (1 / 882) *
   sinc(2 * (1 / 882) * t), t = -L..L; resample_poly multiplies the given window by up.  ceil(n * 100 / 441) samples.
2. remove_silent_frames(x, y, 40, 256, 128): w = np.hanning(258)[1:-1]; frames start at range(0, len - 256, 128) (the last
   possible frame is excluded); energy 20 log10(||w x_frame|| + eps) of the target only; a frame is kept where
   max - 40 - energy < 0, for both signals; the kept windowed frames are overlap-added at hop 128 into (K - 1) * 128 + 256
   samples.
3. STFT of both: window w, frames at range(0, len - 256, 128), rfft(n=512), 257 bins.
4. thirdoct(10000, 512, 15, 150): band k = bins [fl, fh), the nearest bins (first of ties) to 150 * 2^((2k -+ 1) / 6);
   the band value is sqrt(sum |X|^2).
5. For every 30-frame segment (m = 30..M) and band: y <- y * ||x|| / (||y|| + eps); clip y to x * (1 + 10^(15 / 20));
   subtract the means; divide both by (||.|| + eps); correlate.  d = sum of the correlations / (J * 15), J segments.
   With fewer than 30 frames pystoi warns and returns 1e-5.

`VARIANTS` holds deliberately broken restatements (tests/test_speech_metrics_cpu.py shows each one lands far from this one).
"""
import wave

import numpy as np
import scipy.signal

EPS = np.finfo(np.float64).eps
FS, N_FRAME, HOP, NFFT, NUMBAND, MINFREQ, N_SEG, BETA, DYN_RANGE = 10000, 256, 128, 512, 15, 150, 30, -15.0, 40
KEYS = ("sisdr", "stoi")


def octave_window(p: int = 100, q: int = 441):
    """(h, L, beta) of pystoi's _resample_window_oct(p, q) (a port of Octave's resample.m filter), unnormalised."""
    stopband_cutoff_f = 1.0 / (2 * max(p, q))
    roll_off_width = stopband_cutoff_f / 10
    rejection_db = 60.0
    L = int(np.ceil((rejection_db - 8) / (28.714 * roll_off_width)))
    t = np.arange(-L, L + 1, dtype=np.float64)
    ideal = 2 * p * stopband_cutoff_f * np.sinc(2 * stopband_cutoff_f * t)
    beta = 0.1102 * (rejection_db - 8.7)
    return np.kaiser(2 * L + 1, beta) * ideal, L, beta


def resample(x: np.ndarray, fs_sig: int = 44100, filt: str = "octave") -> np.ndarray:
    """pystoi's resample_oct(x, 10000, fs_sig); filt="kaiser5" is scipy's default filter instead (a broken variant)."""
    assert fs_sig == 44100
    if filt == "kaiser5":
        return scipy.signal.resample_poly(x, 100, 441)
    h, _, _ = octave_window()
    return scipy.signal.resample_poly(x, 100, 441, window=h / np.sum(h))


def stoi_window(kind: str = "pystoi") -> np.ndarray:
    return np.hanning(N_FRAME + 2)[1:-1] if kind == "pystoi" else np.hanning(N_FRAME)


def frame_starts(n: int, last_frame: bool = False):
    return range(0, n - N_FRAME + (1 if last_frame else 0), HOP)


def energies(x: np.ndarray, window: str = "pystoi", last_frame: bool = False) -> np.ndarray:
    """20 log10(||w x_frame|| + eps) of every frame of remove_silent_frames."""
    w = stoi_window(window)
    frames = np.array([w * x[i:i + N_FRAME] for i in frame_starts(len(x), last_frame)])
    return 20 * np.log10(np.linalg.norm(frames, axis=1) + EPS)


def overlap_add(frames: np.ndarray) -> np.ndarray:
    """pystoi's _overlap_and_add at hop 128 for 256-sample frames: (K - 1) * 128 + 256 samples."""
    k = len(frames)
    out = np.zeros((k + 1) * HOP)
    out[:k * HOP] += frames[:, :HOP].reshape(-1)
    out[HOP:] += frames[:, HOP:].reshape(-1)
    return out


def remove_silent_frames(x, y, window: str = "pystoi", last_frame: bool = False):
    """(x_sil, y_sil, mask) of pystoi's remove_silent_frames(x, y, 40, 256, 128); the mask is computed on x."""
    w = stoi_window(window)
    starts = frame_starts(len(x), last_frame)
    xf = np.array([w * x[i:i + N_FRAME] for i in starts])
    yf = np.array([w * y[i:i + N_FRAME] for i in starts])
    e = 20 * np.log10(np.linalg.norm(xf, axis=1) + EPS)
    mask = (np.max(e) - DYN_RANGE - e) < 0
    return overlap_add(xf[mask]), overlap_add(yf[mask]), mask


def stft(x, window: str = "pystoi", last_frame: bool = False) -> np.ndarray:
    w = stoi_window(window)
    return np.array([np.fft.rfft(w * x[i:i + N_FRAME], n=NFFT) for i in frame_starts(len(x), last_frame)]).reshape(-1, NFFT // 2 + 1)


def thirdoct():
    """(obm [15, 257], [(fl, fh)] bin ranges) of pystoi's thirdoct(10000, 512, 15, 150)."""
    f = np.linspace(0, FS, NFFT + 1)[:NFFT // 2 + 1]
    k = np.arange(NUMBAND, dtype=np.float64)
    lo, hi = MINFREQ * np.power(2.0, (2 * k - 1) / 6), MINFREQ * np.power(2.0, (2 * k + 1) / 6)
    obm = np.zeros((NUMBAND, len(f)))
    edges = []
    for i in range(NUMBAND):
        fl, fh = int(np.argmin(np.square(f - lo[i]))), int(np.argmin(np.square(f - hi[i])))
        obm[i, fl:fh] = 1
        edges.append((fl, fh))
    return obm, edges


def stoi(x, y, fs_sig: int = 44100, window: str = "pystoi", last_frame: bool = False, clip: bool = True,
         mean_removal: bool = True, filt: str = "octave") -> float:
    """pystoi 0.3.3 stoi(x, y, fs_sig, extended=False), x the clean target and y the estimate, equal lengths.  The keyword
    arguments select the broken variants; their defaults are pystoi."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    assert x.shape == y.shape
    x, y = resample(x, fs_sig, filt), resample(y, fs_sig, filt)
    x, y, _ = remove_silent_frames(x, y, window, last_frame)
    xs, ys = stft(x, window, last_frame).T, stft(y, window, last_frame).T
    if xs.shape[-1] < N_SEG:
        return 1e-5
    obm, _ = thirdoct()
    x_tob, y_tob = np.sqrt(obm @ np.square(np.abs(xs))), np.sqrt(obm @ np.square(np.abs(ys)))
    xseg = np.array([x_tob[:, m - N_SEG:m] for m in range(N_SEG, x_tob.shape[1] + 1)])
    yseg = np.array([y_tob[:, m - N_SEG:m] for m in range(N_SEG, x_tob.shape[1] + 1)])
    norm_const = np.linalg.norm(xseg, axis=2, keepdims=True) / (np.linalg.norm(yseg, axis=2, keepdims=True) + EPS)
    yp = yseg * norm_const
    if clip:
        yp = np.minimum(yp, xseg * (1 + 10 ** (-BETA / 20)))
    if mean_removal:
        yp = yp - np.mean(yp, axis=2, keepdims=True)
        xseg = xseg - np.mean(xseg, axis=2, keepdims=True)
    yp = yp / (np.linalg.norm(yp, axis=2, keepdims=True) + EPS)
    xseg = xseg / (np.linalg.norm(xseg, axis=2, keepdims=True) + EPS)
    return float(np.sum(yp * xseg) / (xseg.shape[0] * xseg.shape[1]))


def sisdr(est, target, mean_removed: bool = False) -> float:
    """speechmetrics' sisdr of equal-length float64 signals; mean_removed=True is a broken variant."""
    e, r = np.asarray(est, np.float64), np.asarray(target, np.float64)
    if mean_removed:
        e, r = e - e.mean(), r - r.mean()
    a = (EPS + np.dot(r, e)) / (np.dot(r, r) + EPS)
    t = a * r
    return float(10 * np.log10((EPS + np.sum(t ** 2)) / (EPS + np.sum((e - t) ** 2))))


def pad_pair(est, target):
    """speechmetrics' zero padding at the end of the shorter signal, float64."""
    n = max(len(est), len(target))
    e, t = np.zeros(n), np.zeros(n)
    e[:len(est)], t[:len(target)] = est, target
    return e, t


def time_scores(est, target, **variant) -> dict:
    """{"sisdr", "stoi"} of one pair of 44.1 kHz signals as speechmetrics computes them (metrics(est, target, rate=44100))."""
    e, t = pad_pair(est, target)
    sd = variant.pop("sisdr_mean_removed", False)
    return {"sisdr": sisdr(e, t, sd), "stoi": stoi(t, e, 44100, **variant)}


def silence_margin(est, target) -> float:
    """Smallest |max - 40 - energy| in dB over the target's frames at 10 kHz, after padding: how far rounding would have to
    move a frame energy to flip STOI's silent-frame mask."""
    _, t = pad_pair(est, target)
    e = energies(resample(t))
    return float(np.min(np.abs(np.max(e) - DYN_RANGE - e)))


U = 2.0 ** -53


def gamma(n: int) -> float:
    """Higham's gamma_n = n u / (1 - n u): the relative error bound of a float64 sum or dot product of n terms, whatever
    its order."""
    return n * U / (1 - n * U)


def sisdr_bar(n: int, snr_db: float) -> float:
    """Bound on |GPU - restatement| for sisdr of a pair padded to n samples whose value is about snr_db (0 when Snn is
    exactly 0 on both sides, as for identical signals).  r.r, r.e, Sss and Snn are n-term sums whose order differs between
    the two (gamma_n each, twice per side of the ratio), and each e - a r is rounded relative to |a r|, which is
    10^(snr_db / 20) times |e - a r|; 10 log10 turns a relative error d into 10 / ln 10 * d dB."""
    return 10 / np.log(10) * (4 * gamma(n) + 4 * U * 10 ** (max(snr_db, 0.0) / 20))


def stoi_bar(n: int) -> float:
    """Bound on |GPU - restatement| for stoi of a pair padded to n samples.  Every band value is the end of a float64
    chain of at most 720 operations (320 resampling taps, a 256-term frame energy, 8 FFT stages, a band of at most 45
    bins, 3 x 30 segment terms), so its relative error is at most gamma_720 ~ 8e-14.  A correlation of two normalised,
    mean-removed 30-vectors can amplify that; 1e4 is the budget allowed for it.  The final sum over J * 15 correlations
    adds gamma(J * 15), with J below n / 441 segments."""
    return 1e4 * gamma(720) + gamma(15 * (n // 441 + 1))


VARIANTS = {   # name -> (est, target) -> {"sisdr", "stoi"}: plausible mistakes a GPU port could make
    "hanning256": lambda e, t: time_scores(e, t, window="hanning256"),
    "last_frame_included": lambda e, t: time_scores(e, t, last_frame=True),
    "no_clipping": lambda e, t: time_scores(e, t, clip=False),
    "no_mean_removal": lambda e, t: time_scores(e, t, mean_removal=False),
    "est_target_swapped": lambda e, t: time_scores(t, e),
    "kaiser5_filter": lambda e, t: time_scores(e, t, filt="kaiser5"),
    "mean_removed_sisdr": lambda e, t: time_scores(e, t, sisdr_mean_removed=True),
}


def load_first_channel(path) -> np.ndarray:
    """soundfile.read(path) of a 16-bit PCM wav, first channel: int16 / 32768 in float64."""
    with wave.open(path, "rb") as w:
        data = np.frombuffer(w.readframes(w.getnframes()), dtype=np.int16).reshape(-1, w.getnchannels())
    return data[:, 0].astype(np.float64) / 32768.0


def evaluation(est_path, target_path) -> dict:
    """AudioMetrics.evaluation(est, target) without pesq, for 44.1 kHz PCM16 wavs: {"sisdr", "stoi", <8 spectral keys>}."""
    from oracle import scoring as S
    if target_path is None:
        return {}
    return {**time_scores(load_first_channel(est_path), load_first_channel(target_path)), **S.evaluation(est_path, target_path)}
