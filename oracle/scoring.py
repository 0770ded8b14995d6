"""CPU restatement of AudioMetrics.evaluation (evaluation_proc/metrics.py:37-106) for 44.1 kHz pairs.  TEST INFRASTRUCTURE.

The reference calls three third-party packages that this image lacks; their arithmetic is restated with numpy / scipy:
* librosa 0.8 `stft(wav, hop_length=441, n_fft=2048)`: np.pad reflect by n_fft / 2, float64 periodic hann
  (scipy.signal.get_window('hann', 2048, fftbins=True)) x float32 frames, np.fft.rfft in float64, stored as complex64.
  (librosa >= 0.10 pads with zeros by default; that is not what the reference's 2021 stack ran.)
* scikit-image 0.18 `structural_similarity(x, y, win_size=7)` on float32 images: data_range 2 (float32's dtype range),
  float64 scipy.ndimage.uniform_filter of size 7, sample covariance (49 / 48), mean over the image cropped by 3.
* librosa.load(path, sr=rate, mono=True) of a PCM16 wav at its own rate: int16 / 32768 averaged over channels.
lsd, sispec, energy_unify, to_log and the mel (MelScale, f_max 22050) are the reference's own torch fp32 arithmetic.
oracle/make_ref_scores.py pins this glue against the reference's unmodified metrics.py (tests/golden/ref_scores.npz).
"""
import wave

import numpy as np
import scipy.ndimage
import scipy.signal
import torch

N_FFT, HOP = 2048, 441
KEYS = ("lsd", "non_log_sispec", "sispec", "ssim", "final_mel_lsd", "final_non_log_mel_sispec", "final_mel_sispec",
        "final_mel_ssim")


def load(path):
    """(float32 mono samples, rate) of a 16-bit PCM wav, as librosa.load(path, sr=<its rate>, mono=True) returns them."""
    with wave.open(path, "rb") as w:
        rate = w.getframerate()
        data = np.frombuffer(w.readframes(w.getnframes()), dtype=np.int16).reshape(-1, w.getnchannels())
    return (data.astype(np.float32) / 32768.0).mean(axis=1).astype(np.float32), rate


def stft(wav: np.ndarray, n_fft: int = N_FFT, hop_length: int = HOP) -> np.ndarray:
    """librosa 0.8 stft (center=True, reflect): complex64 [1 + n_fft // 2, T]."""
    y = np.pad(np.asarray(wav, dtype=np.float32), n_fft // 2, mode="reflect")
    win = scipy.signal.get_window("hann", n_fft, fftbins=True)
    t = 1 + (len(y) - n_fft) // hop_length
    frames = np.lib.stride_tricks.as_strided(y, shape=(n_fft, t), strides=(y.strides[0], hop_length * y.strides[0]))
    return np.fft.rfft(win[:, None] * frames, axis=0).astype(np.complex64)


def spectrogram(wav: np.ndarray) -> np.ndarray:
    """np.abs(stft(wav)) transposed: float32 [T, 1025] (metrics.py:48-49)."""
    return np.ascontiguousarray(np.abs(stft(wav)).T)


def ssim(x: np.ndarray, y: np.ndarray, win_size: int = 7) -> float:
    """scikit-image 0.18 structural_similarity(x, y, win_size=7) of two float32 images."""
    if min(x.shape) < win_size:
        raise ValueError("win_size exceeds image extent")
    x, y = x.astype(np.float64), y.astype(np.float64)
    f = lambda a: scipy.ndimage.uniform_filter(a, size=win_size)
    cov_norm = win_size ** 2 / (win_size ** 2 - 1)
    ux, uy = f(x), f(y)
    uxx, uyy, uxy = f(x * x), f(y * y), f(x * y)
    vx, vy, vxy = cov_norm * (uxx - ux * ux), cov_norm * (uyy - uy * uy), cov_norm * (uxy - ux * uy)
    c1, c2 = (0.01 * 2) ** 2, (0.03 * 2) ** 2
    a1, a2, b1, b2 = 2 * ux * uy + c1, 2 * vxy + c2, ux ** 2 + uy ** 2 + c1, vx + vy + c2
    s = (a1 * a2) / (b1 * b2)
    pad = (win_size - 1) // 2
    return float(s[pad:-pad, pad:-pad].mean())


def mel(sp: torch.Tensor) -> torch.Tensor:
    """MelScale(n_mels=128, sample_rate=44100, n_stft=1025) of [..., T, 1025] (metrics.py:51)."""
    from voicefixer_main_b200.model import melscale_fbanks
    return torch.matmul(sp, melscale_fbanks())


def to_log(x):
    return torch.log10(torch.clip(x, min=1e-8))


def lsd(est, target, eps=1e-12):
    v = torch.log10((target ** 2 / ((est + eps) ** 2)) + eps) ** 2
    return torch.mean(torch.mean(v, dim=3) ** 0.5, dim=2)


def energy_unify(est, original, eps=1e-8):
    """evaluation_proc/utils.py:90-101."""
    dims = list(range(2, est.dim()))
    target = torch.sum(est * original, dim=dims, keepdim=True) * original
    target /= pow_p_norm(original) + eps
    return est, target


def pow_p_norm(x):
    return torch.pow(torch.norm(x, p=2, dim=list(range(1, x.dim())), keepdim=True), 2)


def sispec(est, target, eps=1e-12):
    """metrics.py:89-95."""
    output, target = energy_unify(est, target)
    noise = output - target
    sp_loss = 10 * torch.log10((pow_p_norm(target) / (pow_p_norm(noise) + eps) + eps))
    return torch.sum(sp_loss) / sp_loss.size()[0]


def evaluation_arrays(est: np.ndarray, target: np.ndarray) -> dict:
    """The 8 spectral keys of AudioMetrics.evaluation for two decoded 44.1 kHz signals."""
    est_sp = torch.from_numpy(spectrogram(est))[None, None]
    tgt_sp = torch.from_numpy(spectrogram(target))[None, None]
    est_mel, tgt_mel = mel(est_sp), mel(tgt_sp)
    res = {}
    for pre, e, t in (("", est_sp, tgt_sp), ("final_mel_", est_mel, tgt_mel)):
        names = ("lsd", "non_log_sispec", "sispec", "ssim") if not pre else ("final_mel_lsd", "final_non_log_mel_sispec",
                                                                              "final_mel_sispec", "final_mel_ssim")
        res[names[0]] = float(lsd(e.clone(), t.clone()))
        res[names[1]] = float(sispec(e.clone(), t.clone()))
        res[names[2]] = float(sispec(to_log(e.clone()), to_log(t.clone())))
        res[names[3]] = ssim(e[0, 0].numpy(), t[0, 0].numpy())
    return {k: res[k] for k in KEYS}


def evaluation(est_path, target_path) -> dict:
    """AudioMetrics.evaluation(est, target) restricted to its spectral keys, for 44.1 kHz PCM16 wavs."""
    if target_path is None:
        return {}
    target, rate = load(target_path)
    assert rate == 44100, rate
    est, est_rate = load(est_path)
    assert est_rate == rate, est_rate
    return evaluation_arrays(est, target)


def score_pairs():
    """Seeded PCM16 (est, target) pairs of the golden file: lengths (samples), including a target with leading digital
    silence and a pair whose sample counts differ within one hop."""
    rng = np.random.default_rng(77)
    pairs = []
    for n_e, n_t, silence in ((3100, 3100, 0), (44100, 44100, 0), (20000, 20200, 0), (30000, 30000, 8000)):
        t = np.linspace(0, n_t / 44100, n_t, endpoint=False)
        tgt = 0.3 * np.sin(2 * np.pi * 440 * t) * np.exp(-t) + 0.05 * rng.standard_normal(n_t)
        tgt[:silence] = 0
        est = tgt[:n_e] + 0.05 * rng.standard_normal(n_e) if n_e <= n_t else None
        pairs.append((np.round(np.clip(est, -1, 1) * 32767).astype(np.int16), np.round(np.clip(tgt, -1, 1) * 32767).astype(np.int16)))
    return pairs


def write_pcm16(pcm: np.ndarray, path, rate: int = 44100):
    with wave.open(path, "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(rate)
        w.writeframes(np.ascontiguousarray(pcm, dtype=np.int16).tobytes())
