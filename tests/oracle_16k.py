"""CPU restatement of AudioMetrics.evaluation's 16 kHz branch (evaluation_proc/metrics.py:37-81 with rate 16000).  TEST
INFRASTRUCTURE: the tests of the 16 kHz scoring path import it; run as a script where the reference tree exists, it writes
tests/golden/ref_scores_16k.npz.

It reuses the 44.1 kHz restatements of oracle/scoring.py and oracle/speech_metrics.py and changes only what the rate
changes:
* librosa 0.8 `stft(wav, hop_length=160, n_fft=743)`: reflect padding by 743 // 2 = 371, the float64 periodic hann of
  length 743, a float64 rfft of the prime length 743 (372 bins) stored as complex64.  T = 1 + (N - 1) // 160 frames: with
  an odd n_fft the padded clip is N + 742 samples long.
* MelScale(n_mels=80, sample_rate=16000, n_stft=372) (metrics.py:30): f_max 8000, [372, 80].
* pystoi's resample_oct(x, 10000, 16000): p / q = 5 / 8, Octave's window with cut-off 1 / 16, roll-off 1 / 160 and
  L = 290 (581 taps), ceil(5 n / 8) samples.  Everything at 10 kHz is oracle/speech_metrics.py's.
* sisdr does not depend on the rate.

The keyword arguments of `spectrogram` and `resample` select deliberately broken variants (tests/test_scoring16k_cpu.py
shows each one lands outside the GPU test's bars).
"""
import os
import sys
import tempfile

import numpy as np
import scipy.signal
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import scoring as S            # noqa: E402
from oracle import speech_metrics as M     # noqa: E402

RATE, N_FFT, HOP, BINS, MELS = 16000, 743, 160, 372, 80
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_scores_16k.npz")


def frames(n: int) -> int:
    """librosa's frame count 1 + (N + 2 (n_fft // 2) - n_fft) // hop for n_fft 743, hop 160."""
    return 1 + (n - 1) // HOP


def spectrogram(wav: np.ndarray, n_fft: int = N_FFT, hop: int = HOP, window: str = "periodic") -> np.ndarray:
    """np.abs(librosa.stft(wav, hop_length=160, n_fft=743)) transposed: float32 [T, 372] (metrics.py:43-49).  window=
    "symmetric" is a broken variant."""
    if window == "periodic":
        return np.ascontiguousarray(np.abs(S.stft(wav, n_fft=n_fft, hop_length=hop)).T)
    y = np.pad(np.asarray(wav, dtype=np.float32), n_fft // 2, mode="reflect")
    win = scipy.signal.get_window("hann", n_fft, fftbins=False)
    t = 1 + (len(y) - n_fft) // hop
    fr = np.lib.stride_tricks.as_strided(y, shape=(n_fft, t), strides=(y.strides[0], hop * y.strides[0]))
    return np.ascontiguousarray(np.abs(np.fft.rfft(win[:, None] * fr, axis=0).astype(np.complex64)).T)


def mel_fb() -> torch.Tensor:
    from voicefixer_main_b200.model import melscale_fbanks
    return melscale_fbanks(BINS, 0.0, 8000.0, MELS, RATE)


def mel(sp: torch.Tensor) -> torch.Tensor:
    """MelScale(n_mels=80, sample_rate=16000, n_stft=372) of [..., T, 372] (metrics.py:51)."""
    return torch.matmul(sp, mel_fb())


def evaluation_arrays(est: np.ndarray, target: np.ndarray, spec=spectrogram) -> dict:
    """The 8 spectral keys of AudioMetrics.evaluation for two decoded 16 kHz signals."""
    est_sp = torch.from_numpy(spec(est))[None, None]
    tgt_sp = torch.from_numpy(spec(target))[None, None]
    est_mel, tgt_mel = mel(est_sp), mel(tgt_sp)
    res = {}
    for names, e, t in ((S.KEYS[:4], est_sp, tgt_sp), (S.KEYS[4:], est_mel, tgt_mel)):
        res[names[0]] = float(S.lsd(e.clone(), t.clone()))
        res[names[1]] = float(S.sispec(e.clone(), t.clone()))
        res[names[2]] = float(S.sispec(S.to_log(e.clone()), S.to_log(t.clone())))
        res[names[3]] = S.ssim(e[0, 0].numpy(), t[0, 0].numpy())
    return {k: res[k] for k in S.KEYS}


def evaluation(est_path, target_path, est: np.ndarray = None) -> dict:
    """AudioMetrics(rate=16000).evaluation(est, target) restricted to its spectral keys, for PCM16 wavs with a 16 kHz
    target.  `est` replaces the decoded estimate: pass the est already resampled to 16 kHz when its file is at another
    rate (librosa.load(sr=16000) resamples; the GPU path uses its own resampler)."""
    if target_path is None:
        return {}
    target, rate = S.load(target_path)
    assert rate == RATE, rate
    if est is None:
        est, est_rate = S.load(est_path)
        assert est_rate == RATE, est_rate
    return evaluation_arrays(np.asarray(est, np.float32), target)


# ------------------------------------------------------------------------------------------------------------ sisdr, stoi
def resample(x: np.ndarray, filt: str = "octave") -> np.ndarray:
    """pystoi's resample_oct(x, 10000, 16000): resample_poly(x, 5, 8, window=h / sum(h)) with h = octave_window(5, 8).
    filt="octave441" uses the 44.1 kHz filter (octave_window(100, 441)) instead, a broken variant."""
    h, _, _ = M.octave_window(5, 8) if filt == "octave" else M.octave_window(100, 441)
    return scipy.signal.resample_poly(x, 5, 8, window=h / np.sum(h))


def stoi(x, y, filt: str = "octave") -> float:
    """pystoi 0.3.3 stoi(x, y, 16000, extended=False), x the clean target and y the estimate, equal lengths: the chain of
    oracle/speech_metrics.stoi after its resampling."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    assert x.shape == y.shape
    x, y = resample(x, filt), resample(y, filt)
    x, y, _ = M.remove_silent_frames(x, y)
    xs, ys = M.stft(x).T, M.stft(y).T
    if xs.shape[-1] < M.N_SEG:
        return 1e-5
    obm, _ = M.thirdoct()
    x_tob, y_tob = np.sqrt(obm @ np.square(np.abs(xs))), np.sqrt(obm @ np.square(np.abs(ys)))
    xseg = np.array([x_tob[:, m - M.N_SEG:m] for m in range(M.N_SEG, x_tob.shape[1] + 1)])
    yseg = np.array([y_tob[:, m - M.N_SEG:m] for m in range(M.N_SEG, x_tob.shape[1] + 1)])
    norm_const = np.linalg.norm(xseg, axis=2, keepdims=True) / (np.linalg.norm(yseg, axis=2, keepdims=True) + M.EPS)
    yp = np.minimum(yseg * norm_const, xseg * (1 + 10 ** (-M.BETA / 20)))
    yp = yp - np.mean(yp, axis=2, keepdims=True)
    xseg = xseg - np.mean(xseg, axis=2, keepdims=True)
    yp = yp / (np.linalg.norm(yp, axis=2, keepdims=True) + M.EPS)
    xseg = xseg / (np.linalg.norm(xseg, axis=2, keepdims=True) + M.EPS)
    return float(np.sum(yp * xseg) / (xseg.shape[0] * xseg.shape[1]))


def time_scores(est, target, filt: str = "octave") -> dict:
    """{"sisdr", "stoi"} of one pair of 16 kHz signals as speechmetrics computes them (metrics(est, target, rate=16000))."""
    e, t = M.pad_pair(est, target)
    return {"sisdr": M.sisdr(e, t), "stoi": stoi(t, e, filt)}


def stoi_bar(n: int) -> float:
    """oracle/speech_metrics.stoi_bar re-derived for the 16 kHz chain: a band value ends a float64 chain of at most 520
    operations (117 resampling taps per output: 581 taps over up = 5; then the 256-term frame energy, 8 FFT stages, a band
    of at most 45 bins and 3 x 30 segment terms), with the same 1e4 budget for the correlation; the final sum over J * 15
    correlations adds gamma(J * 15), with J below 5 n / 8 / 128 < n / 160 segments."""
    return 1e4 * M.gamma(520) + M.gamma(15 * (n // HOP + 1))


# ------------------------------------------------------------------------------------------------------- fixture and main
def score_pairs():
    """Seeded PCM16 (est, target) pairs at 16 kHz: lengths (samples), including the 7-frame minimum (961), a length on a
    hop multiple, a pair whose sample counts differ within one hop, and a target with leading digital silence."""
    rng = np.random.default_rng(1600)
    pairs = []
    for n_e, n_t, silence in ((961, 961, 0), (16000, 16000, 0), (16001, 16100, 0), (30000, 30000, 6000)):
        t = np.linspace(0, n_t / RATE, n_t, endpoint=False)
        tgt = 0.3 * np.sin(2 * np.pi * 440 * t) * np.exp(-t) + 0.05 * rng.standard_normal(n_t)
        tgt[:silence] = 0
        est = tgt[:n_e] + 0.05 * rng.standard_normal(n_e)
        pairs.append((np.round(np.clip(est, -1, 1) * 32767).astype(np.int16), np.round(np.clip(tgt, -1, 1) * 32767).astype(np.int16)))
    return pairs


def main():
    from oracle import ref_import
    from oracle.make_ref_scores import reference_metrics
    if not ref_import.available():
        raise SystemExit("reference tree not present at " + ref_import.REFERENCE_ROOT)
    am = reference_metrics()               # evaluation() takes the rate from the target file
    out = {"mel_16k": am.mel_16k.fb.numpy()}
    with tempfile.TemporaryDirectory() as d:
        for i, (est, tgt) in enumerate(score_pairs()):
            pe, pt = os.path.join(d, f"est{i}.wav"), os.path.join(d, f"tgt{i}.wav")
            S.write_pcm16(est, pe, RATE)
            S.write_pcm16(tgt, pt, RATE)
            with torch.no_grad():
                res = am.evaluation(pe, pt)
            keys = [k for k in res if k not in ("sisdr", "stoi", "pesq")]
            out[f"keys{i}"] = np.array(keys)
            out[f"values{i}"] = np.array([res[k] for k in keys], dtype=np.float64)
    np.savez_compressed(GOLDEN, **out)
    print(os.path.basename(GOLDEN), os.path.getsize(GOLDEN), "bytes")


if __name__ == "__main__":
    main()
