"""The pip package's pre-filter, remove_higher_frequency (restore_inmem's mode 1), without a GPU: the oracle's stft ->
istft round trip, the float64 restatement against the package's own dtypes, the edge cases the package's code implies, and
the argument checks of VoiceFixer.remove_higher_frequency_batch, which run before the engine is touched."""
import numpy as np
import pytest
import scipy.signal

from oracle import lowpass as LP
from oracle import prefilter as P
from oracle import vf_oracle as O
from voicefixer_main_b200 import VoiceFixer

SR = 44100
F32 = np.finfo(np.float32).eps


def seeded_set():
    """(name, float32 clip) of the pre-filter test signals: low-passed noise, a sweep, speech-like clips."""
    rng = np.random.default_rng(7)
    out = []
    for k, fc in enumerate((2000, 4000, 8000, 16000)):
        noise = 0.3 * rng.standard_normal(3 * SR + 101 * k)
        out.append((f"noise lp {fc} Hz", LP.lowpass(noise, fc, SR).astype(np.float32)))
    t = np.arange(2 * SR) / SR
    out.append(("sweep", (0.5 * scipy.signal.chirp(t, 50, t[-1], 20000, method="logarithmic")).astype(np.float32)))
    for i, clip in enumerate(O.synth_clips(2, 2 * SR + 333, seed=11).numpy()):
        out.append((f"speech {i}", clip.astype(np.float32)))
    return out


@pytest.mark.parametrize("n", [1025, 44100, 1323000, 7919])
def test_round_trip(n):
    """EPS = 0 and no bin removed: stft -> istft gives back the clip's first 512 * (n // 512) samples.  This pins the
    framing, the reflect padding and librosa's partial window sums at both ends independently of the package's code."""
    x = (0.3 * np.random.default_rng(n).standard_normal(n)).astype(np.float32)
    y, cutoff, _ = P.remove_higher_frequency(x, 1.0, eps=0.0, cutoff=P.BINS)
    assert cutoff == P.BINS and y.shape == (512 * (n // 512),)
    err = np.abs(y - x[:y.shape[0]]).max()
    assert err <= 1e-12 * np.abs(x).max(), err


def test_float64_against_package_dtypes():
    """The float64 path and the package's dtypes pick the same cutoff on the seeded set, and their outputs differ by no
    more than float32 rounding can explain: about ten float32 roundings of each frame's largest possible sample (the sum of
    its bins' magnitudes / 1024), four frames per sample, over a window sum of squares of at least 1."""
    worst = 0.0
    for name, x in seeded_set():
        y64, c64, margin = P.remove_higher_frequency(x)
        y32, c32 = P.remove_higher_frequency_pkg(x)
        assert c64 == c32, (name, c64, c32, margin)
        X = np.fft.rfft(P._frames(x) * P._window(), axis=1)
        frame_peak = (np.abs(X).sum(axis=1) / 1024).max()
        bound = 4 * 10 * F32 * frame_peak
        diff = np.abs(y64 - y32.astype(np.float64)).max()
        worst = max(worst, diff / bound)
        print(f"{name}: cutoff {c64}, largest difference {diff:.3e} (bound {bound:.3e})")
        assert diff <= bound, (name, diff, bound)
    print(f"largest difference / bound: {worst:.3f}")


def test_quiet_clip_is_zeros():
    """Only bins with |X| >= 1 carry energy: a clip of peak 1e-3 has total 0, cutoff 0 and an all-zero output."""
    x = np.random.default_rng(3).standard_normal(SR)
    x = (1e-3 * x / np.abs(x).max()).astype(np.float32)
    y, cutoff, _ = P.remove_higher_frequency(x)
    assert cutoff == 0 and y.shape == (512 * (SR // 512),) and not y.any()
    y32, c32 = P.remove_higher_frequency_pkg(x)
    assert c32 == 0 and not y32.any()


@pytest.mark.parametrize("n", [1, 2, 100, 511])
def test_short_rows_give_empty_outputs(n):
    x = np.random.default_rng(n).standard_normal(n).astype(np.float32)
    y, cutoff, _ = P.remove_higher_frequency(x)
    assert y.shape == (0,) and 0 <= cutoff <= P.BINS


@pytest.mark.parametrize("n", [600, 1000])
def test_repeated_reflection(n):
    """np.pad reflects a clip of n <= 1024 samples more than once: the padded clip is the even periodic extension of
    period 2 (n - 1), the index map the STFT kernel uses, and not a single fold, which would index outside the clip."""
    x = np.random.default_rng(n).standard_normal(n).astype(np.float32)
    s = np.arange(-P.N_FFT // 2, n + P.N_FFT // 2)
    m = np.mod(s, 2 * (n - 1))
    m = np.where(m >= n, 2 * (n - 1) - m, m)
    assert np.array_equal(np.pad(x, P.N_FFT // 2, mode="reflect"), x[m])
    once = np.abs(s)
    assert (np.where(once >= n, 2 * (n - 1) - once, once) < 0).any()
    frames = P._frames(x)
    assert np.array_equal(frames, np.stack([x[m[t * P.HOP:t * P.HOP + P.N_FFT]] for t in range(1 + n // P.HOP)]))
    y, _, _ = P.remove_higher_frequency(x, 1.0, eps=0.0, cutoff=P.BINS)
    assert np.abs(y - x[:512]).max() <= 1e-12 * np.abs(x).max()


@pytest.mark.parametrize("wavs, ratio", [
    ([np.zeros(1000, np.float32)], 0),
    ([np.zeros(1000, np.float32)], 1.5),
    ([np.zeros(1000, np.float32)], float("nan")),
    ([], 0.95),
    ([np.zeros((2, 1000), np.float32)], 0.95),
    ([np.zeros(0, np.float32)], 0.95),
])
def test_argument_checks_before_any_gpu_work(wavs, ratio):
    """The model has no engine at all (never moved to a device): the checks raise before one is needed."""
    with pytest.raises(ValueError):
        VoiceFixer().remove_higher_frequency_batch(wavs, ratio)
    if len(wavs) == 1:
        with pytest.raises(ValueError):
            VoiceFixer().remove_higher_frequency(wavs[0], ratio)
