"""Checks of the sisdr / stoi restatement itself (oracle/speech_metrics.py), without a GPU."""
import numpy as np
import pytest

from oracle import speech_metrics as M


def _pair(n, seed, silences=()):
    """A tonal, amplitude-modulated target with exactly silent stretches and a noisy estimate with a small DC offset: the
    silence mask, the clipping of the quiet high bands and the (absent) mean removal of SI-SDR all matter for this pair."""
    g = np.random.default_rng(seed)
    t = np.arange(n) / 44100
    x = sum(a * np.sin(2 * np.pi * f * t + g.uniform(0, 6)) for a, f in ((0.3, 220), (0.15, 530), (0.05, 1250)))
    x *= 0.6 + 0.4 * np.sin(2 * np.pi * 3 * t)
    for a, b in silences:
        x[int(a * 44100):int(b * 44100)] = 0
    y = x + 0.05 * g.standard_normal(n) + 0.01
    return y, x


def test_filter_taps_beta_and_dc_gain():
    h, L, beta = M.octave_window()
    assert (len(h), L) == (31947, 15973)
    assert beta == pytest.approx(0.1102 * (60 - 8.7), abs=0)
    taps = h / h.sum() * 100
    phases = [taps[p::100].sum() for p in range(100)]          # each output phase's DC gain
    assert np.allclose(phases, 1.0, atol=2e-3)
    y = M.resample(np.ones(44100 * 3))
    assert len(y) == -(-44100 * 3 * 100 // 441)
    assert np.abs(y[5000:25000] - 1).max() < 2e-3


def test_band_edges_are_15_contiguous_ranges():
    obm, edges = M.thirdoct()
    assert len(edges) == 15 and edges[0] == (7, 9) and edges[-1][1] == 219
    for (lo, hi), nxt in zip(edges, edges[1:] + [(edges[-1][1], None)]):
        assert lo < hi and hi == nxt[0]
    for k, (lo, hi) in enumerate(edges):
        assert obm[k].sum() == hi - lo and obm[k, lo:hi].all()


def test_stoi_of_identical_signals_is_one():
    _, x = _pair(44100 * 3, 1, silences=((1.0, 1.5),))
    assert abs(M.stoi(x, x) - 1) < 1e-12


def test_sisdr_scale_invariance_and_known_snr():
    e, t = _pair(44100 * 2, 2)
    assert M.sisdr(3.7 * e, t) == pytest.approx(M.sisdr(e, t), abs=1e-9)
    g = np.random.default_rng(5)
    n = g.standard_normal(len(t))
    n -= np.dot(n, t) / np.dot(t, t) * t                          # orthogonal to the target
    n *= np.sqrt(np.dot(t, t) / np.dot(n, n) / 10)                # 10 dB below it
    assert M.sisdr(t + n, t) == pytest.approx(10.0, abs=1e-9)


def test_silent_stretch_removes_exactly_its_frames_and_not_the_last_frame():
    g = np.random.default_rng(3)
    k = 60
    x = g.standard_normal(256 + 128 * k)            # starts 0, 128, .., 128 k: range(0, len - 256, 128) stops before 128 k
    x[128 * 20:128 * 31 + 256] = 0                  # frames 20 .. 31 are all zeros
    _, _, mask = M.remove_silent_frames(x, x)
    assert len(mask) == k
    want = np.ones(k, bool)
    want[20:32] = False
    assert (mask == want).all()
    _, _, mask_last = M.remove_silent_frames(x, x, last_frame=True)
    assert len(mask_last) == k + 1


def test_fewer_than_30_frames_gives_1e5():
    e, t = _pair(13230, 4)                          # 0.3 s: 3000 samples at 10 kHz, 22 frames
    assert M.stoi(t, e) == 1e-5
    e, t = _pair(44100 * 2, 4, silences=((0.0, 0.9), (1.1, 2.0)))   # 0.2 s of sound: too few frames survive
    assert M.stoi(t, e) == 1e-5


@pytest.mark.parametrize("name", sorted(M.VARIANTS))
def test_broken_variant_lands_far_from_the_restatement(name):
    n = 133217                                      # 30208 = 256 + 128 * 234 samples at 10 kHz: a last frame to include
    e, t = _pair(n, 7, silences=((0.8, 1.3),))
    n10 = len(M.resample(t))
    assert (n10 - 256) % 128 == 0, n10
    want, got = M.time_scores(e, t), M.VARIANTS[name](e, t)
    bars = {"sisdr": M.sisdr_bar(n, want["sisdr"]), "stoi": M.stoi_bar(n)}
    assert max(abs(got[k] - want[k]) / bars[k] for k in M.KEYS) >= 100, (name, got, want)


def test_bars_stay_near_1e9_for_a_minute():
    n = 44100 * 61
    assert M.sisdr_bar(n, 20.0) < 6e-9 and M.stoi_bar(n) < 1e-9
