"""Scoring without a GPU: the CPU restatement of AudioMetrics.evaluation against the reference's own metrics.py (golden), its
SSIM and STFT against direct fp64 loops, and evaluation_batch's checks, which all run before the engine is touched."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import scoring as S
from voicefixer_main_b200.edges import AudioMetrics


def test_oracle_matches_reference_metrics(tmp_path):
    g = load_golden("ref_scores.npz")
    for i, (est, tgt) in enumerate(S.score_pairs()):
        pe, pt = str(tmp_path / f"e{i}.wav"), str(tmp_path / f"t{i}.wav")
        S.write_pcm16(est, pe)
        S.write_pcm16(tgt, pt)
        got = S.evaluation(pe, pt)
        assert list(got) == list(g[f"keys{i}"])
        np.testing.assert_allclose(np.array(list(got.values())), g[f"values{i}"], rtol=1e-6, atol=0)
    assert S.evaluation(pe, None) == {}


def _ssim_direct(x, y):
    """structural_similarity restated pixel by pixel over 7x7 windows, no scipy."""
    x, y = x.astype(np.float64), y.astype(np.float64)
    c1, c2 = 0.02 ** 2, 0.06 ** 2
    vals = []
    for r in range(3, x.shape[0] - 3):
        for c in range(3, x.shape[1] - 3):
            a, b = x[r - 3:r + 4, c - 3:c + 4].ravel(), y[r - 3:r + 4, c - 3:c + 4].ravel()
            ux, uy = a.mean(), b.mean()
            vx, vy = ((a - ux) ** 2).sum() / 48, ((b - uy) ** 2).sum() / 48
            vxy = ((a - ux) * (b - uy)).sum() / 48
            vals.append((2 * ux * uy + c1) * (2 * vxy + c2) / ((ux ** 2 + uy ** 2 + c1) * (vx + vy + c2)))
    return float(np.mean(vals))


@pytest.mark.parametrize("shape", [(7, 7), (7, 128), (11, 9), (23, 40), (40, 131)])
def test_ssim_restatement_is_the_windowed_formula(shape):
    rng = np.random.default_rng(shape[0] * 1000 + shape[1])
    x = rng.random(shape, dtype=np.float32) * 2
    y = (x + 0.3 * rng.standard_normal(shape)).astype(np.float32)
    assert abs(S.ssim(x, y) - _ssim_direct(x, y)) < 1e-12
    assert S.ssim(x, x) == 1.0
    with pytest.raises(ValueError):
        S.ssim(x[:6], y[:6])


def test_stft_restatement_is_the_dft():
    rng = np.random.default_rng(5)
    wav = (rng.standard_normal(9000) * 0.2).astype(np.float32)
    sp = S.spectrogram(wav)
    assert sp.shape == (1 + 9000 // 441, 1025) and sp.dtype == np.float32
    padded = np.pad(wav.astype(np.float64), 1024, mode="reflect")
    win = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(2048) / 2048)
    k = np.arange(1025)[:, None] * np.arange(2048)[None, :]
    dft = np.exp(-2j * np.pi * k / 2048)
    for t in (0, 1, 10, sp.shape[0] - 1):
        want = np.abs(dft @ (win * padded[t * 441:t * 441 + 2048]))
        np.testing.assert_allclose(sp[t], want, rtol=1e-6, atol=1e-6 * want.max())


class StubEngine:
    device = "cpu"

    def __init__(self):
        self.calls = 0

    def __getattr__(self, name):
        raise AssertionError(f"engine touched: {name}")


class StubOwner:
    def __init__(self):
        self.eng = StubEngine()

    def _engine(self):
        return self.eng


def _pair(tmp_path, n_est, n_tgt, rate=44100, name="p"):
    rng = np.random.default_rng(n_est + n_tgt)
    pe, pt = str(tmp_path / f"{name}_est.wav"), str(tmp_path / f"{name}_tgt.wav")
    S.write_pcm16(rng.integers(-9000, 9000, n_est), pe, 44100)
    S.write_pcm16(rng.integers(-9000, 9000, n_tgt), pt, rate)
    return pe, pt


@pytest.mark.parametrize("n_est, n_tgt, rate, exc", [
    (30000, 31000, 44100, ValueError),          # 68 vs 70 frames
    (2600, 2600, 44100, ValueError),            # 6 frames: SSIM's window does not fit
    (30000, 30000, 16000, NotImplementedError),
    (30000, 30000, 8000, ValueError),
])
def test_bad_pair_fails_before_the_engine(tmp_path, n_est, n_tgt, rate, exc):
    am = AudioMetrics(StubOwner())
    good = _pair(tmp_path, 30000, 30000, name="good")
    bad = _pair(tmp_path, n_est, n_tgt, rate, name="bad")
    with pytest.raises(exc, match="bad_"):
        am.evaluation_batch([good, bad])


def test_sample_counts_may_differ_within_a_hop(tmp_path, monkeypatch):
    am = AudioMetrics(StubOwner())
    seen = []

    class Eng:
        device = "cpu"

        def score_varlen(self, e, el, t, tl):
            import torch
            seen.append((list(el), list(tl)))
            return torch.zeros(len(el), 8, dtype=torch.float64)

    am._owner = Eng()
    res = am.evaluation_batch([_pair(tmp_path, 20000, 20200), (str(tmp_path / "x.wav"), None)])
    assert seen == [([20000], [20200])]
    assert list(res[0]) == list(S.KEYS) and res[1] == {}
