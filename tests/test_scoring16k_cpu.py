"""16 kHz scoring without a GPU: the restatement of tests/oracle_16k.py against the reference's own AudioMetrics (golden) and
against direct float64 loops, the deliberately broken variants it must tell apart, and AudioMetrics' rate routing, which
runs before the engine is touched."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import oracle_16k as R
from conftest import load_golden
from oracle import ref_import
from oracle import scoring as S
from oracle import speech_metrics as M
from test_gpu_scoring import _close, _ulp_ok
from test_scoring_cpu import StubOwner, _pair
from voicefixer_main_b200.arch import metric_frames
from voicefixer_main_b200.edges import AudioMetrics
from voicefixer_main_b200.model import mel16k_fbanks


def test_mel_16k_filterbank_is_the_references():
    fb = mel16k_fbanks()
    assert fb.shape == (372, 80) and fb.dtype == torch.float32
    assert torch.equal(fb, torch.from_numpy(load_golden("ref_scores_16k.npz")["mel_16k"]))
    nz = (fb != 0).sum(dim=0)
    assert int(nz.sum()) == 727 and int(nz.min()) == 2 and int(nz.max()) == 24


@pytest.mark.skipif(not ref_import.available(), reason="reference tree not present")
def test_mel_16k_filterbank_is_the_reference_modules():
    path = os.path.join(ref_import.REFERENCE_ROOT, "tools", "pytorch", "mel_scale.py")
    spec = importlib.util.spec_from_file_location("ref_mel_scale", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert torch.equal(mel16k_fbanks(), mod.MelScale(n_mels=80, sample_rate=16000, n_stft=372).fb)


def test_restatement_matches_reference_metrics(tmp_path):
    g = load_golden("ref_scores_16k.npz")
    for i, (est, tgt) in enumerate(R.score_pairs()):
        pe, pt = str(tmp_path / f"e{i}.wav"), str(tmp_path / f"t{i}.wav")
        S.write_pcm16(est, pe, 16000)
        S.write_pcm16(tgt, pt, 16000)
        got = R.evaluation(pe, pt)
        assert list(got) == list(g[f"keys{i}"])
        np.testing.assert_allclose(np.array(list(got.values())), g[f"values{i}"], rtol=1e-6, atol=0)
    assert R.evaluation(pe, None) == {}


def test_stft_restatement_is_the_dft():
    rng = np.random.default_rng(16)
    wav = (rng.standard_normal(5000) * 0.2).astype(np.float32)
    sp = R.spectrogram(wav)
    assert sp.shape == (1 + 4999 // 160, 372) and sp.dtype == np.float32
    padded = np.pad(wav.astype(np.float64), 371, mode="reflect")
    win = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(743) / 743)          # periodic hann of the odd length 743
    k = np.arange(372)[:, None] * np.arange(743)[None, :]
    dft = np.exp(-2j * np.pi * k / 743)
    for t in (0, 1, 10, sp.shape[0] - 1):
        want = np.abs(dft @ (win * padded[t * 160:t * 160 + 743]))
        np.testing.assert_allclose(sp[t], want, rtol=1e-6, atol=1e-6 * want.max())


@pytest.mark.parametrize("n", [961, 1119, 1120, 1121, 15999, 16000, 16001, 16160, 16161])
def test_frame_count_is_np_pad_framing(n):
    padded = np.pad(np.zeros(n, np.float32), 371, mode="reflect")
    want = 1 + (len(padded) - 743) // 160
    assert R.frames(n) == metric_frames(n, 16000) == want == R.spectrogram(np.ones(n, np.float32)).shape[0]
    assert metric_frames(n) == 1 + n // 441


def test_octave_window_for_16k():
    h, L, _ = M.octave_window(5, 8)
    assert L == 290 and h.shape == (581,)
    x = np.random.default_rng(3).standard_normal(1001)
    assert len(R.resample(x)) == (5 * 1001 + 7) // 8


# ------------------------------------------------------------------------------------------ broken variants vs the bars
def _wav(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 16000
    return (0.3 * np.sin(2 * np.pi * 440 * t) + 0.05 * rng.standard_normal(n)).astype(np.float32)


def _outside_spectrogram_bar(got, want):
    return got.shape != want.shape or not _ulp_ok(got, want).all()


def test_broken_spectrograms_land_outside_the_bar():
    wav = _wav(16000, 1)
    want = R.spectrogram(wav)
    assert not _outside_spectrogram_bar(want.copy(), want)
    assert _outside_spectrogram_bar(R.spectrogram(wav, window="symmetric"), want)
    assert _outside_spectrogram_bar(R.spectrogram(wav, n_fft=744), want)
    assert 1 + len(wav) // 160 != want.shape[0]                    # 44.1 kHz's T = 1 + N // hop: one frame too many


def test_44k_octave_filter_lands_outside_the_stoi_bar():
    t = _wav(48000, 2)
    e = t + 0.2 * _wav(48000, 3)
    good, bad = R.time_scores(e, t), R.time_scores(e, t, filt="octave441")
    assert abs(good["stoi"] - bad["stoi"]) > 1e3 * R.stoi_bar(48000)
    assert good["sisdr"] == bad["sisdr"]


def test_unresampled_est_lands_outside_the_bars(tmp_path):
    from voicefixer_main_b200.handler import _rate_len
    t = _wav(32000, 4)
    e44 = np.interp(np.arange(_rate_len(32000, 16000, 44100)) * 16000 / 44100, np.arange(32000), t).astype(np.float32)
    good = R.evaluation_arrays(t + 0.01 * _wav(32000, 5), t)
    bad = R.evaluation_arrays(e44[:32000], t)                      # the 44.1 kHz samples, cut to the target's length
    with pytest.raises(AssertionError):
        _close(bad, good)


# ------------------------------------------------------------------------------------------------- routing (no engine)
@pytest.mark.parametrize("am_rate, n_est, n_tgt, rate, exc", [
    (44100, 30000, 30000, 16000, NotImplementedError),   # the default instance and a 16 kHz target
    (16000, 30000, 30000, 44100, NotImplementedError),   # a 16 kHz instance and a 44.1 kHz target
    (16000, 30000, 30000, 8000, ValueError),             # Bad Samplerate
    (16000, 2600, 900, 16000, ValueError),               # 6 frames at 16 kHz: SSIM's window does not fit
    (16000, 30000, 11200, 16000, ValueError),            # the est resampled to 16 kHz has 69 frames, the target 70
])
def test_bad_pair_fails_before_the_engine(tmp_path, am_rate, n_est, n_tgt, rate, exc):
    am = AudioMetrics(StubOwner(), rate=am_rate)
    good = _pair(tmp_path, 30000, 30000 if am_rate == 44100 else 11000, rate=am_rate, name="good")   # 69 frames at 16 kHz
    bad = _pair(tmp_path, n_est, n_tgt, rate, name="bad")
    with pytest.raises(exc, match="bad_"):
        am.evaluation_batch([good, bad])
    if exc is NotImplementedError:
        with pytest.raises(exc, match=f"rate={rate}"):
            am.evaluation_batch([bad])


def test_16k_instance_calls_the_16k_entry_points(tmp_path):
    am = AudioMetrics(StubOwner(), rate=16000)
    seen = []

    class Eng:
        device = "cpu"

        def score_varlen(self, e, el, t, tl, rate=44100):
            seen.append(("spectral", list(el), list(tl), rate))
            return torch.zeros(len(el), 8, dtype=torch.float64)

        def score_time_varlen(self, e, el, t, tl, rate=44100):
            seen.append(("time", list(el), list(tl), rate))
            return torch.zeros(len(el), 2, dtype=torch.float64)

    am._owner = Eng()
    pe, pt = str(tmp_path / "e.wav"), str(tmp_path / "t.wav")
    S.write_pcm16(np.zeros(16001, np.int16), pe, 16000)
    S.write_pcm16(np.zeros(16100, np.int16), pt, 16000)
    res = am.evaluation_batch([(pe, pt), (pe, None)], time_domain=True)
    assert seen == [("spectral", [16001], [16100], 16000), ("time", [16001], [16100], 16000)]
    assert list(res[0]) == ["sisdr", "stoi"] + list(S.KEYS) and res[1] == {}
    with pytest.raises(ValueError, match="Bad Samplerate"):
        am.wav_to_spectrogram(np.zeros(1000, np.float32), rate=22050)
