"""librosa 0.8's resample(res_type="kaiser_best" / "kaiser_fast") without a GPU: the vectorised restatement of
oracle/resampy.py against a scalar transcription of resampy's loop, its accuracy on a band-limited signal, the broken variants
it must tell apart, librosa's length rule, the host table design of edges.py, and the res_type routing of the handlers and
AudioMetrics, which runs before the engine is touched."""
import numpy as np
import pytest
import torch
from scipy.signal import resample_poly

from oracle import resampy as R
from oracle import scoring as S
from test_scoring_cpu import StubOwner
from voicefixer_main_b200 import edges as E
from voicefixer_main_b200 import handler as H
from voicefixer_main_b200._lib import EngineError
from voicefixer_main_b200.edges import AudioMetrics

RATE_PAIRS = [(16000, 44100), (44100, 16000), (8000, 44100), (22050, 44100), (48000, 44100), (44100, 48000)]


def scalar_resampy(x, orig_sr, target_sr, res_type):
    """resampy's _resample_loop transcribed sample by sample: float64 weights and products, y[t] a float32 register."""
    x = np.asarray(x, np.float32)
    ratio = float(target_sr) / orig_sr
    win, delta, num_table, scale = R.tables(res_type, ratio)
    n_out = int(x.shape[0] * ratio)
    t_out = np.arange(n_out) / ratio
    index_step = int(scale * num_table)
    nwin, n_orig = win.shape[0], x.shape[0]
    y = np.zeros(n_out, np.float32)
    for t in range(n_out):
        time_register = t_out[t]
        n = int(time_register)
        frac = scale * (time_register - n)
        index_frac = frac * num_table
        offset = int(index_frac)
        eta = index_frac - offset
        for i in range(min(n + 1, (nwin - offset) // index_step)):
            weight = win[offset + i * index_step] + eta * delta[offset + i * index_step]
            y[t] = np.float32(np.float64(y[t]) + weight * np.float64(x[n - i]))
        frac = scale - frac
        index_frac = frac * num_table
        offset = int(index_frac)
        eta = index_frac - offset
        for k in range(min(n_orig - n - 1, (nwin - offset) // index_step)):
            weight = win[offset + k * index_step] + eta * delta[offset + k * index_step]
            y[t] = np.float32(np.float64(y[t]) + weight * np.float64(x[n + k + 1]))
    return y


def _noise(n, seed):
    return (0.3 * np.random.default_rng(seed).standard_normal(n)).astype(np.float32)


@pytest.mark.parametrize("res_type", list(R.FILTERS))
@pytest.mark.parametrize("orig_sr, target_sr", [(16000, 44100), (44100, 16000), (44100, 48000)])
def test_vectorised_restatement_is_the_scalar_loop(res_type, orig_sr, target_sr):
    for n in (3, 40, 700):          # 3 and 40 samples: both wing bounds bind (shorter than the filter's half)
        x = _noise(n, n)
        want = scalar_resampy(x, orig_sr, target_sr, res_type)
        got = R.resampy_resample(x, orig_sr, target_sr, res_type)
        assert got.dtype == np.float32 and np.array_equal(got.view(np.int32), want.view(np.int32)), (n, res_type)


def _multisine(n, rate, freqs):
    t = np.arange(n) / rate
    return sum(0.2 * np.sin(2 * np.pi * f * t + k) for k, f in enumerate(freqs))


# (orig_sr, target_sr, res_type): bar on |y - exact| and on |y - resample_poly| away from the ends.  Upsampling with
# kaiser_best is exact to float32 rounding.  Downsampling carries resampy's gain error: its index step int(scale * num_table)
# truncates 185.8 to 185 at 44.1 -> 16 kHz, so the filter's taps sum to about 1.004 (0.3 % here).  kaiser_fast's pass band
# ends near 0.85 Nyquist, close to the 6 kHz tone.
BARS = [(16000, 44100, "kaiser_best", 5e-6, 1e-3), (16000, 44100, "kaiser_fast", 1e-2, 1e-2),
        (44100, 16000, "kaiser_best", 3e-3, 3e-3), (44100, 16000, "kaiser_fast", 1.5e-2, 1.5e-2)]


@pytest.mark.parametrize("orig_sr, target_sr, res_type, bar, poly_bar", BARS)
def test_band_limited_signal_is_reproduced(orig_sr, target_sr, res_type, bar, poly_bar):
    freqs = [220.0, 1000.0, 3100.0, 6000.0]          # inside both filters' pass band at either rate
    n = orig_sr // 2
    x = _multisine(n, orig_sr, freqs).astype(np.float32)
    want = _multisine(R.out_len(n, orig_sr, target_sr), target_sr, freqs)
    edge = target_sr // 20                           # away from the ends, where the filter sees zeros
    poly = resample_poly(x.astype(np.float64), *(np.array([target_sr, orig_sr]) // np.gcd(target_sr, orig_sr)))
    y = R.resample(x, orig_sr, target_sr, res_type)
    assert y.shape == want.shape
    assert np.abs(y[edge:-edge] - want[edge:-edge]).max() < bar
    assert np.abs(y[edge:-edge] - poly[edge:len(y) - edge]).max() < poly_bar


@pytest.mark.parametrize("variant", R.VARIANTS)
def test_every_variant_changes_bits(variant):
    if variant == "fma_weight":
        # the weight itself changes, but on these signals the float32 rounding after every tap absorbs a one-ulp float64
        # change of the weight: no output bit moves (measured), so the GPU's no-FMA rule is pinned by its weights alone
        win, delta, _, _ = R.tables("kaiser_best", 44100 / 16000)
        rng = np.random.default_rng(5)
        idx, eta = rng.integers(0, len(win) - 1, 10000), rng.random(10000)
        assert (R._fma(eta, delta[idx], win[idx]) != win[idx] + eta * delta[idx]).any()
        return
    x = _noise(8000, 9)
    # downsampling, where the window is scaled, then upsampling
    changed = [(R.resample(x, a, b, "kaiser_fast", variant) != R.resample(x, a, b, "kaiser_fast")).sum()
               for a, b in ((44100, 16000), (16000, 44100))]
    assert changed[0] > 0, variant
    if variant != "unscaled_window":
        assert changed[1] > 0, variant


def test_length_rule_is_librosas_float_ceil():
    from fractions import Fraction
    for orig_sr, target_sr in RATE_PAIRS:
        fr = Fraction(target_sr, orig_sr)
        differ = [n for n in range(1, 20000) if R.out_len(n, orig_sr, target_sr) != -(-n * fr.numerator // fr.denominator)]
        if (orig_sr, target_sr) != (44100, 48000):
            assert differ == [], (orig_sr, target_sr)
            continue
        # 44.1 -> 48 kHz: 147 * (48000 / 44100) rounds above 160, so librosa pads to 161 where the exact ceil is 160
        assert differ[:3] == [147, 294, 441]
        for n in differ[:3]:
            y = R.resample(_noise(n, n), orig_sr, target_sr)
            exact = n * fr.numerator // fr.denominator
            assert len(y) == exact + 1 == H._rate_len(n, orig_sr, target_sr, "kaiser_best")
            assert H._rate_len(n, orig_sr, target_sr) == exact
            assert y[-1] == 0 and len(R.resampy_resample(_noise(n, n), orig_sr, target_sr)) == exact


def test_equal_rates_and_too_short_inputs():
    x = _noise(50, 1)
    assert R.resample(x, 16000, 16000) is x or np.array_equal(R.resample(x, 16000, 16000), x)
    assert len(R.resample(x[:1], 16000, 44100)) == 3
    with pytest.raises(ValueError, match="too small"):
        R.resample(x[:2], 44100, 16000)                  # int(2 * 0.3628) = 0
    with pytest.raises(ValueError, match="too small"):
        E.sinc_lengths(2, 44100, 16000)
    with pytest.raises(ValueError, match="too small"):
        H._rate_len(2, 44100, 16000, "kaiser_best")
    assert E.sinc_lengths(3, 44100, 16000) == (1, 2)


@pytest.mark.parametrize("res_type", list(R.FILTERS))
@pytest.mark.parametrize("ratio", [44100 / 16000, 16000 / 44100, 48000 / 44100])
def test_host_table_is_the_restatements(res_type, ratio):
    win, delta, num_table, _ = R.tables(res_type, ratio)
    t = E.sinc_table(res_type, ratio)
    assert t.shape == (len(win), 2) and t.dtype == np.float64
    assert np.array_equal(t[:, 0], win) and np.array_equal(t[:, 1], delta)
    assert num_table == 2 ** E.RES_TYPES[res_type][1] and E.RES_TYPES[res_type] == R.FILTERS[res_type]
    assert len(win) == {"kaiser_best": 32769, "kaiser_fast": 2049}[res_type]


def test_unknown_res_type_raises_naming_it(tmp_path):
    with pytest.raises(ValueError, match="'soxr_hq'"):
        E.check_res_type("soxr_hq")
    with pytest.raises(ValueError, match="'scipy'"):
        E.resample(None, [np.zeros(100, np.float32)], 16000, 44100, "scipy")
    with pytest.raises(ValueError, match="'kaiser'"):
        AudioMetrics(StubOwner(), rate=16000, res_type="kaiser")
    p = str(tmp_path / "x.wav")
    S.write_pcm16(np.zeros(5000, np.int16), p, 44100)
    with pytest.raises(ValueError, match="'fft'"):
        H.load_wav(p, res_type="fft")
    E.check_res_type(None)


# ------------------------------------------------------------------------------------------ routing with stub engines
class StubEngine:
    """Records resample_sinc_varlen calls; its "resampling" is resampy's zero-padded length of zeros."""
    device = torch.device("cpu")

    def __init__(self):
        self.calls = []

    def resample_sinc_varlen(self, x, lengths, filters, rows, out_lengths):
        self.calls.append((list(lengths), [r for _, r, _ in filters], list(rows), list(out_lengths)))
        return torch.zeros(sum(out_lengths))

    def restore_varlen(self, packed, lengths, unify_energy=False, mel_out=None, log_mel_out=None):
        self.calls.append(("restore", list(lengths)))
        return packed.clone()

    def to_pcm16(self, x, saturate=False):
        return (x * 32768.0).to(torch.int32).to(torch.int16)


class StubModel:
    device = torch.device("cpu")

    def __init__(self):
        self._eng = StubEngine()

    def to(self, device):
        return self

    def _engine(self):
        return self._eng


def _write(path, n, rate, seed=0):
    S.write_pcm16(np.random.default_rng(seed).integers(-2000, 2000, n).astype(np.int16), str(path), rate)
    return str(path)


def test_handler_batch_resamples_every_file_in_one_call(tmp_path, monkeypatch):
    m = StubModel()
    monkeypatch.setattr(H, "model", m)
    monkeypatch.setattr(H, "_mel_metrics", lambda *a: {"scored": True})
    items = [(_write(tmp_path / "a.wav", 16000, 16000), str(tmp_path / "oa.wav"), _write(tmp_path / "ta.wav", 16000, 16000)),
             (_write(tmp_path / "b.wav", 44100, 44100), str(tmp_path / "ob.wav"), None),
             (_write(tmp_path / "c.wav", 22050, 22050), str(tmp_path / "oc.wav"), None),
             (_write(tmp_path / "d.wav", 48000, 48000), str(tmp_path / "od.wav"), _write(tmp_path / "td.wav", 48000, 48000))]
    res = H.handler_batch(items, ckpt=None, device="cpu", meta={"res_type": "kaiser_fast"})
    sinc = [c for c in m._eng.calls if c[0] != "restore"]
    assert len(sinc) == 1
    lengths, ratios, rows, out_lengths = sinc[0]
    assert lengths == [16000, 22050, 48000, 16000, 48000]            # inputs, then targets; the 44.1 kHz file stays out
    assert ratios == [44100 / 16000, 44100 / 22050, 44100 / 48000] and rows == [0, 1, 2, 0, 2]
    assert out_lengths == [44100, 44100, 44100, 44100, 44100]
    assert res == [{"scored": True}, {}, {}, {"scored": True}]


@pytest.mark.parametrize("n, res_type, exc, match", [
    (1, None, EngineError, "1 samples"),                   # resample_poly: 1 sample at 44.1 kHz, too short for the front end
    (1, "kaiser_best", ValueError, "too small"),           # resampy: int(1 * 0.91875) = 0 samples
    (1100, "kaiser_best", EngineError, "1011 samples"),    # librosa's ceil(1100 * 0.91875) = 1011
])
def test_check_file_uses_the_res_types_length(tmp_path, monkeypatch, n, res_type, exc, match):
    m = StubModel()
    monkeypatch.setattr(H, "model", m)
    good = (_write(tmp_path / "good.wav", 30000, 44100), str(tmp_path / "good_out.wav"), None)
    bad = (_write(tmp_path / "bad.wav", n, 48000), str(tmp_path / "bad_out.wav"), None)
    with pytest.raises(exc, match=match):
        H.handler_batch([good, bad], ckpt=None, device="cpu", meta={"res_type": res_type})
    assert m._eng.calls == []


def test_44k1_to_48k_target_frames_follow_the_float_length(tmp_path):
    """A 44.1 kHz est of 147 * k samples scored by a 48 kHz-free path: _rate_len's float rule gives one more sample than
    the exact rule, which is what the frame check of evaluation_batch then counts."""
    for n in (147, 294, 441 * 100):
        assert H._rate_len(n, 44100, 48000, "kaiser_best") == H._rate_len(n, 44100, 48000) + 1


def test_evaluation_batch_resamples_ests_in_one_call_and_checks_their_frames(tmp_path):
    am = AudioMetrics(StubOwner(), rate=16000, res_type="kaiser_best")
    seen = []

    class Eng(StubEngine):
        def score_varlen(self, e, el, t, tl, rate=44100):
            seen.append(("spectral", list(el), list(tl), rate))
            return torch.zeros(len(el), 8, dtype=torch.float64)

    am._owner = Eng()
    pairs = []
    for i, (n_e, n_t) in enumerate([(44100, 16000), (88200, 32000), (16000, 16000)]):
        pe = _write(tmp_path / f"e{i}.wav", n_e, 44100 if n_e != n_t else 16000)
        pt = _write(tmp_path / f"t{i}.wav", n_t, 16000)
        pairs.append((pe, pt))
    res = am.evaluation_batch(pairs)
    assert len(res) == 3 and all(list(r) == list(S.KEYS) for r in res)
    sinc = am._owner.calls
    assert len(sinc) == 1 and sinc[0][0] == [44100, 88200] and sinc[0][3] == [16000, 32000]
    assert seen == [("spectral", [16000, 32000, 16000], [16000, 32000, 16000], 16000)]
    # an est whose librosa length lands on another frame count than its target's fails before the engine
    bad = (_write(tmp_path / "bad_e.wav", 44100 + 882, 44100), _write(tmp_path / "bad_t.wav", 16000, 16000))
    with pytest.raises(ValueError, match="bad_e"):
        am.evaluation_batch([pairs[0], bad])
    assert len(am._owner.calls) == 1
