"""voicefixer_main_b200.lowpass without a GPU: the oracle against the reference's goldens, the module's dispatch and
rejections through a stub engine, and the numpy restatement of vf_sosfiltfilt_varlen's chunked scan (oracle/lowpass.py)."""
import os

import numpy as np
import pytest
import torch
from scipy import signal

from oracle import lowpass as O
from voicefixer_main_b200 import lowpass as LP

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "ref_lowpass.npz"))
X = GOLD["x"]


def _case(key):
    kind, rest = key.split("/", 1)
    return kind, rest.split("/")


@pytest.mark.parametrize("key", [k for k in GOLD.files if k != "x"])
def test_oracle_equals_reference(key):
    if key.startswith("lp/"):
        t, o, c = key.split("/")[1:]
        got = O.lowpass(X, float(c), 44100, int(o), _type=t)
    elif key.startswith("bp/"):
        t, o = key.split("/")[1:]
        got = O.bandpass(X, 1000, 8000, 44100, int(o), _type=t)
    elif key == "lpf_cheby2":
        got = O.lowpass_filter(X, 4000, 44100, 6, "cheby2")
    elif key == "bpf_cheby2":
        got = O.bandpass_filter(X, 500, 6000, 44100, 4, "cheby2")
    else:
        got = O.collate_val([X], (int(key.split("/")[1]),))[int(key.split("/")[1])][0]
    ref = GOLD[key]
    assert got.dtype == ref.dtype and got.shape == ref.shape
    if "stft_hard" in key:       # float32 STFT / ISTFT stand-ins: the same ops, summed in whatever order torch picks
        assert np.abs(got - ref).max() < 1e-6
    else:
        assert np.array_equal(got, ref)


class StubEngine:
    """The engine's float64 entry points computed with scipy on the CPU, recording every call."""
    device = torch.device("cpu")

    def __init__(self):
        self.calls = []

    def sosfiltfilt_varlen(self, x, lengths, sos, zi, rows, f32):
        self.calls.append(("sos", list(lengths), [s.shape[0] for s in sos], list(rows), list(f32)))
        for s, z in zip(sos, zi):
            assert np.array_equal(z, signal.sosfilt_zi(s))
        parts = [p.numpy().astype(np.float32) if f else p.numpy() for p, f in zip(torch.split(x, list(lengths)), f32)]
        return torch.cat([torch.from_numpy(signal.sosfiltfilt(sos[r], p).copy()) for p, r in zip(parts, rows)])

    def resample_poly_f64_varlen(self, x, lengths, filters, rows, out_lengths):
        self.calls.append(("resample", list(lengths), [(u, d) for u, d, _ in filters], list(rows), list(out_lengths)))
        outs = []
        for p, r, n in zip(torch.split(x, list(lengths)), rows, out_lengths):
            u, d, taps = filters[r]
            assert np.array_equal(taps.numpy(), signal.firwin(20 * max(u, d) + 1, 1 / max(u, d), window=("kaiser", 5.0)) * u)
            y = signal.resample_poly(p.numpy(), u, d)
            outs.append(torch.from_numpy(O.align_length(np.zeros(n), y)))
        return torch.cat(outs)


@pytest.mark.parametrize("key", [k for k in GOLD.files if k.startswith(("lp/", "bp/", "lpf", "bpf", "sr/"))
                                 and "stft_hard" not in k])
def test_module_dispatch_matches_reference(key):
    eng = StubEngine()
    if "/stft/" in key:       # scipy computes "stft" in the input's dtype: pinned on float64 input, where all versions agree
        t, o, c = key.split("/")[1:]
        x64 = X.astype(np.float64)
        got = LP.lowpass(eng, x64, float(c), 44100, int(o), _type=t)
        assert got.dtype == torch.float64 and np.array_equal(got.numpy(), O.lowpass(x64, float(c), 44100, int(o), _type=t))
        assert np.abs(got.numpy() - GOLD[key]).max() < 1e-6      # the reference's float32 result, one float32 rounding away
        return
    if key.startswith("lp/"):
        t, o, c = key.split("/")[1:]
        got = LP.lowpass(eng, X, float(c), 44100, int(o), _type=t)
    elif key.startswith("bp/"):
        t, o = key.split("/")[1:]
        got = LP.bandpass(eng, torch.from_numpy(X), 1000, 8000, 44100, int(o), _type=t)
    elif key == "lpf_cheby2":
        got = LP.lowpass_filter(eng, X, 4000, 44100, 6, "cheby2")
    elif key == "bpf_cheby2":
        got = LP.bandpass_filter(eng, X, 500, 6000, 44100, 4, "cheby2")
    else:
        c = int(key.split("/")[1])
        got = LP.sr_validation_inputs(eng, [X], (c,))[c][0]
    ref = GOLD[key]
    assert isinstance(got, torch.Tensor) and got.numpy().dtype == ref.dtype
    assert np.array_equal(got.numpy(), ref)


def test_dispatch_is_a_substring_test_in_reference_order():
    eng = StubEngine()
    for t in ("", "b", "e", "butter", "t", "er"):
        LP.lowpass(eng, X, 4000, 44100, 4, _type=t)
        assert eng.calls[-1][0] == "sos" and eng.calls[-1][2] == [2]          # butter order 4
    LP.lowpass(eng, X, 4000, 44100, 4, _type="c")                            # "c" is in "cheby1"
    np.testing.assert_array_equal(eng.calls[-1][2], [2])
    LP.lowpass(eng, X, 4000, 44100, 4, _type="s")                            # "s" is in "bessel"
    LP.lowpass(eng, X, 4000, 44100, 4, _type="ft")                           # stft: down, then up
    assert [c[0] for c in eng.calls[-2:]] == ["resample"] * 2 and eng.calls[-2][2] == [(80, 441)]
    with pytest.raises(ValueError, match="Unexpected filter type cheby2"):
        LP.lowpass(eng, X, 4000, 44100, 4, _type="cheby2")
    with pytest.raises(ValueError, match="Unexpected filter type stft_hard"):
        LP.bandpass(eng, X, 100, 4000, 44100, 4, _type="stft_hard")


def test_order_clamp_and_int_cutoff():
    assert (LP.limit(12, 10, 2), LP.limit(1, 10, 2), LP.limit(5.7, 10, 2)) == (10, 2, 5)
    eng = StubEngine()
    a = LP.lowpass(eng, X, 4000.9, 44100, 30, _type="butter")
    b = LP.lowpass(eng, X, 4000, 44100, 10, _type="butter")
    assert eng.calls[-1][2] == [5] and torch.equal(a, b)
    LP.lowpass(eng, X, 4000, 44100, 5.9, _type="ellip")
    assert eng.calls[-1][2] == [3]                                           # int(5.9) = 5 -> 3 sections
    # "stft": lowpass_ratio = highcut / int(fs / 2) and fs_ori fixed at 44100, whatever fs is
    LP.lowpass(eng, X, 4000, 16000, 8, _type="stft")
    assert eng.calls[-2][2] == [(1, 2)]                                      # int(4000 / 8000 * 44100) = 22050


@pytest.mark.parametrize("order,btype,edge", [(2, "low", 9), (3, "low", 12), (8, "low", 27), (5, "band", 33)])
def test_padlen_even_and_odd_orders(order, btype, edge):
    wn = 0.2 if btype == "low" else [0.1, 0.3]
    sos = signal.butter(order, wn, btype=btype, output="sos")
    assert LP.padlen(sos) == edge
    eng = StubEngine()
    x = np.ones(edge)
    call = (lambda v: LP.lowpass(eng, v, 0.2 * 22050, 44100, order)) if btype == "low" else \
        (lambda v: LP.bandpass(eng, v, 0.1 * 22050, 0.3 * 22050, 44100, order))
    with pytest.raises(ValueError) as e:
        call(x)
    with pytest.raises(ValueError) as e_ref:
        signal.sosfiltfilt(sos, x)
    assert str(e.value) == str(e_ref.value) == f"The length of the input vector x must be greater than padlen, which is {edge}."
    assert not eng.calls
    assert call(np.ones(edge + 1)).numel() == edge + 1


def test_align_length_both_ways():
    for y in (np.arange(5.0), torch.arange(5.0)):
        assert list(LP.align_length(np.zeros(7), y)) == [0, 1, 2, 3, 4, 0, 0]
        assert list(LP.align_length(np.zeros(3), y)) == [0, 1, 2]
        assert LP.align_length(np.zeros(5), y) is y
    eng = StubEngine()                                   # stft: the second resample is cut / padded to the input length
    for n in (2205, 2206, 2207, 1001):
        assert LP.lowpass(eng, np.ones(n), 1000, 44100, _type="stft").numel() == n
        assert eng.calls[-1][-1] == [n]


def _raises_like(call_ref, call_ours):
    with pytest.raises(Exception) as e_ref:
        call_ref()
    eng = StubEngine()
    with pytest.raises(type(e_ref.value)) as e:
        call_ours(eng)
    assert str(e.value) == str(e_ref.value)
    assert not eng.calls


def test_rejections_match_the_reference():
    x2 = np.zeros((100, 1))
    _raises_like(lambda: O.lowpass(x2, 1000, 44100), lambda e: LP.lowpass(e, x2, 1000, 44100))
    _raises_like(lambda: O.bandpass(x2, 100, 1000, 44100), lambda e: LP.bandpass(e, x2, 100, 1000, 44100))
    _raises_like(lambda: O.lowpass(X, 1000, 44100, _type="cheb2"), lambda e: LP.lowpass(e, X, 1000, 44100, _type="cheb2"))
    _raises_like(lambda: O.lowpass(X, 23000, 44100), lambda e: LP.lowpass(e, X, 23000, 44100))            # Wn >= 1
    _raises_like(lambda: O.lowpass(X, 0, 44100, _type="ellip"), lambda e: LP.lowpass(e, X, 0, 44100, _type="ellip"))
    _raises_like(lambda: O.bandpass(X, 3000, 30000, 44100), lambda e: LP.bandpass(e, X, 3000, 30000, 44100))
    _raises_like(lambda: O.lowpass(X, 0.1, 44100, _type="stft"), lambda e: LP.lowpass(e, X, 0.1, 44100, _type="stft"))
    _raises_like(lambda: O.lowpass_filter(X, 1000, 44100, 4, "cheb"), lambda e: LP.lowpass_filter(e, X, 1000, 44100, 4, "cheb"))
    _raises_like(lambda: O.bandpass_filter(X, 1, 900, 44100, 4, "x"), lambda e: LP.bandpass_filter(e, X, 1, 900, 44100, 4, "x"))
    # a bad clip anywhere in a batch fails the whole call before any work
    eng = StubEngine()
    with pytest.raises(ValueError):
        LP.lowpass_batch(eng, [X, X[:20]], [1000, 1000], [8, 8], ["butter", "butter"])
    assert not eng.calls


FILTERS = [("butter", 8, 1000 / 22050), ("ellip", 10, 1000 / 22050), ("cheby1", 3, 0.5), ("bessel", 10, 12000 / 22050),
           ("cheby2", 5, 0.2), ("ellip", 10, [1000 / 22050, 8000 / 22050])]


def _sos(t, o, wn):
    return O.design(t, o, wn, "band" if isinstance(wn, list) else "low")


@pytest.mark.parametrize("f", FILTERS, ids=lambda f: f"{f[0]}{f[1]}")
def test_chunked_scan_matches_scipy(f):
    sos = _sos(*f)
    edge = LP.padlen(sos)
    rng = np.random.default_rng(7)
    worst = 0.0
    for n in (edge + 1, 1024 - 1 - 2 * edge, 1024 - 2 * edge, 1024 + 1 - 2 * edge, 4 * 1024 + 17, 30000):
        for x in (rng.standard_normal(n), np.ones(n), np.eye(1, n, 0)[0], np.eye(1, n, n - 1)[0]):
            err = np.abs(O.chunked_sosfiltfilt(sos, x) - signal.sosfiltfilt(sos, x)).max()
            assert err <= O.iir_bar(x), (n, err)
            worst = max(worst, err / O.iir_bar(x))
    print(f"{f}: worst error {worst:.2e} of the bar, rounding gain {O.rounding_gain(sos):.1f}")


@pytest.mark.parametrize("brk", ["zi_unscaled", "even_ext", "edge+1", "edge-1", "float32_state", "skip_carry", "drop_section"])
def test_broken_scans_land_far_outside_the_bar(brk):
    rng = np.random.default_rng(11)
    x = rng.standard_normal(20000) + 0.5          # a DC offset: the extension and zi carry it
    worst = max(np.abs(O.chunked_sosfiltfilt(_sos(*f), x, break_=brk) - signal.sosfiltfilt(_sos(*f), x)).max()
                for f in FILTERS)
    assert worst > 100 * O.iir_bar(x), (brk, worst)


class PcmStubEngine(StubEngine):
    def to_pcm16(self, x):
        """save_wave's conversion: x * 2^15 truncated through int32, low 16 bits kept."""
        return torch.from_numpy((x.numpy().astype(np.float64) * 32768.0).astype(np.int32).astype(np.int16))


def _write(path, samples, rate=44100):
    from voicefixer_main_b200.handler import save_pcm16
    save_pcm16((np.asarray(samples) * 32768.0).astype(np.int16), str(path), rate)


def test_make_sr_testset_writes_wavs_and_pair_lists(tmp_path):
    from voicefixer_main_b200.handler import read_pcm16
    rng = np.random.default_rng(3)
    paths = []
    for i, n in enumerate((3000, 4410, 5001)):
        p = tmp_path / "clean" / f"c{i}.wav"
        p.parent.mkdir(exist_ok=True)
        _write(p, 0.3 * rng.standard_normal(n).clip(-1, 0.99))
        paths.append(str(p))
    eng = PcmStubEngine()
    lists = LP.make_sr_testset(eng, paths, str(tmp_path / "out"), cutoffs=(1000, 8000))
    assert sorted(lists) == [1000, 8000]
    for c, lst in lists.items():
        assert lst == str(tmp_path / "out" / "cheby1" / f"pair_cheby1_{c}.lst")
        lines = open(lst).read().splitlines()
        assert len(lines) == len(paths)
        for line, clean in zip(lines, paths):
            deg, tgt = line.split(" ")                       # config.py's "input target" line
            assert tgt == os.path.abspath(clean)
            assert deg == os.path.abspath(tmp_path / "out" / "cheby1" / str(c) / os.path.basename(clean))
            x, _ = read_pcm16(clean)
            y, rate = read_pcm16(deg)
            assert rate == 44100 and len(y) == len(x)
            ref = O.collate_val([x], (c,))[c][0]            # the recipe, converted as save_wave converts it
            assert np.array_equal(y, (ref.astype(np.float64) * 32768.0).astype(np.int32).astype(np.int16) / np.float32(32768.0))


def test_make_sr_testset_rejects_before_any_work(tmp_path):
    a, b = tmp_path / "a", tmp_path / "b"
    a.mkdir()
    b.mkdir()
    for d in (a, b):
        _write(d / "same.wav", np.zeros(3000))
    _write(a / "slow.wav", np.zeros(3000), rate=16000)
    eng = PcmStubEngine()
    with pytest.raises(ValueError, match="share the file name same.wav"):
        LP.make_sr_testset(eng, [str(a / "same.wav"), str(b / "same.wav")], str(tmp_path / "out"))
    with pytest.raises(ValueError, match="16000 Hz"):
        LP.make_sr_testset(eng, [str(a / "same.wav"), str(a / "slow.wav")], str(tmp_path / "out"))
    with pytest.raises(ValueError, match="white space"):
        LP.make_sr_testset(eng, [str(a / "same.wav")], str(tmp_path / "o u t"))
    assert not eng.calls and not (tmp_path / "out").exists()
