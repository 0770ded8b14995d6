"""The SR degradations on the GPU (voicefixer_main_b200.lowpass: vf_sosfiltfilt_varlen, vf_resample_poly_f64_varlen)
against oracle/lowpass.py (scipy, float64).  The IIR and "stft" bar is oracle.lowpass.IIR_BAR * max|x| (1e-9; derived in
the oracle's docstring): the scan's only error is fp64 rounding."""
import numpy as np
import pytest
import torch

from oracle import lowpass as O
from oracle import vf_oracle as VO
from voicefixer_main_b200 import _lib as L
from voicefixer_main_b200 import lowpass as LP

pytestmark = pytest.mark.gpu

C = O.IIR_CHUNK
SR = 44100


@pytest.fixture(scope="module")
def eng():
    from voicefixer_main_b200.model import Engine
    e = Engine("cuda:0")
    e.load_state({}, need=())
    yield e
    e.close()
    torch.cuda.empty_cache()


def _signals(edge, seed):
    """(name, float64 signal): the shortest legal row, chunk-boundary rows (C - 1, C, C + 1 extended samples), 1 s and
    60 s of noise and speech-like clips, zeros, DC, impulses at the first and last sample, and +-1 full scale."""
    rng = np.random.default_rng(seed)
    out = [("shortest", rng.standard_normal(edge + 1))]
    for d in (-1, 0, 1):
        if C + d - 2 * edge > edge:
            out.append((f"ext={C + d}", rng.standard_normal(C + d - 2 * edge)))
    out += [("noise1s", 0.3 * rng.standard_normal(SR)), ("synth1s", VO.synth_clips(1, SR, seed=seed)[0].double().numpy()),
            ("zeros", np.zeros(5000)), ("dc", np.full(5000, 0.7)), ("imp0", np.eye(1, 5000, 0)[0]),
            ("imp_last", np.eye(1, 5000, 4999)[0]), ("full", np.where(rng.standard_normal(SR) > 0, 1.0, -1.0)),
            ("noise60s", 0.3 * rng.standard_normal(60 * SR))]
    return out


def _check(got, ref, x, what, worst):
    got = got.cpu().numpy()
    assert got.shape == ref.shape, what
    if not np.any(x):
        assert not np.any(got), what                    # zeros in, exact zeros out
        return
    err = float(np.abs(got - ref).max())
    bar = O.iir_bar(x)
    worst[0] = max(worst[0], err / bar)
    assert err <= bar, (what, err, bar)


@pytest.mark.parametrize("ftype", ["butter", "cheby1", "ellip", "bessel"])
def test_lowpass_iir_matches_scipy(eng, ftype):
    worst = [0.0]
    for order in (2, 3, 8, 10):
        for cutoff in (1000, 4000, 12000, 21000):
            edge = LP.padlen(O.design(ftype, order, cutoff / (0.5 * SR), "low"))
            sigs = _signals(edge, order * cutoff)
            ys = LP.lowpass_batch(eng, [x for _, x in sigs], [cutoff] * len(sigs), [order] * len(sigs), [ftype] * len(sigs))
            for (name, x), y in zip(sigs, ys):
                assert y.dtype == torch.float64
                _check(y, O.lowpass(x, cutoff, SR, order, _type=ftype), x, (ftype, order, cutoff, name), worst)
    print(f"{ftype}: worst IIR error {worst[0]:.2e} of the bar")


@pytest.mark.parametrize("ftype", ["butter", "cheby1", "ellip", "bessel"])
def test_bandpass_matches_scipy(eng, ftype):
    worst = [0.0]
    for order in (2, 5, 10):
        edge = LP.padlen(O.design(ftype, order, [1000 / 22050, 8000 / 22050], "band"))
        for name, x in _signals(edge, order)[:-1]:
            _check(LP.bandpass(eng, x, 1000, 8000, SR, order, _type=ftype), O.bandpass(x, 1000, 8000, SR, order, _type=ftype),
                   x, (ftype, order, name), worst)
    print(f"bandpass {ftype}: worst error {worst[0]:.2e} of the bar")


def test_float32_input_matches_scipy_on_float32(eng):
    """scipy builds the odd extension of float32 input in float32: the kernel rounds it the same way."""
    rng = np.random.default_rng(5)
    for ftype, order, cutoff in (("ellip", 10, 1000), ("butter", 8, 4000)):
        x = (0.5 * rng.standard_normal(30000) + 0.2).astype(np.float32)
        ref = O.lowpass(x, cutoff, SR, order, _type=ftype)
        _check(LP.lowpass(eng, x, cutoff, SR, order, _type=ftype), ref, x, (ftype, "f32"), [0.0])
        _check(LP.lowpass(eng, torch.from_numpy(x).cuda(), cutoff, SR, order, _type=ftype), ref, x, (ftype, "f32 dev"), [0.0])


def test_stft_matches_scipy_on_float64(eng):
    worst = [0.0]
    for cutoff in (1000, 4000, 12000, 21000):
        for name, x in _signals(27, cutoff):
            _check(LP.lowpass(eng, x, cutoff, SR, _type="stft"), O.lowpass(x, cutoff, SR, _type="stft"), x, (cutoff, name), worst)
    print(f"stft: worst error {worst[0]:.2e} of the bar")


def test_sr_validation_inputs_within_one_float32_rounding(eng):
    """The float64 results differ by at most the IIR bar, then each is rounded once to float32: |got - ref| <= one float32
    spacing of ref + the bar (near zero the bar dominates: a float32 spacing there is far below fp64 rounding of the sums)."""
    clips = [VO.synth_clips(1, n, seed=n)[0].numpy() for n in (SR // 2 + 17, 3 * SR + 5, 60 * SR)]
    got = LP.sr_validation_inputs(eng, clips)
    ref = O.collate_val(clips)
    for c in O.SR_CUTOFFS:
        for x, g, r in zip(clips, got[c], ref[c]):
            g = g.cpu().numpy()
            assert g.dtype == np.float32 and g.shape == r.shape
            assert np.all(np.abs(g.astype(np.float64) - r) <= np.spacing(np.abs(r)) + O.iir_bar(x)), c


def test_rows_are_bit_identical_alone_in_a_batch_and_across_a_split(eng):
    rng = np.random.default_rng(9)
    probe = 0.3 * rng.standard_normal(3 * SR + 11)
    alone = LP.lowpass(eng, probe, 2000, SR, 8, _type="ellip")
    alone_stft = LP.lowpass(eng, probe, 2000, SR, _type="stft")
    others = [0.3 * rng.standard_normal(int(n)) for n in rng.integers(300, 50000, 70)]
    for slot in (0, 33, 64, 70):               # 64 rows per sub-batch: slot 64 and 70 land in the second
        wavs = others[:slot] + [probe] + others[slot:]
        cuts = [1000 * int(c) for c in rng.integers(1, 20, len(wavs))]
        cuts[slot] = 2000
        kinds = ["ellip" if i % 3 else "butter" for i in range(len(wavs))]
        kinds[slot] = "ellip"
        ys = LP.lowpass_batch(eng, wavs, cuts, [8] * len(wavs), kinds)
        assert torch.equal(ys[slot], alone), slot
        ys = LP.lowpass_batch(eng, wavs, cuts, [8] * len(wavs), ["stft"] * len(wavs))
        assert torch.equal(ys[slot], alone_stft), slot
    big = [0.1 * rng.standard_normal(60 * SR) for _ in range(6)]       # 6 x 60 s > 2^24 extended samples: split by size
    ys = LP.lowpass_batch(eng, big + [probe], [2000] * 7, [8] * 7, ["ellip"] * 7)
    assert torch.equal(ys[-1], alone)


def test_stft_hard_meets_the_front_end_and_istft_bars(eng):
    for n, ratio_cut in ((SR, 4000), (SR // 3 + 5, 12000)):
        x = VO.synth_clips(1, n, seed=n)[0].numpy()
        got = LP.lowpass(eng, x, ratio_cut, SR, _type="stft_hard")
        ref = O.lowpass(x, ratio_cut, SR, _type="stft_hard")
        assert got.dtype == torch.float32 and got.shape == (n,)
        err = float(np.abs(got.cpu().numpy() - ref).max())
        print(f"stft_hard n={n}: max error {err:.2e}")
        assert err < 1e-4 * np.abs(x).max(), err


def _einval(call):
    with pytest.raises(L.EngineError) as e:
        call()
    assert e.value.code == L.VF_EINVAL


def test_abi_rejections(eng):
    from scipy import signal
    sos = signal.butter(8, 0.1, output="sos")
    zi = signal.sosfilt_zi(sos)
    x = torch.zeros(100, dtype=torch.float64, device="cuda")
    _einval(lambda: eng.sosfiltfilt_varlen(x[:27], [27], [sos], [zi], [0]))          # not longer than padlen 27
    _einval(lambda: eng.sosfiltfilt_varlen(x, [100], [sos], [zi], [1]))              # no filter 1
    _einval(lambda: eng.sosfiltfilt_varlen(x, [100], [sos[:0]], [zi[:0]], [0]))      # zero sections
    bad = sos.copy()
    bad[1, 3] = 2.0
    _einval(lambda: eng.sosfiltfilt_varlen(x, [100], [bad], [zi], [0]))              # a0 != 1
    _einval(lambda: eng.sosfiltfilt_varlen(x, [40, 0, 60], [sos], [zi], [0, 0, 0]))  # an empty row
    taps = torch.ones(5, dtype=torch.float64, device="cuda")
    _einval(lambda: eng.resample_poly_f64_varlen(x, [100], [(1, 2, taps[:4])], [0], [50]))   # even tap count
    _einval(lambda: eng.resample_poly_f64_varlen(x, [100], [(0, 2, taps)], [0], [50]))       # up = 0
    _einval(lambda: eng.resample_poly_f64_varlen(x, [100], [(1, 2, taps)], [3], [50]))       # no filter 3
    with pytest.raises(TypeError):
        eng.sosfiltfilt_varlen(x.float(), [100], [sos], [zi], [0])


def test_non_finite_rows_stay_in_their_row(eng):
    """A NaN or Inf row comes out non-finite where scipy's does, and leaves nothing in the scratch that reaches another
    row: a clean row in a later sub-batch of the same call, or of a later call whose scratch layout differs, keeps the bits
    of its own lowpass()."""
    rng = np.random.default_rng(21)
    probe = 0.3 * rng.standard_normal(2 * SR + 7)
    alone = {t: LP.lowpass(eng, probe, 4000, SR, 4, _type=t) for t in ("butter", "ellip")}
    bad_nan, bad_inf = 0.3 * rng.standard_normal(SR), 0.3 * rng.standard_normal(SR)
    bad_nan[SR // 2] = np.nan
    bad_inf[100] = np.inf
    fill = [0.3 * rng.standard_normal(int(n)) for n in rng.integers(2000, 200000, 80)]
    for t in ("butter", "ellip"):                       # butter 4: 2 sections, so 16 of the 20 carry lanes are unused
        wavs = [bad_nan, bad_inf] + fill[:62] + [probe] + fill[62:]   # the bad rows in sub-batch 1, the probe in 2
        ys = LP.lowpass_batch(eng, wavs, [4000] * len(wavs), [4] * len(wavs), [t] * len(wavs))
        for x, y in zip(wavs[:2], ys[:2]):
            ref = O.lowpass(x, 4000, SR, 4, _type=t)
            assert np.array_equal(np.isfinite(y.cpu().numpy()), np.isfinite(ref)), t
        assert torch.equal(ys[64], alone[t]), t
        assert all(torch.isfinite(y).all() for y in ys[2:])
        short = fill[70:75] + [probe]                   # a later call: smaller rows, so old yf lies under the new state
        ys = LP.lowpass_batch(eng, short, [4000] * 6, [4] * 6, [t] * 6)
        assert torch.equal(ys[-1], alone[t]), t
