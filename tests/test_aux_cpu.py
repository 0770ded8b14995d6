"""The float64 references of tests/test_gpu_aux.py, checked without a GPU: they restate the oracle's ops, and the checks the
GPU tests apply (the same functions, fed a plausibly broken kernel's output instead of the kernel's) fail for each of the
errors a whole-network bar cannot see."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_gpu_aux as A
from oracle import layers as R
from oracle import vf_oracle as O
from voicefixer_main_b200.arch import VocoderConfig


def _bits32(v):
    return np.asarray(v, np.float32).view(np.uint32).copy()


# ------------------------------------------------------------------ the references restate the oracle
def test_conditioning_matches_the_oracle():
    cfg = VocoderConfig()
    g = torch.Generator().manual_seed(1)
    for T in (37, 40):
        mel = torch.exp(torch.randn(2, 1, T, 128, generator=g, dtype=torch.float64) * 4)
        want = O.vocoder_condition(mel, cfg).permute(0, 2, 1).numpy()
        got = R.voc_condition(mel[:, 0].numpy(), 0, O.mel_weight(cfg).double().numpy(), R.voc_frames(T, cfg.tail_pad_base))
        assert got.shape == want.shape == (2, T + T % 2 + 4, 128)
        assert np.abs(got - want).max() <= 1e-12
        # is_log: from_log (pytorch_util.py:161-163) first
        got_log = R.voc_condition(np.log10(mel[:, 0].numpy()), 1, O.mel_weight(cfg).double().numpy(), want.shape[1])
        assert np.abs(got_log - want).max() <= 1e-12


def test_band_sums_match_amp_to_original_f():
    g = torch.Generator().manual_seed(2)
    est = torch.exp(torch.randn(2, 1, 37, 128, generator=g, dtype=torch.float64))
    tgt = torch.exp(torch.randn(2, 1, 37, 128, generator=g, dtype=torch.float64))
    s = R.band_sums(tgt[:, 0].numpy(), np.log10(est[:, 0].numpy()))
    want, _ = O.amp_to_original_f(est, tgt)
    got = est[:, 0].numpy() * (s[:, 0] / s[:, 1])[:, None, None]
    assert np.abs(got - want[:, 0].numpy()).max() <= 1e-12 * float(want.abs().max())


def test_reflect_and_tail_match_the_generator_tail():
    """The last lines of vocoder_generator: ReflectionPad1d(3), Conv1d(C -> 1, k7), tanh."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 64, 300, generator=g, dtype=torch.float64)
    w = torch.randn(1, 64, 7, generator=g, dtype=torch.float64) / 20
    want = torch.tanh(F.conv1d(F.pad(x, (3, 3), mode="reflect"), w, torch.tensor([0.1], dtype=torch.float64)))
    out, _, _ = R.voc_tail(R.reflect_pad(x.permute(0, 2, 1).numpy(), 3), w.numpy(), 0.1, True)
    assert np.abs(out - want[:, 0].numpy()).max() <= 1e-14


def test_first_layer_and_pool_match_the_unet_ops():
    """encoder_block1.conv_block1 of unet_forward (input padded to the UNet's 64 frames, last bin dropped) up to bn2 +
    LeakyReLU, its shortcut, and F.avg_pool2d."""
    g = torch.Generator().manual_seed(4)
    T, W = 101, 127
    x = torch.randn(1, 1, T, W + 1, generator=g, dtype=torch.float64)
    rnd = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    sd = {"bn1.weight": rnd(1), "bn1.bias": rnd(1), "bn1.running_mean": rnd(1), "bn1.running_var": rnd(1).abs() + 0.5,
          "bn2.weight": rnd(32), "bn2.bias": rnd(32), "bn2.running_mean": rnd(32), "bn2.running_var": rnd(32).abs() + 0.5,
          "conv1.weight": rnd(32, 1, 3, 3), "shortcut.weight": rnd(32, 1, 1, 1), "shortcut.bias": rnd(32)}
    Tp = O.padded_frames(T)
    xp = F.pad(x, (0, 0, 0, Tp - T))[..., :W]
    h = F.leaky_relu(O._bn(xp, sd, "bn1"), O.LRELU_SLOPE)
    a_want = F.leaky_relu(O._bn(F.conv2d(h, sd["conv1.weight"], padding=1), sd, "bn2"), O.LRELU_SLOPE)
    r_want = F.conv2d(xp, sd["shortcut.weight"], sd["shortcut.bias"])
    fold = lambda p: (sd[p + ".weight"] / torch.sqrt(sd[p + ".running_var"] + O.BN_EPS),)
    s1, = fold("bn1")
    t1 = sd["bn1.bias"] - sd["bn1.running_mean"] * s1
    s2, = fold("bn2")
    t2 = sd["bn2.bias"] - sd["bn2.running_mean"] * s2
    _, _, a, r = R.unet_first(x[:, 0], Tp, s1, t1, sd["conv1.weight"], s2, t2, sd["shortcut.weight"], sd["shortcut.bias"])
    assert Tp == 128
    assert (a - a_want).abs().max() <= 1e-12 and (r - r_want).abs().max() <= 1e-12
    v, _ = R.pool(a, torch.ones(32), torch.zeros(32))
    assert torch.equal(v, F.avg_pool2d(a, kernel_size=(2, 2))) and v.shape[-1] == W // 2


def test_fused_istft_matches_the_oracle_istft():
    """istft(mag cos, mag sin) with cos / sin of wav_to_spectrogram_phase(exact=True)."""
    g = torch.Generator().manual_seed(5)
    n = 30 * 441 + 123
    wav = torch.randn(1, 1, n, generator=g, dtype=torch.float64) * 0.3
    wav[..., 4000:7000] = 0
    T = 1 + n // 441
    mag = torch.rand(1, 1, T, 1025, generator=g, dtype=torch.float64) * 2
    _, cos, sin = O.wav_to_spectrogram_phase(wav, exact=True)
    want = O.istft(mag * cos, mag * sin, n)[0].numpy()
    got = R.istft_fused(mag[0, 0].numpy(), wav[0, 0].numpy(), T)
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()


def test_lengths_formula_matches_the_plans_geometry():
    off = A.offsets([A.n_for_frames(37), A.n_for_frames(3), A.n_for_frames(16)])
    rows = A.lengths_rows(off, 127)
    assert list(rows[9]) == [42, 8, 20] and list(rows[13]) == [18522, 3528, 8820]
    assert list(rows[1]) == [64, 64, 64] and list(rows[2]) == [64 * 128] * 3


# ------------------------------------------------------------------ the checks fail for each broken kernel
def _first(mutate):
    name = "first.mel_T101_neg_shift"
    c, x, p, Ts, T, a2, sc = A.first_case(name, A.FIRST_CASES[name])
    Tp = (T + 63) // 64 * 64
    c.oc.Tp = Tp
    xb = x[:, :T].astype(np.float64)
    xb[..., -1] = 0
    h, y, a, r = R.unet_first(xb, Tp, p["bn1_scale"], p["bn1_shift"], p["w1"], p["bn2_scale"], p["bn2_shift"], p["w_sc"], p["b_sc"])
    if mutate:          # the padded rows as zeros instead of lrelu(bn1_shift)
        h = h.clone()
        h[:, :, T:] = 0
        y = F.conv2d(h, torch.as_tensor(p["w1"], dtype=torch.float64).reshape(32, 1, 3, 3), padding=1)
        s = lambda v: torch.as_tensor(v, dtype=torch.float64)[None, :, None, None]
        a = R.lrelu(y * s(p["bn2_scale"]) + s(p["bn2_shift"]), 0.01)
    rows = lambda t: R.nchw_to_rows(t.float())
    a2[:] = A.split_bits(rows(a))
    sc[:] = rows(r).numpy().view(np.uint32)
    return A.check_first(name, c, x, p, Ts, T, a2, sc)


def test_first_check_passes_the_reference_and_catches_zero_padded_rows():
    _first(False)
    with pytest.raises(AssertionError):
        _first(True)


def _pool(mode):
    name = "pool.mel_l0"
    c, x, sc, sh, out_r, out_a, out_raw, rv = A.pool_case(name, A.POOL_CASES[name])
    B, H, Wp, C = x.shape
    c.oc.Wpo = Wpo = ((Wp - 1) >> 1) + 1
    xt = torch.as_tensor(np.where(np.isfinite(x) & (np.abs(x) < 1e29), x, 0.5)[:, :, :Wp - 1].astype(np.float64)).permute(0, 3, 1, 2)
    if mode == "ceil":          # ceil pooling: the odd last column makes one more output column
        v = F.avg_pool2d(xt, 2, ceil_mode=True)
    else:
        v = F.avg_pool2d(xt, 2)
    a = R.lrelu(v * torch.as_tensor(sc, dtype=torch.float64)[None, :, None, None] +
                torch.as_tensor(sh, dtype=torch.float64)[None, :, None, None], 0.01)
    lay = lambda t: F.pad(t, (0, Wpo - t.shape[-1])).permute(0, 2, 3, 1).reshape(B, -1, C)
    out_raw[:] = lay(v).numpy().astype(np.float32).view(np.uint32)
    out_r[:] = A.split_bits(lay(v))
    out_a[:] = A.split_bits(lay(a))
    return A.check_pool(name, c, x, sc, sh, out_r, out_a, out_raw, rv)


def test_pool_check_passes_the_reference_and_catches_ceil_pooling():
    _pool("floor")
    with pytest.raises(AssertionError):
        _pool("ceil")


def test_reflect_check_catches_a_symmetric_pad():
    g = np.random.default_rng(7)
    Ls = [42, 20]
    pl = A.planes16((2, 48, 64))
    for b, Lb in enumerate(Ls):
        pl[:, b, 3:3 + Lb] = g.integers(0, 0x7C00, (2, Lb, 64), dtype=np.uint16)
    good, sym = pl.copy(), pl.copy()
    for b, Lb in enumerate(Ls):
        good[:, b, :Lb + 6] = R.reflect_pad(pl[:, b, 3:3 + Lb].astype(np.int32), 3)
        inner = torch.as_tensor(pl[:, b, 3:3 + Lb].astype(np.int64)).permute(0, 2, 1)
        sym[:, b, :Lb + 6] = torch.cat([inner[..., :3].flip(-1), inner, inner[..., -3:].flip(-1)], -1).permute(0, 2, 1).numpy()
    A.check_reflect("reflect.ok", pl, good, Ls)
    with pytest.raises(AssertionError):
        A.check_reflect("reflect.symmetric", pl, sym, Ls)


def _tail(reverse):
    name = "tail.L3528_T3"
    c, bits, w, bias, wav, peak, Ls = A.tail_case(name, A.TAIL_CASES[name], 1, 0)
    c.oc.C, c.oc.L, c.oc.tail_smem = 64, max(Ls), 7 * 64 * 4 + 326 * 72 * 2
    x = R.from_bits(bits[0])
    ww = w[:, :, ::-1] if reverse else w
    for b, Lb in enumerate(Ls):
        out, _, _ = R.voc_tail(x[b:b + 1, :Lb + 6], ww, bias, False)
        wav[b, :Lb] = out[0].astype(np.float32).view(np.uint32)
        peak[b] = np.abs(out[0].astype(np.float32)).max().view(np.uint32)
    return A.check_tail(name, c, bits, w, bias, wav, peak, Ls, 1, 0)


def test_tail_check_passes_the_reference_and_catches_reversed_taps():
    _tail(False)
    with pytest.raises(AssertionError):
        _tail(True)


def _cond(name, drop_odd=False, band=(5, 25)):
    c, mel, tgt, sums, out, Ts, T = A.cond_case(name, A.COND_CASES[name])
    c.oc.Tv = R.voc_frames(T, A.TAIL_BASE)
    w = A.mel_weight64()
    saved = R.BAND
    R.BAND = band
    try:
        for b, Tb in enumerate(Ts):
            s = R.band_sums(tgt[b:b + 1], mel[b:b + 1], [Tb]) if tgt is not None else None
            Tv = Tb + 4 if drop_odd else R.voc_frames(Tb, A.TAIL_BASE)
            want = R.voc_condition(mel[b:b + 1, :Tb], c.oc.is_log, w, Tv, sums=s)[0]
            out[:, b, :Tv] = A.split_bits(want)
            if s is not None:
                sums[b] = _bits32(s[0])
    finally:
        R.BAND = saved
    return A.check_cond(name, c, mel, tgt, sums, out, Ts, T)


def test_cond_check_passes_the_reference_and_catches_a_dropped_odd_frame():
    _cond("cond.log_T37_odd")
    with pytest.raises(AssertionError):
        _cond("cond.log_T37_odd", drop_odd=True)


def test_cond_check_catches_one_band_bin_too_many():
    _cond("cond.log_T37_unify")
    with pytest.raises(AssertionError):
        _cond("cond.log_T37_unify", band=(5, 26))


def test_istft_frame_bar_catches_a_kept_dc_imaginary_part():
    """The fused mode's DC and Nyquist bins carry the phase of a real signal's transform, whose imaginary part is zero, so
    there the mutation cannot show; the inverse it shares with the (real, imag) mode is pinned on a spectrum whose DC and
    Nyquist bins are complex, with the same per-frame bound (phi = 0: the spectrum is given)."""
    g = np.random.default_rng(8)
    Y = g.standard_normal((5, 1025)) + 1j * g.standard_normal((5, 1025))
    good, bad = R.inverse_frames(Y), R.inverse_frames(Y, keep_dc_imag=True)
    E = A.istft_frame_error(np.abs(Y), np.zeros(Y.shape))
    bound = R.hann()[None] * E[:, None] + A.gamma(3) * np.abs(good) + A.FLOOR
    assert (np.abs(bad - good) / bound).max() > 1


def test_peak_test_at_exactly_one_is_output_equivalent():
    """`>=` instead of `>` in the peak test divides a clip whose peak is exactly 1 by 1, which changes no bit: no bar can
    see it, and none needs to.  The GPU tests still run a peak of exactly 1 (finalize and the segmented normalise)."""
    wav = np.random.default_rng(9).uniform(-1, 1, 1000).astype(np.float32)
    wav[10] = 1.0
    ge = wav / np.float32(1.0)
    assert np.array_equal(R.finalize(wav, 1.0, 0, 1000).view(np.uint32), ge.view(np.uint32))
    assert np.array_equal(R.finalize(wav, 2.0, 0, 1000), wav / np.float32(2))
