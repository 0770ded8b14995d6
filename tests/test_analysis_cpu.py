"""The bi_gru and dnn analysis modules without a GPU: key lists against the reference's own state dicts, the float64
restatements against the reference goldens, the float64 GRU-layer reference against torch.nn.GRU (and its known-wrong
variants against the GPU test's bar), and the model's module selection."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import analysis as A
from oracle.make_golden import state_fingerprint
from voicefixer_main_b200.arch import UNET_PREFIX, bigru_keys, dnn_keys
from voicefixer_main_b200.weights import make_bigru_state, make_dnn_state, make_state

KINDS = {"bigru": ("bi_gru", bigru_keys, make_bigru_state), "dnn": ("dnn", dnn_keys, make_dnn_state)}
# the GPU test's bar for one GRU layer (tests/test_gpu_analysis.py)
GRU_TOL = 2e-5


@pytest.mark.parametrize("tag", sorted(KINDS))
def test_keys_match_reference_state_dict(tag):
    _, keys, _ = KINDS[tag]
    g = load_golden(f"stage_b_{tag}_t101.npz")
    ref = [(str(k), tuple(int(v) for v in s.split(",") if v)) for k, s in zip(g["sd_keys"], g["sd_shapes"])]
    assert ref == [(UNET_PREFIX + k, tuple(s)) for k, s in keys()]


@pytest.mark.parametrize("tag", sorted(KINDS))
def test_seeded_state_matches_golden_fingerprint(tag):
    _, _, make = KINDS[tag]
    assert np.allclose(state_fingerprint(make(1234)), load_golden(f"stage_b_{tag}_t101.npz")["fingerprint"], rtol=1e-12)


def test_gru_biases_are_non_zero():
    sd = make_bigru_state(1234)
    for k, v in sd.items():
        if ".gru.bias" in k:
            assert bool((v != 0).all()), k


@pytest.mark.parametrize("t", [101, 1001])
@pytest.mark.parametrize("tag", sorted(KINDS))
def test_float64_restatement_matches_reference(tag, t):
    kind, _, make = KINDS[tag]
    g = load_golden(f"stage_b_{tag}_t{t}.npz")
    mel = torch.from_numpy(g["mel_orig"]).double()
    assert bool((mel == 0).any())                     # to_log's clip is exercised
    with torch.no_grad():
        got = A.generator_forward(make(1234), mel, kind).numpy()
    want = g["log_mel"]
    # float64 goldens: 1e-9.  The T = 1001 ones are stored rounded to float32 (oracle/make_golden_analysis.py): half a
    # float32 ulp of each value, plus the same 1e-9
    tol = 1e-9 + (np.spacing(np.abs(want)) / 2 if want.dtype == np.float32 else 0.0)
    assert bool((np.abs(got - want.astype(np.float64)) <= tol).all()), float(np.abs(got - want).max())


def _gru_case(B, T, seed, layer=0):
    g = torch.Generator().manual_seed(seed)
    gru = torch.nn.GRU(256, 256, num_layers=2, bidirectional=True, batch_first=True).double()
    with torch.no_grad():
        for p in gru.parameters():
            p.copy_((torch.rand(p.shape, generator=g, dtype=torch.float64) * 2 - 1) / 16)
    x = torch.randn(B, T, 256 if layer == 0 else 512, generator=g, dtype=torch.float64)
    return gru, x


@pytest.mark.parametrize("lengths", [None, [40, 3, 39, 17]])
def test_gru_layer_reference_matches_torch_gru(lengths):
    B, T = 4, 40
    gru, x = _gru_case(B, T, seed=5)
    single = torch.nn.GRU(256, 256, bidirectional=True, batch_first=True).double()
    single.load_state_dict({k: v for k, v in gru.state_dict().items() if "_l0" in k})
    G, w, b = A.gru_input(x, gru, 0)
    got = A.gru_layer(G, w, b, lengths)
    with torch.no_grad():
        for i, n in enumerate(lengths or [T] * B):
            want = single(x[i:i + 1, :n])[0][0]
            assert float((got[i, :n] - want).abs().max()) < 1e-12
            assert bool((got[i, n:] == 0).all())


def test_gru_layer_reference_relu():
    gru, x = _gru_case(2, 12, seed=6)
    G, w, b = A.gru_input(x, gru, 0)
    assert torch.equal(A.gru_layer(G, w, b, relu=True), A.gru_layer(G, w, b).clamp(min=0))


@pytest.mark.parametrize("mutation", A.MUTATIONS)
def test_gru_mutations_break_the_gpu_bar(mutation):
    """Each known-wrong variant of the layer differs from the right one by far more than the GPU test allows, on the
    GPU test's own short-clip case (a clip one frame short of its bucket and a 3-frame clip)."""
    B, T, lengths = 3, 64, [63, 3, 64]
    gru, x = _gru_case(B, T, seed=7)
    G, w, b = A.gru_input(x, gru, 0)
    right = A.gru_layer(G, w, b, lengths, relu=True)
    wrong = A.gru_layer(G, w, b, lengths, relu=True, mutation=mutation)
    assert float((right - wrong).abs().max()) > 100 * GRU_TOL


def _sel(**on):
    from voicefixer_main_b200 import default_hparams
    hp = default_hparams()
    sel = hp["task"]["gsr"]["gsr_model"]["voicefixer"]
    for k in ("unet", "unet_small", "bi_gru", "dnn"):
        sel[k] = on.get(k, False)
    return hp


@pytest.mark.parametrize("on, want", [
    ({"unet": True, "unet_small": True, "bi_gru": True, "dnn": True}, "unet"),
    ({"unet_small": True, "bi_gru": True, "dnn": True}, "unet_small"),
    ({"bi_gru": True, "dnn": True}, "bi_gru"),
    ({"dnn": True}, "dnn"),
])
def test_selection_follows_reference_precedence(on, want):
    from voicefixer_main_b200 import VoiceFixer
    m = VoiceFixer(_sel(**on))
    assert m.analysis_module_name == want
    assert m._need() == ("unet" if want.startswith("unet") else want, "vocoder")


def test_nothing_selected_still_fails():
    from voicefixer_main_b200 import VoiceFixer
    with pytest.raises(NotImplementedError):
        VoiceFixer(_sel())


class _FakeLib:
    """Stands in for libb200vf so Engine.load_state's key checks run without a device."""

    def vf_load_weights(self, ctx, descs, n):
        self.names = [descs[i].name.decode() for i in range(n)]
        return 0


def _engine_stub():
    from voicefixer_main_b200.arch import VocoderConfig
    from voicefixer_main_b200.model import Engine
    eng = Engine.__new__(Engine)
    eng.lib, eng.ctx, eng.voc_cfg, eng.loaded = _FakeLib(), None, VocoderConfig(), False
    return eng


def test_unet_checkpoint_for_a_bigru_model_names_the_missing_gru_tensors():
    eng = _engine_stub()
    with pytest.raises(KeyError, match=r"'bi_gru' tensors.*2\.gru\.weight_ih_l0"):
        eng.load_state(make_state(1234), need=("bi_gru", "vocoder"))


@pytest.mark.parametrize("kind, make", [("bi_gru", make_bigru_state), ("dnn", make_dnn_state)])
def test_module_state_loads_with_its_keys(kind, make):
    from voicefixer_main_b200.weights import make_vocoder_state
    eng = _engine_stub()
    sd = make(1234)
    sd.update(make_vocoder_state(seed=1235))
    eng.load_state(sd, need=(kind, "vocoder"))
    sent = [k for k in eng.lib.names if k.startswith(UNET_PREFIX)]
    assert sent == [k for k in sd if k.startswith(UNET_PREFIX) and not k.endswith("num_batches_tracked")]


# ------------------------------------------------------------------------- the Linear layers' float64 references
def test_linear_bn_fold_and_merged_gru_bias_match_the_modules():
    """oracle/layers.py's float64 Linear, BatchNorm2d(1) fold and merged GRU input bias (the GPU layer suite's references
    of the analysis launches) restate the torch modules of oracle/analysis.py: dnn's BatchNorm2d(1) + Linear pairs, and the
    input projection of torch.nn.GRU's layers."""
    import torch.nn.functional as F
    from oracle import layers as R
    s = {k[len(UNET_PREFIX):]: v.double() for k, v in make_dnn_state(1234).items() if k.startswith(UNET_PREFIX)}
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 1, 7, 256, generator=g, dtype=torch.float64).relu()
    for bn, li in (("2", "3"), ("5", "6"), ("8", "9"), ("11", "12")):
        xi = x if s[li + ".weight"].shape[1] == 256 else torch.randn(2, 1, 7, s[li + ".weight"].shape[1], generator=g,
                                                                       dtype=torch.float64).relu()
        s[bn + ".running_mean"].fill_(0.3)           # a non-trivial affine: the seeded state's BatchNorm may be the identity
        s[bn + ".running_var"].fill_(1.7)
        s[bn + ".bias"].fill_(-0.45)
        want = F.linear(A._bn(xi, s, bn), s[li + ".weight"], s[li + ".bias"])
        params = [float(s[bn + k]) for k in (".weight", ".bias", ".running_mean", ".running_var")]
        w, b = R.bn_fold(s[li + ".weight"], s[li + ".bias"], params)
        got = R.linear(xi, w, b)
        assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())
        wrong = R.linear(xi, *R.bn_fold(s[li + ".weight"], s[li + ".bias"], params, shift_sum=False))
        assert float((wrong - want).abs().max()) > 1e-3
    gru = torch.nn.GRU(256, 256, bidirectional=True, batch_first=True).double()
    with torch.no_grad():
        for p in gru.parameters():
            p.copy_(torch.randn(p.shape, generator=g, dtype=torch.float64) / 8)
    xg = torch.randn(3, 9, 256, generator=g, dtype=torch.float64)
    G, _, _ = A.gru_input(xg, gru, 0)
    w_ih = torch.cat([gru.weight_ih_l0, gru.weight_ih_l0_reverse]).detach()
    b_ih = torch.cat([gru.bias_ih_l0, gru.bias_ih_l0_reverse]).detach()
    b_hh = torch.cat([gru.bias_hh_l0, gru.bias_hh_l0_reverse]).detach()
    assert float((R.linear(xg, w_ih, R.gru_ih_bias(b_ih, b_hh)) - G).abs().max()) <= 1e-12 * float(G.abs().max())
    # and the float64 GRU layer built on it is torch.nn.GRU's first layer
    y = gru(xg)[0].detach()
    h = A.gru_layer(G, torch.stack([gru.weight_hh_l0, gru.weight_hh_l0_reverse]).detach(),
                    torch.stack([gru.bias_hh_l0[512:], gru.bias_hh_l0_reverse[512:]]).detach())
    assert float((h - y).abs().max()) <= 1e-12


# ------------------------------------------------------------------------- the input planes (VF_OP_PLANES)
def test_fma32_is_the_exactly_rounded_fused_multiply_add():
    """R.fma32 against rational arithmetic: random operands, and sums constructed on float32 midpoints."""
    from fractions import Fraction
    from oracle import layers as R
    g = np.random.default_rng(9)
    x = (g.standard_normal(4000) * 3).astype(np.float32)
    s = (g.standard_normal(4000) * 2).astype(np.float32)
    t = (g.standard_normal(4000) * 4).astype(np.float32)
    # midpoints: x s = m + half an ulp32 of m exactly, t = 0 or a float32 that keeps the sum on a midpoint ~ 2^-30 apart
    s[:1000] = np.float32(1.0 + 2.0 ** -12)
    x[:1000] = (np.round(x[:1000].astype(np.float64) * 2 ** 11) / 2 ** 11 * (1 + 2.0 ** -12)).astype(np.float32)
    t[:500] = np.float32(2.0 ** -30)
    t[500:1000] = np.float32(-(2.0 ** -30))
    got = R.fma32(x, s, t)
    for i in range(len(x)):
        v = Fraction(float(x[i])) * Fraction(float(s[i])) + Fraction(float(t[i]))
        lo = np.float32(float(v))                       # within one float32 ulp of v; pick the nearest neighbour exactly
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        d = [abs(Fraction(float(c)) - v) for c in cands]
        best = min(d)
        ok = [c for c, e in zip(cands, d) if e == best]
        want = ok[0] if len(ok) == 1 else [c for c in ok if not (c.view(np.uint32) & 1)][0]
        assert got[i] == want, (i, x[i], s[i], t[i], got[i], want)
    assert not np.array_equal(got, (x * s).astype(np.float32) + t)


def test_separate_multiply_and_add_breaks_the_planes_bar():
    """The GPU test compares the planes bit for bit: rounding x * scale before adding shift changes bits of the cases with
    an affine that is not 1 / 0; and every pad row of the varlen cases is zero in the expected planes."""
    import test_gpu_aux as X
    from oracle import layers as R
    for name, spec in X.PLANES_CASES.items():
        x, scale, shift, Ts, off = X.planes_inputs(name)
        want = R.affine_planes(x, scale, shift, Ts if off is not None else None)
        if off is not None:
            for b, T in enumerate(Ts):
                assert not want[:, b, T:].any()
        if spec["scale"] != 1.0 and not spec.get("ties"):
            wrong = R.affine_planes(x, scale, shift, Ts if off is not None else None, fused=False)
            assert (wrong != want).sum() > 10, name
