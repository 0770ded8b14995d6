"""The float64 layer references of tests/test_gpu_layers.py, checked without a GPU: they restate the oracle's ops, their
layouts and write sets are consistent, and the bars the GPU tests apply are tight enough that a plausibly broken kernel
(a dropped or shifted tap, a wrong dilation, bias or prune column, dropped lo products, a doubled residual, one output
row taken from its neighbour) exceeds them."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_gpu_layers as G
from oracle import layers as R
from oracle import vf_oracle as O
from voicefixer_main_b200.arch import VocoderConfig, vocoder_keys


def test_vocoder_chain_of_layer_references_matches_the_oracle():
    """Cond net, stem, up-samplers, residual pairs and tail chained from oracle/layers.py equal vocoder_generator in
    float64 (a small configuration: few channels, two stages)."""
    cfg = VocoderConfig(cond_channels=32, cond_layers=2, channels=64, upsample_scales=[3, 2], resstack_depth=[3, 2],
                        tail_tanh=False)
    g = torch.Generator().manual_seed(3)
    sd = {"vocoder." + k: torch.randn(s, generator=g, dtype=torch.float64) / np.sqrt(np.prod(s[1:]) if len(s) > 1 else 4)
          for k, s in vocoder_keys(cfg)}
    c = torch.randn(2, 128, 19, generator=g, dtype=torch.float64)
    want = O.vocoder_generator(sd, c, cfg)
    w = lambda k: sd["vocoder." + k]
    x = c
    for i in range(cfg.cond_layers):
        x = R.activate(R.conv1d(x, w(f"condnet.{i}.weight"), w(f"condnet.{i}.bias")), 2, 0)
    hk = cfg.stem_kernel // 2
    x = R.lrelu(R.conv1d(F.pad(x, (hk, hk), mode="reflect"), w("stem.weight"), w("stem.bias"), centered=False), cfg.stage_slope)
    for s, (scale, depth) in enumerate(zip(cfg.upsample_scales, cfg.resstack_depth)):
        x = R.conv_transpose1d(x, w(f"up.{s}.weight"), w(f"up.{s}.bias"), scale)
        for i in range(depth):
            x, _ = R.pair(R.lrelu(x, cfg.res_slope), x, w(f"res.{s}.{i}.a.weight"), w(f"res.{s}.{i}.a.bias"),
                          w(f"res.{s}.{i}.b.weight"), w(f"res.{s}.{i}.b.bias"), cfg.dilation(i), cfg.res_slope)
        x = R.lrelu(x, cfg.stage_slope)
    got = R.conv1d(F.pad(x, (hk, hk), mode="reflect"), w("tail.weight"), w("tail.bias"), centered=False)
    assert got.shape == want.shape
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())


@pytest.mark.parametrize("both", [0, 1])
def test_convt2d_prune_matches_the_oracle_decoder(both):
    """vf_oracle.py:187-188 (time-only prune) and :218-219 (both=True)."""
    g = torch.Generator().manual_seed(both)
    x = torch.randn(2, 8, 5, 7, generator=g, dtype=torch.float64)
    w = torch.randn(8, 4, 3, 3, generator=g, dtype=torch.float64)
    y = F.conv_transpose2d(x, w, stride=2)
    want = y[:, :, 0:-1, 0:-1] if both else y[:, :, 0:-1, :]
    assert torch.equal(R.conv_transpose2d(x, w, both), want)


def test_layouts_round_trip():
    x = torch.randn(2, 5, 3, 7, dtype=torch.float64)
    r = R.nchw_to_rows(x)
    assert r.shape == (2, 3 * 8, 5)
    assert (r.reshape(2, 3, 8, 5)[:, :, 7] == 0).all()                  # the pad column
    assert torch.equal(R.rows_to_nchw(r, 3, 7), x)
    cat = torch.cat([torch.zeros_like(r), r], dim=2)                      # concat placement at c_off = C
    assert torch.equal(R.rows_to_nchw(cat, 3, 7, c_off=5, c=5), x)
    y = torch.randn(2, 4, 9, dtype=torch.float64)
    assert torch.equal(R.rows_to_ncl(R.ncl_to_rows(y)), y)
    v = torch.randn(1000, dtype=torch.float64) * 100
    hi, lo = R.split_hi_lo(v.float())
    assert float((hi + lo - v.float().double()).abs().max()) <= 2.0 ** -21 * float(v.abs().max())


@pytest.mark.parametrize("H,W,both", [(3, 4, 0), (3, 4, 1), (1, 1, 1), (2, 16, 1)])
def test_convt2d_write_set_covers_every_output_row_once(H, W, both):
    Wp = W + 1
    ow = 2 * Wp - 1 if both else 2 * Wp
    m = R.write_rows_convt2d(1, 2 * H * ow + 3, 1, H, Wp, ow, 0, 1)[0, :, 0]
    assert m[:2 * H * ow].all() and not m[2 * H * ow:].any()
    hits = np.zeros(2 * H * ow + 3, int)
    for ph in range(2):
        for pw in range(2):
            for h in range(H):
                for w in range(Wp):
                    if 2 * w + pw < ow:
                        hits[(2 * h + ph) * ow + 2 * w + pw] += 1
    assert (hits[:2 * H * ow] == 1).all()
    # the layout of the reference output: 2H rows of ow - 1 bins and the pad column
    y = R.conv_transpose2d(torch.zeros(1, 1, H, W, dtype=torch.float64), torch.zeros(1, 1, 3, 3, dtype=torch.float64), both)
    assert y.shape[2:] == (2 * H, ow - 1)


@pytest.mark.parametrize("L,s", [(42, 7), (5, 3), (1, 2)])
def test_convt1d_write_set_is_the_reference_length(L, s):
    m = R.write_rows_convt1d(1, L * s + 4, 1, 2, L + 1, s, L * s, 0, 1)[0, :, 0]
    assert m[2:2 + L * s].all() and m.sum() == L * s
    y = R.conv_transpose1d(torch.zeros(1, 1, L, dtype=torch.float64), torch.zeros(1, 1, 2 * s, dtype=torch.float64), None, s)
    assert y.shape[2] == L * s


# ------------------------------------------------------------------ the bars can fail
def _bar_ratio(b, y_mut):
    """max |y_mut - y64| / bound over the layer's outputs, with the bound the GPU test applies to its first output
    (rows the layer zeroes excluded)."""
    y, M = G.reference(b).numpy(), G.reference(b, abs_=True).numpy()
    keep = ~G.zero_rows_mask(b)[..., None]
    tol = G.TOL[b.terms]
    first = G.BY_NAME[b.c["name"]].get("outs", "a").split(",")[0]
    rel = {"raw": 0.0, "r": 2.0 ** -21}.get(first, 2.0 ** -21 if b.terms == 3 else 2.0 ** -11)
    bound = tol * M + rel * np.abs(y) + G.FLOOR
    return float((np.abs(np.asarray(y_mut) - y) / bound * keep).max())


def _mutated(case, **kw):
    """The reference of a built case with some of its operands (or its spec `c`) replaced."""
    saved = {k: getattr(case, k) for k in kw}
    for k, v in kw.items():
        setattr(case, k, v)
    try:
        return G.reference(case).numpy()
    finally:
        for k, v in saved.items():
            setattr(case, k, v)


def _case(name):
    return G.build(G.BY_NAME[name])


def test_bar_catches_a_dropped_tap():
    b = _case("conv1.mel_l0")
    w = b.w.clone()
    w[:, :, 1, 2] = 0
    assert _bar_ratio(b, _mutated(b, w=w)) > 1


def test_bar_catches_a_tap_shifted_by_one_row():
    b = _case("gemm.2x300_32to32_k9_d1_t1")
    w = torch.zeros(b.w.shape[0], b.w.shape[1], 11, dtype=torch.float64)
    w[:, :, 1:10] = b.w
    w[:, :, 0], w[:, :, 1] = w[:, :, 1].clone(), 0                     # tap 0 reads one row further up
    assert _bar_ratio(b, _mutated(b, w=w)) > 1


def test_bar_catches_a_dilation_off_by_one():
    b = _case("res_a.d27_c128")
    assert _bar_ratio(b, _mutated(b, c=dict(b.c, dilation=28))) > 1


def test_bar_catches_the_neighbouring_channels_bias():
    b = _case("cond.tv42_t1")
    assert _bar_ratio(b, _mutated(b, b=torch.roll(b.b, 1))) > 1


def test_bar_catches_the_wrong_prune_column():
    b = _case("convt2d.v2_both")
    x = R.rows_to_nchw(b.x, b.c["H"], b.c["W"])
    y = F.conv_transpose2d(x, b.w, stride=2)[:, :, :-1, 1:]              # drops the first column instead of the last
    assert _bar_ratio(b, R.nchw_to_rows(y).numpy()) > 1


def test_bar_catches_dropped_lo_products_in_3_term_mode():
    b = _case("conv2_res.c384")
    x_hi = R.fp16(b.x)
    w_hi = R.fp16(b.w)
    assert _bar_ratio(b, _mutated(b, x=x_hi, w=w_hi)) > 1


def test_bar_catches_the_residual_added_twice():
    b = _case("res_b.planes_c256")
    assert _bar_ratio(b, _mutated(b, resid=2 * b.resid)) > 1


def test_bar_catches_one_row_of_one_image_replaced_by_its_neighbours():
    b = _case("gemm.2x200_64to32_k3_d1_t3")
    y = G.reference(b).numpy().copy()
    y[1, 150] = y[1, 151]
    assert _bar_ratio(b, y) > 1


# ------------------------------------------------------------------ the analysis modules' Linear layers
def _act_ratio(b, y_mut):
    """max |act(y_mut) - act(y64)| / bound with the bound the GPU test applies to the case's 3-term outputs (out_a after
    its affine and activation, or the raw fp32 output), rows the layer zeroes excluded."""
    c = b.c
    y, M = G.reference(b).numpy(), G.reference(b, abs_=True).numpy()
    keep = ~G.zero_rows_mask(b)[..., None]
    tol = G.TOL[b.terms]
    if c["outs"] == "raw":
        want, got, bound = y, np.asarray(y_mut), tol * M + G.FLOOR
    else:
        sc = np.abs(b.scale) if c.get("affine") else 1.0
        f = lambda v: R.activate(torch.as_tensor(v * b.scale + b.shift if c.get("affine") else v), c["act"],
                                 c.get("slope", 0.0)).numpy()
        want, got = f(y), f(np.asarray(y_mut))
        bound = sc * tol * M + 2.0 ** -21 * np.abs(want) + G.FLOOR
    return float((np.abs(got - want) / bound * keep).max())


def test_linear_cases_pass_their_own_reference():
    for c in G.CASES:
        if c["kind"] == G.LINEAR:
            b = _case(c["name"])
            assert _act_ratio(b, G.reference(b).numpy()) == 0.0


def test_bar_catches_the_bn_fold_without_the_weight_sums():
    for name in ("dnn.lin1_bn", "dnn.lin3_bn_k1024", "dnn.lin3_bn_k1024.varlen"):
        b = _case(name)
        _, bias = R.bn_fold(b.w_raw, b.b_raw, b.bn, shift_sum=False)
        assert _act_ratio(b, _mutated(b, b=bias)) > 1, name


def test_bar_catches_b_hn_merged_into_the_gru_input_projection():
    for name in ("bigru.gru0.ih", "bigru.gru1.ih", "bigru.gru0.ih.varlen"):
        b = _case(name)
        assert _act_ratio(b, _mutated(b, b=R.gru_ih_bias(b.b_raw, b.b_hh, merge_n=True))) > 1, name


def test_bar_catches_the_log_mel_residual_on_the_first_n_tile_only():
    """linear_out's N = 128 is two 64-column tiles in 3-term mode; the residual left off the second one."""
    for name in ("bigru.lin6", "dnn.lin5", "bigru.lin6.varlen", "dnn.lin5.T3"):
        b = _case(name)
        resid = b.resid.clone()
        resid[..., 64:] = 0
        assert _act_ratio(b, _mutated(b, resid=resid)) > 1, name


def test_pad_rows_of_a_3_frame_clip_are_nonzero_unless_written_as_zeros():
    """The GPU test demands exact zeros at rows t >= 3 of the 3-frame clips: the GEMM's value there (the bias, with the
    residual and the activation) is not zero, so a pad row left as computed fails it."""
    for name in ("bigru.lin1.varlen", "bigru.gru0.ih.varlen", "bigru.lin4.varlen", "bigru.lin6.varlen", "dnn.lin3_bn_k1024.varlen"):
        b = _case(name)
        img = list(b.rv).index(3)
        y = G.reference(b).numpy()[img, 3:]
        c = b.c
        if c["outs"] == "a":
            v = y * b.scale + b.shift if c.get("affine") else y
            y = R.activate(torch.as_tensor(v), c["act"], c.get("slope", 0.0)).numpy()
        assert G.zero_rows_mask(b)[img, 3:].all() and (y != 0).any(axis=-1).all(), name
