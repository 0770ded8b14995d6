"""The fp16 range guard (DESIGN.md §3) at every launch that splits values into fp16 planes.

The restore calls never synchronise, so the sticky device flag behind `vf_check_errors` -> VF_EDEVICE is the only way a
caller learns that a plane overflowed.  On the self-test hooks of test_gpu_layers.py / test_gpu_aux.py, with operand bits
chosen so that chosen output elements take chosen values, this file checks for every GEMM configuration signature the
plans build, for the fused pair and for the split-writing non-GEMM ops:
  (a) each fp16 plane a launch writes, overflowed on its own, raises VF_EDEVICE: the raw r planes with the activated value
      in range (LeakyReLU slope 0.01), the activated planes with r in range (BN scale > 1), the (a, r) stream's |v|, the
      3-term hi + lo, the pair's output and its shared-memory intermediate h;
  (b) a NaN or an infinity in an operand or a residual word raises VF_EDEVICE;
  (c) the boundary: |v| = 65504 is VF_OK and stored exactly, 65504 < |v| < 65520 (fp16 rounds it to 65504) is VF_EDEVICE;
  (d) NaN and out-of-range values where the layer writes zeros or stores nothing leave the flag clear, and the outputs are
      those of the clean case bit for bit (which test_gpu_layers.py checks against float64) - here also checked against
      float64: the pad column, rows at or past row_valid (also whole empty tiles), rows past rows_in in the last tile in
      both halves of a warp's 16-row fragment band, the pair's halo rows and rows past its clip;
  (e) after every flagged case the clean case on the same context gives the bits of its first run;
  (f) every plan signature and every split-writing op kind has an (a) and a (d) case."""
import ctypes

import numpy as np
import pytest
import torch

import test_gpu_aux as A
import test_gpu_layers as G
from oracle import layers as R
from voicefixer_main_b200 import _lib as VL

pytestmark = pytest.mark.gpu

CONV2D, CONVT2D, CONV1D, CONVT1D, PAIR, LINEAR = G.CONV2D, G.CONVT2D, G.CONV1D, G.CONVT1D, G.PAIR, G.LINEAR
NAN16, PINF16, NINF16, MAX16 = 0x7E00, 0x7C00, 0xFC00, 0x7BFF
COVER = {}            # signature or op kind -> set of parts ("a", "b", "c", "d") with a passing case
SIGS = {}             # case name -> configuration signature
CLEAN = {}            # case name -> output bits of its first clean run


def fp16_bits(v):
    return np.float16(v).view(np.uint16)


def flag(eng):
    """VF_OK, or the code check_errors raised (and cleared)."""
    try:
        eng.check_errors()
    except VL.EngineError as e:
        return e.code
    return VL.VF_OK


def held(b, field, lc=None):
    """The host array of b.keep (or b.buf) the case's pointer `field` points at."""
    p = getattr(lc or b.lc, field)
    for a in list(b.keep) + list(getattr(b, "buf", {}).values()):
        if isinstance(a, np.ndarray) and a.ctypes.data == p:
            return a
    raise KeyError(field)


def outputs(b):
    out = {k: v.copy() for k, v in b.buf.items()}
    if b.c.get("head"):
        out["head"] = b.head_out.copy()
    return out


def fp16_outs(c):
    if c["kind"] == PAIR:
        return {"a"}
    if c.get("head"):
        return set()
    return {"r", "a"} & set(c.get("outs", "a").split(","))


def record(key, part):
    COVER.setdefault(key, set()).add(part)


# ------------------------------------------------------------------ the clean case, and (e)
def run_clean(eng, name):
    """Runs case `name` as test_gpu_layers builds it; the first run records its signature and output bits, later runs must
    reproduce them (the flag of a preceding case has been cleared)."""
    b = G.build(G.BY_NAME[name])
    eng.selftest_layer(b.lc)
    assert flag(eng) == VL.VF_OK, (name, "the clean case raised the flag")
    out = outputs(b)
    if name not in CLEAN:
        CLEAN[name] = out
        SIGS[name] = b.lc.sig.decode()
    else:
        for k, v in out.items():
            bad = np.argwhere(v != CLEAN[name][k])
            assert not len(bad), (name, k, f"{len(bad)} elements differ from the first clean run, first {bad[:4].tolist()}")
    return b


def expect_flag(eng, name, b, want, what):
    eng.selftest_layer(b.lc)
    got = flag(eng)
    assert got == want, (name, what, f"check_errors -> {got}, want {want}")
    if want != VL.VF_OK:
        run_clean(eng, name)         # (e)


# ------------------------------------------------------------------ operand geometry
def valid_img_row(b):
    """(image, input row, output row) of a valid element away from every edge: the image with the most valid rows."""
    c, kind = b.c, b.c["kind"]
    img = 0 if b.rv is None else int(np.argmax(b.rv))
    if kind in (CONV2D, CONVT2D):
        H, W = c["H"], c["W"]
        Wp = W + 1
        h = (H if b.rv is None else min(H, int(b.rv[img]) // Wp)) // 2
        r = h * Wp + W // 2
        return img, r, r
    if kind == CONVT1D:
        lim = c["L"] if b.rv is None else min(c["L"], -(-int(b.rv[img]) // c["stride"]))
        return img, lim // 2, (lim // 2) * c["stride"]
    lim = c["L"] if b.rv is None else min(c["L"], int(b.rv[img]))
    return img, lim // 2, lim // 2


def out_channel(b, min_scale=0.0):
    """An output channel whose BN scale (if the layer has one) is positive and above min_scale."""
    if getattr(b, "scale", None) is None or not b.c.get("affine"):
        return 0
    ok = np.flatnonzero(b.scale > min_scale)
    assert len(ok), (b.c["name"], "no BN scale above", min_scale)
    return int(ok[0])


def w_column(b, w, co, ci):
    """The view of weight array w (the layer's host layout) that multiplies input channel ci into output channel co."""
    kind = b.c["kind"]
    if kind in (CONVT2D, CONVT1D):
        return w[ci, co]
    if kind == LINEAR:
        return w[co, ci:ci + 1]
    return w[co, ci]


def inject_product(b, X, Wv, co, ci=0, img=None, row=None, taps=None, alone=False):
    """x[img, row, ci] = X (fp16, lo plane 0) and the weights of (co, ci) = Wv: every output element of channel co that reads
    that x element gets X * Wv plus the layer's ordinary terms.  With `taps` (flat indices into the kernel of (co, ci)),
    only those kernel entries are Wv and the others 0, so only the outputs those taps map the element to read it; with
    `alone`, input channel ci is zero everywhere else.  The float64 operands of the case (b.x, b.w) follow."""
    if img is None:
        img, row, _ = valid_img_row(b)
    xb = held(b, "x")
    if alone:
        xb[..., ci] = 0
        if hasattr(b, "x"):
            b.x[..., ci] = 0
    xb[0, img, row, ci], xb[1, img, row, ci] = fp16_bits(X), 0
    w = held(b, "w")
    col = w_column(b, w, co, ci)
    if taps is None:
        col[...] = Wv
    else:
        col[...] = 0
        col.reshape(-1)[list(taps)] = Wv
    if hasattr(b, "x"):
        b.x[img, row, ci] = X
    if torch.is_tensor(getattr(b, "w", None)) and b.c["kind"] != LINEAR:
        w_column(b, b.w, co, ci).copy_(torch.from_numpy(np.ascontiguousarray(col, np.float64)))


def x_word(b, img, row, ci, bits, plane=0):
    xb = held(b, "x")
    xb[plane, img, row, ci] = bits
    if plane == 0:
        xb[1, img, row, ci] = 0


# ------------------------------------------------------------------ (a), (b)
# a hi-only (a, r) residual layer whose CTAs run an empty tile (image 0 past its 1000 rows) before a live one (image 1): the
# fragment epilogue's residual barrier parity advances on live tiles only
EXTRA = [G.C("res_b.ar_c128_varlen_empty_then_live", CONV1D, terms=1, n_img=2, L=40000, cin=128, cout=128, k=3, resid="ar",
             outs="a", out_ar=True, row_valid=[1000, 40000])]
for _c in EXTRA:
    G.BY_NAME.setdefault(_c["name"], _c)

# every layer case that writes an fp16 plane (the windowed decode case aside: its reference covers two windows only); their
# signatures are those of every fp16-writing launch the plans build (test_gpu_layers.py::test_cases_cover_every_kernel_configuration)
NAMES = [c["name"] for c in G.CASES + EXTRA if fp16_outs(c) and not c.get("windows")]


@pytest.fixture(scope="module")
def eng():
    from voicefixer_main_b200.model import Engine
    e = Engine("cuda:0")
    yield e
    e.check_errors()
    e.close()


def overflow_variants(c):
    """(what, X, Wv, min BN scale): operand products that put one plane of the case out of range on its own."""
    outs = fp16_outs(c)
    v = []
    if "r" in outs:        # v ~ -2.6e5: r = fp16(v) = -inf; lrelu_0.01(s v) <= 5.3e3 (s <= 2)
        v.append(("r alone", 64.0, -4096.0, 0.0))
    if "a" in outs and "r" in outs and c.get("affine"):       # v ~ 6.1e4 in range, s v > 6.7e4 (s > 1.1)
        v.append(("a alone", 16.0, 3840.0, 1.1))
    elif "a" in outs:      # v ~ 2.6e5 (the (a, r) stream: |v|; 3-term: hi + lo)
        v.append(("ar |v|" if c.get("out_ar") else "a" + (" (hi + lo)" if c.get("terms", 1) == 3 else ""), 64.0, 4096.0, 0.0))
    return v


@pytest.mark.parametrize("name", [n for n in NAMES if G.BY_NAME[n]["kind"] != PAIR])
def test_each_plane_out_of_range_alone_raises_the_flag(eng, name):
    """(a) + (e)"""
    run_clean(eng, name)
    for what, X, Wv, smin in overflow_variants(G.BY_NAME[name]):
        b = G.build(G.BY_NAME[name])
        inject_product(b, X, Wv, out_channel(b, smin))
        expect_flag(eng, name, b, VL.VF_EDEVICE, what)
    record(SIGS[name], "a")


@pytest.mark.parametrize("name", NAMES)
def test_nan_and_inf_operands_raise_the_flag(eng, name):
    """(b) + (e): fp16 NaN / +Inf / -Inf in one element of x, and a NaN residual word, at a valid row."""
    c = G.BY_NAME[name]
    run_clean(eng, name)
    for bits, what in ((NAN16, "x NaN"), (PINF16, "x +Inf"), (NINF16, "x -Inf")):
        b = G.build(c)
        img, row, _ = valid_img_row(b) if c["kind"] != PAIR else (0, min(c["L"], *(c.get("row_valid") or [c["L"]])) // 2, 0)
        x_word(b, img, row, 0, bits)
        expect_flag(eng, name, b, VL.VF_EDEVICE, what)
    if c["kind"] == PAIR:          # the correction plane r of the (a, r) input: read only by E2, as the residual
        b = G.build(c)
        held(b, "x")[1, 0, min(c["L"], *(c.get("row_valid") or [c["L"]])) // 2, 5] = NAN16
        expect_flag(eng, name, b, VL.VF_EDEVICE, "x.r NaN")
    if c.get("resid"):
        b = G.build(c)
        img, _, orow = valid_img_row(b)
        rarr = held(b, "resid")
        if c["resid"] == "fp32":
            rarr[img, orow, 3] = np.float32("nan")
        else:
            rarr[0, img, orow, 3] = NAN16
        expect_flag(eng, name, b, VL.VF_EDEVICE, "residual NaN")
    record(SIGS[name], "b")


# ------------------------------------------------------------------ (c) the boundary
BOUNDARY = ["res_a.d243_c64", "res_b.planes_c128", "res_b.ar_c256", "up.s3_r_stg", "up.s7_ar_tma", "cond.tv42_t3",
            "res_b.planes_c64_t3", "up.s3_t3", "dnn.lin0"]


def bias_only_channel(b, co, value):
    """Output channel co = bias exactly: its weights (and residual column) zero, its bias `value`."""
    w = held(b, "w")
    if b.c["kind"] == CONVT1D:
        w[:, co] = 0
    else:
        w[co] = 0
    held(b, "b")[co] = value
    if b.c.get("resid"):
        rarr = held(b, "resid")
        rarr[..., co] = 0


@pytest.mark.parametrize("name", BOUNDARY)
def test_the_boundary_is_65504(eng, name):
    """(c): v = 65504 exactly in every valid row of one channel is VF_OK and stored as 65504 (lo 0) in each fp16 plane; v =
    65510, which fp16 rounds to the finite 65504, raises the flag."""
    c = G.BY_NAME[name]
    run_clean(eng, name)
    b = G.build(c)
    bias_only_channel(b, 7, 65504.0)
    eng.selftest_layer(b.lc)
    assert flag(eng) == VL.VF_OK, (name, "65504 raised the flag")
    zr = G.zero_rows_mask(b)
    rows = slice(b.out_row0, b.out_row0 + zr.shape[1])
    for key in fp16_outs(c):
        buf = b.buf[key]
        live = G.write_mask(b, buf.shape[-1], b.c_off, c["cout"])[:, rows, b.c_off + 7] & ~zr
        assert live.sum() > 0
        hi, lo = buf[0][:, rows, b.c_off + 7][live], buf[1][:, rows, b.c_off + 7][live]
        assert (hi == MAX16).all(), (name, key, "hi plane is not 65504", np.unique(hi)[:4])
        if key == "r" or c.get("terms", 1) == 3 or c.get("out_ar"):         # 0 or -0: the split writes -(hi - v)
            assert (lo.view(np.float16) == 0).all(), (name, key, "lo plane is not 0", np.unique(lo)[:4])
    b = G.build(c)
    bias_only_channel(b, 7, 65510.0)
    expect_flag(eng, name, b, VL.VF_EDEVICE, "65510")
    record(SIGS[name], "c")


# ------------------------------------------------------------------ (d) must-zero places
def reach(b):
    """(before, after): output rows m read input rows m - before .. m + after (GEMM rows for the transposed convs)."""
    c, kind = b.c, b.c["kind"]
    if kind == CONV2D:
        return c["W"] + 2, c["W"] + 2
    if kind == CONVT2D:
        return 0, c["W"] + 2
    if kind == CONV1D:
        span = (c["k"] - 1) * c.get("dilation", 1)
        return (span // 2, span // 2) if c.get("centered", 1) else (0, span)
    if kind == CONVT1D:
        return 1, 1
    return 0, 0


def product_targets(c):
    """[(what, img, input row, taps, alone)]: paths (inject_product) from a valid input element to output elements the layer
    must zero or not store, and to no other output of that channel:
      CONV2D   the pad column of an image row: output (h, W) reads the valid pixel (h, W - 1) through tap (1, 0) alone;
      CONVT2D  (both=True) the pad column 2 W: pixel (h, W - 1) reaches it through the kernel column kw = 2 alone;
      CONVT1D  the outputs t = -pad (kernel entry 0 of input row 0) and t = L s + s - 1 - pad (entry 2 s - 1 of row L - 1),
               never stored;
      CONV1D   rows past rows_in that the last tile computes, one in each half (hh) of a warp's 16-row fragment band where
               the taps reach both, through the tap of the most negative offset."""
    kind = c["kind"]
    n = c.get("n_img", 1)
    if kind == CONV2D:
        H, W = c["H"], c["W"]
        Wp = W + 1
        return [(f"pad column of image row {h}", n - 1, h * Wp + W - 1, [3], False) for h in sorted({0, H - 1})
                if c.get("row_valid") is None or (h + 1) * Wp <= min(c["row_valid"])]
    if c.get("row_valid") is not None:
        return []
    if kind == CONVT2D:          # output column 2 w + kw reads input column w through the kernel column kw
        if not c["both"]:
            return []            # the pad column 2 W + 1 reads only the input's pad column: nothing reaches it
        H, W = c["H"], c["W"]
        return [(f"pad column 2 W of output rows 2 h .. 2 h + 2, h = {h}", n - 1, h * (W + 1) + W - 1, [2, 5, 8], True)
                for h in sorted({0, H - 1})]
    if kind == CONVT1D:
        s_ = c["stride"]
        return [("output t = -pad", n - 1, 0, [0], True), ("output past L s", n - 1, c["L"] - 1, [2 * s_ - 1], True)]
    if kind != CONV1D:
        return []
    L, k, d = c["L"], c["k"], c.get("dilation", 1)
    centered = c.get("centered", 1)
    if centered and k % 2 == 0:
        return []
    offs = [(t - (k - 1) // 2) * d if centered else t * d for t in range(k)]
    t0 = int(np.argmin(offs))
    top = -(-L // 128) * 128
    got = {}
    for m in range(max(L, -offs[t0]), min(top, L + c.get("x_extra", 0) - offs[t0])):
        got.setdefault(m % 16 >= 8, m)
    return [(f"row {m} past rows_in = {L} (fragment half {int(m % 16 >= 8)})", n - 1, m + offs[t0], [t0], False)
            for m in sorted(got.values())]


def zero_rows_of(b):
    """[(img, row)] of rows the layer writes as zeros: per image the first, the 64th and the last such row (pad column and
    rows at or past row_valid)."""
    zr = G.zero_rows_mask(b)
    out = []
    for i in range(b.n):
        rows = np.flatnonzero(zr[i])
        if len(rows):
            out += [(i, int(r)) for r in sorted({rows[0], rows[min(63, len(rows) - 1)], rows[-1]})]
    return out


def check_like_clean(eng, name, b, what):
    """Flag clear, and every output the clean run's bit for bit."""
    assert flag(eng) == VL.VF_OK, (name, what, "raised the flag")
    for k, v in outputs(b).items():
        bad = np.argwhere(v != CLEAN[name][k])
        assert not len(bad), (name, what, k, f"{len(bad)} elements differ from the clean run, first {bad[:4].tolist()}")


def check_float64(name, b, what):
    G.check_outputs(b, G.Checker(f"{name} {what}"), G.reference(b), G.reference(b, abs_=True))


@pytest.mark.parametrize("name", [n for n in NAMES if G.BY_NAME[n]["kind"] != PAIR])
def test_must_zero_places_leave_the_flag_clear(eng, name):
    """(d): NaN and out-of-range residual words in rows the layer writes as zeros (pad column, rows at or past row_valid;
    the first, a middle and the last channel); NaN x rows that only such rows read (varlen); 2.6e5 through chosen taps into
    outputs that are zeroed or not stored (product_targets).  Each leaves the flag clear and the outputs right."""
    c = G.BY_NAME[name]
    run_clean(eng, name)
    b0 = G.build(c)
    cases = 0
    if c.get("resid") and c["kind"] in (CONV2D, CONV1D) and zero_rows_of(b0):
        cout = c["cout"]
        for word in ("NaN", "out of range"):
            b = G.build(c)
            rarr = held(b, "resid")
            for (i, r) in zero_rows_of(b):
                for co in (0, cout // 2 + 1, cout - 1):
                    nan = word == "NaN"
                    if c["resid"] == "fp32":
                        rarr[i, r, co] = np.float32("nan") if nan else np.float32(1e30)
                    elif c["resid"] == "ar":
                        rarr[0, i, r, co] = NAN16 if nan else 0xFBFF          # a = -65504: U(a) = -6.5e6
                    else:
                        rarr[0, i, r, co], rarr[1, i, r, co] = (NAN16, 0) if nan else (MAX16, MAX16)
            eng.selftest_layer(b.lc)
            check_like_clean(eng, name, b, f"residual {word} in zero rows")
            cases += 1
    if b0.rv is not None:
        _, after = reach(b0)
        b = G.build(c)
        xb = held(b, "x")
        rows_x = xb.shape[2]
        for i in range(b.n):
            rv = int(b.rv[i])
            first = rv + after if c["kind"] != CONVT1D else -(-rv // c["stride"]) + 2
            for r in sorted({first, rows_x - 1}):
                if first <= r < rows_x:
                    for ci in (0, xb.shape[3] - 1):
                        xb[0, i, r, ci], xb[1, i, r, ci] = NAN16, 0
                    cases += 1
        if cases:
            eng.selftest_layer(b.lc)
            check_like_clean(eng, name, b, "NaN x rows read only by zero rows")
    if c["kind"] == LINEAR and b0.rv is None and not c.get("in_bn") and c["L"] % 128:
        # rows past rows_in read only the zero fill, so they hold the bias alone: bias 2^18 on channel 5, cancelled exactly in
        # every valid row by x[:, 0] = 64 times w[5, 0] = -4096 (channel 5's other weights 0)
        b = G.build(c)
        xb, w = held(b, "x"), held(b, "w")
        xb[0, ..., 0], xb[1, ..., 0] = fp16_bits(64.0), 0
        w[5], w[5, 0] = 0, -4096.0
        held(b, "b")[5] = 262144.0
        b.x[..., 0] = 64.0
        b.w[5], b.w[5, 0], b.b[5] = 0, -4096.0, 262144.0
        eng.selftest_layer(b.lc)
        assert flag(eng) == VL.VF_OK, (name, "2.6e5 in the rows past rows_in raised the flag")
        check_float64(name, b, "2.6e5 in the rows past rows_in")
        cases += 1
    for what, img, r_x, taps, alone in product_targets(c):
        b = G.build(c)
        inject_product(b, 64.0, 4096.0, 5, img=img, row=r_x, taps=taps, alone=alone)
        eng.selftest_layer(b.lc)
        assert flag(eng) == VL.VF_OK, (name, f"2.6e5 in the {what} raised the flag")
        check_float64(name, b, f"2.6e5 in the {what}")
        cases += 1
    if cases:
        record(SIGS[name], "d")


# ------------------------------------------------------------------ the fused pair: (a), (c), (d)
PAIR_NAMES = [n for n in NAMES if G.BY_NAME[n]["kind"] == PAIR]


def pair_single_path(b, row, from_top):
    """Channel 9 of h is 240 x_a[row, 0] and nothing else; output channel 5 reads it through one conv_b tap: the row above
    it (from_top) or below it.  x_a[:, 0] is zero in every clip except at `row` of the last one, where it is 240 (an fp16
    value, r = 0)."""
    xb = held(b, "x")
    img = b.n - 1
    xb[:, :, :, 0] = 0
    xb[0, img, row, 0], xb[1, img, row, 0] = fp16_bits(240.0), 0
    wa, ba, wb = held(b, "w"), held(b, "b"), held(b, "w2")
    wa[9] = 0
    wa[9, 0, 1] = 240.0
    ba[9] = 0
    wb[5, 9] = 0
    wb[5, 9, 2 if from_top else 0] = 4096.0       # y[m] reads h[m + 1] (tap 2) or h[m - 1] (tap 0)
    a, r = xb[0].view(np.float16), xb[1].view(np.float16)
    b.x_stream = torch.from_numpy(R.ar_decode(a, r, G.RES_SLOPE))
    b.x_act = torch.from_numpy(a.astype(np.float64))
    b.wa[9], b.ba[9] = 0, 0
    b.wa[9, 0, 1] = 240.0
    b.wb[5, 9] = 0
    b.wb[5, 9, 2 if from_top else 0] = 4096.0


@pytest.mark.parametrize("name", PAIR_NAMES)
def test_pair_planes_boundary_and_halo(eng, name):
    c = G.BY_NAME[name]
    run_clean(eng, name)
    L = c["L"]
    Lv = L if c.get("row_valid") is None else c["row_valid"][-1]
    # (a) the intermediate h alone: channel 9 of h = 65510 in every row (fp16: 65504), and conv_b does not read it
    b = G.build(c)
    held(b, "w")[9] = 0
    held(b, "b")[9] = 65510.0
    held(b, "w2")[:, 9] = 0
    expect_flag(eng, name, b, VL.VF_EDEVICE, "h alone")
    # (c) h = 65504 exactly is in range
    b = G.build(c)
    held(b, "w")[9] = 0
    held(b, "b")[9] = 65504.0
    held(b, "w2")[:, 9] = 0
    eng.selftest_layer(b.lc)
    assert flag(eng) == VL.VF_OK, (name, "h = 65504 raised the flag")
    # (a) the output alone: x = U(a) = -3e6 in one element (conv_a reads a = -30000: |h| stays below 2e4)
    b = G.build(c)
    xb = held(b, "x")
    xb[0, 0, min(L, Lv) // 2, 3], xb[1, 0, min(L, Lv) // 2, 3] = fp16_bits(-30000.0), 0
    expect_flag(eng, name, b, VL.VF_EDEVICE, "output alone")
    record(SIGS[name], "a")
    record(SIGS[name], "c")
    # (d) 2.4e8 in the halo row above the clip (accumulator row 0 of the first tile) and in the row just past the clip (a row
    # of the last tile, or its bottom halo row when the clip ends on a tile boundary): h is in range, and only that row of the
    # output reads it
    for row, from_top, what in ((0, True, "halo row above the clip"), (Lv - 1, False, "row past the clip")):
        b = G.build(c)
        pair_single_path(b, row, from_top)
        eng.selftest_layer(b.lc)
        assert flag(eng) == VL.VF_OK, (name, what, "raised the flag")
        ck = G.Checker(f"{name} {what}")
        G.check_pair(b, ck)
        record(SIGS[name], "d")


# ------------------------------------------------------------------ the non-GEMM ops
def run_op(eng, case):
    eng.selftest_op(case.oc)
    return flag(eng)


def test_unet_first_and_pool(eng):
    """(a), (b) on valid elements; (d): the aux cases' NaN pad columns and rows past a clip (never read) leave the flag clear
    and the outputs match float64."""
    spec = A.FIRST_CASES["first.mel_varlen_T130_T3"]
    for what, val in (("overflow", 1e6), ("NaN", np.nan), ("+Inf", np.inf)):
        args = A.first_case("first.mel_varlen_T130_T3", spec)
        args[1][0, 5, 7] = val
        assert run_op(eng, args[0]) == VL.VF_EDEVICE, ("first", what)
    args = A.first_case("first.mel_varlen_T130_T3", spec)
    assert run_op(eng, args[0]) == VL.VF_OK
    A.check_first("first.after_flag", *args)
    record("first", "a"); record("first", "b"); record("first", "d")
    spec = A.POOL_CASES["pool.mel_l1_varlen"]
    for what, val in (("overflow", 1e6), ("NaN", np.nan), ("-Inf", -np.inf)):
        args = A.pool_case("pool.mel_l1_varlen", spec)
        args[1][0, 4, 6, 3] = val
        assert run_op(eng, args[0]) == VL.VF_EDEVICE, ("pool", what)
    # the raw plane r alone: the 2 x 2 block of output (2, 3) at -1e6 in a channel of positive BN scale s: r = -1e6, and
    # a = lrelu_0.01(s r + t) is about -1e4
    args = A.pool_case("pool.mel_l1_varlen", spec)
    ch = int(np.flatnonzero(args[2] > 0)[0])
    args[1][0, 4:6, 6:8, ch] = -1e6
    assert run_op(eng, args[0]) == VL.VF_EDEVICE, ("pool", "r alone")
    args = A.pool_case("pool.mel_l1_varlen", spec)
    assert run_op(eng, args[0]) == VL.VF_OK
    A.check_pool("pool.after_flag", *args)
    record("pool", "a"); record("pool", "b"); record("pool", "d")


def planes_case(name, edit=None):
    x, scale, shift, Ts, off = A.planes_inputs(name)
    if edit:
        edit(x)
    B, T = x.shape[:2]
    out = A.planes16((B, T, 128))
    return A.Case(A.PLANES, B, off, T=T, x=x, bn1_scale=scale, bn1_shift=shift, planes=out), x, scale, shift, Ts, off, out


def test_input_planes(eng):
    """affine_planes_kernel (the bi_gru / dnn input): (a) 1e6, (b) NaN / -Inf at a valid frame, (c) 65504 exact and 65510
    flagged (scale 1, shift 0), (d) NaN and 1e30 at frames past a clip: flag clear, and the planes bit-exact."""
    def at(v, b=0, t=1, ch=5):
        return lambda x: x.__setitem__((b, t, ch), v)
    for what, v in (("1e6", 1e6), ("NaN", np.nan), ("-Inf", -np.inf), ("65510", 65510.0)):
        c = planes_case("planes.dnn_T101", at(v))[0]
        assert run_op(eng, c) == VL.VF_EDEVICE, ("planes", what)
    c, x, scale, shift, Ts, off, out = planes_case("planes.dnn_T101", at(65504.0))
    assert run_op(eng, c) == VL.VF_OK
    assert out[0, 0, 1, 5] == MAX16 and out[1, 0, 1, 5] == 0
    record("planes", "a"); record("planes", "b"); record("planes", "c")

    def past(x):
        for b, t in enumerate(A.PLANES_CASES["planes.bn0_varlen"]["Ts"]):
            if t < x.shape[1]:
                x[b, t:, ::2] = np.nan
                x[b, t:, 1::2] = 1e30
    c, x, scale, shift, Ts, off, out = planes_case("planes.bn0_varlen", past)
    assert run_op(eng, c) == VL.VF_OK, "planes: values past a clip raised the flag"
    want = R.affine_planes(np.nan_to_num(x, nan=0.0), scale, shift, Ts)
    assert np.array_equal(out, want)
    record("planes", "d")


def _gru(eng, G_, w, bh, lengths, T):
    B = G_.shape[0]
    Gf, wf, bf = (torch.as_tensor(v).float().contiguous() for v in (G_, w, bh))
    out = np.full((2, B, T, 512), 0x7E00, np.uint16)
    lens = (ctypes.c_int * B)(*lengths)
    case = VL.VfGruCase(batch=B, T=T, G=Gf.data_ptr(), w_hh=wf.data_ptr(), b_hn=bf.data_ptr(), lengths=ctypes.addressof(lens),
                        relu=1, out=out.ctypes.data)
    eng.selftest_gru(case)
    return flag(eng), out


def test_gru_hidden_state(eng):
    """The GRU's h split: |h| < 1 by the recurrence, so the guard meets only what G carries: (b) a NaN (with relu, which
    would store relu(NaN) = 0) raises the flag; (d) NaN in G at frames past a clip, never read, leaves it clear and the
    planes equal the clean run's; (e) the clean run after the flag reproduces its bits."""
    from test_gpu_analysis import _gru_inputs
    T, lengths = 24, [24, 9, 17]
    G0, w, bh = _gru_inputs(len(lengths), T, seed=21)
    code, clean = _gru(eng, G0, w, bh, lengths, T)
    assert code == VL.VF_OK
    for what, (b, t, col) in (("forward", (1, 4, 3)), ("reverse n gate", (2, 16, 768 + 512 + 7))):
        Gn = G0.clone()
        Gn[b, t, col] = float("nan")
        code, _ = _gru(eng, Gn, w, bh, lengths, T)
        assert code == VL.VF_EDEVICE, ("gru", what)
        code, again = _gru(eng, G0, w, bh, lengths, T)
        assert code == VL.VF_OK and np.array_equal(again, clean), ("gru", "clean run after the flag")
    Gp = G0.clone()
    for b, n in enumerate(lengths):
        Gp[b, n:] = float("nan")
    code, out = _gru(eng, Gp, w, bh, lengths, T)
    assert code == VL.VF_OK and np.array_equal(out, clean), "gru: NaN past a clip's frames"
    record("gru", "a"); record("gru", "b"); record("gru", "d")


def test_conditioning_clamps_a_nan_mel_bin(eng):
    """voc_condition_kernel clamps instead of flagging (DESIGN.md §3): a NaN log-mel bin goes through fminf(x, 5) and a
    NaN linear bin through fmaxf(v, floor), so the planes stay finite and the call is VF_OK; every other element is the
    clean run's."""
    for name in ("cond.log_T37_odd", "cond.lin_T40_even"):
        args = A.cond_case(name, A.COND_CASES[name])
        assert run_op(eng, args[0]) == VL.VF_OK
        clean = args[4].copy()
        args = A.cond_case(name, A.COND_CASES[name])
        args[1][0, 11, 40] = np.nan
        assert run_op(eng, args[0]) == VL.VF_OK, (name, "NaN mel bin")
        got = args[4]
        assert np.isfinite(A.hi_lo(got)).all(), (name, "non-finite conditioning")
        diff = np.argwhere(got != clean)
        assert {(int(d[1]), int(d[2]), int(d[3])) for d in diff} <= {(0, 11, 40)}, (name, diff[:4].tolist())
    record("cond", "clamp")


# ------------------------------------------------------------------ (f) coverage
def test_every_signature_and_op_kind_has_an_overflow_and_a_must_zero_case(eng):
    """Every GEMM / pair configuration the plans build (test_gpu_layers.plan_sweep) that writes an fp16 plane has an (a)
    and a (d) case above, and so has every split-writing op kind.  Launches that write only fp32 (the GRU input projection,
    the analysis modules' last Linear, the fused head) have no fp16 plane to guard."""
    for n in NAMES:
        c = G.BY_NAME[n]
        if n not in SIGS:
            run_clean(eng, n)
        need = {"a", "d"}
        if not need <= COVER.get(SIGS[n], set()):
            if c["kind"] == PAIR:
                test_pair_planes_boundary_and_halo(eng, n)
            else:
                test_each_plane_out_of_range_alone_raises_the_flag(eng, n)
                test_must_zero_places_leave_the_flag_clear(eng, n)
    fp16_sigs = {SIGS[n] for n in NAMES}
    for c in G.CASES:
        if c["name"] not in SIGS and not c.get("windows"):
            b = G.build(c)
            eng.selftest_layer(b.lc)
            assert flag(eng) == VL.VF_OK
            SIGS[c["name"]] = b.lc.sig.decode()
    fp32_only = {SIGS[c["name"]] for c in G.CASES if c["name"] in SIGS and not fp16_outs(c)} - fp16_sigs
    sweep = G.plan_sweep()
    missing = {}
    for plan, label, sig in sweep:
        if sig in fp32_only:
            continue
        lack = {"a", "d"} - COVER.get(sig, set())
        if lack:
            missing.setdefault(sig, (sorted(lack), []))[1].append(f"{plan}:{label}")
    for sig in sorted({s for _, _, s in sweep}):
        print(f"{sig}: {'fp32 only' if sig in fp32_only else ' '.join(sorted(COVER.get(sig, set())))}")
    assert not missing, "plan signatures without a range-guard case:\n" + "\n".join(
        f"{sig} lacks {lack}: {', '.join(labels[:4])}" for sig, (lack, labels) in sorted(missing.items()))
    if not {"a", "d"} <= COVER.get("planes", set()):
        test_input_planes(eng)
    if "d" not in COVER.get("gru", set()):
        test_gru_hidden_state(eng)
    if "d" not in COVER.get("first", set()):
        test_unet_first_and_pool(eng)
    lacking = [k for k in ("first", "pool", "planes", "gru") if not {"a", "d"} <= COVER.get(k, set())]
    assert not lacking, ("split-writing op kinds without a range-guard case", lacking)
