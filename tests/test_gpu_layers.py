"""Every conv GEMM configuration the plans build, one layer at a time, against a float64 reference (oracle/layers.py).

vf_selftest_layer builds one layer the way plan.cu does (the product's packers, tap lists, Builder::gemm and the fused
pair's set-up), runs it on operands whose every bit the test chose, and copies the outputs back.  Each output element is
checked against |y - y64| <= tol * M, M being the same op on |x| and |w| plus |bias| and |residual|; elements the layer
must zero are checked for exact zeros, and every element outside the layer's write set must still hold its sentinel."""
import ctypes
import zlib

import numpy as np
import pytest
import torch

from oracle import layers as R
from voicefixer_main_b200 import _lib as VL

pytestmark = pytest.mark.gpu

SENT16 = np.uint16(0x7E5A)        # fp16 NaN payloads: no layer output is a NaN
SENT32 = np.uint32(0x7FC0BEEF)
TOL = {3: 2.0 ** -16, 1: 2.0 ** -14}
FLOOR = 2.0 ** -24                # fp16 subnormal spacing: the absolute floor of every plane bound
RES_SLOPE, STAGE_SLOPE, UNET_SLOPE = 0.01, 0.2, 0.01
CONV2D, CONVT2D, CONV1D, CONVT1D, PAIR = range(5)                            # vf_layer_case kinds (include/b200vf.h)
RESID = {"fp32": 1, "planes": 2, "ar": 3, "identity": 4}

REPORTS = {}          # case name -> reported launch configuration (product kernel)


def C(name, kind, **kw):
    kw["name"], kw["kind"] = name, kind
    return kw


def unet_conv1(name, H, W, cin, cout, n_img=1, row_valid=None):
    return C(name, CONV2D, terms=3, n_img=n_img, H=H, W=W, cin=cin, cout=cout, outs="a", affine=True, act=1,
             slope=UNET_SLOPE, row_valid=row_valid)


CASES = [
    # ---- UNet conv1 (plan.cu: conv1 lambda): 3-term, out_a = bn2 affine + LeakyReLU
    unet_conv1("conv1.mel_l0", 4, 127, 32, 32),
    unet_conv1("conv1.v2_l0", 2, 1024, 32, 32),
    unet_conv1("conv1.v2_l1", 2, 512, 64, 64),
    unet_conv1("conv1.v2_l6", 2, 16, 384, 384),
    unet_conv1("conv1.mel_l6", 1, 1, 384, 384),
    unet_conv1("conv1.varlen", 8, 63, 64, 64, n_img=3, row_valid=[512, 200, 100]),
    # ---- conv2 + 1x1 shortcut (BK = 64 with the 32-channel tail zero-padded; the decoder's 2C shortcut); bias = shortcut's
    C("conv2_sc.enc2_b1", CONV2D, terms=3, H=4, W=63, cin=64, cout=64, sc_cin=32, outs="raw,a", affine=True, act=1, slope=UNET_SLOPE),
    C("conv2_sc.dec_b2", CONV2D, terms=3, H=4, W=31, cin=64, cout=64, sc_cin=128, outs="raw,a", affine=True, act=1, slope=UNET_SLOPE),
    # ---- conv2 + fp32 residual (run-ahead ring of 2 and of 1 residual tiles; many tiles per CTA)
    C("conv2_res.c32_many_tiles", CONV2D, terms=3, H=32, W=1024, cin=32, cout=32, resid="fp32", outs="raw,a", affine=True, act=1, slope=UNET_SLOPE),
    C("conv2_res.c384", CONV2D, terms=3, H=2, W=16, cin=384, cout=384, resid="fp32", outs="raw,a", affine=True, act=1, slope=0.0),
    C("conv2_res.varlen_empty_tiles", CONV2D, terms=3, n_img=2, H=16, W=63, cin=64, cout=64, resid="fp32", outs="raw,a",
      affine=True, act=1, slope=UNET_SLOPE, row_valid=[1024, 70]),
    # ---- skip into the decoder's concat buffer: raw + the r / a halves at c_off = C, ld = 2C
    C("skip_concat.enc_b4", CONV2D, terms=3, H=4, W=63, cin=64, cout=64, resid="fp32", outs="raw,r,a", concat=True,
      affine=True, act=1, slope=UNET_SLOPE),
    # ---- decoder up: ConvTranspose2d k3 s2 + prune + concat placement
    C("convt2d.mel_time_only", CONVT2D, terms=3, H=4, W=31, cin=128, cout=64, both=0, outs="r,a", concat_low=True,
      affine=True, act=1, slope=UNET_SLOPE),
    C("convt2d.v2_both", CONVT2D, terms=3, H=2, W=512, cin=64, cout=32, both=1, outs="r,a", concat_low=True, affine=True,
      act=1, slope=UNET_SLOPE),
    C("convt2d.c384_to_32_odd_wp_varlen", CONVT2D, terms=3, n_img=2, H=4, W=16, cin=384, cout=32, both=1, outs="r,a",
      concat_low=True, affine=True, act=1, slope=UNET_SLOPE, row_valid=[68, 40], out_slack=3),
    C("convt2d.time_only_varlen", CONVT2D, terms=3, n_img=2, H=4, W=15, cin=64, cout=32, both=0, outs="r,a", concat_low=True,
      affine=True, act=1, slope=UNET_SLOPE, row_valid=[64, 23], out_slack=3),
    # ---- post block conv2 + fused 1x1 head (+ the log-mel residual of the mel UNet)
    C("head.mel", CONV2D, terms=3, n_img=2, H=8, W=127, cin=32, cout=32, resid="fp32", head=True, head_in=True, head_T=7,
      head_valid=[7, 3]),
    C("head.v2", CONV2D, terms=3, H=4, W=1024, cin=32, cout=32, resid="fp32", head=True, head_in=False, head_T=4),
    # ---- vocoder condition net (ELU) and stem (k = 7, not centred, LeakyReLU 0.2)
    C("cond.tv42_t1", CONV1D, terms=1, L=42, cin=128, cout=512, k=3, outs="a", act=2),
    C("cond.tv42_t3", CONV1D, terms=3, L=42, cin=128, cout=512, k=3, outs="a", act=2),
    C("cond.tv1006_t1", CONV1D, terms=1, n_img=2, L=1006, cin=512, cout=512, k=3, outs="a", act=2),
    C("cond.last_row0_3", CONV1D, terms=1, L=128, cin=512, cout=512, k=3, outs="a", act=2, out_row0=3, out_slack=6),
    C("cond.L129_t3", CONV1D, terms=3, L=129, cin=128, cout=512, k=3, outs="a", act=2),
    C("stem.k7", CONV1D, terms=1, L=42, x_extra=6, cin=512, cout=1024, k=7, centered=0, outs="a", act=1, slope=STAGE_SLOPE),
    C("stem.k7_t3", CONV1D, terms=3, L=127, x_extra=6, cin=512, cout=1024, k=7, centered=0, outs="a", act=1, slope=STAGE_SLOPE),
    # ---- up-sampler: ConvTranspose1d stride s
    C("up.s7_ar_tma", CONVT1D, terms=1, L=42, cin=1024, cout=512, stride=7, outs="a", out_ar=True),
    C("up.s7_ar_tma_2img", CONVT1D, terms=1, n_img=2, L=294, cin=512, cout=256, stride=7, outs="a", out_ar=True),
    C("up.s3_r_stg", CONVT1D, terms=1, L=2058, cin=256, cout=128, stride=3, outs="r,a", act=1, slope=RES_SLOPE),
    C("up.s3_t3", CONVT1D, terms=3, L=300, cin=128, cout=64, stride=3, outs="r,a", act=1, slope=RES_SLOPE),
    C("up.s3_ar_varlen", CONVT1D, terms=1, n_img=3, L=200, cin=128, cout=64, stride=3, outs="a", out_ar=True,
      row_valid=[600, 385, 100]),
    # ---- res.a: k = 3 dilated, LeakyReLU 0.01
    C("res_a.d1_c512", CONV1D, terms=1, L=294, cin=512, cout=512, k=3, dilation=1, outs="a", act=1, slope=RES_SLOPE),
    C("res_a.d3_c256", CONV1D, terms=1, L=2058, cin=256, cout=256, k=3, dilation=3, outs="a", act=1, slope=RES_SLOPE),
    C("res_a.d27_c128", CONV1D, terms=1, L=1500, cin=128, cout=128, k=3, dilation=27, outs="a", act=1, slope=RES_SLOPE),
    C("res_a.d243_c64", CONV1D, terms=1, L=1000, cin=64, cout=64, k=3, dilation=243, outs="a", act=1, slope=RES_SLOPE),
    C("res_a.d2187_gt_L", CONV1D, terms=1, L=1000, cin=64, cout=64, k=3, dilation=2187, outs="a", act=1, slope=RES_SLOPE),
    # ---- res.b: k = 3 + the residual stream
    C("res_b.ar_c512", CONV1D, terms=1, L=294, cin=512, cout=512, k=3, resid="ar", outs="a", out_ar=True),
    C("res_b.ar_c256", CONV1D, terms=1, L=2058, cin=256, cout=256, k=3, resid="ar", outs="a", out_ar=True),
    C("res_b.ar_c128_varlen", CONV1D, terms=1, n_img=3, L=700, cin=128, cout=128, k=3, resid="ar", outs="a", out_ar=True,
      row_valid=[700, 300, 50]),
    C("res_b.identity_c128", CONV1D, terms=1, L=1000, cin=128, cout=128, k=3, resid="identity", outs="r,a", act=1, slope=RES_SLOPE),
    C("res_b.identity_c64_t3", CONV1D, terms=3, L=500, cin=64, cout=64, k=3, resid="identity", outs="r,a", act=1, slope=RES_SLOPE),
    C("res_b.planes_c256", CONV1D, terms=1, L=800, cin=256, cout=256, k=3, resid="planes", outs="r,a", act=1, slope=RES_SLOPE),
    C("res_b.planes_c512_t3", CONV1D, terms=3, L=300, cin=512, cout=512, k=3, resid="planes", outs="r,a", act=1, slope=RES_SLOPE),
    C("res_b.last_of_stack", CONV1D, terms=1, L=500, cin=128, cout=128, k=3, resid="ar", outs="a", act=1, slope=STAGE_SLOPE,
      out_row0=3, out_slack=6),
    # ---- fused residual pair (C = 64)
    C("pair.L18522", PAIR, L=18522, dilation=1),
    C("pair.L46746_d27", PAIR, L=46746, dilation=27),
    *[C(f"pair.L{L}", PAIR, L=L, dilation=3) for L in (1, 125, 126, 127, 252, 253)],
    C("pair.varlen", PAIR, n_img=3, L=1000, dilation=9, row_valid=[1000, 378, 127]),
    C("pair.last", PAIR, L=1000, dilation=243, last=True, out_row0=3, out_slack=6),
    C("pair.d2187", PAIR, L=5000, dilation=2187),
    # ---- the tile decode's division fallback: SSR 60 s level 0 (6016 x 1025 rows, two images), windows only
    C("decode_fallback", CONV1D, terms=1, n_img=2, L=6016 * 1025, cin=32, cout=32, k=1, outs="a", act=1, slope=RES_SLOPE,
      windows=True),
]
# the configurations of the former tensor-core vs SIMT self-test (centred 1-D taps), now against float64
for (n, rows, cin, cout, ntaps, dil) in [(2, 300, 32, 32, 9, 1), (1, 128, 32, 64, 3, 1), (1, 257, 32, 128, 1, 1),
                                         (2, 200, 64, 32, 3, 1), (1, 129, 64, 64, 9, 1), (2, 500, 128, 128, 3, 27),
                                         (3, 40, 384, 384, 9, 2), (1, 1000, 64, 192, 2, 1), (2, 700, 128, 512, 3, 3)]:
    for terms in (3, 1):
        CASES.append(C(f"gemm.{n}x{rows}_{cin}to{cout}_k{ntaps}_d{dil}_t{terms}", CONV1D, terms=terms, n_img=n, L=rows,
                       cin=cin, cout=cout, k=ntaps, dilation=dil, outs="raw" if terms == 3 else "r"))
BY_NAME = {c["name"]: c for c in CASES}


# ------------------------------------------------------------------ case set-up
class Built:
    pass


def _rng(name):
    return np.random.default_rng(zlib.crc32(name.encode()))


def _planes_bits(x_rows):
    """[n, rows, C] fp32-valued -> ([2, n, rows, C] uint16 hi/lo bits, hi + lo, hi)"""
    hi, lo = R.split_hi_lo(x_rows)
    return np.stack([R.to_bits(hi), R.to_bits(lo)]), hi + lo, hi


def _ptr(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def build(c, impl):
    """Inputs, the ctypes case and the float64 expectations of case c."""
    g = _rng(c["name"])
    b = Built()
    kind, terms, n = c["kind"], c.get("terms", 1), c.get("n_img", 1)
    cin, cout = c.get("cin", 64), c.get("cout", 64)
    b.c, b.n, b.terms, b.impl = c, n, terms, impl
    lc = VL.VfLayerCase()
    lc.kind, lc.impl, lc.terms, lc.n_img = kind, impl, terms, n
    lc.cin, lc.cout = cin, cout
    keep = []                                     # host arrays the case points at
    rv = c.get("row_valid")
    b.rv = None if rv is None else np.asarray(rv, np.int32)
    if b.rv is not None:
        keep.append(b.rv)
        lc.row_valid = _ptr(b.rv)

    def eff(hi_lo_sum, hi):
        return hi_lo_sum if terms == 3 else hi

    def weights(shape, fan_in):
        w = (g.standard_normal(shape) / np.sqrt(fan_in)).astype(np.float32)
        keep.append(w)
        h, l = R.split_hi_lo(torch.from_numpy(w))
        return w, (h + l if terms == 3 else h)

    def bias():
        v = (g.standard_normal(cout) * 0.5).astype(np.float32)
        keep.append(v)
        return v

    windows = c.get("windows", False)
    b.xbits = None
    # ---- operand x in rows layout
    if kind in (CONV2D, CONVT2D):
        H, W = c["H"], c["W"]
        Wp = W + 1
        rows = H * Wp
        lc.H, lc.W = H, W
        x = torch.from_numpy(g.standard_normal((n, cin, H, W)).astype(np.float32))
        xr = R.nchw_to_rows(x)
    else:
        L = c["L"]
        lc.L = L
        rows = L + c.get("x_extra", 0)
        xr = None if windows else torch.from_numpy(g.standard_normal((n, rows, cin)).astype(np.float32))
    if windows:        # too large for a whole-tensor reference: random rows in the reference windows (k = 1), zeros elsewhere
        assert c["k"] == 1
        xbits = np.zeros((2, n, rows, cin), np.uint16)
        for (i, r0, r1) in windows_of(b):
            hi, lo = R.split_hi_lo(torch.from_numpy(g.standard_normal((r1 - r0, cin)).astype(np.float32)))
            xbits[0, i, r0:r1], xbits[1, i, r0:r1] = R.to_bits(hi), R.to_bits(lo)
        b.xbits = xbits
    elif b.rv is not None:                        # a varlen plan's activations are zero past each clip's rows
        lim = b.rv if kind != CONVT1D else (b.rv + c["stride"] - 1) // c["stride"]
        for i in range(n):
            xr[i, lim[i]:] = 0
    b.rows = rows
    if windows:
        pass
    elif kind == PAIR:
        # the (a, r) stream x: a = fp16(lrelu(x)) is also conv_a's input
        xs = xr.numpy().astype(np.float32) * 2
        a, r = R.ar_encode(xs, RES_SLOPE)
        xbits = np.stack([a.view(np.uint16), r.view(np.uint16)])
        b.x_stream = torch.from_numpy(R.ar_decode(a, r, RES_SLOPE))
        b.x_act = torch.from_numpy(a.astype(np.float64))
    else:
        xbits, xsum, xhi = _planes_bits(xr)
        b.x = eff(xsum, xhi)                      # the operand as the kernel contracts it
    lc.x = _ptr(xbits)
    lc.x_img_rows, lc.x_row0 = rows, 0
    keep.append(xbits)

    # ---- weights
    if kind == CONV2D:
        w, b.w = weights((cout, cin, 3, 3), 9 * cin)
        lc.w = _ptr(w)
        if c.get("sc_cin"):
            sc = c["sc_cin"]
            lc.sc_cin = sc
            scw, b.sc_w = weights((cout, sc), sc)
            b.sc_b = torch.from_numpy(bias()).to(torch.float64)
            lc.sc_w, lc.sc_b = _ptr(scw), _ptr(keep[-1])
            sx = torch.from_numpy(g.standard_normal((n, sc, H, W)).astype(np.float32))
            sbits, ssum, shi = _planes_bits(R.nchw_to_rows(sx))
            keep.append(sbits)
            lc.sc_x = _ptr(sbits)
            b.sc_x = eff(ssum, shi)
    elif kind == CONVT2D:
        w, b.w = weights((cin, cout, 3, 3), 4 * cin)
        lc.w = _ptr(w)
        lc.both = c["both"]
    elif kind == CONV1D:
        lc.k, lc.dilation, lc.centered = c["k"], c.get("dilation", 1), c.get("centered", 1)
        w, b.w = weights((cout, cin, c["k"]), c["k"] * cin)
        lc.w = _ptr(w)
        lc.b = _ptr(bias())
        b.b = torch.from_numpy(keep[-1]).to(torch.float64)
    elif kind == CONVT1D:
        lc.stride = c["stride"]
        w, b.w = weights((cin, cout, 2 * c["stride"]), 2 * cin)
        lc.w = _ptr(w)
        lc.b = _ptr(bias())
        b.b = torch.from_numpy(keep[-1]).to(torch.float64)
    else:
        lc.terms = b.terms = terms = 1
        lc.dilation = c["dilation"]
        wa, b.wa = weights((64, 64, 3), 3 * 64)
        lc.w, lc.b = _ptr(wa), _ptr(bias())
        b.ba = torch.from_numpy(keep[-1]).to(torch.float64)
        wb, b.wb = weights((64, 64, 3), 3 * 64)
        lc.w2, lc.b2 = _ptr(wb), _ptr(bias())
        b.bb = torch.from_numpy(keep[-1]).to(torch.float64)
        lc.pair_slope_h = RES_SLOPE
        lc.pair_slope_out = STAGE_SLOPE if c.get("last") else RES_SLOPE
        lc.pair_last = int(bool(c.get("last")))
        lc.ar_slope = RES_SLOPE

    # ---- residual
    rk = c.get("resid")
    b.resid = None
    if rk:
        rrows = rows if kind != CONV1D else c["L"]
        rv32 = torch.from_numpy((g.standard_normal((n, rrows, cout)) * 2).astype(np.float32))
        if b.rv is not None:
            for i in range(n):
                rv32[i, b.rv[i]:] = 0
        if kind == CONV2D:
            rv32 = R.nchw_to_rows(R.rows_to_nchw(rv32, H, W))       # zero pad column, as the plans' fp32 streams
        if rk == "fp32":
            lc.resid_kind = RESID["fp32"]
            rarr = rv32.numpy().copy()
            b.resid = rv32.to(torch.float64)
        elif rk == "ar":
            lc.resid_kind = RESID["ar"]
            a, r = R.ar_encode(rv32.numpy(), RES_SLOPE)
            rarr = np.stack([a.view(np.uint16), r.view(np.uint16)])
            b.resid = torch.from_numpy(R.ar_decode(a, r, RES_SLOPE))
            lc.ar_slope = RES_SLOPE
        else:
            lc.resid_kind = RESID[rk]
            rarr, rsum, _ = _planes_bits(rv32)
            b.resid = rsum
        keep.append(rarr)
        lc.resid = _ptr(rarr)
    if c.get("out_ar"):
        lc.ar_slope = RES_SLOPE
    b.lc, b.keep = lc, keep
    _set_outputs(b)
    return b


def _out_geometry(b):
    c, kind = b.c, b.c["kind"]
    if kind in (CONV2D, CONVT2D):
        Wp = c["W"] + 1
        if kind == CONV2D:
            return b.rows, Wp
        ow = 2 * Wp - 1 if c["both"] else 2 * Wp
        return 2 * c["H"] * ow, ow
    if kind == CONVT1D:
        return c["L"] * c["stride"], 0
    return c["L"], 0


def _set_outputs(b):
    c, lc, n, cout = b.c, b.lc, b.n, b.lc.cout
    out_rows, _ = _out_geometry(b)
    b.out_row0 = c.get("out_row0", 0)
    b.out_img_rows = out_rows + c.get("out_slack", 0)
    lc.out_row0, lc.out_img_rows = b.out_row0, b.out_img_rows
    outs = set(c.get("outs", "a").split(",")) if c["kind"] != PAIR else {"a"}
    if c.get("head"):
        outs = set()
    ld = 2 * cout if (c.get("concat") or c.get("concat_low")) else cout
    c_off = cout if c.get("concat") else 0
    b.ld, b.c_off = ld, c_off
    b.buf = {}
    if "raw" in outs:
        raw = np.full((n, b.out_img_rows, cout), SENT32, np.uint32)
        b.buf["raw"] = raw
        lc.out_raw, lc.raw_ld = _ptr(raw), raw.shape[2]
    if "r" in outs:
        r = np.full((2, n, b.out_img_rows, ld), SENT16, np.uint16)
        b.buf["r"] = r
        lc.out_r, lc.r_ld, lc.r_c_off = _ptr(r), ld, c_off
    if "a" in outs:
        a = np.full((2, n, b.out_img_rows, ld if c["kind"] != PAIR else 64), SENT16, np.uint16)
        b.buf["a"] = a
        lc.out_a, lc.a_ld, lc.a_c_off = _ptr(a), a.shape[3], c_off
        lc.act, lc.slope = c.get("act", 1), c.get("slope", RES_SLOPE)
        lc.out_ar = int(bool(c.get("out_ar")))
        if c.get("out_ar"):
            lc.act, lc.slope = 1, RES_SLOPE
        if c.get("affine"):
            g = _rng(c["name"] + ".affine")
            b.scale = (g.uniform(0.5, 2.0, cout) * np.where(g.random(cout) < 0.2, -1, 1)).astype(np.float32)
            b.shift = (g.standard_normal(cout) * 0.3).astype(np.float32)
            b.keep += [b.scale, b.shift]
            lc.a_scale, lc.a_shift = _ptr(b.scale), _ptr(b.shift)
    if c.get("head"):
        g = _rng(c["name"] + ".head")
        b.head_w = (g.standard_normal(32) / 6).astype(np.float32)
        T, Wp = c["head_T"], c["W"] + 1
        b.head_in = (g.standard_normal((n, T, Wp)) * 3).astype(np.float32) if c.get("head_in") else None
        b.head_out = np.full((n, T, Wp), SENT32, np.uint32)
        b.head_valid = None if c.get("head_valid") is None else np.asarray(c["head_valid"], np.int32)
        b.keep += [b.head_w, b.head_in, b.head_out, b.head_valid]
        lc.head_w, lc.head_b, lc.head_T = _ptr(b.head_w), 0.375, T
        lc.head_in, lc.head_out, lc.head_valid = _ptr(b.head_in), _ptr(b.head_out), _ptr(b.head_valid)


# ------------------------------------------------------------------ float64 expectations
def reference(b, abs_=False):
    """(y, M) in output-row layout [n, out_rows, cout] before the activation: y64 and the magnitude bound's M."""
    c, kind = b.c, b.c["kind"]
    ab = (lambda t: t.abs()) if abs_ else (lambda t: t)
    if kind == CONV2D:
        H, W = c["H"], c["W"]
        x = R.rows_to_nchw(b.x, H, W)
        sc = {}
        if c.get("sc_cin"):
            sc = dict(sc_x=ab(R.rows_to_nchw(b.sc_x, H, W)), sc_w=ab(b.sc_w), sc_b=ab(b.sc_b))
        y = R.nchw_to_rows(R.conv2d(ab(x), ab(b.w), **sc))
    elif kind == CONVT2D:
        x = R.rows_to_nchw(b.x, c["H"], c["W"])
        y = R.nchw_to_rows(R.conv_transpose2d(ab(x), ab(b.w), c["both"]))
    elif kind == CONV1D:
        y = R.ncl_to_rows(R.conv1d(ab(R.rows_to_ncl(b.x)), ab(b.w), ab(b.b), c.get("dilation", 1), c.get("centered", 1)))
    else:
        y = R.ncl_to_rows(R.conv_transpose1d(ab(R.rows_to_ncl(b.x)), ab(b.w), ab(b.b), c["stride"]))
    if b.resid is not None:
        y = y + ab(b.resid)
    return y


def zero_rows_mask(b):
    """[n, out_rows] True where the layer must write zeros: the pad column and rows at or past row_valid."""
    c, kind = b.c, b.c["kind"]
    out_rows, ow = _out_geometry(b)
    z = np.zeros((b.n, out_rows), bool)
    if kind == CONV2D:
        z[:, np.arange(out_rows) % ow == ow - 1] = True
        if b.rv is not None:
            for i in range(b.n):
                z[i, b.rv[i]:] = True
    elif kind == CONVT2D:
        z[:, np.arange(out_rows) % ow == ow - 1] = True
        if b.rv is not None:
            Wp = c["W"] + 1
            oh, oc = np.divmod(np.arange(out_rows), ow)
            gemm_row = (oh // 2) * Wp + oc // 2
            for i in range(b.n):
                z[i, gemm_row >= b.rv[i]] = True
    elif b.rv is not None:
        for i in range(b.n):
            z[i, b.rv[i]:] = True
    return z


def write_mask(b, ld, c_off, cout):
    c, kind = b.c, b.c["kind"]
    if kind in (CONV2D, CONV1D, PAIR):
        return R.write_rows_plain(b.n, b.out_img_rows, ld, b.out_row0, _out_geometry(b)[0], c_off, cout)
    if kind == CONVT2D:
        _, ow = _out_geometry(b)
        return R.write_rows_convt2d(b.n, b.out_img_rows, ld, c["H"], c["W"] + 1, ow, c_off, cout)
    L, s = c["L"], c["stride"]
    return R.write_rows_convt1d(b.n, b.out_img_rows, ld, b.out_row0, L + 1, s, L * s, c_off, cout)


def windows_of(b):
    """Large cases: the output rows the reference is evaluated on - the first and the last tiles of each image, which
    make a window around every image boundary.  None: all of them."""
    if not b.c.get("windows"):
        return None
    out_rows = _out_geometry(b)[0]
    return [(i, r0, r1) for i in range(b.n) for (r0, r1) in ((0, 384), (out_rows - 384, out_rows))]


# ------------------------------------------------------------------ checks
class Checker:
    def __init__(self, name):
        self.name, self.worst = name, 0.0

    def values(self, what, got, want, bound, exact_zero):
        got = np.asarray(got, np.float64)
        want = np.asarray(want, np.float64)
        bound = np.asarray(bound, np.float64)
        assert np.isfinite(got).all(), (self.name, what, "non-finite output")
        zr = np.broadcast_to(exact_zero, got.shape)
        assert (got[zr] == 0).all(), (self.name, what, "nonzero where the layer must write zeros", int((got[zr] != 0).sum()))
        err = np.abs(got - want)
        ratio = np.where(zr, 0.0, err / np.maximum(bound, 1e-300))
        if ratio.size:
            self.worst = max(self.worst, float(ratio.max()))
            i = np.unravel_index(int(ratio.argmax()), ratio.shape)
            assert ratio.max() <= 1.0, (self.name, what, "err / bound", float(ratio.max()), "at", i, float(got[i]), float(want[i]))


def _f32(bits):
    return bits.view(np.float32).astype(np.float64)


def check_sentinels(name, what, bits, mask, sentinel):
    """Every element of the write set was written, and every other one still holds its sentinel."""
    written = bits != sentinel
    if not np.array_equal(written, mask):
        bad = np.argwhere(written != mask)
        raise AssertionError((name, what, f"{len(bad)} elements break the write set, first {bad[:4].tolist()}",
                              "touched outside" if written[tuple(bad[0])] else "not written inside"))


def run_and_check(eng, c, impl):
    b = build(c, impl)
    eng.selftest_layer(b.lc)
    eng.check_errors()
    lc = b.lc
    rep = {k: getattr(lc, k) for k in ("bn", "bk", "stages", "resid_tma", "tma_out", "grid", "tiles", "div_fallback")}
    rep["terms"] = b.terms
    ck = Checker(c["name"] + ("/simt" if impl else ""))
    if c["kind"] == PAIR:
        check_pair(b, ck)
        return ck.worst, rep
    tol = TOL[b.terms]
    cout = lc.cout
    wins = windows_of(b)
    y = reference(b) if wins is None else None
    M = reference(b, abs_=True) if wins is None else None
    zr = zero_rows_mask(b)

    def views():
        if wins is None:
            yield slice(None), 0, zr.shape[1], y, M
        else:
            for (i, r0, r1) in wins:
                yy, mm = window_reference(b, i, r0, r1)
                yield slice(i, i + 1), r0, r1, yy, mm

    for key, buf in b.buf.items():
        ld = buf.shape[-1]
        off = b.c_off if key != "raw" else 0
        m = write_mask(b, ld, off, cout)
        if key == "raw":
            check_sentinels(ck.name, key, buf, m, SENT32)
        else:
            check_sentinels(ck.name, key + ".hi", buf[0], m, SENT16)
            lo_written = key == "r" or b.terms == 3 or lc.out_ar or impl == 1
            check_sentinels(ck.name, key + ".lo", buf[1], m if lo_written else np.zeros_like(m), SENT16)
        del m
        for si, r0, r1, yy, mm in views():
            yy, mm = np.asarray(yy), np.asarray(mm)
            z = zr[si, r0:r1][..., None]
            rs, cs = slice(b.out_row0 + r0, b.out_row0 + r1), slice(off, off + cout)
            if key == "raw":
                ck.values("raw", _f32(buf[si, rs, cs]), yy, tol * mm + FLOOR, z)
                continue
            hi, lo = R.from_bits(buf[0][si, rs, cs]), R.from_bits(buf[1][si, rs, cs])
            if key == "r":
                ck.values("r", hi + lo, yy, tol * mm + 2.0 ** -21 * np.abs(yy) + FLOOR, z)
            elif lc.out_ar:
                ck.values("ar.x", R.ar_decode(hi.astype(np.float16), lo.astype(np.float16), RES_SLOPE), yy,
                          tol * mm + 2.0 ** -20 * np.abs(yy) + FLOOR, z)
                a_ref = R.lrelu(torch.as_tensor(yy), RES_SLOPE).numpy()
                ck.values("ar.a", hi, a_ref, tol * mm + _ulp16(a_ref) + FLOOR, z)
            else:
                sc = np.abs(b.scale) if c.get("affine") else 1.0
                v = torch.as_tensor(yy)
                if c.get("affine"):
                    v = v * torch.from_numpy(b.scale).double() + torch.from_numpy(b.shift).double()
                a_ref = R.activate(v, lc.act, lc.slope).numpy()
                if b.terms == 3:
                    ck.values("a", hi + lo, a_ref, sc * tol * mm + 2.0 ** -21 * np.abs(a_ref) + FLOOR, z)
                else:
                    ck.values("a", hi, a_ref, sc * tol * mm + 2.0 ** -11 * np.abs(a_ref) + FLOOR, z)
    if c.get("head"):
        check_head(b, ck, y, M, zr, tol)
    return ck.worst, rep


def _ulp16(v):
    v16 = np.abs(np.asarray(v, np.float64)).astype(np.float16)
    return np.spacing(v16).astype(np.float64)


def window_reference(b, img, r0, r1):
    """CONV1D k = 1 on the fp16 input planes: (y, M) of rows [r0, r1) of one image."""
    hi = torch.from_numpy(R.from_bits(b.xbits[0, img, r0:r1]))
    x = hi + torch.from_numpy(R.from_bits(b.xbits[1, img, r0:r1])) if b.terms == 3 else hi
    y = x @ b.w[:, :, 0].T + b.b
    m = x.abs() @ b.w[:, :, 0].abs().T + b.b.abs()
    return y[None].numpy(), m[None].numpy()


def check_head(b, ck, y, M, zr, tol):
    c = b.c
    T, Wp = c["head_T"], c["W"] + 1
    got = _f32(b.head_out)
    hw = torch.from_numpy(b.head_w).double()
    v = torch.where(torch.from_numpy(zr)[..., None], torch.zeros(()), y.clone() if torch.is_tensor(y) else torch.as_tensor(y))
    h = (v @ hw).reshape(b.n, -1, Wp)[:, :T]
    hm = (M @ hw.abs()).reshape(b.n, -1, Wp)[:, :T]
    h[:, :, :Wp - 1] += 0.375
    h[:, :, Wp - 1] = 0
    bound = tol * (hm + 0.375)
    if b.head_in is not None:
        h = h + torch.from_numpy(b.head_in).double()
        bound = bound + 2.0 ** -23 * torch.from_numpy(np.abs(b.head_in)).double()
    mask = np.zeros((b.n, T, Wp), bool)
    for i in range(b.n):
        mask[i, :T if b.head_valid is None else b.head_valid[i]] = True
    check_sentinels(ck.name, "head", b.head_out, mask, SENT32)
    ck.values("head", np.where(mask, got, 0), np.where(mask, h.numpy(), 0), bound.numpy() + FLOOR, np.zeros(1, bool))


def check_pair(b, ck):
    c = b.c
    L, n = c["L"], b.n
    a = b.buf["a"]
    orow0 = b.out_row0
    mask = R.write_rows_plain(n, b.out_img_rows, 64, orow0, L, 0, 64)
    check_sentinels(ck.name, "a", a[0], mask, SENT16)
    last = bool(c.get("last"))
    check_sentinels(ck.name, "r", a[1], np.zeros_like(mask) if last else R.write_rows_plain(n, b.out_img_rows, 64, 0, L, 0, 64), SENT16)
    tol = TOL[1]
    slope_out = STAGE_SLOPE if last else RES_SLOPE
    for i in range(n):
        Lv = L if b.rv is None else int(b.rv[i])
        xa = R.rows_to_ncl(b.x_act[i:i + 1, :Lv])
        xs = R.rows_to_ncl(b.x_stream[i:i + 1, :Lv])
        y, h = R.pair(xa, xs, b.wa, b.ba, b.wb, b.bb, c["dilation"], RES_SLOPE, fp16_h=True)
        mh = R.conv1d(xa.abs(), b.wa.abs(), b.ba.abs(), c["dilation"])
        conv_h = R.conv1d(h.abs(), b.wb.abs(), None, 1)
        M = xs.abs() + conv_h + b.bb.abs()[None, :, None] + R.conv1d(mh, b.wb.abs(), None, 1)
        bound = tol * M + 2.0 ** -11 * conv_h
        y, bound = R.ncl_to_rows(y)[0].numpy(), R.ncl_to_rows(bound)[0].numpy()
        hi = R.from_bits(a[0, i, orow0:orow0 + L])
        zero = np.zeros((L, 1), bool)
        zero[Lv:] = True
        yp = np.zeros((L, 64))
        yp[:Lv] = y
        bp = np.zeros((L, 64))
        bp[:Lv] = bound
        a_ref = R.lrelu(torch.from_numpy(yp), slope_out).numpy()
        ck.values("pair.a", hi, a_ref, bp + _ulp16(a_ref) + FLOOR, zero)
        if not last:
            r = R.from_bits(a[1, i, :L])
            x_new = R.ar_decode(hi.astype(np.float16), r.astype(np.float16), RES_SLOPE)
            ck.values("pair.x", x_new, yp, bp + 2.0 ** -20 * np.abs(yp) + FLOOR, zero)


# ------------------------------------------------------------------ tests
@pytest.fixture(scope="module")
def eng():
    from voicefixer_main_b200.model import Engine
    e = Engine("cuda:0")
    yield e
    e.check_errors()
    e.close()


def _simt_ok(c):
    return c["kind"] != PAIR and not c.get("out_ar") and c.get("resid") != "ar"


@pytest.mark.parametrize("name", [c["name"] for c in CASES])
def test_layer_matches_float64(eng, name):
    c = BY_NAME[name]
    worst, rep = run_and_check(eng, c, 0)
    REPORTS[name] = rep
    print(f"{name}: max err / bound = {worst:.3e} (tol {TOL[rep['terms']]:.1e})  config {rep}")


@pytest.mark.parametrize("name", [c["name"] for c in CASES if _simt_ok(c)])
def test_layer_simt_matches_float64(eng, name):
    worst, _ = run_and_check(eng, BY_NAME[name], 1)
    print(f"{name}/simt: max err / bound = {worst:.3e}")


@pytest.mark.parametrize("name", [c["name"] for c in CASES if c["kind"] == PAIR])
def test_pair_two_launch_path_matches_float64(eng, name):
    """The same residual pair as the two launches the plans use without the fused kernel: res.a (CONV1D, dilation d),
    then res.b (CONV1D + the (a, r) residual, (a, r) out); each checked against float64 on its own."""
    c = BY_NAME[name]
    L, n = c["L"], c.get("n_img", 1)
    common = dict(n_img=n, L=L, cin=64, cout=64, k=3, terms=1, row_valid=c.get("row_valid"))
    a_case = C(name + ".a", CONV1D, dilation=c["dilation"], outs="a", act=1, slope=RES_SLOPE, **common)
    b_case = C(name + ".b", CONV1D, dilation=1, resid="ar",
               **(dict(outs="a", act=1, slope=STAGE_SLOPE, out_row0=c.get("out_row0", 0), out_slack=c.get("out_slack", 0))
                  if c.get("last") else dict(outs="a", out_ar=True)), **common)
    for cc in (a_case, b_case):
        worst, _ = run_and_check(eng, cc, 0)
        print(f"{cc['name']}: max err / bound = {worst:.3e}")


def test_fp16_overflow_is_reported_and_the_next_case_passes(eng):
    from voicefixer_main_b200._lib import EngineError
    c = dict(BY_NAME["res_a.d243_c64"], name="overflow")
    b = build(c, 0)
    xb = np.stack([np.full_like(b.keep[0][0], 0x7800), np.zeros_like(b.keep[0][1])])   # x = 32768 everywhere
    b.lc.x = _ptr(xb)
    b.keep.append(xb)
    eng.selftest_layer(b.lc)
    with pytest.raises(EngineError) as ei:
        eng.check_errors()
    assert ei.value.code == VL.VF_EDEVICE
    run_and_check(eng, BY_NAME["res_a.d243_c64"], 0)


def test_cases_cover_every_kernel_configuration(eng):
    for c in CASES:
        if c["name"] not in REPORTS:
            REPORTS[c["name"]] = run_and_check(eng, c, 0)[1]
    reps = [r for k, r in REPORTS.items() if BY_NAME[k]["kind"] != PAIR]
    assert {32, 64, 128} <= {r["bn"] for r in reps}
    assert {32, 64} <= {r["bk"] for r in reps}
    assert {1, 3} <= {r["terms"] for r in reps}
    assert {1, 2} <= {r["resid_tma"] for r in reps}
    assert {0, 1} <= {r["tma_out"] for r in reps}
    assert any(r["tiles"] > r["grid"] for r in reps)
    assert any(r["div_fallback"] for r in REPORTS.values())
