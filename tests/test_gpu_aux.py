"""The non-GEMM kernels of the restore chains (aux.cu, istft.cu), one launch at a time, against float64 references
(oracle/layers.py).

vf_selftest_op sets each op up with the helpers the plan builders and restore paths use (first_op, pool_op, cond_op,
unify_energy, reflect_op / memset_op / tail_op, finalize_params, istft_params) and launches it as they do.  Every case
checks three things:
  1. every value against a bound derived from the kernel's arithmetic (each case's docstring gives its derivation;
     u = 2^-24, gamma_k = k u / (1 - k u), M = the same op on absolute values);
  2. exact zeros where the kernel must write zeros;
  3. every element outside the kernel's write set still holds its sentinel.
Outputs in hi/lo planes are read as hi + lo and carry 2^-21 |y| for the split; FLOOR = 2^-24 is the absolute floor of
every bound.  CUDA's documented accuracy: log10f and exp10f 2 ulp, tanhf 2 ulp; `/` is IEEE (no fast-math)."""
import ctypes
import zlib

import numpy as np
import pytest
import torch

import test_gpu_layers as G
from oracle import layers as R
from voicefixer_main_b200 import _lib as VL

pytestmark = pytest.mark.gpu

SENT16, SENT32, FLOOR = G.SENT16, G.SENT32, G.FLOOR
U = 2.0 ** -24
SPLIT = 2.0 ** -21
FIRST, POOL, COND, REFLECT, TAIL, FINALIZE, ISTFT, PEAK_NORM = range(8)     # VF_OP_* (include/b200vf.h)
HOP, TAIL_BASE, SCALES = 441, 4, (7, 7, 3, 3)
WORST = {}            # case -> worst err / bound
COVER = set()         # (kind, terms, varlen) reached


def gamma(k):
    return k * U / (1 - k * U)


def _rng(name):
    return np.random.default_rng(zlib.crc32(name.encode()))


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def n_for_frames(T, extra=100):
    """A clip length whose frame count 1 + n // 441 is T."""
    return (T - 1) * HOP + extra


def offsets(ns):
    return np.concatenate([[0], np.cumsum(ns)]).astype(np.int64)


def lengths_rows(off, w0):
    """The lengths table (kernels.cuh: VL_*) from the host formula, [18][batch]."""
    ns = np.diff(off)
    rows = np.zeros((18, len(ns)), np.int32)
    for b, n in enumerate(ns):
        T = 1 + int(n) // HOP
        Tp = (T + 63) // 64 * 64
        rows[0, b], rows[1, b] = T, Tp
        for l in range(7):
            rows[2 + l, b] = (Tp >> l) * ((w0 >> l) + 1)
        Tv = R.voc_frames(T, TAIL_BASE)
        rows[9, b] = Tv
        L = Tv
        for s, sc in enumerate(SCALES):
            L *= sc
            rows[10 + s, b] = L
    return rows


class Case:
    """A vf_op_case plus the host arrays it points at."""

    def __init__(self, kind, batch, clip_off=None, w0=127, **fields):
        self.oc = VL.VfOpCase()
        self.keep = []
        self.oc.kind, self.oc.batch = kind, batch
        if clip_off is not None:
            self.off = np.asarray(clip_off, np.int64)
            self.rows = np.zeros((18, batch), np.int32)
            self.oc.clip_off, self.oc.unet_w0, self.oc.vl_rows = self.ptr(self.off), w0, self.ptr(self.rows)
        else:
            self.off = None
        for k, v in fields.items():
            setattr(self.oc, k, self.ptr(v) if isinstance(v, np.ndarray) else v.item() if isinstance(v, np.generic) else v)

    def ptr(self, a):
        self.keep.append(a)
        return _p(a)

    def run(self, eng, name):
        eng.selftest_op(self.oc)
        eng.check_errors()
        COVER.add((self.oc.kind, self.oc.terms if self.oc.kind == TAIL else 0, self.off is not None))
        if self.off is not None:        # the lengths table every varlen kernel reads, row by row (rows past the last
            want = lengths_rows(self.off, self.oc.unet_w0)      # vocoder stage are not part of it)
            for r in range(10 + len(SCALES)):
                assert np.array_equal(self.rows[r], want[r]), (name, "lengths table row", r, self.rows[r], want[r])
        return self


def planes16(n, fill=SENT16):
    return np.full((2,) + tuple(n), fill, np.uint16)


def hi_lo(bits):
    return R.from_bits(bits[0]) + R.from_bits(bits[1])


def split_bits(x):
    hi, lo = R.split_hi_lo(torch.as_tensor(np.asarray(x, np.float32)))
    return np.stack([R.to_bits(hi), R.to_bits(lo)])


def report(name, ck):
    WORST[name] = ck.worst
    print(f"{name}: max err / bound = {ck.worst:.3e}")


@pytest.fixture(scope="module")
def eng():
    from voicefixer_main_b200.model import Engine
    e = Engine("cuda:0")
    yield e
    e.check_errors()
    e.close()


# ------------------------------------------------------------------ FIRST: unet_first_kernel
FIRST_CASES = {
    "first.mel_T101_neg_shift": dict(W=127, Ts=[101], shift=-0.7),
    "first.mel_T64_pos_shift": dict(W=127, Ts=[64], shift=0.9),
    "first.v2_T71": dict(W=1024, Ts=[71], shift=-0.3),
    "first.mel_varlen_T130_T3": dict(W=127, Ts=[130, 3], shift=-0.5, varlen=True),
}


def first_case(name, spec, x_scale=2.0):
    g = _rng(name)
    W, Ts = spec["W"], spec["Ts"]
    B = len(Ts)
    varlen = spec.get("varlen", False)
    T = (max(Ts) + 63) // 64 * 64 if varlen else Ts[0]          # a varlen plan's frames: the bucket
    x = (g.standard_normal((B, T, W + 1)) * x_scale).astype(np.float32)
    x[:, :, W] = np.nan                                         # the unused last bin: never read
    for b, t in enumerate(Ts):
        x[b, t:] = np.nan                                       # rows past a clip's frames: never read
    p = dict(bn1_scale=np.float32(g.uniform(0.5, 1.5)), bn1_shift=np.float32(spec["shift"]),
             w1=(g.standard_normal((32, 9)) / 3).astype(np.float32),
             bn2_scale=(g.uniform(0.5, 2.0, 32) * np.where(g.random(32) < 0.2, -1, 1)).astype(np.float32),
             bn2_shift=(g.standard_normal(32) * 0.3).astype(np.float32),
             w_sc=g.standard_normal(32).astype(np.float32), b_sc=(g.standard_normal(32) * 0.5).astype(np.float32))
    Tp = (T + 63) // 64 * 64
    a2 = planes16((B, Tp * (W + 1), 32))
    sc = np.full((B, Tp * (W + 1), 32), SENT32, np.uint32)
    off = offsets([n_for_frames(t) for t in Ts]) if varlen else None
    c = Case(FIRST, B, off, w0=W, T=T, W=W, x=x, a2=a2, sc_raw=sc, **p)
    return c, x, p, Ts, T, a2, sc


def check_first(name, c, x, p, Ts, T, a2, sc):
    """y = 9-tap fp32 fmaf chain on h = lrelu(fmaf(x, s1, t1)): |dy| <= gamma_10 M_y, M_y = conv(|x s1| + |t1|, |w|).
    a = lrelu(fmaf(y, s2, t2)) in hi/lo: gamma_11 (|s2| M_y + |t2|) + 2^-21 |a|.  sc_raw = fmaf(x, w_sc, b_sc) in fp32:
    gamma_1 (|x w_sc| + |b_sc|).  Zeros: the pad column and, varlen, rows t >= Tp_b."""
    W = c.oc.W
    Tp = c.oc.Tp
    assert Tp == (T + 63) // 64 * 64
    ck = G.Checker(name)
    Wp = W + 1
    ahl = hi_lo(a2).reshape(len(Ts), Tp, Wp, 32)
    scv = sc.view(np.float32).astype(np.float64).reshape(len(Ts), Tp, Wp, 32)
    assert not (a2 == SENT16).any() and not (sc == SENT32).any(), (name, "an element of the output was not written")
    ab = lambda v: np.abs(np.asarray(v, np.float64))
    for b, Tb in enumerate(Ts):
        Tpb = (Tb + 63) // 64 * 64
        xb = x[b:b + 1, :Tb].astype(np.float64)
        xb[..., W] = 0
        _, y, a, r = R.unet_first(xb, Tpb, p["bn1_scale"], p["bn1_shift"], p["w1"], p["bn2_scale"], p["bn2_shift"],
                                  p["w_sc"], p["b_sc"])
        xp = np.zeros((1, 1, Tpb, W))
        xp[0, 0, :Tb] = xb[0, :, :W]
        hm = torch.as_tensor(ab(xp * p["bn1_scale"]) + abs(float(p["bn1_shift"])))
        My = torch.nn.functional.conv2d(hm, torch.as_tensor(ab(p["w1"])).reshape(32, 1, 3, 3), padding=1).numpy()[0]
        s2, t2 = ab(p["bn2_scale"])[:, None, None], ab(p["bn2_shift"])[:, None, None]
        a, r = a.numpy()[0], r.numpy()[0]
        ba = gamma(11) * (s2 * My + t2) + SPLIT * np.abs(a) + FLOOR
        br = gamma(1) * (ab(xp[0]) * ab(p["w_sc"])[:, None, None] + ab(p["b_sc"])[:, None, None]) + FLOOR
        got_a = ahl[b].transpose(2, 0, 1)           # [32, Tp, Wp]
        got_r = scv[b].transpose(2, 0, 1)
        zero = np.zeros((1, Tp, Wp), bool)
        zero[:, :, W] = True
        zero[:, Tpb:] = True
        pad = lambda v: np.pad(v, ((0, 0), (0, Tp - Tpb), (0, 1)))
        ck.values("a", got_a, pad(a), pad(ba), zero)
        ck.values("sc_raw", got_r, pad(r), pad(br), zero)
    return ck


@pytest.mark.parametrize("name", list(FIRST_CASES))
def test_first_layer_matches_float64(eng, name):
    args = first_case(name, FIRST_CASES[name])
    args[0].run(eng, name)
    report(name, check_first(name, *args))


# ------------------------------------------------------------------ POOL: pool_kernel
POOL_CASES = {
    "pool.mel_l0": dict(W=127, H=64, C=32, level=0),
    "pool.mel_l5_one_column": dict(W=3, H=4, C=384, level=5),
    "pool.v2_l0": dict(W=1024, H=16, C=32, level=0),
    "pool.v2_l4": dict(W=64, H=8, C=384, level=4),
    "pool.mel_l1_varlen": dict(W=63, H=96, C=64, level=1, Ts=[130, 3], w0=127),
}


def pool_case(name, spec, scale=3.0):
    g = _rng(name)
    W, H, C, level = spec["W"], spec["H"], spec["C"], spec["level"]
    Ts = spec.get("Ts")
    B = len(Ts) if Ts else 2
    Wp = W + 1
    x = (g.standard_normal((B, H, Wp, C)) * scale).astype(np.float32)
    x[:, :, W] = np.nan                                          # pad column: never read
    if W % 2:
        x[:, :, W - 1] = np.float32(1e30)                        # floor pooling: the odd last column is never read
    rv = None
    if Ts:
        for b, t in enumerate(Ts):
            x[b, ((t + 63) // 64 * 64) >> level:] = np.nan      # rows past the clip at this level: never read
    sc = (g.uniform(0.5, 2.0, C) * np.where(g.random(C) < 0.2, -1, 1)).astype(np.float32)
    sh = (g.standard_normal(C) * 0.3).astype(np.float32)
    Wpo = (W >> 1) + 1
    n = (B, (H // 2) * Wpo, C)
    out_r, out_a = planes16(n), planes16(n)
    out_raw = np.full(n, SENT32, np.uint32)
    off = offsets([n_for_frames(t) for t in Ts]) if Ts else None
    c = Case(POOL, B, off, w0=spec.get("w0", 127), H=H, W=W, C=C, level=level, pin=x.reshape(B, H * Wp, C),
             a_scale=sc, a_shift=sh, out_r=out_r, out_a=out_a, out_raw=out_raw)
    if Ts:
        rv = lengths_rows(off, spec.get("w0", 127))[2 + level + 1]
    return c, x, sc, sh, out_r, out_a, out_raw, rv


def check_pool(name, c, x, sc, sh, out_r, out_a, out_raw, rv):
    """v = 0.25 * (4 fp32 adds): gamma_3 M, M = avg_pool(|x|).  a = lrelu(fmaf(v, s, t)): gamma_4 (|s| M + |t|).  Planes +
    2^-21 |y|.  Zeros: the output pad column (and with it the one column of an output pitch of 2) and rows past row_valid."""
    B, H, Wp, C = x.shape
    W = Wp - 1
    Wpo = c.oc.Wpo
    assert Wpo == (W >> 1) + 1
    ck = G.Checker(name)
    for arr, s in ((out_r, SENT16), (out_a, SENT16), (out_raw, SENT32)):
        assert not (arr == s).any(), (name, "an element of the output was not written")
    xin = np.nan_to_num(x[:, :, :W].astype(np.float64), nan=0.0, posinf=0.0)
    xin = np.where(np.abs(xin) > 1e29, 0, xin)
    xt = torch.as_tensor(xin).permute(0, 3, 1, 2)
    v, a = R.pool(xt, sc, sh)
    M = torch.nn.functional.avg_pool2d(xt.abs(), 2)
    v, a, M = (t.permute(0, 2, 3, 1).numpy() for t in (v, a, M))       # [B, H/2, W//2, C]
    pad = lambda t: np.pad(t, ((0, 0), (0, 0), (0, 1), (0, 0)))
    v, a, M = pad(v), pad(a), pad(M)
    zero = np.zeros((B, H // 2, Wpo, 1), bool)
    zero[:, :, Wpo - 1] = True
    if rv is not None:
        for b in range(B):
            zero[b].reshape(-1)[rv[b]:] = True
    sh_ = lambda t: t.reshape(B, H // 2, Wpo, C)
    bv = gamma(3) * M + FLOOR
    ba = gamma(4) * (np.abs(sc) * M + np.abs(sh)) + SPLIT * np.abs(a) + FLOOR
    ck.values("raw", sh_(out_raw.view(np.float32).astype(np.float64)), v, bv, zero)
    ck.values("r", sh_(hi_lo(out_r)), v, bv + SPLIT * np.abs(v), zero)
    ck.values("a", sh_(hi_lo(out_a)), a, ba, zero)
    return ck


@pytest.mark.parametrize("name", list(POOL_CASES))
def test_pool_matches_float64(eng, name):
    args = pool_case(name, POOL_CASES[name])
    args[0].run(eng, name)
    report(name, check_pool(name, *args))


# ------------------------------------------------------------------ COND (+ BAND): voc_condition_kernel, band_energy_kernel
def mel_weight64():
    cfg = VL.VfConfig()
    VL.load_library().vf_default_config(ctypes.byref(cfg))
    return cfg.voc_mel_weight_a * np.exp(cfg.voc_mel_weight_b * np.arange(128))


COND_CASES = {
    "cond.log_T37_odd": dict(Ts=[37, 37], is_log=1),
    "cond.lin_T40_even": dict(Ts=[40], is_log=0),
    "cond.log_T37_unify": dict(Ts=[37, 37], is_log=1, unify=True),
    "cond.log_varlen_unify": dict(Ts=[37, 10, 61], is_log=1, unify=True, varlen=True),
}


def cond_case(name, spec):
    g = _rng(name)
    Ts = spec["Ts"]
    B = len(Ts)
    varlen = spec.get("varlen", False)
    T = (max(Ts) + 63) // 64 * 64 if varlen else Ts[0]
    if spec["is_log"]:
        mel = g.uniform(-10.0, 7.0, (B, T, 128)).astype(np.float32)     # below the amp floor .. past from_log's clamp at 5
    else:
        mel = (np.exp(g.uniform(-14, 9, (B, T, 128))) * np.where(g.random((B, T, 128)) < 0.2, -1, 1)).astype(np.float32)
    for b, t in enumerate(Ts):
        mel[b, t:] = np.nan                                              # rows past a clip: never read
    tgt = None
    sums = None
    kw = {}
    if spec.get("unify"):
        tgt = np.exp(g.uniform(-6, 4, (B, T, 128))).astype(np.float32)
        for b, t in enumerate(Ts):
            tgt[b, t:] = np.nan
        sums = np.full((B, 2), SENT32, np.uint32)
        kw = dict(unify=1, mel_target=tgt, band_sums=sums)
    Tv = R.voc_frames(T, TAIL_BASE)
    out = planes16((B, Tv, 128))
    off = offsets([n_for_frames(t) for t in Ts]) if varlen else None
    c = Case(COND, B, off, T=T, is_log=spec["is_log"], mel=mel, cond=out, **kw)
    return c, mel, tgt, sums, out, Ts, T


def band_bound(tgt, mel, Tb):
    """Each sum is fp32: per-thread strided partial sums (ceil(20 T_b / 256) terms), a 5-level shuffle tree, then 8 warp
    sums: gamma_(k + 13) of the sum of |terms|; each estimate term carries exp10f's 2 ulp (2^-22 relative)."""
    k = -(-20 * Tb // 256) + 13
    lo, hi = R.BAND
    st = np.abs(tgt[:Tb, lo:hi].astype(np.float64)).sum()
    se = (10.0 ** np.minimum(mel[:Tb, lo:hi].astype(np.float64), 5.0)).sum()
    return np.array([gamma(k) * st, (gamma(k) + 2.0 ** -22) * se])


def check_cond(name, c, mel, tgt, sums, out, Ts, T):
    """m = exp10f(min(x, 5)) (2^-22 relative) [* ratio: relative 2 sum bounds + u]; v = |m| / w (IEEE, and w is the
    context's fp32 table of the float64 weight: 2u); s = 20 log10f(max(v, floor)) - ref: 20 (dv / ln 10 + 2^-22 |log10 v|)
    + gamma_3 (20 |log10 v| + |ref|); c = clip((s - min) / -min): (ds + gamma_2 (|s| + |min|)) / 115.  Plus 2^-21 |c|.
    Rows T_b <= t < Tv_b hold the tail value -4 exactly; varlen rows t >= Tv_b exact zeros."""
    B = len(Ts)
    Tv = c.oc.Tv
    assert Tv == R.voc_frames(T, TAIL_BASE)
    ck = G.Checker(name)
    assert not (out == SENT16).any(), (name, "an element of the output was not written")
    got = hi_lo(out)
    w = mel_weight64()
    is_log = c.oc.is_log
    for b, Tb in enumerate(Ts):
        Tvb = R.voc_frames(Tb, TAIL_BASE) if c.off is not None else Tv
        m = mel[b:b + 1, :Tb]
        rel = 2.0 ** -22 if is_log else 0.0
        s64 = None
        if tgt is not None:
            s64 = R.band_sums(tgt[b:b + 1], mel[b:b + 1], [Tb])
            bb = band_bound(tgt[b], mel[b], Tb)
            gs = sums[b].view(np.float32).astype(np.float64)
            ck.values("band", gs, s64[0], bb + FLOOR, np.zeros(1, bool))
            rel += bb[0] / s64[0, 0] + bb[1] / s64[0, 1] + U
        want = R.voc_condition(m, is_log, w, Tvb, sums=s64)[0]
        mm = 10.0 ** np.minimum(m[0].astype(np.float64), 5.0) if is_log else np.abs(m[0].astype(np.float64))
        if s64 is not None:
            mm = mm * s64[0, 0] / s64[0, 1]
        v = np.maximum(mm / w, 1e-5)
        lg = np.abs(np.log10(v))
        ds = 20.0 * ((rel + 2 * U) / np.log(10.0) + 2.0 ** -22 * lg) + gamma(3) * (20.0 * lg + 20.0)
        s = 20.0 * np.log10(v) - 20.0
        bnd = np.zeros((Tv, 128))
        bnd[:Tb] = (ds + gamma(2) * (np.abs(s) + 115.0)) / 115.0
        bnd += SPLIT * np.abs(np.pad(want, ((0, Tv - Tvb), (0, 0)))) + FLOOR
        zero = np.zeros((Tv, 1), bool)
        zero[Tvb:] = True
        wantp = np.pad(want, ((0, Tv - Tvb), (0, 0)))
        ck.values("cond", got[b], wantp, bnd, zero)
        assert (got[b, Tb:Tvb] == -4.0).all(), (name, "tail rows")
    return ck


@pytest.mark.parametrize("name", list(COND_CASES))
def test_conditioning_matches_float64(eng, name):
    args = cond_case(name, COND_CASES[name])
    args[0].run(eng, name)
    report(name, check_cond(name, *args))


def test_band_sums_are_reproducible_and_varlen_equals_its_own_launch(eng):
    """kernels.cuh: clip b of a varlen launch sums its first T_b frames in the order of a T = T_b launch.  T_b * 20 is not a
    multiple of 256 for any clip here."""
    spec = COND_CASES["cond.log_varlen_unify"]
    c1, mel, tgt, sums1, *_ = cond_case("cond.log_varlen_unify", spec)
    c1.run(eng, "band.varlen.1")
    c2, _, _, sums2, *_ = cond_case("cond.log_varlen_unify", spec)
    c2.run(eng, "band.varlen.2")
    assert np.array_equal(sums1, sums2)
    for b, Tb in enumerate(spec["Ts"]):
        assert (20 * Tb) % 256
        m = np.ascontiguousarray(mel[b:b + 1, :Tb])
        t = np.ascontiguousarray(tgt[b:b + 1, :Tb])
        s = np.full((1, 2), SENT32, np.uint32)
        Case(COND, 1, T=Tb, is_log=1, mel=m, mel_target=t, band_sums=s, unify=1,
             cond=planes16((1, R.voc_frames(Tb, TAIL_BASE), 128))).run(eng, f"band.T{Tb}")
        assert np.array_equal(s[0], sums1[b]), (b, s[0].view(np.float32), sums1[b].view(np.float32))


# ------------------------------------------------------------------ REFLECT: reflect_fill_kernel (bit-exact)
REFLECT_CASES = {
    "reflect.c512_Tv42": dict(C=512, Ls=[42, 42], cond_pad=1),
    "reflect.c64_L46746": dict(C=64, Ls=[46746], cond_pad=0),
    "reflect.c64_varlen": dict(C=64, Ts=[37, 3, 16], cond_pad=0),
    "reflect.c512_varlen_cond": dict(C=512, Ts=[37, 10], cond_pad=1),
}


def clip_lengths(spec):
    """Per clip rows of a REFLECT / TAIL case: the given lengths, or those the lengths table gives the clips' frames."""
    if "Ts" not in spec:
        return spec["Ls"], None
    off = offsets([n_for_frames(t) for t in spec["Ts"]])
    rows = lengths_rows(off, 127)
    return list(rows[9 if spec.get("cond_pad") else 13]), off


@pytest.mark.parametrize("name", list(REFLECT_CASES))
def test_reflect_fill_is_exact(eng, name):
    spec = REFLECT_CASES[name]
    g = _rng(name)
    Ls, off = clip_lengths(spec)
    C, B, L = spec["C"], len(Ls), max(Ls)
    pl = planes16((B, L + 6, C))
    for b, Lb in enumerate(Ls):
        pl[:, b, 3:3 + Lb] = g.integers(0, 0x7C00, (2, Lb, C), dtype=np.uint16)
    before = pl.copy()
    Case(REFLECT, B, off, L=L, C=C, cond_pad=spec["cond_pad"], planes=pl).run(eng, name)
    check_reflect(name, before, pl, Ls)
    WORST[name] = 0.0
    print(f"{name}: bit-exact")


def check_reflect(name, before, after, Ls, pad=R.reflect_pad):
    """Rows [0, L_b + 6) of each clip are the reflection of its rows [3, L_b + 3), bit for bit; the rest is untouched."""
    for b, Lb in enumerate(Ls):
        want = pad(before[:, b, 3:3 + Lb].astype(np.int32), 3).astype(np.uint16)     # the two planes as two images
        assert np.array_equal(after[:, b, :Lb + 6], want), (name, b)
        assert np.array_equal(after[:, b, Lb + 6:], before[:, b, Lb + 6:]), (name, b, "rows past the clip touched")


# ------------------------------------------------------------------ TAIL: voc_tail_kernel<1/3-term> + the peak memset
TAIL_CASES = {
    "tail.L18522_T37": dict(Ls=[18522, 18522]),
    "tail.L3528_T3": dict(Ls=[3528]),
    "tail.L300_lt_one_tile": dict(Ls=[300, 300]),
    "tail.varlen": dict(Ts=[37, 3, 16]),
}


def tail_case(name, spec, terms, tanh):
    g = _rng(f"{name}.{terms}.{tanh}")
    Ls, off = clip_lengths(spec)
    C, B, L = 64, len(Ls), max(Ls)
    x = np.full((B, L + 6, C), np.nan, np.float32)                 # rows past a clip's padded rows: never read
    for b, Lb in enumerate(Ls):
        x[b, :Lb + 6] = R.reflect_pad(g.standard_normal((1, Lb, C)).astype(np.float32), 3)[0]
    bits = split_bits(x)
    bits[:, np.isnan(x)] = 0x7E00
    w = (g.standard_normal((1, C, 7)) * (1.0 if tanh else 3.0) / np.sqrt(7 * C)).astype(np.float32)
    bias = np.float32(0.125)
    wav = np.full((B, L), SENT32, np.uint32)
    peak = np.full(B, SENT32, np.uint32)
    c = Case(TAIL, B, off, L=L, C=C, terms=terms, tanh_out=int(tanh), tail_in=bits, tail_w=w, tail_b=bias, wav=wav,
             peak_bits=peak)
    return c, bits, w, bias, wav, peak, Ls


def check_tail(name, c, bits, w, bias, wav, peak, Ls, terms, tanh):
    """y = a fp32 fmaf chain of 7 C products from 0 (the operand is hi, or hi + lo which fp32 holds exactly; the weights
    are exact) + the bias: |dy| <= gamma_(7C + 1) M, M = conv(|x|, |w|) + |b|.  tanh: + tanhf's 2 ulp (2^-22 |out|), and
    |tanh'| <= 1.  Peak bits == max |out| of the kernel's own output, bit for bit."""
    ck = G.Checker(name)
    C, L = c.oc.C, c.oc.L
    assert c.oc.tail_smem == 7 * C * 4 + (2 if terms == 3 else 1) * 326 * (C + 8) * 2 <= 200 * 1024
    x = R.from_bits(bits[0]) + (R.from_bits(bits[1]) if terms == 3 else 0)
    got = wav.view(np.float32).astype(np.float64)
    for b, Lb in enumerate(Ls):
        out, _, M = R.voc_tail(x[b:b + 1, :Lb + 6], w, bias, tanh)
        bnd = gamma(7 * C + 1) * M[0] + (2.0 ** -22 * np.abs(out[0]) if tanh else 0) + FLOOR
        ck.values("wav", got[b, :Lb], out[0], bnd, np.zeros(1, bool))
        assert (wav[b, Lb:] == SENT32).all(), (name, b, "samples past the clip written")
        pk = np.abs(wav[b, :Lb].view(np.float32)).max()
        assert peak[b] == pk.view(np.uint32), (name, b, peak[b], pk)
        if not tanh:
            assert pk > 1
    return ck


@pytest.mark.parametrize("tanh", [1, 0])
@pytest.mark.parametrize("terms", [1, 3])
@pytest.mark.parametrize("name", list(TAIL_CASES))
def test_tail_matches_float64(eng, name, terms, tanh):
    args = tail_case(name, TAIL_CASES[name], terms, tanh)
    args[0].run(eng, name)
    report(f"{name}.t{terms}.tanh{tanh}", check_tail(name, *args, terms, tanh))


# ------------------------------------------------------------------ FINALIZE: finalize_kernel (bit-exact)
def test_finalize_uniform_is_exact(eng):
    g = _rng("finalize.uniform")
    B, L, n = 3, 3528, 3000
    wav = g.uniform(-1, 1, (B, L)).astype(np.float32)
    peaks = np.array([0.5, 1.0, 2.5], np.float32)
    out = np.full((B, n), SENT32, np.uint32)
    c = Case(FINALIZE, B, L=L, n=n, in_wav=wav, peak_bits=peaks.view(np.uint32).copy(), out=out).run(eng, "finalize.uniform")
    skip = c.oc.skip
    assert skip == (L - n) // 2 > 0
    for b in range(B):
        assert np.array_equal(out[b], R.finalize(wav[b], peaks[b], skip, n).view(np.uint32)), b
    WORST["finalize.uniform"] = 0.0


def test_finalize_varlen_is_exact(eng):
    g = _rng("finalize.varlen")
    ns = [16000, 1000, 7000]
    off = offsets(ns)
    Ls = list(lengths_rows(off, 127)[13])
    B, L = len(ns), max(Ls)
    wav = g.uniform(-3, 3, (B, L)).astype(np.float32)
    peaks = np.array([0.75, 3.0, 1.5], np.float32)
    out = np.full(off[-1], SENT32, np.uint32)
    Case(FINALIZE, B, off, L=L, n=max(ns), in_wav=wav, peak_bits=peaks.view(np.uint32).copy(), out=out).run(eng, "finalize.varlen")
    skips = set()
    for b, (nb, Lb) in enumerate(zip(ns, Ls)):
        skip = (Lb - nb) // 2
        skips.add(skip)
        assert np.array_equal(out[off[b]:off[b + 1]], R.finalize(wav[b], peaks[b], skip, nb).view(np.uint32)), b
    assert len(skips) == B
    WORST["finalize.varlen"] = 0.0


# ------------------------------------------------------------------ ISTFT: istft_frames_kernel (fused) + istft_ola_kernel
def istft_frame_error(mg, phi):
    """E_t of the fused ISTFT (see the test's docstring): per-sample bound of frame t before the window, from the bin
    magnitudes mg [T, 1025] and the phase bounds phi [T, 1025]."""
    return (2 * (mg * (phi + 3 * U)).sum(axis=1) + 8 * U * np.log2(2048) * mg.sum(axis=1)) / 1024


ISTFT_NS = [1025, 30 * 441 + 123, 70 * 441 + 17]


def test_fused_istft_varlen_matches_float64(eng):
    """Per frame t: the STFT X of the input frame is fp32 radix-2: |dX_k| <= 4 u log2(2048) S_t, S_t = sum |x w|, so the
    phase (cos, sin) moves by phi_k = min(2, 4 u log2(2048) S_t / max(|X_k|, 1e-4)) (the 1e-4 is the 1e-8 power clamp; two
    unit vectors differ by at most 2), and |dY_k| <= mag_k (phi_k + 3u).  The packed inverse (1024-point FFT, /1024) of Y gives
    |dx| <= E_t = (2 sum_k |dY_k| + 8 u log2(2048) sum_k mag_k) / 1024 per sample; the window multiply adds gamma_3 |f|.
    Overlap-add: (sum_t w E_t + gamma_8 sum_t |f_t|) / wsum + gamma_8 |y|.  The silent stretch holds whole frames of exact
    zeros: their X is exactly 0 in both, the clamp gives cos = sin = 0 and their frames must be exact zeros."""
    name = "istft.fused_varlen"
    g = _rng(name)
    ns = ISTFT_NS
    off = offsets(ns)
    Ts = [1 + n // HOP for n in ns]
    B, T = len(ns), (max(Ts) + 63) // 64 * 64
    wav = (g.standard_normal(off[-1]) * 0.3).astype(np.float32)
    sil = slice(off[2] + 8000, off[2] + 14000)
    wav[sil] = 0.0
    mag = np.abs(g.standard_normal((B, T, 1025)) * 2).astype(np.float32)
    mag[g.random(mag.shape) < 0.1] = 0.0
    for b, Tb in enumerate(Ts):
        mag[b, Tb:] = np.nan                                     # frames past a clip: never read
    frames = np.full((B, T, 2048), SENT32, np.uint32)
    out = np.full(off[-1], SENT32, np.uint32)
    Case(ISTFT, B, off, w0=1024, T=T, n=max(ns), mag=mag, in_wav=wav, frames=frames, out=out).run(eng, name)
    ck = G.Checker(name)
    win = R.hann()
    c_fft = 4 * U * np.log2(2048)
    silent_frames = 0
    for b, (nb, Tb) in enumerate(zip(ns, Ts)):
        x = wav[off[b]:off[b + 1]]
        X, S = R.stft64(x, Tb)
        cs, sn = R.phase(X)
        mg = mag[b, :Tb].astype(np.float64)
        Y = mg * (cs + 1j * sn)
        f64 = R.inverse_frames(Y)
        E = istft_frame_error(mg, np.minimum(2.0, c_fft * S[:, None] / np.maximum(np.abs(X), 1e-4)))
        gf = frames[b, :Tb].view(np.float32).astype(np.float64)
        zero = (S == 0)[:, None]
        silent_frames += int(zero.sum())
        ck.values("frames", gf, f64, win[None] * E[:, None] + gamma(3) * np.abs(f64) + FLOOR, zero)
        assert (frames[b, Tb:] == SENT32).all(), (name, b, "frames past the clip written")
        y, ws, ab = R.overlap_add(f64, nb)
        EO = np.zeros((Tb - 1) * HOP + 2048)
        for t in range(Tb):
            EO[t * HOP:t * HOP + 2048] += win * E[t]
        EO = EO[1024:1024 + nb]
        bnd = (EO + gamma(8) * ab) / ws + gamma(8) * np.abs(y) + FLOOR
        ck.values("out", out[off[b]:off[b + 1]].view(np.float32).astype(np.float64), y, bnd, np.zeros(1, bool))
    assert silent_frames > 0
    report(name, ck)


# ------------------------------------------------------------------ PEAK_NORM: peak_varlen_kernel + scale_varlen_kernel
def test_peak_normalise_varlen_is_exact(eng):
    """Clip 0 is longer than 128 blocks x 2048 samples, so each thread strides over it; its peak sits near the end.  Peaks
    below 1 (left alone), exactly 1 (left alone: the test is `> 1`), above 1, and a negative sample as the peak."""
    g = _rng("peak_norm")
    ns = [300000, 5000, 4000, 6000]
    off = offsets(ns)
    wav = (g.uniform(-0.5, 0.5, off[-1])).astype(np.float32)
    wav[off[0] + 299000] = 3.0
    wav[off[1] + 17] = 0.7
    wav[off[2] + 3999] = -1.0
    wav[off[3] + 100] = -2.5
    wav[off[3] + 200] = 2.0
    before = wav.copy()
    peak = np.full(4, SENT32, np.uint32)
    Case(PEAK_NORM, 4, off, n=max(ns), wav=wav, peak_bits=peak).run(eng, "peak_norm")
    for b in range(4):
        seg = before[off[b]:off[b + 1]]
        pk = np.abs(seg).max()
        assert peak[b] == pk.view(np.uint32), b
        want = seg / pk if pk > np.float32(1) else seg
        assert np.array_equal(wav[off[b]:off[b + 1]].view(np.uint32), want.view(np.uint32)), b
    assert [np.abs(before[off[b]:off[b + 1]]).max() for b in range(4)] == [np.float32(v) for v in (3.0, 0.7, 1.0, 2.5)]
    WORST["peak_norm"] = 0.0


# ------------------------------------------------------------------ the lengths table, the range flag, coverage
def test_lengths_table_matches_the_host_formula(eng):
    """Every row of the table (kernels.cuh) for both UNets' bins, clips from one frame to a 60 s clip."""
    for w0 in (127, 1024):
        ns = [1025, 1323, 441 * 63, 441 * 64 + 5, 44100 * 60, 4410]
        off = offsets(ns)
        L = int(lengths_rows(off, w0)[9].max())                  # the conditioning's rows: the longest clip's Tv
        pl = planes16((len(ns), L + 6, 64), 0)
        Case(REFLECT, len(ns), off, w0=w0, L=L, C=64, cond_pad=1, planes=pl).run(eng, f"lengths.w0_{w0}")


def test_fp16_range_flag_is_reported_and_the_next_case_passes(eng):
    from voicefixer_main_b200._lib import EngineError
    for nm, mk in (("first.mel_T64_pos_shift", lambda: first_case("first.overflow", FIRST_CASES["first.mel_T64_pos_shift"], 1e5)),
                   ("pool.mel_l0", lambda: pool_case("pool.overflow", POOL_CASES["pool.mel_l0"], 1e6))):
        c = mk()[0]
        eng.selftest_op(c.oc)
        with pytest.raises(EngineError) as ei:
            eng.check_errors()
        assert ei.value.code == VL.VF_EDEVICE
    args = first_case("first.mel_T64_pos_shift", FIRST_CASES["first.mel_T64_pos_shift"])
    args[0].run(eng, "first.after_flag")
    check_first("first.after_flag", *args)
    args = pool_case("pool.mel_l0", POOL_CASES["pool.mel_l0"])
    args[0].run(eng, "pool.after_flag")
    check_pool("pool.after_flag", *args)


def test_cases_cover_every_kind_both_tails_and_every_varlen_table(eng):
    want = {(k, 0, v) for k in (FIRST, POOL, COND, REFLECT) for v in (False, True)}
    want |= {(TAIL, t, v) for t in (1, 3) for v in (False, True)}
    want |= {(FINALIZE, 0, False), (FINALIZE, 0, True), (ISTFT, 0, True), (PEAK_NORM, 0, True)}
    if not want <= COVER:            # run on its own: run every case once
        for name in FIRST_CASES:
            test_first_layer_matches_float64(eng, name)
        for name in POOL_CASES:
            test_pool_matches_float64(eng, name)
        for name in COND_CASES:
            test_conditioning_matches_float64(eng, name)
        for name in REFLECT_CASES:
            test_reflect_fill_is_exact(eng, name)
        for name in TAIL_CASES:
            for terms in (1, 3):
                test_tail_matches_float64(eng, name, terms, 1)
        test_finalize_uniform_is_exact(eng)
        test_finalize_varlen_is_exact(eng)
        test_fused_istft_varlen_matches_float64(eng)
        test_peak_normalise_varlen_is_exact(eng)
    assert want <= COVER, sorted(want - COVER)
    for k, v in sorted(WORST.items()):
        print(f"worst {k}: {v:.3e}")
