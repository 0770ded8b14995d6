"""Every launch of the restore plans, replayed against float64 on the plans' own weights and activations.

vf_selftest_plan_trace runs one restore on a fresh plan one launch at a time and describes each launch as the builder set it
up.  Around every launch this file
  1. snapshots every buffer of the plan, and afterwards checks that no byte outside the launch's declared outputs changed
     (inside a GEMM's or a pair's outputs, no element outside its write set either);
  2. checks every output value against the float64 reference of the same op, computed from the launch's own inputs as they
     were just before it ran, with the weights the test maps from the launch's label to the state dict.  Each op starts from
     the engine's inputs, so errors do not carry from op to op and every op is held to the bound the layer suite
     (test_gpu_layers.py) or the non-GEMM suite (test_gpu_aux.py) derives for it, at every element;
  3. checks each GEMM's and pair's wiring: every operand, shortcut operand and residual was last written by the launch the
     network's dataflow names (expected_producers), and in a varlen plan its row_valid is the lengths-table row of its
     geometry, computed from the clip lengths;
  4. in a varlen plan, checks that the rows past each clip of every GEMM and pair input are zeros (of either sign), the
     precondition of the layer suite's varlen cases (rows past a clip in each output are checked as exact zeros by step 2).
Then the traced output must equal the product call's bit for bit (eager and graph replay), and every op kind and every
GEMM / pair configuration of the plan must have been replayed.

Inputs: seeded synthetic speech and one clip that widens the activations' range (digital silence, a full-scale click and
a DC offset).  The UNet launches are the same for every vocoder mode, so the GSR plans pair the vocoder's 1- and 3-term
modes with unify_energy off and on once each, uniform and varlen."""
import ctypes
import time
import types

import numpy as np
import pytest
import torch

import test_gpu_aux as A
import test_gpu_layers as G
from oracle import layers as R
from oracle import vf_oracle as O
from voicefixer_main_b200 import _lib as VL
from voicefixer_main_b200.arch import SSR_PREFIX, UNET_PREFIX

pytestmark = pytest.mark.gpu

GEMM, FIRST, POOL, COND, REFLECT, TAIL, FINALIZE, MEMSET, PAIR = range(9)       # VF_TRACE_* (include/b200vf.h)
KIND_NAMES = ["gemm", "first", "pool", "cond", "reflect", "tail", "finalize", "memset", "pair"]
SR, HOP = 44100, 441
# 1 s, 0.5 s and the shortest clip a restore takes: a varlen bucket of 128 frames pads two of its three clips
N_LONG, N_MID, N_MIN = SR, SR // 2, 1025
CLAMP = np.float32(np.log10(np.float32(1e-8)))     # the front end's log10(max(mel, 1e-8))
PLANS = {                                          # name -> (plan kind, vocoder terms, unify_energy)
    "gsr.voc1": (0, 1, False),
    "gsr.voc3.unify": (0, 3, True),
    "gsr_varlen.voc1.unify": (2, 1, True),
    "gsr_varlen.voc3": (2, 3, False),
    "ssr": (1, 3, False),
    "ssr_varlen": (3, 3, False),
}
RESULTS = {}          # plan -> (kinds replayed, signatures replayed)


# ------------------------------------------------------------------ inputs
def wide_clip(n, seed):
    """Speech with a stretch of digital silence, one full-scale click and a DC offset."""
    x = O.synth_clips(1, n, seed=seed)[0].double()
    x[n // 4:n // 2] = 0.0
    x[n // 3] = 1.0
    x[n // 2:] += 0.25
    return x.clamp(-1, 1).float()


def inputs(kind):
    """(wav on the device, lengths or None)."""
    if kind in (0, 1):
        wav = torch.stack([O.synth_clips(1, N_LONG, seed=11)[0].float(), wide_clip(N_LONG, 12)])
        return wav.cuda(), None
    clips = [O.synth_clips(1, N_MIN, seed=13)[0].float(), wide_clip(N_MID, 14), O.synth_clips(1, N_LONG, seed=15)[0].float()]
    return torch.cat(clips).cuda(), [len(c) for c in clips]


# ------------------------------------------------------------------ device buffers
class _Dev:
    """A device byte range as a torch view (no copy)."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False), "strides": None,
                                        "version": 2}


def dev(ptr, nbytes):
    return torch.as_tensor(_Dev(ptr, nbytes), device="cuda")


def host(ptr, dtype, shape):
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    return dev(ptr, n).cpu().numpy().view(dtype).reshape(shape)


def planes(ptr, n, rows, C):
    return host(ptr, np.uint16, (2, n, rows, C))


def rows_of(p, n):
    return None if not p else np.ctypeslib.as_array(ctypes.cast(p, ctypes.POINTER(ctypes.c_int)), (n,)).copy()


def vl_table(t, B):
    return None if not t.vl_rows else np.ctypeslib.as_array(ctypes.cast(t.vl_rows, ctypes.POINTER(ctypes.c_int)), (18, B)).copy()


# ------------------------------------------------------------------ the state dict behind each label
def bn32(sd, key, sl=slice(None)):
    """fold_bn (pack.cu): scale = fp32(w / sqrt(v + eps)), shift = fp32(b - m * scale64)."""
    w, b, m, v = (sd[f"{key}.{k}"].double()[sl] for k in ("weight", "bias", "running_mean", "running_var"))
    s = w / torch.sqrt(v + 1e-5)
    return s.float().numpy(), (b - m * s).float().numpy()


def unet_spec(label, sd, pre, C):
    """What plan.cu's build_unet gives the GEMM `label` (without its "ssr." tag): its weights, the affine of its activated
    output (the consumer's BatchNorm) and the activation slope.  C: the op's output channels."""
    P = lambda k: sd[pre + k]
    parts = label.split(".")
    blk = None
    if parts[0] == "bottleneck":
        blk, nxt, slope = "conv_block7", ("decoder_block1.bn1", slice(None)), 0.0
    elif parts[0] == "post":
        blk, nxt, slope = "after_conv_block1", None, None
    elif parts[1] == "convT":
        k = int(parts[0][3:])
        return dict(w=P(f"decoder_block{k}.conv1.weight"), bn=bn32(sd, pre + f"decoder_block{k}.conv_block2.bn1", slice(0, C)),
                    slope=G.UNET_SLOPE)
    else:
        lvl, j = int(parts[0][3:]), int(parts[1][1:])
        if parts[0].startswith("enc"):
            blk = f"encoder_block{lvl}.conv_block{j}"
            nxt = ((f"encoder_block{lvl}.conv_block{j + 1}.bn1", slice(None)) if j < 4 else
                   (f"decoder_block{7 - lvl}.conv_block2.bn1", slice(C, 2 * C)))
            slope = G.UNET_SLOPE
        else:
            blk = f"decoder_block{lvl}.conv_block{j}"
            nxt, slope = (f"decoder_block{lvl}.conv_block{j + 1}.bn1", slice(None)), G.UNET_SLOPE
            if j == 5:
                nxt, slope = ((f"decoder_block{lvl + 1}.bn1", slice(None)), 0.0) if lvl < 6 else (("after_conv_block1.bn1", slice(None)), G.UNET_SLOPE)
    if parts[-1] == "conv1":
        return dict(w=P(blk + ".conv1.weight"), bn=bn32(sd, pre + blk + ".bn2"), slope=G.UNET_SLOPE)
    spec = dict(w=P(blk + ".conv2.weight"))
    if parts[-1] == "conv2+sc":
        spec.update(sc_w=P(blk + ".shortcut.weight")[:, :, 0, 0], sc_b=P(blk + ".shortcut.bias"))
    if nxt is None:
        spec.update(head_w=P("after_conv2.weight").reshape(-1), head_b=float(P("after_conv2.bias")[0]))
    else:
        spec.update(bn=bn32(sd, pre + nxt[0], nxt[1]), slope=slope)
    return spec


def voc_spec(label, sd, cfg):
    P = lambda k: sd["vocoder." + k]
    parts = label.split(".")
    if parts[1].startswith("cond"):
        i = int(parts[1][4:])
        return dict(w=P(f"condnet.{i}.weight"), b=P(f"condnet.{i}.bias"), act=2)
    if parts[1] == "stem":
        return dict(w=P("stem.weight"), b=P("stem.bias"), act=1, slope=cfg.voc_stage_slope)
    if parts[1].startswith("up"):
        s = int(parts[1][2:])
        return dict(w=P(f"up.{s}.weight"), b=P(f"up.{s}.bias"), act=1, slope=cfg.voc_res_slope, stride=cfg.voc_scales[s])
    s, i = int(parts[1][3:]), int(parts[2])
    last = i == cfg.voc_depth[s] - 1
    dil = 3 ** (i % 10)
    key = f"res.{s}.{i}"
    if parts[3] == "pair":
        return dict(w=P(key + ".a.weight"), b=P(key + ".a.bias"), w2=P(key + ".b.weight"), b2=P(key + ".b.bias"), dilation=dil,
                    last=last)
    ab = parts[3]
    return dict(w=P(f"{key}.{ab}.weight"), b=P(f"{key}.{ab}.bias"), act=1, dilation=dil if ab == "a" else 1,
                slope=cfg.voc_stage_slope if (ab == "b" and last) else cfg.voc_res_slope)


def spec_of(label, sd, cfg, C):
    if label.startswith("voc."):
        return voc_spec(label, sd, cfg)
    if label.startswith("ssr."):
        return unet_spec(label[4:], sd, SSR_PREFIX, C)
    return unet_spec(label, sd, UNET_PREFIX, C)


# ------------------------------------------------------------------ one op: capture, reference, check
class Replay:
    """The checks of one traced plan; on_op is vf_selftest_plan_trace's callback."""

    def __init__(self, name, sd, cfg, varlen):
        self.name, self.sd, self.cfg, self.varlen = name, sd, cfg, varlen
        self.views = None
        self.snap = None
        self.cap = {}
        self.ops = 0
        self.kinds, self.sigs = set(), set()
        self.worst, self.worst_op = 0.0, ""
        self.per_kind = {}
        self.t_ref = self.t_snap = 0.0
        self.arena = 0
        self.clamped = []
        self.writers = []         # (first byte, end, label) of every launch's outputs so far, in launch order
        self.lengths = None

    # ---- containment
    def on_op(self, after, t):
        t0 = time.perf_counter()
        if self.views is None:
            allocs = [(t.alloc_ptr[i], t.alloc_bytes[i]) for i in range(t.n_allocs)]
            self.arena = sum(n for _, n in allocs)
            self.views = [(p, n, dev(p, n)) for p, n in allocs]
        label = t.label.decode()
        if not after:
            torch.cuda.synchronize()
            self.snap = [v.clone() for _, _, v in self.views]
            torch.cuda.synchronize()
            self.t_snap += time.perf_counter() - t0
            self.cap = self.capture(t, label)
            return
        torch.cuda.synchronize()
        outs = [(t.out_ptr[i], t.out_bytes[i]) for i in range(t.n_out)]
        for i, ((p, n, v), s) in enumerate(zip(self.views, self.snap)):
            moved = (v != s).nonzero().flatten()
            if moved.numel() == 0:
                continue
            inside = torch.zeros_like(moved, dtype=torch.bool)
            for (q, m) in outs:
                inside |= (moved >= q - p) & (moved < q - p + m)
            assert bool(inside.all()), (self.name, label, f"buffer {i} ({n} bytes) changed at byte {int(moved[~inside][0])}, "
                                                          "outside the launch's outputs")
        self.snap = None
        self.t_snap += time.perf_counter() - t0
        t1 = time.perf_counter()
        ck = G.Checker(f"{self.name}:{label}")
        CHECKS[t.kind](self, t, label, ck)
        self.t_ref += time.perf_counter() - t1
        self.writers += [(t.out_ptr[i], t.out_ptr[i] + t.out_bytes[i], label) for i in range(t.n_out)]
        self.ops += 1
        self.kinds.add(t.kind)
        if t.kind in (GEMM, PAIR):
            self.sigs.add(t.layer.sig.decode())
        k = KIND_NAMES[t.kind]
        self.per_kind[k] = max(self.per_kind.get(k, 0.0), ck.worst)
        if ck.worst >= self.worst:
            self.worst, self.worst_op = ck.worst, label

    # ---- inputs (and the outputs as they were) before the launch
    def capture(self, t, label):
        cap = {}
        if t.kind in (GEMM, PAIR):
            lc = t.layer
            n = lc.n_img
            cap["x"] = planes(lc.x, n, lc.x_img_rows, lc.cin)
            if lc.sc_x:
                cap["sc_x"] = planes(lc.sc_x, n, lc.H * (lc.W + 1), lc.sc_cin)
            rows_in = lc.H * (lc.W + 1) if lc.kind == G.CONV2D else lc.L
            if lc.resid_kind == 1:
                cap["resid"] = host(lc.resid, np.float32, (n, rows_in, lc.cout))
            elif lc.resid_kind in (2, 3):
                cap["resid"] = planes(lc.resid, n, rows_in, lc.cout)
            if lc.head_in:
                cap["head_in"] = host(lc.head_in, np.float32, (n, lc.head_T, lc.W + 1))
            cap["before"] = self.outputs(t)
            self.check_wiring(t, label)
            if self.varlen and lc.row_valid:
                self.check_zero_input(t, label, cap)
        elif t.kind == FIRST:
            o = t.op
            cap["x"] = host(o.x, np.float32, (o.batch, o.T, o.W + 1))
        elif t.kind == POOL:
            o = t.op
            cap["x"] = host(o.pin, np.float32, (o.batch, o.H, o.W + 1, o.C))
        elif t.kind == COND:
            o = t.op
            cap["mel"] = host(o.mel, np.float32, (o.batch, o.T, 128))
            if o.unify:
                cap["tgt"] = host(o.mel_target, np.float32, (o.batch, o.T, 128))
        elif t.kind == REFLECT:
            cap["before"] = planes(t.op.planes, t.op.batch, t.op.L + 6, t.op.C)
        elif t.kind == TAIL:
            o = t.op
            cap["bits"] = planes(o.tail_in, o.batch, o.L + 6, o.C)
            cap["wav"] = host(o.wav, np.uint32, (o.batch, o.L))
        elif t.kind == FINALIZE:
            o = t.op
            cap["wav"] = host(o.in_wav, np.float32, (o.batch, o.L))
            cap["peak"] = host(o.peak_bits, np.uint32, (o.batch,))
        return cap

    def outputs(self, t):
        """The GEMM's / pair's output buffers, keyed as test_gpu_layers' b.buf."""
        lc = t.layer
        n, rows = lc.n_img, lc.out_img_rows
        out = {}
        if lc.out_raw:
            out["raw"] = host(lc.out_raw, np.uint32, (n, rows, lc.raw_ld))
        if lc.out_r:
            out["r"] = planes(lc.out_r, n, rows, lc.r_ld)
        if lc.out_a:
            out["a"] = planes(lc.out_a, n, rows, lc.a_ld)
        if lc.head_w:
            out["head"] = host(lc.head_out, np.uint32, (n, lc.head_T, lc.W + 1))
        return out

    def producer(self, ptr):
        """The label of the last launch whose outputs hold device address ptr ("input": none, the front end's)."""
        for lo, hi, label in reversed(self.writers):
            if lo <= ptr < hi:
                return label
        return "input"

    def check_wiring(self, t, label):
        """Each operand, shortcut operand and residual of a GEMM or pair was last written by the launch the network says
        produces it (expected_producers), and in a varlen plan its row_valid / head_valid are the lengths-table rows of its
        geometry, computed here from the clip lengths."""
        lc = t.layer
        want = expected_producers(label, self.cfg)
        got = {"x": self.producer(lc.x)}
        if lc.sc_x:
            got["sc_x"] = self.producer(lc.sc_x)
        if lc.resid_kind:
            got["resid"] = self.producer(lc.resid)
        assert got == want, (self.name, label, "reads", got, "expected", want)
        if not self.varlen:
            assert not lc.row_valid and not lc.head_valid, (self.name, label)
            return
        off = np.concatenate([[0], np.cumsum(self.lengths)])
        table = A.lengths_rows(off, 1024 if self.name.startswith("ssr") else 127)
        if label.startswith("voc.cond") or label == "voc.stem":
            row = 9
        elif label.startswith("voc."):
            row = 10 + int(label.split(".")[1][-1])
        else:
            Tp = int(table[1].max())
            row = 2 + [Tp >> l for l in range(7)].index(lc.H)
        assert np.array_equal(rows_of(lc.row_valid, lc.n_img), table[row]), (self.name, label, "row_valid is not lengths row", row)
        if lc.head_w:
            assert np.array_equal(rows_of(lc.head_valid, lc.n_img), table[0]), (self.name, label, "head_valid")

    def check_zero_input(self, t, label, cap):
        """The layer suite's varlen precondition (test_gpu_layers.build): the operand and the residual are zeros past each
        clip's rows (CONVT1D: past its input rows).  The stem's input rows past a clip hold the reflection padding and rows
        no launch writes; it reads rows t .. t + 6 of valid output rows t only, and is not held to it."""
        lc = t.layer
        if lc.kind == G.CONV1D and not lc.centered:
            return
        rv = rows_of(lc.row_valid, lc.n_img)
        lim = rv if lc.kind != G.CONVT1D else (rv + lc.stride - 1) // lc.stride
        for i in range(lc.n_img):
            x = R.from_bits(cap["x"][:, i, lc.x_row0 + lim[i]:])         # zeros of either sign
            assert not x.any(), (self.name, label, "operand rows past clip", i, "are not zero")
            if "resid" in cap:
                r = cap["resid"][i, rv[i]:] if cap["resid"].ndim == 3 else R.from_bits(cap["resid"][:, i, rv[i]:])
                assert not r.any(), (self.name, label, "residual rows past clip", i, "are not zero")


def expected_producers(label, cfg):
    """{input: label of the launch that must have written it last} for the GEMM or pair `label` (plan.cu's dataflow: each
    block's conv1 reads the previous block's activated output, conv2 reads its conv1, the residual stream runs from block
    to block; the non-GEMM producers carry their kind's name)."""
    if label.startswith("voc."):
        p = label.split(".")
        if p[1].startswith("cond"):
            i = int(p[1][4:])
            return {"x": "voc_condition" if i == 0 else f"voc.cond{i - 1}"}
        if p[1] == "stem":
            return {"x": "reflect_fill"}
        last = lambda s: (f"voc.res{s}.{cfg.voc_depth[s] - 1}." + ("pair" if PAIR_STAGE.get(s) else "b"))
        if p[1].startswith("up"):
            s = int(p[1][2:])
            return {"x": "voc.stem" if s == 0 else last(s - 1)}
        s, i = int(p[1][3:]), int(p[2])
        stream = f"voc.up{s}" if i == 0 else f"voc.res{s}.{i - 1}.{p[3] if p[3] == 'pair' else 'b'}"
        if p[3] == "pair":
            return {"x": stream}
        if p[3] == "a":
            return {"x": stream}
        return {"x": f"voc.res{s}.{i}.a", "resid": stream}
    tag = "ssr." if label.startswith("ssr.") else ""
    p = label[len(tag):].split(".")
    T = lambda x: tag + x
    if p[0] == "post":
        return {"x": T("dec6.b5.conv2")} if p[1] == "conv1" else {"x": T("post.conv1"), "resid": T("dec6.b5.conv2")}
    if p[0] == "bottleneck":
        return {"x": "pool"} if p[1] == "conv1" else {"x": T("bottleneck.conv1"), "resid": "pool"}
    if p[1] == "convT":
        k = int(p[0][3:])
        return {"x": T("bottleneck.conv2") if k == 1 else T(f"dec{k - 1}.b5.conv2")}
    lvl, j = int(p[0][3:]), int(p[1][1:])
    enc = p[0].startswith("enc")
    first_j = 1 if enc else 2
    prev = lambda jj: T(f"{p[0]}.b{jj}.conv2" + ("+sc" if (enc and jj == 1 and lvl not in (1, 6)) or (not enc and jj == 2) else ""))
    if p[2] == "conv1":
        if j == first_j:
            return {"x": "pool" if enc else T(f"dec{lvl}.convT")}
        return {"x": prev(j - 1)}
    want = {"x": "unet_first" if (enc and lvl == 1 and j == 1) else T(f"{p[0]}.b{j}.conv1")}
    if p[2] == "conv2+sc":
        want["sc_x"] = "pool" if enc else T(f"dec{lvl}.convT")
    elif j == first_j:
        want["resid"] = "unet_first" if lvl == 1 else "pool"
    else:
        want["resid"] = prev(j - 1)
    return want


PAIR_STAGE = {}       # vocoder stages run as fused pairs in the plan being replayed (set per plan)


def _w(x, terms, device="cuda"):
    """fp32 weights as the kernel contracts them: hi + lo (3-term) or hi."""
    h, l = R.split_hi_lo(torch.as_tensor(x).float())
    return (h + l if terms == 3 else h).to(device)


def check_gemm(rp, t, label, ck):
    lc = t.layer
    n, terms, kind = lc.n_img, lc.terms, lc.kind
    sp = spec_of(label, rp.sd, rp.cfg, lc.cout)
    c = dict(name=label, kind=kind, terms=terms, n_img=n, H=lc.H, W=lc.W, L=lc.L, k=lc.k, dilation=lc.dilation,
             centered=lc.centered, stride=lc.stride, both=lc.both, sc_cin=lc.sc_cin)
    b = G.Built()
    b.c, b.n, b.terms, b.lc = c, n, terms, lc
    b.rv = rows_of(lc.row_valid, n)
    b.out_row0, b.out_img_rows = lc.out_row0, lc.out_img_rows
    b.rows = lc.x_img_rows - lc.x_row0
    x = rp.cap["x"][:, :, lc.x_row0:]
    b.x = torch.from_numpy(R.from_bits(x[0]) + (R.from_bits(x[1]) if terms == 3 else 0)).cuda()
    b.w = _w(sp["w"], terms)
    if "dilation" in sp:
        assert lc.dilation == sp["dilation"], (label, "dilation", lc.dilation)
    if "stride" in sp:
        assert lc.stride == sp["stride"], (label, "stride", lc.stride)
    if "b" in sp:
        b.b = torch.as_tensor(sp["b"]).double().cuda()
    if lc.sc_cin:
        b.sc_w, b.sc_b = _w(sp["sc_w"], terms), torch.as_tensor(sp["sc_b"]).double().cuda()
        s = rp.cap["sc_x"]
        b.sc_x = torch.from_numpy(R.from_bits(s[0]) + (R.from_bits(s[1]) if terms == 3 else 0)).cuda()
    b.resid = None
    if lc.resid_kind == 1:
        b.resid = torch.from_numpy(rp.cap["resid"].astype(np.float64)).cuda()
    elif lc.resid_kind == 2:
        b.resid = torch.from_numpy(A.hi_lo(rp.cap["resid"])).cuda()
    elif lc.resid_kind == 3:
        assert lc.ar_slope == np.float32(G.RES_SLOPE)
        r = rp.cap["resid"]
        b.resid = torch.from_numpy(R.ar_decode(r[0].view(np.float16), r[1].view(np.float16), G.RES_SLOPE)).cuda()
    # the outputs, as the layer suite keys them
    b.buf = rp.outputs(t)
    before = dict(rp.cap["before"])
    if lc.out_r and lc.out_a:
        assert lc.r_c_off == lc.a_c_off, (label, "r and a halves at different channel offsets")
    b.c_off = lc.a_c_off if lc.out_a else lc.r_c_off
    if lc.out_a:
        if lc.out_ar:
            assert lc.ar_slope == np.float32(G.RES_SLOPE) and sp["slope"] == np.float32(G.RES_SLOPE), label
        else:
            assert (lc.act, lc.slope) == (sp.get("act", 1), np.float32(sp["slope"] if "slope" in sp else 0)), (label, lc.act, lc.slope)
        if "bn" in sp:
            c["affine"] = True
            b.scale, b.shift = sp["bn"]
            assert lc.a_scale and lc.a_shift, (label, "no affine")
        else:
            assert not lc.a_scale, (label, "an affine the network does not have")
    if lc.head_w:
        c.update(head=True, head_T=lc.head_T)
        b.head_w = sp["head_w"].float().numpy()
        b.head_b = sp["head_b"]
        assert lc.head_b == np.float32(b.head_b), label
        b.head_in = rp.cap.get("head_in")
        b.head_out = b.buf.pop("head")
        b.head_valid = rows_of(lc.head_valid, n)
    y = G.reference(b).cpu()
    M = G.reference(b, abs_=True).cpu()
    G.check_outputs(b, ck, y, M, before)


def check_pair(rp, t, label, ck):
    lc = t.layer
    sp = spec_of(label, rp.sd, rp.cfg, lc.cout)
    assert (lc.dilation, bool(lc.pair_last)) == (sp["dilation"], sp["last"]), (label, lc.dilation, lc.pair_last)
    assert lc.pair_slope_h == np.float32(G.RES_SLOPE) and lc.ar_slope == np.float32(G.RES_SLOPE), label
    assert lc.pair_slope_out == np.float32(G.STAGE_SLOPE if sp["last"] else G.RES_SLOPE), label
    b = G.Built()
    b.c = dict(name=label, kind=G.PAIR, L=lc.L, dilation=lc.dilation, last=sp["last"])
    b.n, b.terms, b.lc = lc.n_img, 1, lc
    b.rv = rows_of(lc.row_valid, lc.n_img)
    b.out_row0, b.out_img_rows = lc.out_row0, lc.out_img_rows
    x = rp.cap["x"]
    b.x_act = torch.from_numpy(R.from_bits(x[0, :, :lc.L])).cuda()
    b.x_stream = torch.from_numpy(R.ar_decode(x[0, :, :lc.L].view(np.float16), x[1, :, :lc.L].view(np.float16), G.RES_SLOPE)).cuda()
    b.wa, b.wb = _w(sp["w"], 1), _w(sp["w2"], 1)
    b.ba, b.bb = torch.as_tensor(sp["b"]).double().cuda(), torch.as_tensor(sp["b2"]).double().cuda()
    b.buf = rp.outputs(t)
    G.check_pair(b, ck, rp.cap["before"])


def check_first(rp, t, label, ck):
    o = t.op
    pre = SSR_PREFIX if o.W == 1024 else UNET_PREFIX
    blk = pre + "encoder_block1.conv_block1"
    s1, t1 = bn32(rp.sd, blk + ".bn1")
    s2, t2 = bn32(rp.sd, blk + ".bn2")
    p = dict(bn1_scale=np.float32(s1[0]), bn1_shift=np.float32(t1[0]), w1=rp.sd[blk + ".conv1.weight"].reshape(32, 9).numpy(),
             bn2_scale=s2, bn2_shift=t2, w_sc=rp.sd[blk + ".shortcut.weight"].reshape(32).numpy(),
             b_sc=rp.sd[blk + ".shortcut.bias"].numpy())
    assert (o.bn1_scale, o.bn1_shift) == (p["bn1_scale"], p["bn1_shift"]), label
    B, T = o.batch, o.T
    vl = vl_table(t, B)
    Ts = [T] * B if vl is None else list(vl[0])
    x = rp.cap["x"]
    if o.W == 127:
        rp.clamped = [int((x[i, :Ts[i], :128] <= CLAMP).sum()) for i in range(B)]
    rows = o.Tp * (o.W + 1)
    a2 = planes(o.a2, B, rows, 32)
    sc = host(o.sc_raw, np.uint32, (B, rows, 32))
    ck.worst = max(ck.worst, A.check_first(ck.name, types.SimpleNamespace(oc=o), x, p, Ts, T, a2, sc).worst)


def check_pool(rp, t, label, ck):
    o = t.op
    pre = SSR_PREFIX if rp.name.startswith("ssr") else UNET_PREFIX
    nxt = pre + (f"encoder_block{o.level + 2}.conv_block1.bn1" if o.level < 5 else "conv_block7.bn1")
    sc, sh = bn32(rp.sd, nxt)
    B, rows = o.batch, (o.H // 2) * o.Wpo
    out_r, out_a = planes(o.out_r, B, rows, o.C), planes(o.out_a, B, rows, o.C)
    out_raw = host(o.out_raw, np.uint32, (B, rows, o.C)) if o.out_raw else None
    vl = vl_table(t, B)
    rv = None if vl is None else vl[2 + o.level + 1]
    res = A.check_pool(ck.name, types.SimpleNamespace(oc=o), rp.cap["x"], sc, sh, out_r, out_a, out_raw, rv)
    ck.worst = max(ck.worst, res.worst)


def check_cond(rp, t, label, ck):
    o = t.op
    B = o.batch
    vl = vl_table(t, B)
    Ts = [o.T] * B if vl is None else list(vl[0])
    sums = host(o.band_sums, np.uint32, (B, 2)) if o.unify else None
    out = planes(o.cond, B, o.Tv, 128)
    c = types.SimpleNamespace(oc=o, off=None if vl is None else True)
    ck.worst = max(ck.worst, A.check_cond(ck.name, c, rp.cap["mel"], rp.cap.get("tgt"), sums, out, Ts, o.T).worst)


def check_reflect(rp, t, label, ck):
    o = t.op
    vl = vl_table(t, o.batch)
    Ls = [o.L] * o.batch if vl is None else list(vl[9 if o.cond_pad else 10 + rp.cfg.voc_num_stages - 1])
    A.check_reflect(ck.name, rp.cap["before"], planes(o.planes, o.batch, o.L + 6, o.C), Ls)


def check_memset(rp, t, label, ck):
    assert not bool(dev(t.op.planes, t.op.n).any()), (ck.name, "not cleared")


def check_tail(rp, t, label, ck):
    o = t.op
    B = o.batch
    vl = vl_table(t, B)
    Ls = [o.L] * B if vl is None else list(vl[10 + rp.cfg.voc_num_stages - 1])
    w = rp.sd["vocoder.tail.weight"].numpy()
    bias = np.float32(rp.sd["vocoder.tail.bias"][0])
    assert o.tail_b == bias, label
    wav, peak = host(o.wav, np.uint32, (B, o.L)), host(o.peak_bits, np.uint32, (B,))
    res = A.check_tail(ck.name, types.SimpleNamespace(oc=o), rp.cap["bits"], w, bias, wav, peak, Ls, o.terms, o.tanh_out,
                       rp.cap["wav"])
    ck.worst = max(ck.worst, res.worst)


def check_finalize(rp, t, label, ck):
    """Bit-exact: R.finalize of each clip's vocoder output with its peak."""
    o = t.op
    B = o.batch
    vl = vl_table(t, B)
    wav, peak = rp.cap["wav"], rp.cap["peak"].view(np.float32)
    if vl is None:
        out = host(o.out, np.uint32, (B, o.n))
        for i in range(B):
            assert np.array_equal(out[i], R.finalize(wav[i], peak[i], o.skip, o.n).view(np.uint32)), (ck.name, i)
        return
    ns = rp.lengths
    off = np.concatenate([[0], np.cumsum(ns)])
    out = host(o.out, np.uint32, (int(off[-1]),))
    for i, (nb, Lb) in enumerate(zip(ns, vl[10 + rp.cfg.voc_num_stages - 1])):
        want = R.finalize(wav[i], peak[i], (int(Lb) - nb) // 2, nb).view(np.uint32)
        assert np.array_equal(out[off[i]:off[i + 1]], want), (ck.name, i)


CHECKS = {GEMM: check_gemm, PAIR: check_pair, FIRST: check_first, POOL: check_pool, COND: check_cond, REFLECT: check_reflect,
          MEMSET: check_memset, TAIL: check_tail, FINALIZE: check_finalize}


# ------------------------------------------------------------------ tests
@pytest.fixture(scope="module")
def setup():
    from voicefixer_main_b200.model import Engine
    from voicefixer_main_b200.weights import make_ssr_state, make_state
    sd = {**make_state(1234), **make_ssr_state(1234)}
    e = Engine("cuda:0")
    e.load_state(sd, need=("unet", "vocoder", "ssr"))
    cfg = VL.VfConfig()
    VL.load_library().vf_default_config(ctypes.byref(cfg))
    yield e, sd, cfg
    e.check_errors()
    e.close()


def product(e, kind, wav, lengths, unify):
    if kind == 0:
        return e.restore(wav, unify_energy=unify)
    if kind == 1:
        return e.ssr_forward(None, wav)
    if kind == 2:
        return e.restore_varlen(wav, lengths, unify_energy=unify)
    return e.ssr_restore_varlen(wav, lengths)


def replay(setup, name):
    e, sd, cfg = setup
    kind, terms, unify = PLANS[name]
    e.set_option("vocoder_terms", terms)
    wav, lengths = inputs(kind)
    rp = Replay(name, sd, cfg, lengths is not None)
    rp.lengths = lengths
    PAIR_STAGE.clear()
    if terms == 1:
        PAIR_STAGE[cfg.voc_num_stages - 1] = True          # the C = 64 stack of the (a, r) stream (plan.cu: fused)
    t0 = time.perf_counter()
    got = e.selftest_plan_trace(kind, wav, lengths, rp.on_op, unify_energy=unify)
    wall = time.perf_counter() - t0
    e.check_errors()
    # the product call on the same input, eager then from its graph, equals the traced run bit for bit
    for _ in range(2):
        want = product(e, kind, wav, lengths, unify)
        torch.cuda.synchronize()
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (name, "traced output differs from the product call")
    # every GEMM / pair configuration of the plan was replayed
    n = len(lengths) if lengths else wav.shape[0]
    T = (1 + max(lengths) // HOP + 63) // 64 * 64 if lengths else 1 + wav.shape[1] // HOP
    sigs = {sg for _, sg in e.selftest_plan_gemms(kind, n, T)}
    assert sigs == rp.sigs, (name, "configurations not replayed", sigs - rp.sigs)
    assert rp.kinds == ({GEMM, FIRST, POOL} if kind in (1, 3) else {GEMM, FIRST, POOL, COND, REFLECT, MEMSET, TAIL, FINALIZE, PAIR}
                        if terms == 1 else {GEMM, FIRST, POOL, COND, REFLECT, MEMSET, TAIL, FINALIZE}), (name, rp.kinds)
    RESULTS[name] = (rp.kinds, rp.sigs)
    print(f"{name}: {rp.ops} ops, worst err / bound {rp.worst:.3e} at {rp.worst_op}; arena {rp.arena / 2 ** 20:.1f} MiB; "
          f"snapshots + containment {rp.t_snap:.1f} s, float64 references + checks {rp.t_ref:.1f} s, wall {wall:.1f} s")
    print(f"    worst err / bound per kind: " + ", ".join(f"{k} {v:.3e}" for k, v in sorted(rp.per_kind.items())))
    if rp.clamped:
        print(f"    log-mel values at the to_log clamp per clip: {rp.clamped}")


@pytest.mark.parametrize("name", list(PLANS))
def test_plan_replays_against_float64(setup, name):
    replay(setup, name)


def test_replays_cover_every_op_kind(setup):
    """Every op kind the plans launch and both (a, r) and hi / lo vocoder stacks were replayed."""
    for name in PLANS:
        if name not in RESULTS:
            replay(setup, name)
    kinds = set().union(*(k for k, _ in RESULTS.values()))
    assert kinds == set(CHECKS), kinds
    sigs = set().union(*(s for _, s in RESULTS.values()))
    assert any("resid=ar" in s for s in sigs) and any("resid=planes" in s for s in sigs)
    assert any("varlen=1" in s for s in sigs) and any(s.startswith("pair") for s in sigs)
