"""Every launch of the restore plans, replayed against float64 on the plans' own weights and activations.

vf_selftest_plan_trace runs one restore on a fresh plan one step at a time and describes each step as the builder or the
restore path set it up: every launch of the analysis module's and the vocoder's lists, the finalize, and the launches the
restore makes itself (the front end, unify_energy's band sums, the SSR ISTFT).  Around every step this file
  1. snapshots every buffer of the plan, and afterwards checks that no byte outside the step's declared outputs changed
     (inside a GEMM's or a pair's outputs, no element outside its write set either);
  2. checks every output value against the float64 reference of the same op, computed from the step's own inputs as they
     were just before it ran, with the weights the test maps from the step's label to the state dict.  Each op starts from
     the engine's inputs, so errors do not carry from op to op and every op is held to the bound the layer suite
     (test_gpu_layers.py), the non-GEMM suite (test_gpu_aux.py), the front-end suite (test_gpu_frontend.py) or the GRU
     suite (test_gpu_analysis.py) derives for it, at every element;
  3. checks each step's wiring: every operand, shortcut operand and residual of a GEMM or pair, and what the GRU, the
     input planes, the conditioning, the band sums, the UNet's first layer and the ISTFT read, was last written by the
     step the network's dataflow names (expected_producers, expected_reads), and in a varlen plan a GEMM's row_valid is
     the lengths-table row of its geometry, computed from the clip lengths;
  4. in a varlen plan, checks that the rows past each clip of every GEMM and pair input are zeros (of either sign), the
     precondition of the layer suite's varlen cases (rows past a clip in each output are checked as exact zeros by step 2).
Then the traced output must equal the product call's bit for bit (eager and graph replay), and every op kind and every
GEMM / pair configuration of the plan must have been replayed.  The accounting test traces every plan kind each context
builds and checks that the traced steps are every launch the product call makes, but for the lengths table.

Inputs: seeded synthetic speech and one clip that widens the activations' range (digital silence, a full-scale click and
a DC offset).  The UNet launches are the same for every vocoder mode, so the GSR plans pair the vocoder's 1- and 3-term
modes with unify_energy off and on once each, uniform and varlen; the bi_gru and dnn plans do the same with the other
pairings.  Their varlen calls hold five clips, so that the GRU's groups of four clips split 4 + 1, and the shortest clip
is 3 frames of a 128-frame bucket."""
import ctypes
import time
import types

import numpy as np
import pytest
import torch

import test_gpu_analysis as AN
import test_gpu_aux as A
import test_gpu_frontend as FE
import test_gpu_layers as G
from oracle import analysis as AO
from oracle import layers as R
from oracle import vf_oracle as O
from voicefixer_main_b200 import _lib as VL
from voicefixer_main_b200.arch import DNN_LINEARS, SSR_PREFIX, UNET_PREFIX

pytestmark = pytest.mark.gpu

# VF_TRACE_* (include/b200vf.h)
GEMM, FIRST, POOL, COND, REFLECT, TAIL, FINALIZE, MEMSET, PAIR, PLANES, GRU, FRONTEND, BAND, ISTFT = range(14)
KIND_NAMES = ["gemm", "first", "pool", "cond", "reflect", "tail", "finalize", "memset", "pair", "planes", "gru", "frontend",
              "band", "istft"]
SR, HOP = 44100, 441
# 1 s, 0.5 s and the shortest clip a restore takes: a varlen bucket of 128 frames pads two of its three clips
N_LONG, N_MID, N_MIN = SR, SR // 2, 1025
CLAMP = np.float32(np.log10(np.float32(1e-8)))     # the front end's log10(max(mel, 1e-8))
PLANS = {                                          # name -> (plan kind, vocoder terms, unify_energy, analysis module)
    "gsr.voc1": (0, 1, False, "unet"),
    "gsr.voc3.unify": (0, 3, True, "unet"),
    "gsr_varlen.voc1.unify": (2, 1, True, "unet"),
    "gsr_varlen.voc3": (2, 3, False, "unet"),
    "ssr": (1, 3, False, "unet"),
    "ssr_varlen": (3, 3, False, "unet"),
    "bigru.voc1": (0, 1, False, "bi_gru"),
    "bigru_varlen.voc3.unify": (2, 3, True, "bi_gru"),
    "dnn.voc3.unify": (0, 3, True, "dnn"),
    "dnn_varlen.voc1": (2, 1, False, "dnn"),
}
RESULTS = {}          # plan -> (kinds replayed, signatures replayed)
# what the plan's conditioning (and the band sums) read as the restored mel: the analysis module's last launch, or the front
# end's linear mel in a vocoder-only plan
MEL_PRODUCER = {"unet": "post.conv2", "bi_gru": "bigru.lin6", "dnn": "dnn.lin5", "voc": "frontend"}


def module_of(name):
    """The network a replay's plan name stands for: "unet", "bi_gru", "dnn", "ssr" or "voc" (vocoder only)."""
    for prefix, module in (("bigru", "bi_gru"), ("dnn", "dnn"), ("ssr", "ssr"), ("voc", "voc")):
        if name.startswith(prefix):
            return module
    return "unet"


def want_kinds(module, terms, unify):
    """The step kinds a traced plan of `module` must go through."""
    if module == "ssr":
        return {FRONTEND, GEMM, FIRST, POOL, ISTFT}
    kinds = {FRONTEND, GEMM, COND, REFLECT, MEMSET, TAIL, FINALIZE}
    kinds |= {"unet": {FIRST, POOL}, "bi_gru": {PLANES, GRU}, "dnn": {PLANES}, "voc": set()}[module]
    if terms == 1:
        kinds.add(PAIR)
    if unify:
        kinds.add(BAND)
    return kinds


# ------------------------------------------------------------------ inputs
def wide_clip(n, seed):
    """Speech with a stretch of digital silence, one full-scale click and a DC offset."""
    x = O.synth_clips(1, n, seed=seed)[0].double()
    x[n // 4:n // 2] = 0.0
    x[n // 3] = 1.0
    x[n // 2:] += 0.25
    return x.clamp(-1, 1).float()


def inputs(kind, five=False):
    """(wav on the device, lengths or None).  five: the varlen call of the bi_gru / dnn plans, two more clips (a GRU
    cluster takes four)."""
    if kind in (0, 1, 4):
        wav = torch.stack([O.synth_clips(1, N_LONG, seed=11)[0].float(), wide_clip(N_LONG, 12)])
        return wav.cuda(), None
    clips = [O.synth_clips(1, N_MIN, seed=13)[0].float(), wide_clip(N_MID, 14), O.synth_clips(1, N_LONG, seed=15)[0].float()]
    if five:
        clips += [O.synth_clips(1, 30001, seed=16)[0].float(), wide_clip(20000, 17)]
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


def scalar_bn(sd, key):
    """A BatchNorm2d(1) of the state dict as (weight, bias, running_mean, running_var) float32, the layer suite's in_bn."""
    return np.array([float(sd[f"{key}.{k}"].reshape(-1)[0]) for k in ("weight", "bias", "running_mean", "running_var")],
                    np.float32)


def analysis_spec(label, sd):
    """What plan.cu's build_bigru / build_dnn give the Linear `label`, as pack.cu packs it: weights [cout, cin, 1] (a one-tap
    GEMM), bias, the epilogue's affine and activation.  A BatchNorm2d(1) before a dnn Linear is folded as pack_linear folds
    it (R.bn_fold, rounded to the fp32 weights the loader uploads); BN_GRU.bn is bigru.lin1's epilogue affine, its fp32
    scalar repeated over the channels."""
    P = lambda k: sd[UNET_PREFIX + k].double()
    spec = {}
    if label.startswith("bigru.gru"):
        l = int(label[len("bigru.gru")])
        g = lambda n: torch.cat([P(f"2.gru.{n}_l{l}"), P(f"2.gru.{n}_l{l}_reverse")])
        w, b = g("weight_ih"), R.gru_ih_bias(g("bias_ih"), g("bias_hh"))
    elif label.startswith("bigru."):
        idx = {"bigru.lin1": 1, "bigru.lin4": 4, "bigru.lin6": 6}[label]
        w, b = P(f"{idx}.weight"), P(f"{idx}.bias")
        if idx == 1:
            s, t = R.bn_scalar(scalar_bn(sd, UNET_PREFIX + "2.bn"))
            spec.update(bn=(np.full(w.shape[0], s, np.float32), np.full(w.shape[0], t, np.float32)), act=0, slope=0.0)
        elif idx == 4:
            spec.update(act=1, slope=0.0)
    else:
        i = int(label[len("dnn.lin"):])
        idx = DNN_LINEARS[i]
        w, b = P(f"{idx}.weight"), P(f"{idx}.bias")
        if 1 <= i <= 4:
            w, b = R.bn_fold(w.float(), b.float(), scalar_bn(sd, UNET_PREFIX + str(idx - 1)))
            w = w.float().double()
        if i < 5:
            spec.update(act=1, slope=0.0)
    spec.update(w=w[:, :, None], b=b)
    return spec


def spec_of(label, sd, cfg, C):
    if label.startswith(("bigru.", "dnn.")):
        return analysis_spec(label, sd)
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
        self.writers = []         # (first byte, end, label) of every step's outputs so far, in launch order
        self.lengths = None
        self.module = module_of(name)
        self.launches = 0         # what the traced steps added to vf_launch_count

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
        self.launches += t.launches
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
        elif t.kind == PLANES:
            o = t.op
            cap["x"] = host(o.x, np.float32, (o.batch, o.T, 128))
        elif t.kind == GRU:
            g = t.gru
            cap["G"] = host(g.G, np.float32, (g.batch, g.T, 1536))
        elif t.kind == FRONTEND:
            o = t.op
            cap["wav"] = host(o.in_wav, np.float32, (self.samples(o),))
            cap["before"] = {k: host(getattr(o, k), np.uint32, (o.batch, o.T, FE.WIDTH[k])) for k in FE.OUTS if getattr(o, k)}
        elif t.kind == BAND:
            o = t.op
            cap["mel"] = host(o.mel, np.float32, (o.batch, o.T, 128))
            cap["tgt"] = host(o.mel_target, np.float32, (o.batch, o.T, 128))
        elif t.kind == ISTFT:
            o = t.op
            cap["mag"] = host(o.mag, np.float32, (o.batch, o.T, 1025))
            cap["wav"] = host(o.in_wav, np.float32, (self.samples(o),))
            cap["frames"] = host(o.frames, np.uint32, (o.batch, o.T, 2048))
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
        if t.kind not in (GEMM, PAIR):
            self.check_reads(t, label)
        return cap

    def samples(self, o):
        """Samples of the call's input (and of the ISTFT's output): packed clips, or batch x n."""
        return sum(self.lengths) if self.lengths else o.batch * o.n

    def clips(self, wav, o):
        """The call's input as a list of clips."""
        if not self.lengths:
            return [wav[i * o.n:(i + 1) * o.n] for i in range(o.batch)]
        off = np.concatenate([[0], np.cumsum(self.lengths)])
        return [wav[off[i]:off[i + 1]] for i in range(len(self.lengths))]

    def check_reads(self, t, label):
        """What a step other than a GEMM or a pair reads was last written by the step the plan's dataflow names
        (expected_reads)."""
        o = t.op
        ptrs = {PLANES: lambda: {"x": o.x}, GRU: lambda: {"G": t.gru.G}, FIRST: lambda: {"x": o.x},
                COND: lambda: {"mel": o.mel, **({"band_sums": o.band_sums} if o.unify else {})},
                BAND: lambda: {"mel": o.mel, "mel_target": o.mel_target}, ISTFT: lambda: {"mag": o.mag}}
        if t.kind not in ptrs:
            return
        got = {k: self.producer(p) for k, p in ptrs[t.kind]().items()}
        want = expected_reads(t.kind, label, self.module, t.kind == COND and bool(o.unify))
        assert got == want, (self.name, label, "reads", got, "expected", want)

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
        if label.startswith(("bigru.", "dnn.")):
            row = 0
        elif label.startswith("voc.cond") or label == "voc.stem":
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
        no launch writes; it reads rows t .. t + 6 of valid output rows t only, and is not held to it.  Nor is the front
        end's log-mel, the residual of an analysis module's last Linear: the front end leaves the rows past a clip as they
        were, and the epilogue writes zeros to those output rows whatever it adds there (checked by the replay)."""
        lc = t.layer
        if lc.kind == G.CONV1D and not lc.centered:
            return
        if "resid" in cap and self.producer(lc.resid) == "frontend":
            cap = {k: v for k, v in cap.items() if k != "resid"}
        rv = rows_of(lc.row_valid, lc.n_img)
        lim = rv if lc.kind != G.CONVT1D else (rv + lc.stride - 1) // lc.stride
        for i in range(lc.n_img):
            x = R.from_bits(cap["x"][:, i, lc.x_row0 + lim[i]:])         # zeros of either sign
            assert not x.any(), (self.name, label, "operand rows past clip", i, "are not zero")
            if "resid" in cap:
                r = cap["resid"][i, rv[i]:] if cap["resid"].ndim == 3 else R.from_bits(cap["resid"][:, i, rv[i]:])
                assert not r.any(), (self.name, label, "residual rows past clip", i, "are not zero")


def expected_reads(kind, label, module, unify=False):
    """{input: label of the step that must have written it last} for a step other than a GEMM or a pair: the input planes
    and the UNet's first layer read the front end's log-mel (SSR: its magnitudes), each GRU layer the G of its own input
    projection (both layers share one G buffer), the conditioning and the band sums the restored log-mel (a vocoder-only
    plan: the front end's linear mel), the band sums also the front end's linear mel, the ISTFT the SSR UNet's magnitudes."""
    if kind in (PLANES, FIRST):
        return {"x": "frontend"}
    if kind == GRU:
        return {"G": label + ".ih"}
    if kind == COND:
        return {"mel": MEL_PRODUCER[module], **({"band_sums": "band_energy"} if unify else {})}
    if kind == BAND:
        return {"mel": MEL_PRODUCER[module], "mel_target": "frontend"}
    return {"mag": "ssr.post.conv2"}


def expected_producers(label, cfg):
    """{input: label of the launch that must have written it last} for the GEMM or pair `label` (plan.cu's dataflow: each
    block's conv1 reads the previous block's activated output, conv2 reads its conv1, the residual stream runs from block
    to block; the non-GEMM producers carry their kind's name).  The analysis modules' Linear layers read the previous
    launch's output; their last one adds the front end's log-mel."""
    if label.startswith("bigru."):
        x = {"bigru.lin1": "analysis.in_planes", "bigru.gru0.ih": "bigru.lin1", "bigru.gru1.ih": "bigru.gru0",
             "bigru.lin4": "bigru.gru1", "bigru.lin6": "bigru.lin4"}[label]
        return {"x": x, **({"resid": "frontend"} if label == "bigru.lin6" else {})}
    if label.startswith("dnn."):
        i = int(label[len("dnn.lin"):])
        return {"x": "analysis.in_planes" if i == 0 else f"dnn.lin{i - 1}", **({"resid": "frontend"} if i == 5 else {})}
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


def clip_frames(rp, t, B, T):
    vl = vl_table(t, B)
    return [T] * B if vl is None else [int(v) for v in vl[0]]


def check_planes(rp, t, label, ck):
    """Bit-exact, as test_gpu_aux.test_input_planes_are_exact: BN0's scale and shift as load_bigru folds them (dnn: 1, 0)."""
    o = t.op
    B = o.batch
    s, sh = (R.bn_scalar(scalar_bn(rp.sd, UNET_PREFIX + "0")) if rp.module == "bi_gru" else (1.0, 0.0))
    assert (o.bn1_scale, o.bn1_shift) == (np.float32(s), np.float32(sh)), (ck.name, o.bn1_scale, o.bn1_shift)
    Ts = clip_frames(rp, t, B, o.T)
    want = R.affine_planes(rp.cap["x"], o.bn1_scale, o.bn1_shift, Ts if rp.varlen else None)
    bad = np.argwhere(planes(o.planes, B, o.T, 128) != want)
    assert not len(bad), (ck.name, f"{len(bad)} elements differ, first [plane, clip, row, channel] {bad[:4].tolist()}")


def check_gru(rp, t, label, ck):
    """oracle/analysis.gru_layer from the captured G with the state dict's weight_hh / bias_hh (the device copies must be
    those fp32 tensors bit for bit), ReLU on layer 1 only, each clip over its own frames: |err| < GRU_TOL
    (test_gpu_analysis.py) and exact zeros past each clip."""
    g = t.gru
    l = int(label[len("bigru.gru")])
    key = lambda n, d: UNET_PREFIX + f"2.gru.{n}_l{l}" + ("_reverse" if d else "")
    w = torch.stack([rp.sd[key("weight_hh", d)].float() for d in range(2)])
    bh = torch.stack([rp.sd[key("bias_hh", d)].float()[512:] for d in range(2)])
    for d in range(2):
        assert np.array_equal(host(g.w_hh[d], np.uint32, (768, 256)), w[d].numpy().view(np.uint32)), (ck.name, "w_hh", d)
        assert np.array_equal(host(g.b_hn[d], np.uint32, (256,)), bh[d].numpy().view(np.uint32)), (ck.name, "b_hn", d)
    assert g.relu == l, (ck.name, "relu", g.relu)
    B, T = g.batch, g.T
    Ts = clip_frames(rp, t, B, T)
    if rp.varlen:
        assert list(rows_of(g.lengths, B)) == Ts, (ck.name, "lengths are not the frames row")
    else:
        assert not g.lengths, ck.name
    want = AO.gru_layer(torch.from_numpy(rp.cap["G"]).double(), w.double(), bh.double(), Ts, relu=bool(l)).numpy()
    got = A.hi_lo(planes(g.out, B, T, 512))
    zero = np.zeros((B, T, 1), bool)
    for i, Tb in enumerate(Ts):
        zero[i, Tb:] = True
    ck.values("gru", got, want, np.full(got.shape, AN.GRU_TOL), zero)


def check_frontend(rp, t, label, ck):
    """test_gpu_frontend.check_frontend's bounds on every output the restore asks for; rows past a varlen clip are not
    written."""
    o = t.op
    outs = {}
    for k in FE.OUTS:
        full = np.full((o.batch, o.T, FE.WIDTH[k]), G.SENT32, np.uint32)
        if getattr(o, k):
            got = host(getattr(o, k), np.uint32, full.shape)
            for b, x in enumerate(rp.clips(rp.cap["wav"], o)):
                Tb = 1 + len(x) // HOP
                assert np.array_equal(got[b, Tb:], rp.cap["before"][k][b, Tb:]), (ck.name, k, b, "rows past the clip written")
                full[b, :Tb] = got[b, :Tb]
        outs[k] = full
    want = [k for k in FE.OUTS if getattr(o, k)]
    res = FE.check_frontend(ck.name, rp.clips(rp.cap["wav"], o), outs, O.mel_filterbank().numpy(), want)
    ck.worst = max(ck.worst, res.worst)


def check_band(rp, t, label, ck):
    """unify_energy's sums against R.band_sums within test_gpu_aux.band_bound."""
    o = t.op
    sums = host(o.band_sums, np.float32, (o.batch, 2)).astype(np.float64)
    for b, Tb in enumerate(clip_frames(rp, t, o.batch, o.T)):
        s64 = R.band_sums(rp.cap["tgt"][b:b + 1], rp.cap["mel"][b:b + 1], [Tb])
        ck.values("band", sums[b], s64[0], A.band_bound(rp.cap["tgt"][b], rp.cap["mel"][b], Tb) + G.FLOOR, np.zeros(1, bool))


def check_istft(rp, t, label, ck):
    """The fused ISTFT's frames and overlap-add within test_gpu_aux.fused_istft's bounds, from the captured magnitudes and
    the input's phase; frames past a varlen clip are not written."""
    o = t.op
    wav, mag = rp.cap["wav"], rp.cap["mag"]
    frames = host(o.frames, np.uint32, (o.batch, o.T, 2048))
    out = host(o.out, np.uint32, (rp.samples(o),))
    c_fft = 4 * A.U * np.log2(2048)
    win = R.hann()
    start = 0
    for b, x in enumerate(rp.clips(wav, o)):
        nb, Tb = len(x), 1 + len(x) // HOP
        X, S = R.stft64(x, Tb)
        cs, sn = R.phase(X)
        mg = mag[b, :Tb].astype(np.float64)
        f64 = R.inverse_frames(mg * (cs + 1j * sn))
        E = A.istft_frame_error(mg, np.minimum(2.0, c_fft * S[:, None] / np.maximum(np.abs(X), 1e-4)))
        ck.values("frames", frames[b, :Tb].view(np.float32).astype(np.float64), f64,
                  win[None] * E[:, None] + A.gamma(3) * np.abs(f64) + G.FLOOR, (S == 0)[:, None])
        assert np.array_equal(frames[b, Tb:], rp.cap["frames"][b, Tb:]), (ck.name, b, "frames past the clip written")
        y, bnd = A.ola_bound(f64, E, nb)
        ck.values("out", out[start:start + nb].view(np.float32).astype(np.float64), y, bnd, np.zeros(1, bool))
        start += nb


CHECKS = {GEMM: check_gemm, PAIR: check_pair, FIRST: check_first, POOL: check_pool, COND: check_cond, REFLECT: check_reflect,
          MEMSET: check_memset, TAIL: check_tail, FINALIZE: check_finalize, PLANES: check_planes, GRU: check_gru,
          FRONTEND: check_frontend, BAND: check_band, ISTFT: check_istft}


# ------------------------------------------------------------------ tests
@pytest.fixture(scope="module")
def setup():
    """engine(module) -> (Engine, state dict, config): one context per analysis module, loaded once.  "unet" also holds the
    SSR UNet; "bi_gru" and "dnn" hold their module and the vocoder (test_gpu_analysis.py's states)."""
    from voicefixer_main_b200.model import Engine
    from voicefixer_main_b200.weights import make_bigru_state, make_dnn_state, make_ssr_state, make_state, make_vocoder_state
    cfg = VL.VfConfig()
    VL.load_library().vf_default_config(ctypes.byref(cfg))
    engines = {}

    def engine(module):
        if module not in engines:
            if module == "unet":
                sd, need = {**make_state(1234), **make_ssr_state(1234)}, ("unet", "vocoder", "ssr")
            else:
                sd = {**(make_bigru_state if module == "bi_gru" else make_dnn_state)(1234), **make_vocoder_state(seed=1235)}
                need = (module, "vocoder")
            e = Engine("cuda:0")
            e.load_state(sd, need=need)
            engines[module] = (e, sd, cfg)
        return engines[module]

    yield engine
    for e, _, _ in engines.values():
        e.check_errors()
        e.close()


def product(e, kind, wav, lengths, unify):
    if kind == 0:
        return e.restore(wav, unify_energy=unify)
    if kind == 1:
        return e.ssr_forward(None, wav)
    if kind == 2:
        return e.restore_varlen(wav, lengths, unify_energy=unify)
    if kind == 3:
        return e.ssr_restore_varlen(wav, lengths)
    return e.resynth(wav) if kind == 4 else e.resynth_varlen(wav, lengths)


def replay(setup, name):
    kind, terms, unify, module = PLANS[name]
    e, sd, cfg = setup(module)
    e.set_option("vocoder_terms", terms)
    wav, lengths = inputs(kind, five=module != "unet")
    rp = Replay(name, sd, cfg, lengths is not None)
    rp.lengths = lengths
    PAIR_STAGE.clear()
    if terms == 1:
        PAIR_STAGE[cfg.voc_num_stages - 1] = True          # the C = 64 stack of the (a, r) stream (plan.cu: fused)
    t0 = time.perf_counter()
    got = e.selftest_plan_trace(kind, wav, lengths, rp.on_op, unify_energy=unify, direct_steps=True)
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
    assert rp.kinds == want_kinds("ssr" if kind in (1, 3) else module, terms, unify), (name, sorted(rp.kinds))
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


# the plan kinds each context builds: GSR 0 / 2 (with unify_energy), SSR 1 / 3, vocoder-only 4 / 5
ACCOUNTING = [("unet", k, u) for k, u in ((0, True), (2, True), (1, False), (3, False), (4, False), (5, False))] + \
             [(m, k, k in (0, 2)) for m in ("bi_gru", "dnn") for k in (0, 2, 4, 5)]
SETUP_LAUNCHES = {"lengths table": lambda varlen: int(varlen)}     # launches a call makes that the trace does not replay


def test_traced_steps_are_every_launch_of_the_product_call(setup):
    """For every plan kind of every context: the trace runs to completion and goes through every GEMM / pair configuration
    vf_selftest_plan_gemms reports, and with graphs off the product call's launch count is the traced steps' plus
    SETUP_LAUNCHES.  Without direct_steps the trace goes through the same steps but those of list 3.  Every step kind the
    plans have is among CHECKS."""
    seen = set()
    for module, kind, unify in ACCOUNTING:
        e, _, _ = setup(module)
        e.set_option("vocoder_terms", 1)
        wav, lengths = inputs(kind, five=module != "unet")
        steps = {"kinds": set(), "sigs": set(), "launches": 0, "order": []}

        def on_op(after, t):
            if after:
                steps["order"].append((t.list, t.label.decode()))
                steps["kinds"].add(t.kind)
                steps["launches"] += t.launches
                if t.kind in (GEMM, PAIR):
                    steps["sigs"].add(t.layer.sig.decode())

        got = e.selftest_plan_trace(kind, wav, lengths, on_op, unify_energy=unify, direct_steps=True)
        listed = []
        plain = e.selftest_plan_trace(kind, wav, lengths, lambda after, t: listed.append((t.list, t.label.decode())) if after
                                      else None, unify_energy=unify)
        e.set_option("graphs", 0)
        try:
            n0 = e.launch_count()
            want = product(e, kind, wav, lengths, unify)
            torch.cuda.synchronize()
            launches = e.launch_count() - n0
        finally:
            e.set_option("graphs", 1)
        e.check_errors()
        tag = (module, kind, unify)
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), tag
        assert torch.equal(plain.view(torch.int32), want.view(torch.int32)), tag
        assert listed == [s for s in steps["order"] if s[0] != 3], (tag, "steps without direct_steps")
        n = len(lengths) if lengths else wav.shape[0]
        T = (1 + max(lengths) // HOP + 63) // 64 * 64 if lengths else 1 + wav.shape[1] // HOP
        assert {sg for _, sg in e.selftest_plan_gemms(kind, n, T)} == steps["sigs"], tag
        setup_launches = sum(f(lengths is not None) for f in SETUP_LAUNCHES.values())
        assert launches == steps["launches"] + setup_launches, (tag, launches, steps["launches"], setup_launches)
        mod = "ssr" if kind in (1, 3) else "voc" if kind in (4, 5) else module
        assert steps["kinds"] == want_kinds(mod, 1, unify), (tag, sorted(steps["kinds"]))
        print(f"{module} plan {kind}{' unify' if unify else ''}: {launches} launches = {steps['launches']} traced + "
              f"{setup_launches} set-up")
        seen |= steps["kinds"]
    assert seen == set(CHECKS), sorted(seen)
