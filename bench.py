#!/usr/bin/env python
"""Benchmark of the VoiceFixer inference hot path (BASELINE.json metric: clips/sec on 44.1 kHz 10 s clips).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl b200|reference]
                    [--workload gsr|ssr|longform] [--batch B] [--seconds S] [--minutes M] [--dump-outputs DIR]

Default workload `gsr`: a step = one pass of the whole hot path (STFT+mel -> ResUNet ->
vocoder -> peak-normalise -> trim) over one batch of B synthetic clips per GPU (configs[1] of BASELINE.json: batch
32 x 10 s, 1 x H100; at N GPUs each rank runs its own 32 clips = configs[3], weak scaling, the only collective being
the start-up weight broadcast).  `ssr` = BASELINE configs[2] (SSR_UNet denoising, unet_v2 + ISTFT, batch 64);
`longform` = configs[4] (one 30-minute stream as 60 s segments, handler() hard cuts and the margin mode).

Prints ONE JSON line (rank 0).  `value` = clips/s with inputs resident in HBM; `e2e` = the same metric through the
host-buffer entry point (pinned host buffers, H2D + D2H inside the timed region); `roofline` = the dominant kernel
(live CUDA events) plus one entry per stage against SURVEY.md 8(d)'s algorithmic work; `parity` = the reference's
golden clip riding in row 0 of the benchmarked batch; `cpu_baseline` = the oracle timed on host cores.
`--impl reference` times the reference algorithm on the host CPU (the oracle port of the reference's Python code) on a
bounded sample of the same workload.
`--dump-outputs DIR` writes what the last timed step returned to its caller as DIR/<name>.npy (float32; at most 64 MB in
all - a larger output is written as a fixed, seeded sample of its elements plus DIR/<name>_index.npy).  The inputs are
seeded, so two builds run with the same arguments can be compared output for output.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

SR, HOP = 44100, 441
METRIC = "clips_per_sec_10s_44k1"
UNET_GFLOP_PER_CLIP_T1024 = 190.16          # SURVEY.md 8(d): mel UNet, T' = 1024
SSR_GFLOP_PER_CLIP_T1024 = 1597.95          # SURVEY.md 8(d): unet_v2, T' = 1024
REF_STEP_BUDGET_S = 150.0                   # --impl reference: bound on timed CPU work (the whole run must end in minutes)


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return {"hbm_gbs": d["hbm_gbs"], "tflops": d.get("bf16_tflops_sustained", d["bf16_tflops"]),
                "tflops_burst": d["bf16_tflops"], "source": "measured"}
    # H100 SXM data sheet (700 W card): 3.35 TB/s HBM3, 989 TFLOP/s dense fp16 - not reached figures, the denominators
    return {"hbm_gbs": 3350.0, "tflops": 989.0, "tflops_burst": 989.0, "source": "H100 SXM data sheet"}


class ClockSampler(threading.Thread):
    """nvidia-smi clocks / throttle reasons sampled during the timed region (read-only queries)."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.rows, self.stop_flag = index, [], False

    def run(self):
        while not self.stop_flag:
            try:
                out = subprocess.run(["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits"],
                                     capture_output=True, text=True, timeout=5).stdout.strip()
                if out:
                    self.rows.append([x.strip() for x in out.split(",")])
            except Exception:
                pass
            time.sleep(0.2)

    def summary(self):
        sm = sorted(float(r[0]) for r in self.rows if r and r[0].replace(".", "").isdigit())
        reasons = set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            for n, v in zip(names, r[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        mx = [float(r[1]) for r in self.rows if len(r) > 1 and r[1].replace(".", "").isdigit()]
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx[0] if mx else None,
                "reasons": sorted(reasons), "samples": len(self.rows)}


DUMP_LIMIT_BYTES = 64 << 20


def dump_outputs(out_dir, arrays):
    """Write {name: tensor} as out_dir/<name>.npy in float32; past DUMP_LIMIT_BYTES in all, every array is replaced by the
    same fraction of its elements, chosen by a fixed seed and stored with their flat indices (<name>_index.npy)."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    arrays = {k: v.detach().float().cpu().contiguous() for k, v in arrays.items()}
    total = sum(v.numel() * 4 for v in arrays.values())
    for name, v in arrays.items():
        if total > DUMP_LIMIT_BYTES:
            keep = max(1, int(v.numel() * (DUMP_LIMIT_BYTES / 2) / total))        # index + value both stored
            g = torch.Generator().manual_seed(12345)
            idx = torch.randperm(v.numel(), generator=g)[:keep].sort().values
            np.save(os.path.join(out_dir, f"{name}_index.npy"), idx.numpy().astype(np.int64 if v.numel() >= 2**31 else np.int32))
            v = v.reshape(-1)[idx]
        np.save(os.path.join(out_dir, f"{name}.npy"), v.numpy())


def synth_batch(batch, n, seed):
    """Speech-like synthetic clips (SURVEY.md 8(d)): harmonic stack x slow envelope + noise floor, peak in [0.3, 1]."""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(n, dtype=torch.float32) / SR
    f0 = 80 + 220 * torch.rand(batch, 1, generator=g)
    sig = torch.zeros(batch, n)
    for h in range(1, 13):
        amp = torch.rand(batch, 1, generator=g) / h
        ph = 6.2831853 * torch.rand(batch, 1, generator=g)
        sig += amp * torch.sin(6.2831853 * f0 * h * t[None, :] + ph)
    env = 0.55 + 0.45 * torch.sin(6.2831853 * (0.5 + torch.rand(batch, 1, generator=g)) * t[None, :])
    sig = sig * env + 0.003 * torch.randn(batch, n, generator=g)
    return sig / sig.abs().amax(dim=1, keepdim=True) * (0.3 + 0.7 * torch.rand(batch, 1, generator=g))


def load_golden(name):
    import numpy as np
    p = os.path.join(ROOT, "tests", "golden", name)
    return np.load(p) if os.path.exists(p) else None


# ---------------------------------------------------------------------------------------------- CPU reference arm
def best_cpu_threads(fn, candidates):
    """torch CPU convs do not scale to every core of a big host; give the reference its best thread count."""
    best, best_t = None, None
    for th in candidates:
        torch.set_num_threads(th)
        with torch.no_grad():
            fn()
            t0 = time.perf_counter()
            fn()
            dt = time.perf_counter() - t0
        if best is None or dt < best:
            best, best_t = dt, th
    return best_t


def cpu_reference(workload, seconds, steps, warmup, threads=None):
    """The reference algorithm (oracle port, pinned against the reference's own modules where they import) on the host
    CPU, one clip per step as the reference runs it (batch 1, eval_gsr_voicefixer.py:19-21), warm-up on the FULL clip.
    Returns (clips/s, s/step, threads, steps actually timed, note)."""
    from oracle import vf_oracle as O
    from voicefixer_main_b200.weights import make_ssr_state, make_state
    n = int(seconds * SR)
    if workload == "ssr":
        state = make_ssr_state(1234)
        step = lambda w: O.ssr_forward(state, w[:, None, :])
    else:
        state = make_state(1234)
        step = lambda w: O.restore(state, w)
    cores = os.cpu_count() or 1
    probe = synth_batch(1, SR, 98)
    if threads is None:
        threads = best_cpu_threads(lambda: step(probe), sorted({min(cores, c) for c in (8, 16, 32, 64, cores)}))
    torch.set_num_threads(threads)
    wav = synth_batch(1, n, 99)
    note = ""
    with torch.no_grad():
        t0 = time.perf_counter()
        step(wav)                                     # first warm-up step on the full clip (allocations, thread pools)
        one = time.perf_counter() - t0
        for _ in range(max(0, warmup - 1)):
            if one * 2 > REF_STEP_BUDGET_S / 4:
                note = f"warm-up capped at 1 of {warmup} full-clip steps ({one:.1f} s each)"
                break
            step(wav)
        t0 = time.perf_counter()
        step(wav)
        one = time.perf_counter() - t0
        k = max(1, min(steps, int(REF_STEP_BUDGET_S / max(one, 1e-3))))
        if k < steps:
            note = (note + "; " if note else "") + f"timed steps capped at {k} of {steps}: one step takes {one:.1f} s and the run is bounded to ~{REF_STEP_BUDGET_S:.0f} s of CPU work"
        dt = one
        t0 = time.perf_counter()
        for _ in range(k - 1):
            step(wav)
        dt += time.perf_counter() - t0
    return k / dt, dt / k, threads, k, note


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    seconds = args.seconds if args.seconds else (3.0 if args.workload == "ssr" else 10.0)
    wl = "ssr" if args.workload == "ssr" else "gsr"
    cps, spc, threads, k, note = cpu_reference(wl, seconds, max(1, args.steps), max(1, args.warmup))
    what = ("ssr_unet (unet_v2 + ISTFT) forward" if wl == "ssr" else "gsr_voicefixer handler path")
    line = {
        "impl": "reference", "metric": METRIC if wl == "gsr" and seconds == 10.0 else f"clips_per_sec_{seconds:g}s_44k1", "value": cps, "unit": "clips/s",
        "n_gpus": args.gpus, "steps": k, "warmup": max(1, args.warmup),
        "ms_per_step": spc * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic", "rtf": cps * seconds,
        "config": {"workload": f"{what}, 1 x {seconds:g} s 44.1 kHz clip per step on host CPU (batch 1 as the reference runs)",
                   "clip_seconds": seconds, "steps_requested": args.steps, "warmup_requested": args.warmup, "note": note},
        "cpu_baseline": {"value": cps, "unit": "clips/s", "cores": threads, "kind": "port",
                         "sample": f"{k} x one {seconds:g} s clip, torch CPU fp32, best of 8/16/32/64/all threads = {threads} of {os.cpu_count()} host cores"},
        "e2e": {"value": cps, "unit": "clips/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line))


# ---------------------------------------------------------------------------------------------- roofline helpers
def stage_of(label):
    if label.startswith("voc") or label in ("voc_condition", "reflect_fill", "voc_tail", "memset"):
        return "C"
    return "B"


def stage_roofline(prof, stage_ms, peaks, clips, n_samples, frames, ssr=False):
    """One entry per stage against SURVEY.md 8(d): algorithmic work of the reference op counts (not this design's
    traffic), the live stage time, and the fraction of the measured peak - raw and counting the MMAs executed."""
    tp = (frames + 63) // 64 * 64
    out = []
    a_bytes = clips * (n_samples * 4 + (frames * 1025 * 4 if ssr else frames * 128 * 4))
    a_ms = stage_ms["frontend_ms"]
    out.append({"stage": "A", "what": "STFT magnitude" + (" [B,T,1025]" if ssr else " + mel + log10 (spectrogram never materialised)"),
                "bound": "hbm (nominal; FFT-latency bound in practice, DESIGN.md)", "algorithmic_gb": a_bytes / 1e9, "ms": a_ms,
                "achieved_gbs": a_bytes / (a_ms * 1e-3) / 1e9 if a_ms > 0 else None, "peak_gbs": peaks["hbm_gbs"],
                "frac": a_bytes / (a_ms * 1e-3) / 1e9 / peaks["hbm_gbs"] if a_ms > 0 else None})
    for st, key, name in (("B", "unet_ms", "ResUNet"), ("C", "vocoder_ms", "vocoder")):
        ops = [r for r in prof if stage_of(r["label"]) == st]
        if not ops:
            continue
        fl = sum(r["flops"] for r in ops)
        ex = sum(r.get("exec_flops", 0.0) for r in ops)
        ms = stage_ms[key]
        e = {"stage": st, "what": name, "bound": "tensor", "algorithmic_tflop": fl / 1e12, "executed_tflop": ex / 1e12, "ms": ms,
             "achieved_tflops": fl / (ms * 1e-3) / 1e12, "peak_tflops": peaks["tflops"],
             "frac_raw": fl / (ms * 1e-3) / 1e12 / peaks["tflops"], "frac_executed": ex / (ms * 1e-3) / 1e12 / peaks["tflops"],
             "launches": len(ops), "min_hbm_gb": sum(r["bytes"] for r in ops) / 1e9,
             "hbm_frac_of_design_traffic": sum(r["bytes"] for r in ops) / (ms * 1e-3) / 1e9 / peaks["hbm_gbs"]}
        if st == "B":
            per_clip = (SSR_GFLOP_PER_CLIP_T1024 if ssr else UNET_GFLOP_PER_CLIP_T1024) * tp / 1024
            e["survey_8d_gflop_per_clip"] = per_clip
            e["engine_vs_survey"] = fl / 1e9 / clips / per_clip
            # SURVEY.md 8(d) secondary floor: weights once + input / output / skips written and read once per clip
            e["survey_8d_hbm_floor_gb"] = (248.5e6 + clips * (0.52e6 + 0.51e6 + 2 * 31.8e6) * (tp / 1024) * (8.0 if ssr else 1.0)) / 1e9
        else:
            # SURVEY.md 8(d): weights (~130 MB) + 0.5 MB in + 1.77 MB out per clip - the stage is tensor-bound there; the
            # `min_hbm_gb` above is THIS design's layer-by-layer traffic (activations round-trip through HBM between launches)
            e["survey_8d_hbm_floor_gb"] = (130e6 + clips * 2.27e6 * (n_samples / 441000.0)) / 1e9
        out.append(e)
    return out


def dominant_kernel(prof, peaks):
    groups = {}
    for r in prof:
        if r["bn"]:
            key = (r["bn"], r["bk"], r.get("terms", 0))
            g = groups.setdefault(key, {"ms": 0.0, "flops": 0.0, "exec": 0.0, "bytes": 0.0, "n": 0, "ops": []})
            g["ms"] += r["ms"]; g["flops"] += r["flops"]; g["exec"] += r.get("exec_flops", 0.0); g["bytes"] += r["bytes"]; g["n"] += 1; g["ops"].append(r)
    total_ms = sum(r["ms"] for r in prof)

    def rates(g):
        tf = g["flops"] / (g["ms"] * 1e-3) / 1e12
        gb = g["bytes"] / (g["ms"] * 1e-3) / 1e9
        return tf, gb, tf / peaks["tflops"], gb / peaks["hbm_gbs"]

    (bn, bk, terms), top = max(groups.items(), key=lambda kv: kv[1]["ms"])
    tf, gb, f_t, f_h = rates(top)
    bound = "hbm" if f_h > f_t else "tensor"
    labels = [r["label"] for r in top["ops"]]
    kname = f"gemm_tc_kernel<BN={bn},BK={bk},{'3-term' if terms == 3 else 'hi-only'}> (wgmma flat-shift conv GEMM; layers: {labels[0]} ... {labels[-1]})"
    return {
        "kernel": kname,
        "bound": bound,
        "achieved": gb if bound == "hbm" else tf, "peak": peaks["hbm_gbs"] if bound == "hbm" else peaks["tflops"],
        "unit": "GB/s" if bound == "hbm" else "TFLOP/s", "frac": f_h if bound == "hbm" else f_t,
        "peak_source": peaks["source"] + (" STREAM copy" if bound == "hbm" else " bf16 dense (== fp16 rate), sustained"),
        "launches": top["n"], "avg_launch_ms": top["ms"] / top["n"], "share_of_step": top["ms"] / total_ms,
        "algorithmic_gflop_per_launch": top["flops"] / top["n"] / 1e9, "algorithmic_gb_per_launch": top["bytes"] / top["n"] / 1e9,
        "tensor_frac": f_t, "tensor_frac_executed": top["exec"] / (top["ms"] * 1e-3) / 1e12 / peaks["tflops"], "hbm_frac": f_h,
        "all_kernels": {f"gemm<{k[0]},{k[1]},{'3t' if k[2] == 3 else '1t'}>": {"ms": v["ms"], "launches": v["n"], "tflops": rates(v)[0], "min_gbs": rates(v)[1],
                                                                   "tensor_frac": rates(v)[2], "hbm_frac": rates(v)[3]}
                        for k, v in sorted(groups.items(), key=lambda kv: -kv[1]["ms"])},
    }


def timed_loop(fn, steps, barrier, dev, vdist):
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    barrier()
    return vdist.max_over_ranks(e0.elapsed_time(e1), dev)


# ---------------------------------------------------------------------------------------------- GSR (default) and SSR
def run_b200(args):
    from voicefixer_main_b200 import SSR_UNet, VoiceFixer
    from voicefixer_main_b200 import dist as vdist
    from voicefixer_main_b200.weights import make_ssr_state, make_state
    import torch.distributed as tdist

    ssr = args.workload == "ssr"
    t0 = time.perf_counter()
    rank, world, local = vdist.init_from_env()
    if not torch.cuda.is_available():
        raise SystemExit("bench.py --impl b200 needs a CUDA device (there is no CPU fallback)")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    seconds = args.seconds if args.seconds else (3.0 if ssr else 10.0)
    n = int(seconds * SR)
    B = args.batch if args.batch else (64 if ssr else 32)
    frames = 1 + n // HOP

    # weights: built on rank 0 only, one broadcast over NCCL/NVLink, packed per rank inside libb200vf
    state0 = (make_ssr_state(1234) if ssr else make_state(1234)) if rank == 0 else None
    if ssr:
        from voicefixer_main_b200.arch import SSR_PREFIX, unet_keys
        items = [(SSR_PREFIX + k, tuple(s)) for k, s in unet_keys() if not k.endswith("num_batches_tracked")]
        layout = [(k, s, int(torch.tensor(s).prod()) if s else 1) for k, s in sorted(items)]
    else:
        layout = vdist.layout_from_arch()
    if world > 1:
        tdist.barrier()                      # NCCL communicator creation happens here, not in the weight broadcast
    torch.cuda.synchronize()
    t_init = time.perf_counter()
    state = vdist.broadcast_state(state0, layout, dev)
    torch.cuda.synchronize()
    bcast_ms = (time.perf_counter() - t_init) * 1e3
    model = (SSR_UNet() if ssr else VoiceFixer()).load_state_dict(state).eval().to(dev)
    eng = model._engine()
    if args.vocoder_terms and not ssr:
        eng.set_option("vocoder_terms", args.vocoder_terms)
    if args.no_graphs:
        eng.set_option("graphs", 0)

    host_in = synth_batch(B, n, 1000 + rank)
    # parity rides along: the reference-generated golden clip is row 0 of the benchmarked batch (rank 0)
    gold = None
    if rank == 0 and not ssr and n == 441000:
        gold = load_golden("e2e_10s.npz")
        if gold is not None:
            host_in[0] = torch.from_numpy(gold["wav"])[0]
    host_in = host_in.pin_memory()
    host_out = torch.empty_like(host_in).pin_memory()
    dev_in = host_in.to(dev)
    dev_out = torch.empty_like(dev_in)
    step_dev = (lambda: model.restore(dev_in, dev_out))
    step_host = (lambda: model.restore_host(host_in, host_out))

    def barrier():
        if world > 1:
            tdist.barrier()
        torch.cuda.synchronize()

    # ---- device-resident throughput
    for _ in range(args.warmup):
        step_dev()
    eng.check_errors()
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    l0 = eng.launch_count()
    ms = timed_loop(step_dev, args.steps, barrier, dev, vdist)
    launches = eng.launch_count() - l0
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, {"wav": dev_out})        # restore()'s result in the last timed step
    # ---- end to end through the public host API (pinned host in/out, copies inside the timed region)
    for _ in range(min(2, args.warmup)):
        step_host()
    ms_e2e = timed_loop(step_host, args.steps, barrier, dev, vdist)
    sampler.stop_flag = True
    eng.check_errors()
    assert torch.isfinite(host_out).all()

    if rank != 0:
        return
    parity = None
    if gold is not None:
        _, log_mel = eng.restore_stages(B, n)
        parity = {"golden": "tests/golden/e2e_10s.npz (generated by the reference's own modules, oracle/make_golden.py)", "row": 0, "batch": B,
                  "wav_rms": float((host_out[0] - torch.from_numpy(gold["out"])[0]).double().pow(2).mean().sqrt()), "wav_rms_bar": 1e-3,
                  "logmel_max_e2e": float((log_mel[0].cpu() - torch.from_numpy(gold["log_mel"])[0, 0]).abs().max()),
                  "logmel_note": "end-to-end log-mel also carries the reference's fp32 conv-DFT noise in quiet bins; the 1e-4 stage-B bar is "
                                 "tested on identical mel input at this batch in tests/test_gpu_round2.py"}
    # ---- per-stage and per-launch profile (outside the timed regions)
    eng.enable_stage_timing(True)
    step_dev()
    stage = eng.stage_times()
    eng.enable_stage_timing(False)
    eng.enable_op_timing(True)
    step_dev()
    prof = eng.op_profile()
    eng.enable_op_timing(False)
    if args.profile_out:
        os.makedirs(os.path.dirname(os.path.abspath(args.profile_out)), exist_ok=True)
        json.dump({"stage_ms": stage, "ops": prof}, open(args.profile_out, "w"), indent=0)
    peaks = load_peaks()
    roofline = dominant_kernel(prof, peaks)
    roofline["stages"] = stage_roofline(prof, stage, peaks, B, n, frames, ssr=ssr)
    slow = sorted(prof, key=lambda r: -r["ms"])[:8]
    clips = B * world
    value = clips * args.steps / (ms * 1e-3)
    e2e = clips * args.steps / (ms_e2e * 1e-3)
    cpu = None
    if not args.no_cpu_baseline:
        cps, spc, threads, k, note = cpu_reference("ssr" if ssr else "gsr", seconds, 2, 1)
        cpu = {"value": cps, "unit": "clips/s", "cores": threads, "kind": "port",
               "sample": f"{k} x one {seconds:g} s clip (batch 1), oracle port of the reference, torch CPU fp32, best thread count {threads} of {os.cpu_count()} host cores",
               "rtf": cps * seconds}
    wl = (f"ssr_unet denoising (unet_v2 + ISTFT), batch {B} x {seconds:g} s synthetic 44.1 kHz clips per GPU (BASELINE configs[2])" if ssr else
          f"gsr_voicefixer inference, batch {B} x {seconds:g} s synthetic 44.1 kHz clips per GPU (BASELINE configs[1]; configs[3] at 8 GPUs)")
    line = {
        "metric": METRIC if (not ssr and seconds == 10.0) else f"{'ssr_' if ssr else ''}clips_per_sec_{seconds:g}s_44k1",
        "value": value, "unit": "clips/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": ("f16 tensor-core (hi/lo split, fp32-grade), f32 accumulate" if ssr else
                  "f16 tensor-core (UNet: hi/lo split, fp32-grade; vocoder: " + ("hi/lo split" if args.vocoder_terms == 3 else "hi-only") + "), f32 accumulate"),
        "data": "synthetic", "rtf": value * seconds,
        "config": {"workload": wl, "global_batch": clips, "per_gpu_batch": B, "clip_seconds": seconds, "frames": frames,
                   "parallelism": f"dp{world} (independent clips, one NCCL weight broadcast at start-up)",
                   "startup": {"weight_broadcast_ms": bcast_ms, "process_group_init_and_first_barrier_ms": (t_init - t0) * 1e3,
                               "payload_mb": sum(x[2] for x in layout) * 4 / 1e6},
                   "l2": "activation working set per step (GBs) far exceeds the 50 MB L2; no explicit flush needed",
                   "weights": "seeded synthetic (no checkpoint/network)", "workspace_gb": eng.workspace_bytes(B, n) / 1e9 if not ssr else eng.plan_cache_info()["bytes"] / 1e9,
                   "cuda_graphs": not args.no_graphs},
        "e2e": {"value": e2e, "unit": "clips/s", "h2d_bytes_per_step": B * n * 4, "d2h_bytes_per_step": B * n * 4,
                "ms_per_step": ms_e2e / args.steps, "rtf": e2e * seconds},
        "gpu_launches": int(launches),
        "stage_ms": stage,
        "parity": parity,
        "roofline": roofline,
        "slowest_launches": [{"label": r["label"], "ms": r["ms"], "tflops": (r["flops"] / (r["ms"] * 1e-3) / 1e12) if r["ms"] > 0 else 0} for r in slow],
        "cpu_baseline": cpu,
        "clocks": sampler.summary(),
    }
    print(json.dumps(line))


# ---------------------------------------------------------------------------------------------- long form (configs[4])
def run_longform(args):
    """BASELINE configs[4]: one 30-minute stream on 1 x H100.  Three schedules over the same engine:
    (a) handler(): independent 60 s segments one at a time, hard cuts (eval_gsr_voicefixer.py:47-75) - bit-compatible;
    (b) the same segments batched `--batch` at a time (they are independent, so the bits do not change);
    (c) 30 s windows with 2 s context margins (tools/dsp/overlapadd_boxcar.py:416-510), middle windows batched."""
    from voicefixer_main_b200 import VoiceFixer
    from voicefixer_main_b200 import handler as H
    from voicefixer_main_b200.longform import restore_longform
    from voicefixer_main_b200.weights import make_state
    from oracle import vf_oracle as O
    if not torch.cuda.is_available():
        raise SystemExit("bench.py --workload longform needs a CUDA device")
    dev = torch.device("cuda", 0)
    seg = 60 * SR
    n_seg = int(args.minutes)
    n = n_seg * seg
    state = make_state(1234)
    model = VoiceFixer().load_state_dict(state).eval().to(dev)
    eng = model._engine()
    gb = args.batch if args.batch else 6
    host = torch.cat([synth_batch(1, seg, 500 + i) for i in range(n_seg)], dim=1)[0].pin_memory()     # [N]
    out_host = torch.empty_like(host).pin_memory()

    def hard_cuts():      # (a): what handler() does, segment by segment, through the host entry point
        for i in range(n_seg):
            model.restore_host(host[None, i * seg:(i + 1) * seg], out_host[None, i * seg:(i + 1) * seg])

    def batched():        # (b)
        for i in range(0, n_seg, gb):
            k = min(gb, n_seg - i)
            model.restore_host(host[i * seg:(i + k) * seg].view(k, seg), out_host[i * seg:(i + k) * seg].view(k, seg))

    res = {}
    sampler = ClockSampler(0)
    sampler.start()
    for name, fn in (("handler_hard_cuts_batch1", hard_cuts), (f"segments_batched_{gb}", batched)):
        fn()                                              # warm-up (plans, graphs)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        res[name] = {"ms_per_stream": ms, "rtf": n / SR / (ms * 1e-3), "keep": out_host.clone() if name.startswith("handler") else None}
        if not name.startswith("handler"):
            res[name]["bit_identical_to_hard_cuts"] = bool(torch.equal(out_host, res["handler_hard_cuts_batch1"]["keep"]))
    ref_out = res["handler_hard_cuts_batch1"].pop("keep")
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, {"wav": ref_out})           # the handler schedule's stream, last timed step
    res[f"segments_batched_{gb}"].pop("keep")
    ws_seg = eng.workspace_bytes(1, seg) / 1e9
    ws_b = eng.workspace_bytes(gb, seg) / 1e9
    # (c) margins: device-resident input (the OLA wrapper slices on the device)
    dev_in = host.to(dev)[None]
    restore_longform(model, dev_in, max_batch=gb)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out_m = restore_longform(model, dev_in, max_batch=gb)
    e1.record()
    torch.cuda.synchronize()
    ms_m = e0.elapsed_time(e1)
    res["margins_30s_windows_2s_context"] = {"ms_per_stream": ms_m, "rtf": n / SR / (ms_m * 1e-3), "windows": (n + 30 * SR - 1) // (30 * SR)}
    sampler.stop_flag = True
    eng.check_errors()
    # parity of one 60 s segment against the oracle (the reference's handler on the CPU)
    parity = None
    if not args.no_cpu_baseline:
        torch.set_num_threads(min(16, os.cpu_count() or 1))
        t0 = time.perf_counter()
        with torch.no_grad():
            ref = O.restore(state, host[None, :seg].clone())
        cpu_s = time.perf_counter() - t0
        parity = {"segment": 0, "wav_rms_vs_oracle": float((ref_out[:seg] - ref[0]).double().pow(2).mean().sqrt()), "bar": 1e-3,
                  "oracle_cpu_seconds_for_60s": cpu_s, "cpu_rtf": 60.0 / cpu_s}
    best = max(res.values(), key=lambda r: r["rtf"])
    line = {"metric": "rtf_30min_longform_44k1", "value": res["handler_hard_cuts_batch1"]["rtf"], "unit": "x real time", "n_gpus": 1, "steps": args.steps, "warmup": 1,
            "ms_per_step": res["handler_hard_cuts_batch1"]["ms_per_stream"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f16 tensor-core (UNet hi/lo split; vocoder hi-only), f32 accumulate", "data": "synthetic",
            "config": {"workload": f"{n_seg}-minute long-form restoration as {n_seg} x 60 s segments (T = 6001 -> T' = 6016), 1 x H100 (BASELINE configs[4]); value = handler() schedule "
                                   "through the host entry point (H2D + D2H inside)", "minutes": n_seg, "segment_batch": gb,
                       "workspace_gb_batch1": ws_seg, f"workspace_gb_batch{gb}": ws_b, "plan_cache": eng.plan_cache_info()},
            "schedules": res, "best_rtf": best["rtf"], "parity": parity,
            "e2e": {"value": res["handler_hard_cuts_batch1"]["rtf"], "unit": "x real time", "h2d_bytes_per_step": n * 4, "d2h_bytes_per_step": n * 4},
            "gpu_launches": int(eng.launch_count()), "clocks": sampler.summary()}
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--workload", default="gsr", choices=["gsr", "ssr", "longform"])
    ap.add_argument("--batch", type=int, default=0, help="clips per GPU per step (default 32 gsr / 64 ssr; longform: segments per call, default 6)")
    ap.add_argument("--seconds", type=float, default=0.0, help="clip length (default 10 gsr / 3 ssr = the SSR config's input_segment_length)")
    ap.add_argument("--minutes", type=float, default=30.0, help="longform: stream length")
    ap.add_argument("--vocoder-terms", type=int, default=0, choices=[0, 1, 3])
    ap.add_argument("--no-graphs", action="store_true", help="launch every kernel individually instead of replaying CUDA graphs")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--profile-out", default="", help="write the per-launch profile (JSON) to this file")
    ap.add_argument("--dump-outputs", default="", metavar="DIR",
                    help="write what the last timed step computed as DIR/<name>.npy (float32, at most 64 MB in all)")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3) if args.impl == "b200" else args.warmup
    if args.impl == "reference":
        run_reference(args)
    elif args.workload == "longform":
        run_longform(args)
    else:
        run_b200(args)
    import torch.distributed as tdist
    if tdist.is_available() and tdist.is_initialized():
        tdist.destroy_process_group()


if __name__ == "__main__":
    main()
