#!/usr/bin/env python
"""Benchmark of clips of different lengths (vf_restore_varlen / VoiceFixer.restore_batch) on one GPU.

    python tools/bench_varlen.py [--workload gsr|ssr] [--batch B] [--seconds S] [--steps K] [--warmup W] [--dump-outputs DIR]

A step restores `--batch` clips of seeded lengths, uniform in [1 s, `--seconds`] (default 32 clips, 10 s), the way a test
set or a request queue arrives.  `--workload ssr` runs the same on the SSR / GSR-UNet path (SSR_UNet.restore_batch,
vf_ssr_restore_varlen) with lengths up to 3 s by default, the SSR config's input_segment_length.  Alternating in one process, it times ONE restore_batch call (one launch chain) and one
restore() per clip (what handler() does), checks that the two return the same bits, and prints one JSON line with clips/s
and audio-seconds/s of both arms plus the card's name and power limit.  The synthetic clips, the clock sampler and the
output dump are bench.py's.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import SR, ClockSampler, dump_outputs, synth_batch  # noqa: E402


def card_info(index):
    """Name and power limit of the card the numbers were taken on (read-only query)."""
    try:
        out = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        name, limit = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": limit}
    except Exception:
        return {"name": torch.cuda.get_device_name(index), "power_limit": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=("gsr", "ssr"), default="gsr",
                    help="gsr: VoiceFixer.restore_batch; ssr: SSR_UNet.restore_batch (unet_v2 + ISTFT)")
    ap.add_argument("--batch", type=int, default=32, help="clips per step")
    ap.add_argument("--seconds", type=float, default=None,
                    help="longest clip (lengths are uniform in [1 s, this]); default 10 (gsr) or 3 (ssr)")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dump-outputs", default="", metavar="DIR", help="write the varlen arm's last output as DIR/wav.npy")
    args = ap.parse_args()
    from voicefixer_main_b200 import SSR_UNet, VoiceFixer
    from voicefixer_main_b200.weights import make_ssr_state, make_state
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_varlen.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    ssr = args.workload == "ssr"
    B, top = args.batch, args.seconds if args.seconds is not None else (3.0 if ssr else 10.0)
    g = torch.Generator().manual_seed(2024)
    lengths = [int(SR * (1.0 + (top - 1.0) * float(u))) for u in torch.rand(B, generator=g)]
    clips = [synth_batch(1, n, 900 + i)[0].to(dev) for i, n in enumerate(lengths)]
    if ssr:
        model = SSR_UNet().load_state_dict(make_ssr_state(1234)).eval().to(dev)
    else:
        model = VoiceFixer().load_state_dict(make_state(1234)).eval().to(dev)
    eng = model._engine()

    arms = {"varlen_one_call": lambda: model.restore_batch(clips),
            "restore_per_clip": lambda: [model.restore(c[None])[0] for c in clips]}
    for fn in arms.values():                              # warm-up: plans, graph capture
        for _ in range(args.warmup):
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    outs = {}
    sampler = ClockSampler(0)
    sampler.start()
    for _ in range(args.steps):
        for k, fn in arms.items():                        # alternating: both arms see the same clocks and neighbours
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            outs[k] = fn()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1))
    sampler.stop_flag = True
    eng.check_errors()
    same = all(torch.equal(a, b) for a, b in zip(outs["varlen_one_call"], outs["restore_per_clip"]))
    audio_s = sum(lengths) / SR
    res = {}
    for k, v in ms.items():
        med = sorted(v)[len(v) // 2]
        res[k] = {"ms_per_step_median": med, "ms_min": min(v), "ms_max": max(v), "clips_per_sec": B / (med * 1e-3),
                  "audio_seconds_per_sec": audio_s / (med * 1e-3)}
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, {"wav": torch.cat(outs["varlen_one_call"])})
    entry = "SSR_UNet, vf_ssr_restore_varlen" if ssr else "vf_restore_varlen"
    line = {"metric": ("ssr_" if ssr else "") + "clips_per_sec_varlen_44k1", "value": res["varlen_one_call"]["clips_per_sec"],
            "unit": "clips/s", "steps": args.steps, "warmup": args.warmup, "ms_per_step": res["varlen_one_call"]["ms_per_step_median"],
            "higher_is_better": True, "data": "synthetic",
            "config": {"workload": f"{B} clips of seeded lengths uniform in [1, {top:g}] s, 44.1 kHz, device-resident; value = one "
                                   f"{entry} call per step", "batch": B, "total_audio_seconds": audio_s,
                       "lengths": lengths, "plan_cache": eng.plan_cache_info()},
            "arms": res, "speedup_vs_per_clip": res["restore_per_clip"]["ms_per_step_median"] / res["varlen_one_call"]["ms_per_step_median"],
            "bit_identical_to_per_clip": bool(same), "card": card_info(0), "gpu_launches": int(eng.launch_count()),
            "clocks": sampler.summary()}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
