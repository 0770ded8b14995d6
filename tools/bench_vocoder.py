#!/usr/bin/env python
"""Benchmark of the stand-alone vocoder (voicefixer_main_b200.vocoder.Vocoder) on one GPU.

    python tools/bench_vocoder.py [--clips N] [--steps K] [--warmup W]

A step vocodes N seeded mels of lengths uniform in [1 s, 10 s] plus one of 60 s (the mels of synthetic speech), and
resynthesises the same clips.  It times
  - forward_batch: one vf_vocoder_varlen call per group of similar lengths (vocoder.length_groups), against one call for
    all mels in their given order (every sub-batch on the bucket of its longest mel) and Vocoder.forward per mel;
  - resynth_batch: one vf_resynth_varlen call per group of similar lengths, against the composed per-clip calls vf_frontend ->
    vf_vocoder -> vf_finalize on a context that also holds the analysis module (what a caller without the packed call
    does),
each pair of arms alternating on contexts of their own (the one-call arm alone).  It checks that all arms give the same
bits and prints one JSON line with audio-seconds/s of every arm, the plan bytes per clip and padded frame of a
vocoder-only plan (both vocoder modes) against the restore plan's, the sub-batch each allows at a 10 s bucket, and the
card's name and power limit.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from bench import SR, ClockSampler, synth_batch  # noqa: E402
from bench_varlen import card_info  # noqa: E402


def plan_bytes_per_frame(make_engine, call, batch, bucket):
    """Plan bytes per clip and padded frame of the one plan `call(engine)` builds for `batch` clips at `bucket` frames."""
    e = make_engine()
    try:
        call(e)
        torch.cuda.synchronize()
        info = e.plan_cache_info()
        assert info["plans"] == 1, info
        return info["bytes"] / (batch * bucket)
    finally:
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=16, help="mels of 1-10 s per step, plus one of 60 s")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    from voicefixer_main_b200.model import Engine
    from voicefixer_main_b200.vocoder import Vocoder, packing
    from voicefixer_main_b200.weights import make_state
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_vocoder.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    state = make_state(1234)
    voc_sd = {k: v for k, v in state.items() if k.startswith("vocoder.")}
    g = torch.Generator().manual_seed(2026)
    lengths = [int(SR * (1.0 + 9.0 * float(u))) for u in torch.rand(args.clips, generator=g)] + [60 * SR]
    clips = [synth_batch(1, n, 700 + i)[0].to(dev) for i, n in enumerate(lengths)]

    full = Engine(dev)
    full.load_state(state, need=("unet", "vocoder"))
    mels = [full.frontend(c[None])[0][0] for c in clips]
    frames = [m.shape[0] for m in mels]
    packed = torch.cat(mels)
    _, s_off = packing(frames)

    def timed(arms):
        """Median ms per step of each arm (warm-up first, then the arms alternate step by step) and each arm's last output"""
        for fn in arms.values():                          # warm-up: plans, graph capture
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        ms, outs = {k: [] for k in arms}, {}
        for _ in range(args.steps):
            for k, fn in arms.items():                    # alternating: every arm sees the same clocks and neighbours
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                outs[k] = fn()
                e1.record()
                torch.cuda.synchronize()
                ms[k].append(e0.elapsed_time(e1))
        return ms, outs

    # Each phase on contexts of its own, closed after it: the arms of one context share its plan cache, and one arm's
    # plans would evict another's (a process serving one kind of call keeps its own plans cached).
    sampler = ClockSampler(0)
    sampler.start()
    voc = Vocoder().load_state_dict(voc_sd).eval().to(dev)
    ms, outs = timed({"forward_batch": lambda: voc.forward_batch(mels),
                      "forward_per_clip": lambda: [voc.forward(m[None, None])[0, 0] for m in mels]})
    voc._engine().check_errors()
    voc._engine().close()
    one = Vocoder().load_state_dict(voc_sd).eval().to(dev)
    m1, o1 = timed({"forward_one_call": lambda: list(torch.split(one._engine().vocoder_varlen(packed, frames),
                                                                 [s_off[i + 1] - s_off[i] for i in range(len(frames))]))})
    one._engine().check_errors()
    one._engine().close()
    voc = Vocoder().load_state_dict(voc_sd).eval().to(dev)
    m2, o2 = timed({"resynth_batch": lambda: voc.resynth_batch(clips),
                    "composed_per_clip": lambda: [full.finalize(full.vocoder(m[None]), c.numel())[0] for m, c in zip(mels, clips)]})
    sampler.stop_flag = True
    ms.update(m1); ms.update(m2); outs.update(o1); outs.update(o2)
    voc._engine().check_errors()
    full.check_errors()
    same = {"forward": all(torch.equal(a, b) and torch.equal(a, c) for a, b, c in
                           zip(outs["forward_batch"], outs["forward_per_clip"], outs["forward_one_call"])),
            "resynth": all(torch.equal(a, b) for a, b in zip(outs["resynth_batch"], outs["composed_per_clip"]))}
    audio_s = sum(lengths) / SR
    res = {}
    for k, v in ms.items():
        med = sorted(v)[len(v) // 2]
        res[k] = {"ms_per_step_median": med, "ms_min": min(v), "ms_max": max(v), "audio_seconds_per_sec": audio_s / (med * 1e-3)}
    plans = {"vocoder_only": voc._engine().plan_cache_info(), "full": full.plan_cache_info()}
    voc._engine().close()
    full.close()

    # plan bytes per clip and padded frame: 8 clips of 10 s (bucket 1024) on fresh contexts
    ten = torch.cat([c[:10 * SR] for c in [synth_batch(1, 10 * SR, 50 + i)[0].to(dev) for i in range(8)]])

    def engine(need, terms):
        def make():
            e = Engine(dev)
            e.load_state(state if "unet" in need else voc_sd, need=need)
            e.set_option("vocoder_terms", terms)
            return e
        return make

    per_frame = {
        "restore_voc1": plan_bytes_per_frame(engine(("unet", "vocoder"), 1), lambda e: e.restore_varlen(ten, [10 * SR] * 8), 8, 1024),
        "vocoder_only_voc1": plan_bytes_per_frame(engine(("vocoder",), 1), lambda e: e.resynth_varlen(ten, [10 * SR] * 8), 8, 1024),
        "vocoder_only_voc3": plan_bytes_per_frame(engine(("vocoder",), 3), lambda e: e.resynth_varlen(ten, [10 * SR] * 8), 8, 1024),
    }
    sub = {}
    for name, need, kind in (("restore", ("unet", "vocoder"), 2), ("vocoder_only", ("vocoder",), 5)):
        e = engine(need, 1)()
        e.set_option("plan_cache_mb", 16 * 1024)
        sub[name] = e.selftest_sub_batch(kind, 256, 1024)
        e.close()
    line = {"metric": "audio_seconds_per_sec_vocoder_forward_batch_44k1", "value": res["forward_batch"]["audio_seconds_per_sec"],
            "unit": "audio-s/s", "steps": args.steps, "warmup": args.warmup, "higher_is_better": True, "data": "synthetic",
            "config": {"workload": f"{args.clips} mels of seeded lengths uniform in [1, 10] s and one of 60 s (the front end's "
                                   "mels of synthetic speech), device-resident", "total_audio_seconds": audio_s,
                       "lengths": lengths, "frames": frames},
            "arms": res,
            "speedup_forward_batch_vs_per_clip": res["forward_per_clip"]["ms_per_step_median"] / res["forward_batch"]["ms_per_step_median"],
            "speedup_resynth_batch_vs_composed": res["composed_per_clip"]["ms_per_step_median"] / res["resynth_batch"]["ms_per_step_median"],
            "bit_identical": same, "plan_cache_after_run": plans, "plan_bytes_per_clip_frame": per_frame,
            "sub_batch_at_10s_bucket_16GiB": sub, "card": card_info(0), "clocks": sampler.summary()}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
