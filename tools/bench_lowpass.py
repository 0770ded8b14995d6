#!/usr/bin/env python
"""Benchmark of building the SR validation inputs (lowpass.sr_validation_inputs, collate_fn_val's recipe) on one GPU.

    python tools/bench_lowpass.py [--clips N] [--steps K]

Makes N seeded speech-like clips (default 64) of 3-10 s at 44.1 kHz plus one 60 s clip, then times two arms, alternating,
for K rounds (after one untimed warm-up of each): one sr_validation_inputs() call over all clips and the five cutoffs
(ending in a device synchronise), and the CPU recipe (oracle/lowpass.py: scipy sosfiltfilt + two resample_poly calls per
clip and cutoff, float64), which is a single-threaded loop: one host core.  It reports the largest difference between the
arms (float32 outputs: at most one float32 rounding is expected) and prints one JSON line with every round's time, audio
seconds per second per arm (best round), and the card's name and power limit.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_varlen import card_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--steps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lowpass needs a CUDA device")
    from oracle import lowpass as O
    from oracle import vf_oracle as VO
    from voicefixer_main_b200 import lowpass as LP
    from voicefixer_main_b200.model import Engine

    g = np.random.default_rng(17)
    lengths = [int(44100 * g.uniform(3.0, 10.0)) for _ in range(a.clips)] + [44100 * 60]
    clips = [VO.synth_clips(1, n, seed=i)[0].numpy() for i, n in enumerate(lengths)]
    seconds = sum(lengths) / 44100 * len(O.SR_CUTOFFS)
    eng = Engine("cuda:0")

    def gpu():
        out = LP.sr_validation_inputs(eng, clips)
        torch.cuda.synchronize()
        return out

    gpu_out, cpu_out = gpu(), O.collate_val(clips)
    times = {"gpu": [], "cpu": []}
    for _ in range(a.steps):
        t0 = time.perf_counter()
        gpu_out = gpu()
        times["gpu"].append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        cpu_out = O.collate_val(clips)
        times["cpu"].append(time.perf_counter() - t0)
    diff = max(float(np.abs(gg.cpu().numpy() - cc).max()) for c in O.SR_CUTOFFS for gg, cc in zip(gpu_out[c], cpu_out[c]))
    ulps = max(float((np.abs(gg.cpu().numpy() - cc) / np.spacing(np.abs(cc))).max())
               for c in O.SR_CUTOFFS for gg, cc in zip(gpu_out[c], cpu_out[c]))
    res = {"clips": len(clips), "audio_s_per_cutoff": round(sum(lengths) / 44100, 2), "cutoffs": list(O.SR_CUTOFFS),
           "gpu_s": [round(t, 4) for t in times["gpu"]], "cpu_s": [round(t, 4) for t in times["cpu"]],
           "gpu_audio_s_per_s": round(seconds / min(times["gpu"]), 1),
           "cpu_audio_s_per_s": round(seconds / min(times["cpu"]), 1),
           "max_abs_diff": diff, "max_diff_float32_ulps": ulps, "cpu_arm_cores": 1, "host_cores": os.cpu_count(),
           "card": card_info(0)}
    print(json.dumps(res))
    eng.close()


if __name__ == "__main__":
    main()
