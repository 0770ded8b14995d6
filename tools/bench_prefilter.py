"""The pip package's mode-1 pre-filter on the GPU (VoiceFixer.remove_higher_frequency_batch, vf_remove_higher_frequency_varlen)
against the per-file numpy restatement in the package's dtypes (oracle/prefilter.py) on the host cores, and what it adds to a
restore: restore_batch of the same files with and without it.

Twelve seeded speech-like files of 10-30 s (the package filters 30 s segments, so these are one segment each).  GPU times
are CUDA-event medians after a warm-up call; a separate torch.profiler pass gives each kernel's share.  The card's name and
power limit are read in the same run.

    python tools/bench_prefilter.py [--files 12] [--reps 10] [--host-files 12]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from oracle import prefilter as P                                # noqa: E402
from oracle import vf_oracle as O                                # noqa: E402
from voicefixer_main_b200 import VoiceFixer                      # noqa: E402
from voicefixer_main_b200.weights import make_state              # noqa: E402


def _files(n, seed):
    rng = np.random.default_rng(seed)
    lengths = [int(rng.integers(10 * 44100, 30 * 44100 + 1)) for _ in range(n)]
    return [O.synth_clips(1, m, seed=seed + i)[0].numpy() for i, m in enumerate(lengths)]


def _gpu_time(fn, reps):
    fn()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(reps):
        start.record()
        fn()
        stop.record()
        stop.synchronize()
        times.append(start.elapsed_time(stop))
    return float(np.median(times)), float(np.min(times)), float(np.max(times))


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=12)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--host-files", type=int, default=12)
    a = ap.parse_args()
    print(json.dumps({"card": _card(), "host_cores": os.cpu_count()}))
    xs = _files(a.files, 2024)
    audio_s = sum(len(x) for x in xs) / 44100
    model = VoiceFixer().load_state_dict(make_state(1234)).eval().to("cuda:0")
    eng = model._engine()
    dev = [torch.from_numpy(x).cuda() for x in xs]
    frames = sum(1 + len(x) // 512 for x in xs)
    res = {"files": len(xs), "audio_s": round(audio_s, 2), "frames": frames}
    med, lo, hi = _gpu_time(lambda: model.remove_higher_frequency_batch(dev), a.reps)
    res.update(prefilter_ms=round(med, 3), prefilter_ms_min=round(lo, 3), prefilter_ms_max=round(hi, 3),
               prefilter_ms_per_30s=round(med / audio_s * 30, 3), prefilter_audio_s_per_s=round(audio_s / med * 1e3, 1))
    # HBM traffic: each frame's 16.4 KB slot is written (spectrum), read twice (cutoff, inverse), written (frame) and read
    # once more by the overlap-add; each input sample is read by four frames and each output sample written once
    traffic = frames * 1025 * 16 * 5 + sum(len(x) for x in xs) * 4 * 5
    res["prefilter_traffic_gb"] = round(traffic / 1e9, 3)
    res["prefilter_gb_per_s"] = round(traffic / (med * 1e-3) / 1e9, 1)
    k = min(a.host_files, len(xs))
    t0 = time.perf_counter()
    for i in range(k):
        P.remove_higher_frequency_pkg(xs[i])
    dt = time.perf_counter() - t0
    res["host_numpy_pkg_dtypes_ms_per_30s"] = round(dt * 1e3 / (sum(len(xs[i]) for i in range(k)) / 44100) * 30, 1)
    filtered, cut = model.remove_higher_frequency_batch(dev)
    res["cutoffs"] = [int(c) for c in cut.cpu()]
    med_r, _, _ = _gpu_time(lambda: model.restore_batch(dev, unify_energy=True), a.reps)
    med_f, _, _ = _gpu_time(lambda: model.restore_batch(model.remove_higher_frequency_batch(dev)[0], unify_energy=True),
                            a.reps)
    res.update(restore_batch_ms=round(med_r, 2), prefilter_then_restore_batch_ms=round(med_f, 2),
               restore_ms_per_30s=round(med_r / audio_s * 30, 2))
    eng.check_errors()
    print(json.dumps(res))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            model.remove_higher_frequency_batch(dev)
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        m = re.search(r"prefilter_\w+_kernel", e.key)
        if m:
            kernels[m.group(0)] = round(e.device_time_total / 3 / 1e3, 3)
    print(json.dumps({"prefilter_kernel_ms_per_call": kernels}))
    model._eng.close()


if __name__ == "__main__":
    main()
