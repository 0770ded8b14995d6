#!/usr/bin/env python
"""Benchmark of a test-set evaluation: handler() once per file against one handler_batch() call, on one GPU.

    python tools/bench_testset.py --out DIR [--files F] [--steps K] [--workload gsr|ssr]

Writes a seeded synthetic test set under DIR/set: F PCM16 files (default 64) of lengths uniform in [1 s, 10 s] at 44.1 kHz,
plus one 61 s file (two segments) and two 22.05 kHz files, with clean targets for every other file.  In one process it
times evaluation_proc/eval.py's schedule (handler() per file, outputs under DIR/per_file) against handler_batch() over the
whole set (DIR/batch).  Both include decoding, resampling, the metrics and writing the wav files.  Each arm's first run
over the set, which builds its plans, is timed on its own (first_run_*: one evaluation of a test set in a fresh process,
after one warm-up file); then the two arms alternate for --steps runs with their plans cached as far as the plan budget
allows.  It checks that the two arms wrote byte-identical files and equal metrics, and prints one JSON line with files/s
and audio-seconds/s of both arms, the plans each evicted per run, and the card's name and power limit.
--workload gsr (the default) runs VoiceFixer through handler.py; --workload ssr runs SSR_UNet through handler_unet.py
(eval_gsr_unet.py / eval_ssr_unet.py's handler) on the same set.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_varlen import card_info  # noqa: E402


def write_set(H, d, n_files, seed):
    """(input, output name, target) items and the audio seconds of the seeded test set written under d."""
    from oracle import vf_oracle as O
    g = np.random.default_rng(seed)
    spec = [(int(44100 * g.uniform(1.0, 10.0)), 44100) for _ in range(n_files)]
    spec += [(44100 * 61, 44100), (int(22050 * 2.5), 22050), (int(22050 * 7.3), 22050)]
    os.makedirs(d, exist_ok=True)
    items, seconds = [], 0.0
    for i, (n, rate) in enumerate(spec):
        src = os.path.join(d, f"in{i}.wav")
        H.save_pcm16(O.to_int16(O.synth_clips(1, n, seed=seed + i)[0].clamp(-0.99, 0.99).numpy()), src, sample_rate=rate)
        tgt = None
        if i % 2 == 0:
            tgt = os.path.join(d, f"tgt{i}.wav")
            H.save_pcm16(O.to_int16(O.synth_clips(1, n, seed=seed + 10000 + i)[0].clamp(-0.99, 0.99).numpy()), tgt, sample_rate=rate)
        items.append((src, f"out{i}.wav", tgt))
        seconds += n / rate
    return items, seconds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the test set and both arms' outputs")
    ap.add_argument("--files", type=int, default=64, help="files of 1 - 10 s (plus the 61 s and the two 22.05 kHz files)")
    ap.add_argument("--steps", type=int, default=3, help="timed runs of each arm")
    ap.add_argument("--seed", type=int, default=4242)
    ap.add_argument("--workload", choices=("gsr", "ssr"), default="gsr",
                    help="gsr: VoiceFixer through handler.py; ssr: SSR_UNet through handler_unet.py")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_testset.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    if args.workload == "ssr":
        from voicefixer_main_b200 import SSR_UNet
        from voicefixer_main_b200 import handler_unet as H
        from voicefixer_main_b200.weights import make_ssr_state
        H.model = SSR_UNet().load_state_dict(make_ssr_state(1234)).eval().to(dev)
    else:
        from voicefixer_main_b200 import VoiceFixer
        from voicefixer_main_b200 import handler as H
        from voicefixer_main_b200.weights import make_state
        H.model = VoiceFixer().load_state_dict(make_state(1234)).eval().to(dev)
    items, audio_s = write_set(H, os.path.join(args.out, "set"), args.files, args.seed)
    dirs = {k: os.path.join(args.out, k) for k in ("per_file", "batch")}
    for d in dirs.values():
        os.makedirs(d, exist_ok=True)
    arms = {
        "per_file": lambda: [H.handler(s, os.path.join(dirs["per_file"], o), t, None, dev) for s, o, t in items],
        "batch": lambda: H.handler_batch([(s, os.path.join(dirs["batch"], o), t) for s, o, t in items], None, dev),
    }
    eng = H.model._engine()
    metrics, secs, evicted = {}, {k: [] for k in arms}, {k: 0 for k in arms}

    def run(k):
        torch.cuda.synchronize()
        ev0, t0 = eng.plan_cache_info()["evicted"], time.perf_counter()
        metrics[k] = arms[k]()
        torch.cuda.synchronize()
        evicted[k] += eng.plan_cache_info()["evicted"] - ev0
        return time.perf_counter() - t0

    # the kernels' first launches (module loading, function attributes) on a file outside the set, so that each arm's
    # first run over the set - what one evaluation of a test set costs, plan builds included - is timed on its own
    from oracle import vf_oracle as O
    warm = os.path.join(args.out, "warmup_in.wav")
    H.save_pcm16(O.to_int16(O.synth_clips(1, 66150, seed=args.seed - 1)[0].clamp(-0.99, 0.99).numpy()), warm)
    H.handler(warm, os.path.join(args.out, "warmup_out.wav"), None, None, dev)
    first = {k: run(k) for k in arms}
    evicted = {k: 0 for k in arms}
    for _ in range(args.steps):
        for k in arms:                                      # alternating: both arms see the same clocks and neighbours
            secs[k].append(run(k))
    eng.check_errors()

    def read(arm, name):
        with open(os.path.join(dirs[arm], name), "rb") as f:
            return f.read()

    same_files = all(read("per_file", o) == read("batch", o) for _, o, _ in items)
    res = {}
    for k, v in secs.items():
        med = sorted(v)[len(v) // 2]
        res[k] = {"s_median": med, "s_min": min(v), "s_max": max(v), "files_per_sec": len(items) / med,
                  "audio_seconds_per_sec": audio_s / med, "plans_evicted_per_run": evicted[k] / len(v),
                  "first_run_s": first[k], "first_run_files_per_sec": len(items) / first[k]}
    line = {"metric": "files_per_sec_testset_44k1" + ("_ssr" if args.workload == "ssr" else ""), "value": res["batch"]["files_per_sec"], "unit": "files/s",
            "steps": args.steps, "higher_is_better": True, "data": "synthetic",
            "config": {"workload": f"{len(items)} PCM16 files ({args.files} of 1 - 10 s, one of 61 s, two at 22.05 kHz), "
                                   f"targets on every other file; value = one "
                                   f"{'handler_unet.' if args.workload == 'ssr' else ''}handler_batch call", "files": len(items),
                       "total_audio_seconds": audio_s, "plan_cache": H.model._engine().plan_cache_info()},
            "arms": res, "speedup_vs_per_file": res["per_file"]["s_median"] / res["batch"]["s_median"],
            "first_run_speedup_vs_per_file": first["per_file"] / first["batch"],
            "files_identical": bool(same_files), "metrics_equal": metrics["per_file"] == metrics["batch"],
            "card": card_info(0)}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
