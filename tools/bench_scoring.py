#!/usr/bin/env python
"""Benchmark of scoring a test set (AudioMetrics.evaluation over (restored, target) pairs) on one GPU.

    python tools/bench_scoring.py [--files F] [--steps K] [--dir DIR]

Writes a seeded set of F PCM16 pairs (default 64) of 1-10 s at 44.1 kHz plus one 61 s pair to DIR (default: a temporary
directory), then times three arms, alternating, for K rounds: one evaluation_batch() call over the set, evaluation() per
pair, and the CPU restatement (oracle/scoring.py: numpy / scipy / torch, the arithmetic of librosa 0.8 and scikit-image
0.18) per pair, on the host's cores.  All arms include decoding the wavs.  It checks that the arms agree (GPU arms
exactly; GPU vs CPU within 1e-3 relative for lsd / sispec - the CPU arm sums up to millions of values in torch fp32, the
kernels in fp64 - and 1e-6 absolute for ssim), reports the largest deviation per key, and prints one JSON line with files/s
and audio seconds/s per arm, the host's core count, and the card's name and power limit.
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_varlen import card_info  # noqa: E402


def write_pairs(d, n_files, seed):
    from oracle import scoring as S
    from oracle import vf_oracle as O
    g = np.random.default_rng(seed)
    lengths = [int(44100 * g.uniform(1.0, 10.0)) for _ in range(n_files)] + [44100 * 61]
    pairs = []
    for i, n in enumerate(lengths):
        t = O.synth_clips(1, n, seed=seed + i)[0].clamp(-0.9, 0.9).numpy()
        e = t + 0.05 * O.synth_clips(1, n, seed=seed + 10000 + i)[0].numpy()
        pe, pt = os.path.join(d, f"est{i}.wav"), os.path.join(d, f"tgt{i}.wav")
        S.write_pcm16(O.to_int16(np.clip(e, -0.99, 0.99)), pe)
        S.write_pcm16(O.to_int16(t), pt)
        pairs.append((pe, pt))
    return pairs, sum(lengths) / 44100


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=64)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--dir", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_scoring needs a CUDA device")
    from oracle import scoring as S
    from voicefixer_main_b200.edges import AudioMetrics
    from voicefixer_main_b200.model import Engine
    eng = Engine("cuda:0")
    eng.load_state({}, need=())
    am = AudioMetrics(eng)
    with tempfile.TemporaryDirectory() as tmp:
        d = args.dir or tmp
        os.makedirs(d, exist_ok=True)
        pairs, seconds = write_pairs(d, args.files, 4242)
        arms = {
            "gpu_batch": lambda: am.evaluation_batch(pairs),
            "gpu_per_file": lambda: [am.evaluation(pe, pt) for pe, pt in pairs],
            "cpu_per_file": lambda: [S.evaluation(pe, pt) for pe, pt in pairs],
        }
        am.evaluation_batch(pairs[:2])          # warm-up: module load, scratch
        times = {k: [] for k in arms}
        results = {}
        for _ in range(args.steps):
            for k, fn in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                results[k] = fn()
                torch.cuda.synchronize()
                times[k].append(time.perf_counter() - t0)
    assert results["gpu_batch"] == results["gpu_per_file"], "evaluation_batch differs from evaluation"
    worst = dict.fromkeys(S.KEYS, 0.0)            # ssim: absolute; the others: relative (absolute below 1)
    for g, c in zip(results["gpu_batch"], results["cpu_per_file"]):
        for k in S.KEYS:
            d = abs(g[k] - c[k]) if k.endswith("ssim") else abs(g[k] - c[k]) / max(1.0, abs(c[k]))
            worst[k] = max(worst[k], d)
    assert all(v < (1e-6 if k.endswith("ssim") else 1e-3) for k, v in worst.items()), worst
    n = len(pairs)
    res = {"files": n, "audio_s": round(seconds, 1), "host_cores": os.cpu_count(), "torch_threads": torch.get_num_threads(),
           "max_deviation_vs_cpu": worst, **card_info(0)}
    for k, ts in times.items():
        res[f"{k}_files_per_s"] = [round(n / t, 2) for t in ts]
        res[f"{k}_audio_s_per_s"] = [round(seconds / t, 1) for t in ts]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
