#!/usr/bin/env python
"""Decoding a test set of 24-bit stereo 48 kHz WAV files to librosa.load's mono float32 samples, on the host and on the GPU.

    python tools/bench_wav_decode.py [--files 32] [--seconds 10] [--reps 7] [--warmup 2]

The files are seeded and held in memory, parsed once (voicefixer_main_b200.wavfile), so neither arm reads a disk.  Two arms
run alternately on the same files and must give the same bits:
- "host_numpy": the numpy restatement (oracle/wavfile.py: libsndfile's conversion, then numpy's channel mean) of every
  file, then one copy of the packed float32 mono samples to the device (where every consumer of them runs);
- "gpu": Engine.decode_pcm_varlen on every file in one call: the data chunks into one pinned staging buffer, one
  host-to-device copy of the raw 3-byte samples, one decode launch.
Each rep is timed with CUDA events after a device synchronise (the host arm's events enclose its host work and its copy);
medians are reported, with audio seconds decoded per second.  A separate pass under torch.profiler sums the device time of
decode_pcm_kernel alone.  Prints one JSON line with the card's name and power limit, read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_varlen import card_info                     # noqa: E402
from oracle import wavfile as O                        # noqa: E402
from voicefixer_main_b200 import wavfile as W          # noqa: E402
from voicefixer_main_b200.model import Engine          # noqa: E402

RATE = 48000


def make_files(n_files, seconds, seed=0):
    """Seeded 24-bit stereo files as parsed WavInfos: two detuned tones in noise, about -6 dBFS."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n_files):
        n = int(seconds * RATE) + int(rng.integers(0, RATE))
        t = np.arange(n) / RATE
        x = np.stack([0.3 * np.sin(2 * np.pi * (220 + 7 * i + 3 * c) * t) + 0.05 * rng.standard_normal(n) for c in range(2)], 1)
        raw = O.wav_bytes(O.encode(np.round(x * (2 ** 23 - 1)).astype(np.int64), W.S24), RATE, 2, W.S24)
        path = f"<memory {i}>"
        out.append(W.WavInfo(path, RATE, 2, W.S24, n, memoryview(raw)[len(raw) - n * 6:]))
    return out


def host_arm(files, device):
    mono = np.concatenate([O.downmix(O.samples(w.data, w.channels, w.format)) for w in files])
    return torch.from_numpy(mono).to(device)


def gpu_arm(eng, files):
    return eng.decode_pcm_varlen(files)[0]


def timed(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_wav_decode needs a CUDA device")
    eng = Engine("cuda:0")
    files = make_files(args.files, args.seconds)
    audio_s = sum(w.frames for w in files) / RATE
    arms = {"host_numpy": lambda: host_arm(files, eng.device), "gpu": lambda: gpu_arm(eng, files)}
    for _ in range(args.warmup):
        outs = {k: fn() for k, fn in arms.items()}
    if not torch.equal(outs["host_numpy"].view(torch.int32), outs["gpu"].view(torch.int32)):
        raise SystemExit("the two arms disagree")
    times = {k: [] for k in arms}
    for _ in range(args.reps):
        for k, fn in arms.items():
            times[k].append(timed(fn)[0])
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            gpu_arm(eng, files)
        torch.cuda.synchronize()
    kernel_us = sum(e.device_time_total for e in prof.key_averages() if "decode_pcm_kernel" in e.key) / args.reps
    eng.check_errors()
    res = {"files": args.files, "audio_seconds": round(audio_s, 2), "bytes_per_call": sum(len(w.data) for w in files),
           "bits_identical": True, "card": card_info(0)}
    for k, ts in times.items():
        med = statistics.median(ts)
        res[k] = {"median_ms": round(med, 3), "min_ms": round(min(ts), 3), "max_ms": round(max(ts), 3),
                  "audio_s_per_s": round(audio_s / (med / 1e3), 1)}
    res["decode_kernel_ms_per_call"] = round(kernel_us / 1e3, 4)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
