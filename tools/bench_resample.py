"""librosa.load's resampling on the GPU (vf_resample_sinc_varlen, res_type kaiser_best / kaiser_fast) against the numpy
restatement (oracle/resampy.py) on the host cores and the default resample_poly path, in audio-seconds per second.

Two seeded sets: 16 / 22.05 / 48 kHz files going up to 44.1 kHz (the inputs and targets of a restore), and 44.1 kHz files
going down to 16 kHz (the ests of a 16 kHz scoring).  Also prints the largest sample difference between kaiser_best and
resample_poly, and how much the 16 kHz spectral scores of a set of 44.1 kHz ests move between the two resamplers.

    python tools/bench_resample.py [--files 12] [--seconds 10] [--reps 5] [--host-files 2]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from oracle import resampy as R                                  # noqa: E402
from oracle import scoring as S                                  # noqa: E402
from voicefixer_main_b200.edges import AudioMetrics, resample, resample_to   # noqa: E402
from voicefixer_main_b200.model import Engine                    # noqa: E402


def _signals(rates, seconds, seed):
    rng = np.random.default_rng(seed)
    out = []
    for i, r in enumerate(rates):
        n = int(seconds * r) + int(rng.integers(0, r))
        t = np.arange(n) / r
        x = 0.3 * np.sin(2 * np.pi * (200 + 50 * i) * t) * (1 + 0.5 * np.sin(2 * np.pi * 3 * t)) + 0.05 * rng.standard_normal(n)
        out.append(np.clip(x, -0.99, 0.99).astype(np.float32))
    return out


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
        times.append(start.elapsed_time(stop) / 1e3)
    return float(np.median(times))


def _run_set(eng, name, xs, rates, target, reps, host_files):
    audio_s = sum(len(x) / r for x, r in zip(xs, rates))
    dev = [torch.from_numpy(x).cuda() for x in xs]
    res = {"set": name, "files": len(xs), "audio_s": round(audio_s, 2)}
    for rt in ("kaiser_best", "kaiser_fast"):
        t = _gpu_time(lambda: resample(eng, dev, rates, target, rt), reps)
        res[f"gpu_{rt}_audio_s_per_s"] = round(audio_s / t, 1)
        res[f"gpu_{rt}_ms"] = round(1e3 * t, 3)
    t = _gpu_time(lambda: [resample_to(eng, d[None], r, target) for d, r in zip(dev, rates)], reps)
    res["gpu_resample_poly_audio_s_per_s"] = round(audio_s / t, 1)
    k = min(host_files, len(xs))
    t0 = time.perf_counter()
    host = [R.resample(xs[i], rates[i], target, "kaiser_best") for i in range(k)]
    dt = time.perf_counter() - t0
    res["host_numpy_kaiser_best_audio_s_per_s"] = round(sum(len(xs[i]) / rates[i] for i in range(k)) / dt, 2)
    gpu = resample(eng, dev[:k], rates[:k], target, "kaiser_best")
    res["gpu_equals_restatement"] = all(np.array_equal(g.cpu().numpy(), h) for g, h in zip(gpu, host))
    best = resample(eng, dev, rates, target, "kaiser_best")
    poly = [resample_to(eng, d[None], r, target)[0] for d, r in zip(dev, rates)]
    res["max_abs_kaiser_best_minus_resample_poly"] = max(float((b - p[:len(b)]).abs().max()) for b, p in zip(best, poly))
    e = target // 10                      # 100 ms from either end: where the two filters see the signal's edges differently
    res["max_abs_kaiser_best_minus_resample_poly_interior"] = max(float((b - p[:len(b)])[e:-e].abs().max())
                                                                  for b, p in zip(best, poly))
    return res


def _score_shift(eng, d, n_pairs, seconds):
    """16 kHz spectral scores of 44.1 kHz ests (target + noise, written at 44.1 kHz) under both resamplers."""
    tgts = _signals([16000] * n_pairs, seconds, 7)
    pairs = []
    for i, t in enumerate(tgts):
        e16 = t + 0.05 * np.random.default_rng(100 + i).standard_normal(len(t)).astype(np.float32)
        n44 = int(np.ceil(len(t) * 44100 / 16000))
        e44 = np.interp(np.arange(n44) * 16000 / 44100, np.arange(len(t)), e16)
        pe, pt = os.path.join(d, f"e{i}.wav"), os.path.join(d, f"t{i}.wav")
        S.write_pcm16(np.round(np.clip(e44, -1, 1) * 32767).astype(np.int16), pe, 44100)
        S.write_pcm16(np.round(np.clip(t, -1, 1) * 32767).astype(np.int16), pt, 16000)
        pairs.append((pe, pt))
    a = AudioMetrics(eng, rate=16000).evaluation_batch(pairs)
    b = AudioMetrics(eng, rate=16000, res_type="kaiser_best").evaluation_batch(pairs)
    return {k: float(max(abs(x[k] - y[k]) for x, y in zip(a, b))) for k in a[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=12)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-files", type=int, default=2)
    a = ap.parse_args()
    eng = Engine("cuda:0")
    eng.load_state({}, need=())
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "host_cores": os.cpu_count()}))
    up_rates = [(16000, 22050, 48000)[i % 3] for i in range(a.files)]
    print(json.dumps(_run_set(eng, "up_to_44100", _signals(up_rates, a.seconds, 1), up_rates, 44100, a.reps, a.host_files)))
    down = [44100] * a.files
    print(json.dumps(_run_set(eng, "44100_down_to_16000", _signals(down, a.seconds, 2), down, 16000, a.reps, a.host_files)))
    with tempfile.TemporaryDirectory() as d:
        shift = _score_shift(eng, d, 4, a.seconds)
    print(json.dumps({"max_16k_score_change_kaiser_best_vs_resample_poly": shift}))
    eng.check_errors()
    eng.close()


if __name__ == "__main__":
    main()
