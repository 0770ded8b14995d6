"""Time handler.decode_wavs on a seeded set of FLAC files and on WAV copies of the same samples.

The set: 32 files of 10 - 11 s, 16- and 24-bit, mono and stereo, 44.1 and 48 kHz, written by oracle/flac.py's vectorised
FIXED-2 encoder (4096-sample blocks).  Both arms run in the same process, alternating, each from its own files (so each
stages its own bytes), timed with CUDA events around the whole decode_wavs call, median of --reps.  --profile runs one
more decode of each arm under torch.profiler and prints the per-kernel CUDA times.  Prints one JSON line, with the card's name and power limit.
Usage: python tools/bench_flac_decode.py [--files 32] [--reps 15] [--profile]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import flac as F                                     # noqa: E402
from oracle import wavfile as OW                                 # noqa: E402
from voicefixer_main_b200 import wavfile as W                    # noqa: E402
from voicefixer_main_b200.handler import decode_wavs             # noqa: E402
from voicefixer_main_b200.model import Engine                    # noqa: E402


def make_set(d, n_files, seed=0):
    rng = np.random.default_rng(seed)
    flac, wav, audio = [], [], 0.0
    for i in range(n_files):
        bits, channels, rate = (16, 24)[i % 2], (1, 2)[(i // 2) % 2], (44100, 48000)[(i // 4) % 2]
        n = int(rate * rng.uniform(10, 11))
        t = np.arange(n) / rate
        x = np.stack([0.3 * np.sin(2 * np.pi * (180 + 40 * c) * t * (1 + 0.1 * np.sin(t))) + 0.003 * rng.standard_normal(n)
                      for c in range(channels)], axis=1)
        x = np.round(np.clip(x, -1, 1) * (2 ** (bits - 1) - 1)).astype(np.int64)
        f, w = os.path.join(d, f"{i}.flac"), os.path.join(d, f"{i}.wav")
        with open(f, "wb") as fh:
            fh.write(F.encode_fast(x, rate, bits))
        with open(w, "wb") as fh:
            fh.write(OW.wav_bytes(F.wav_bytes(x, bits), rate, channels, {16: W.S16, 24: W.S24}[bits]))
        flac.append(f)
        wav.append(w)
        audio += n / rate
    return flac, wav, audio


def power_limit():
    """The power limit of GPU 0 in watts, read with a query of nvidia-smi (changes nothing), or None without one."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30, check=True).stdout
        return float(out.strip().splitlines()[0])
    except (OSError, subprocess.SubprocessError, ValueError, IndexError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=32)
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    eng = Engine("cuda:0")
    with tempfile.TemporaryDirectory() as d:
        flac, wav, audio = make_set(d, a.files)
        sizes = [sum(os.path.getsize(p) for p in paths) for paths in (flac, wav)]
        for paths in (flac, wav):                                # warm-up, and the two arms agree
            decode_wavs(paths, eng)
        out_f, out_w = decode_wavs(flac, eng), decode_wavs(wav, eng)
        same = all(np.array_equal(x.view(np.uint32), y.view(np.uint32)) for (x, _), (y, _) in zip(out_f, out_w))
        times = {"flac": [], "wav": []}
        for _ in range(a.reps):
            for arm, paths in (("flac", flac), ("wav", wav)):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                s.record()
                decode_wavs(paths, eng)
                e.record()
                torch.cuda.synchronize()
                times[arm].append(s.elapsed_time(e))
        kernels = {}
        if a.profile:
            from torch.profiler import ProfilerActivity, profile
            for arm, paths in (("flac", flac), ("wav", wav)):
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    decode_wavs(paths, eng)
                    torch.cuda.synchronize()
                kernels[arm] = {ev.key: round(ev.device_time_total / 1000, 4) for ev in prof.key_averages()
                                if ev.device_time_total > 0}
    eng.check_errors()
    props = torch.cuda.get_device_properties(0)
    print(json.dumps({"bench": "flac_decode", "device": props.name, "power_limit_w": power_limit(), "files": a.files,
                      "audio_s": round(audio, 1),
                      "flac_bytes": sizes[0], "wav_bytes": sizes[1], "same_bits": same,
                      "flac_ms_median": round(float(np.median(times["flac"])), 3),
                      "wav_ms_median": round(float(np.median(times["wav"])), 3), "kernels_ms": kernels}))


if __name__ == "__main__":
    main()
