#!/usr/bin/env python
"""Benchmark of live-stream restoration (StreamingRestorer / vf_restore_chunks, vf_ssr_restore_chunks) on one GPU.

    python tools/bench_stream.py [--workload gsr|ssr] [--ola boxcar|windowed [--hop-div 2]] [--streams 1,8,64,256]
                                 [--windows 1,2] [--steps K] [--warmup W]
    python tools/bench_stream.py --input-rate 8000,16000,48000 [--res-type kaiser_best] [--streams 64] [--windows 1]

--workload gsr (the default) streams through VoiceFixer (ResUNet + vocoder, vf_restore_chunks); ssr through SSR_UNet
(unet_v2 + ISTFT, vf_ssr_restore_chunks), whose baseline arm calls SSR_UNet.restore_batch (vf_ssr_restore_varlen).

For every window W (seconds) and stream count S: S streams of seeded speech-like audio each push W of samples per step, with
M = W / 4 samples of context on each side of every window (BoxcarOverlapAdd geometry), so after the first step every step
restores S middle chunks of W + 2M.  Two arms run alternately in one process on the same chunks:
- "streaming": S pushes (device to device, one copy each) + StreamingRestorer.step(): one gather launch, the varlen restore
  chain, one crop launch ("streaming_step_only": the step without the pushes);
- "torch_slicing": what a server does without it: slices each stream's chunk out of its (device-resident) history, one
  restore_batch call per GROUP streams (torch.cat of the slices + the varlen restore), and crops every result.
  Its histories are resident from the start, so it pays nothing for receiving the audio.
With --ola windowed the streams run WindowedStreamingRestorer (vf_restore_windows / vf_ssr_restore_windows) instead:
hann-weighted windows of W every hop = W / hop_div, each stream still pushing W per step, so a steady-state step restores
hop_div windows per stream and emits W samples of each.  Its baseline arm ("torch_windowed") slices the ready windows out of
the zero-led resident histories, restores them with restore_batch GROUP at a time, multiplies them by the synthesis window
and adds them into per-stream output buffers in ascending window order with torch, then cuts out the finished samples.
Both must give the same bits.  A step is timed with CUDA events around it after a device synchronise; medians are
reported.  A step is real time when it takes at most W seconds (it restores W of audio per stream).  Prints one JSON line:
per (W, S) the step times, audio seconds restored per second and the plans built and evicted; per W the largest S that
stays real time; the card's name and power limit, read in the same run.

With --input-rate R (a comma-separated list), each case is S streams at R Hz through StreamingRestorer (VoiceFixer, boxcar,
M = W / 4; --res-type picks the resampler, default resample_poly): each step pushes W R / 44100 samples per stream and the
step first resamples the newly final samples into the 44.1 kHz rings (one vf_resample_rings launch), then restores.  Its
baseline arm ("pre_resampled") is the same audio resampled whole beforehand with edges.resample_to and pushed at 44.1 kHz,
exactly the samples the first arm made final in that step, so both restore the same chunks and must give the same bits.
Only step() is timed in both arms.  A third pass, run separately under torch.profiler, sums the device time of
stream_resample_kernel per step and its share of the step's kernel time.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from bench import SR, synth_batch  # noqa: E402
from bench_varlen import card_info  # noqa: E402

BANK = 8            # distinct synthetic signals; stream s plays signal s % BANK shifted by s * 997 samples
# restore_batch calls of the baseline take at most this many streams.  gsr: the sub-batch the streaming arm's plan-shape rule
# picks for 1 - 2 s windows on an 80 GB card, so both arms run on the same cached plans.  ssr (about 1.4 times the plan bytes
# per frame): a group whose plans stay cached beside the streaming arm's at 1 s windows (at S = 64 on an 80 GB H100, one plan
# was evicted in the whole run: the first step's).  Left to its own split, restore_batch of 256 chunks picks other shapes,
# and the two arms' plans would evict each other on every alternation.
GROUP = {"gsr": 64, "ssr": 16}


def timed(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0, e1


def run_case(workload, state, bank, W, M, S, steps, warmup):
    """One (W, S) case on a model of its own: a fresh plan cache, so that plans of earlier cases neither crowd the budget nor
    enter its size estimates."""
    from voicefixer_main_b200 import SSR_UNet, VoiceFixer
    from voicefixer_main_b200.streaming import StreamingRestorer
    model = (SSR_UNet if workload == "ssr" else VoiceFixer)().load_state_dict(state).eval().to(bank.device)
    group = GROUP[workload]
    eng = model._engine()
    xs = [torch.roll(bank[s % BANK], s * 997) for s in range(S)]
    sr = StreamingRestorer(model, W, M, max_streams=S)
    ids = [sr.open() for _ in range(S)]

    def chunk(i):
        return (0, W + M, 0, M) if i == 0 else (i * W - M, W + 2 * M, M, M)

    pushed = torch.cuda.Event(enable_timing=True)

    def streaming(i):
        lo, hi = (0, W + M) if i == 0 else (i * W + M, (i + 1) * W + M)
        for sid, x in zip(ids, xs):
            sr.push(sid, x[lo:hi])
        pushed.record()
        out = sr.step()
        return [out[sid] for sid in ids]

    def torch_slicing(i):
        start, length, cl, cr = chunk(i)
        outs = []
        for g in range(0, S, group):
            outs += model.restore_batch([x[start:start + length] for x in xs[g:g + group]])
        return [o[cl:length - cr] for o in outs]

    info0 = eng.plan_cache_info()
    ms = {"streaming": [], "streaming_step_only": [], "torch_slicing": []}
    same = True
    for i in range(warmup + steps):
        a, a0, a1 = timed(lambda: streaming(i))
        b, b0, b1 = timed(lambda: torch_slicing(i))
        same = same and all(torch.equal(p, q) for p, q in zip(a, b))
        if i >= warmup:
            ms["streaming"].append(a0.elapsed_time(a1))
            ms["streaming_step_only"].append(pushed.elapsed_time(a1))
            ms["torch_slicing"].append(b0.elapsed_time(b1))
    eng.check_errors()
    info1 = eng.plan_cache_info()
    launches = eng.launch_count()
    eng.close()
    audio_s = S * W / SR                                      # kept audio per steady-state step
    res = {}
    for k, v in ms.items():
        med = sorted(v)[len(v) // 2]
        res[k] = {"ms_per_step_median": med, "ms_min": min(v), "ms_max": max(v), "audio_seconds_per_sec": audio_s / (med * 1e-3),
                  "real_time": med <= 1e3 * W / SR}
    return {"window_s": W / SR, "margin_s": M / SR, "streams": S, "arms": res,
            "speedup_vs_torch_slicing": res["torch_slicing"]["ms_per_step_median"] / res["streaming"]["ms_per_step_median"],
            "bit_identical": bool(same), "baseline_group": group,
            "plans_built": (info1["plans"] + info1["evicted"]) - (info0["plans"] + info0["evicted"]),
            "plans_evicted": info1["evicted"] - info0["evicted"], "plan_cache": info1, "gpu_launches": launches}


def run_case_windowed(workload, state, bank, W, hop, S, steps, warmup):
    """One (W, S) case of the windowed scheme on a model of its own (see run_case)."""
    import torch.nn.functional as F
    from voicefixer_main_b200 import SSR_UNet, VoiceFixer
    from voicefixer_main_b200.streaming import WindowedStreamingRestorer
    model = (SSR_UNet if workload == "ssr" else VoiceFixer)().load_state_dict(state).eval().to(bank.device)
    group = GROUP[workload]
    eng = model._engine()
    xs = [torch.roll(bank[s % BANK], s * 997) for s in range(S)]
    sr = WindowedStreamingRestorer(model, W, hop, max_streams=S)
    ids = [sr.open() for _ in range(S)]
    syn = sr.synthesis
    xps = [F.pad(x, (W, 0)) for x in xs]                    # window k = xp[k hop : k hop + W]
    accs = [torch.zeros(x.numel(), device=bank.device) for x in xs]
    state_b = {"next": 1, "emitted": 0}
    pushed = torch.cuda.Event(enable_timing=True)

    def streaming(i):
        for sid, x in zip(ids, xs):
            sr.push(sid, x[i * W:(i + 1) * W])
        pushed.record()
        out = sr.step()
        return [out[sid] for sid in ids]

    def torch_windowed(i):
        k0, k1 = state_b["next"], (i + 1) * W // hop + 1           # the windows ready once (i + 1) W samples are in
        slices = [xp[k * hop:k * hop + W] for xp in xps for k in range(k0, k1)]
        ys = []
        for g in range(0, len(slices), group):
            ys += model.restore_batch(slices[g:g + group])
        nk = k1 - k0
        for s in range(S):
            for j, k in enumerate(range(k0, k1)):
                lo, hi = max(0, k * hop - W), k * hop
                y = ys[s * nk + j] * syn
                accs[s][lo:hi] = accs[s][lo:hi] + y[lo - (k * hop - W):]
        a, b = state_b["emitted"], max(0, k1 * hop - W)
        state_b["next"], state_b["emitted"] = k1, b
        return [acc[a:b] for acc in accs]

    info0 = eng.plan_cache_info()
    ms = {"streaming": [], "streaming_step_only": [], "torch_windowed": []}
    same = True
    for i in range(warmup + steps):
        a, a0, a1 = timed(lambda: streaming(i))
        b, b0, b1 = timed(lambda: torch_windowed(i))
        same = same and all(torch.equal(p, q) for p, q in zip(a, b))
        if i >= warmup:
            ms["streaming"].append(a0.elapsed_time(a1))
            ms["streaming_step_only"].append(pushed.elapsed_time(a1))
            ms["torch_windowed"].append(b0.elapsed_time(b1))
    eng.check_errors()
    info1 = eng.plan_cache_info()
    launches = eng.launch_count()
    eng.close()
    audio_s = S * W / SR                                      # emitted audio per steady-state step
    res = {}
    for k, v in ms.items():
        med = sorted(v)[len(v) // 2]
        res[k] = {"ms_per_step_median": med, "ms_min": min(v), "ms_max": max(v), "audio_seconds_per_sec": audio_s / (med * 1e-3),
                  "real_time": med <= 1e3 * W / SR}
    return {"window_s": W / SR, "hop_s": hop / SR, "streams": S, "arms": res,
            "speedup_vs_torch_windowed": res["torch_windowed"]["ms_per_step_median"] / res["streaming"]["ms_per_step_median"],
            "bit_identical": bool(same), "baseline_group": group,
            "plans_built": (info1["plans"] + info1["evicted"]) - (info0["plans"] + info0["evicted"]),
            "plans_evicted": info1["evicted"] - info0["evicted"], "plan_cache": info1, "gpu_launches": launches}


def run_case_rates(state, W, M, S, rate, res_type, steps, warmup, seed=4242):
    """S streams at `rate` Hz (see the module docstring) on a VoiceFixer of its own."""
    from torch.profiler import ProfilerActivity, profile
    from voicefixer_main_b200 import VoiceFixer
    from voicefixer_main_b200.edges import resample_to
    from voicefixer_main_b200.streaming import StreamingRestorer
    dev = torch.device("cuda", 0)
    model = VoiceFixer().load_state_dict(state).eval().to(dev)
    eng = model._engine()
    P = W * rate // SR                                        # input samples per stream per step
    rounds = warmup + 2 * steps + 2
    bank = synth_batch(BANK, rounds * P + 1, seed).to(dev)
    xs = [torch.roll(bank[s % BANK], s * 997) for s in range(S)]
    x44 = [resample_to(eng, x[None], rate, SR, res_type)[0] for x in xs]
    a = StreamingRestorer(model, W, M, max_streams=S, res_type=res_type)
    b = StreamingRestorer(model, W, M, max_streams=S)
    ia, ib = [a.open(rate) for _ in range(S)], [b.open() for _ in range(S)]
    assert P <= a.max_push(rate)

    def step_pair(i):
        for sid, x in zip(ia, xs):
            a.push(sid, x[i * P:(i + 1) * P])
        out_a, a0, a1 = timed(a.step)
        for j, (sid, x) in enumerate(zip(ib, x44)):
            done = a._streams[ia[j]].pushed                   # the 44.1 kHz samples arm a has made final
            b.push(sid, x[b._streams[sid].pushed:done])
        out_b, b0, b1 = timed(b.step)
        same = all((p in out_a) == (q in out_b) and (p not in out_a or torch.equal(out_a[p], out_b[q])) for p, q in zip(ia, ib))
        return same, a0.elapsed_time(a1), b0.elapsed_time(b1)

    ms_a, ms_b, same = [], [], True
    for i in range(warmup + steps):
        ok, ta, tb = step_pair(i)
        same = same and ok
        if i >= warmup:
            ms_a.append(ta)
            ms_b.append(tb)
    # the resample kernel's share, in a pass of its own under the profiler
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(warmup + steps, warmup + 2 * steps):
            for sid, x in zip(ia, xs):
                a.push(sid, x[i * P:(i + 1) * P])
            a.step()
        torch.cuda.synchronize()
    kern = [e for e in prof.events() if e.device_type.name == "CUDA"]
    rs_us = sum(e.device_time for e in kern if "stream_resample_kernel" in e.name)
    all_us = sum(e.device_time for e in kern)
    eng.check_errors()
    eng.close()
    med = lambda v: sorted(v)[len(v) // 2]
    return {"input_rate": rate, "res_type": res_type, "window_s": W / SR, "margin_s": M / SR, "streams": S,
            "input_samples_per_stream_per_step": P,
            "arms": {"streaming_at_input_rate": {"step_ms_median": med(ms_a), "ms_min": min(ms_a), "ms_max": max(ms_a)},
                     "pre_resampled": {"step_ms_median": med(ms_b), "ms_min": min(ms_b), "ms_max": max(ms_b)}},
            "step_ms_ratio": med(ms_a) / med(ms_b), "bit_identical": bool(same),
            "resample_kernel_us_per_step": rs_us / steps, "resample_share_of_step_kernel_time": rs_us / all_us if all_us else None,
            "profiled_steps": steps}


def main_rates(args):
    from voicefixer_main_b200.weights import make_state
    state = make_state(1234)
    streams = [int(s) for s in args.streams.split(",")]
    cases = []
    for w_s in [float(w) for w in args.windows.split(",")]:
        W = int(round(w_s * SR)) // 2 * 2
        for rate in [int(r) for r in args.input_rate.split(",")]:
            for S in streams:
                cases.append(run_case_rates(state, W, W // 4, S, rate, args.res_type, args.steps, args.warmup))
    line = {"metric": "stream_resample_step_ms_ratio", "value": max(c["step_ms_ratio"] for c in cases),
            "unit": "step time at the input rate / step time pre-resampled", "higher_is_better": False, "data": "synthetic",
            "steps": args.steps, "warmup": args.warmup,
            "config": {"workload": "S streams of seeded speech-like audio at the input rate, each pushing W of audio per step, "
                                   "M = W / 4, VoiceFixer (vf_resample_rings + vf_restore_chunks); value = the worst case",
                       "res_type": args.res_type},
            "cases": cases, "card": card_info(0)}
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=("gsr", "ssr"), default="gsr",
                    help="gsr: VoiceFixer (vf_restore_chunks); ssr: SSR_UNet (vf_ssr_restore_chunks)")
    ap.add_argument("--ola", choices=("boxcar", "windowed"), default="boxcar",
                    help="boxcar: StreamingRestorer, M = W / 4; windowed: WindowedStreamingRestorer, hann, hop = W / hop-div")
    ap.add_argument("--hop-div", type=int, default=2, help="windowed: hop = W / hop-div")
    ap.add_argument("--streams", default="1,8,64,256")
    ap.add_argument("--windows", default="1,2", help="window lengths in seconds; the margin is a quarter of the window")
    ap.add_argument("--steps", type=int, default=5, help="timed steady-state steps per case")
    ap.add_argument("--warmup", type=int, default=2, help="untimed steps per case (the first is the streams' first chunk)")
    ap.add_argument("--input-rate", default=None, help="streams at these rates (Hz, comma-separated) through the resampler")
    ap.add_argument("--res-type", default=None, choices=("kaiser_best", "kaiser_fast"),
                    help="with --input-rate: librosa 0.8's resampy filter instead of resample_poly")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_stream.py needs a CUDA device")
    if args.input_rate:
        return main_rates(args)
    from voicefixer_main_b200.weights import make_ssr_state, make_state
    dev = torch.device("cuda", 0)
    state = (make_ssr_state if args.workload == "ssr" else make_state)(1234)
    streams = [int(s) for s in args.streams.split(",")]
    cases, best = [], {}
    for w_s in [float(w) for w in args.windows.split(",")]:
        W = int(round(w_s * SR)) // 2 * 2
        M = W // 4
        n = (args.warmup + args.steps + 1) * W + M
        bank = synth_batch(BANK, n, 4242).to(dev)
        for S in streams:
            if args.ola == "windowed":
                c = run_case_windowed(args.workload, state, bank, W, W // args.hop_div, S, args.steps, args.warmup)
            else:
                c = run_case(args.workload, state, bank, W, M, S, args.steps, args.warmup)
            cases.append(c)
            if c["arms"]["streaming"]["real_time"]:
                best[f"{w_s:g}"] = max(best.get(f"{w_s:g}", 0), S)
        del bank
    top = max(cases, key=lambda c: c["arms"]["streaming"]["audio_seconds_per_sec"])
    line = {"metric": "stream_audio_seconds_per_sec", "value": top["arms"]["streaming"]["audio_seconds_per_sec"], "unit": "audio s/s",
            "higher_is_better": True, "data": "synthetic", "steps": args.steps, "warmup": args.warmup,
            "config": {"workload": "S streams of seeded speech-like audio, each pushing W per step, "
                                   + (f"hann windows every W / {args.hop_div}" if args.ola == "windowed" else "M = W / 4")
                                   + ", 44.1 kHz; value = the best streaming arm over the cases",
                       "best_case": {"window_s": top["window_s"], "streams": top["streams"]}, "ola": args.ola,
                       "model": ("SSR_UNet (vf_ssr_restore_" if args.workload == "ssr" else "VoiceFixer (vf_restore_")
                                + ("windows)" if args.ola == "windowed" else "chunks)")},
            "largest_real_time_streams": {"window_s=" + k: v for k, v in best.items()},
            "cases": cases, "card": card_info(0)}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
