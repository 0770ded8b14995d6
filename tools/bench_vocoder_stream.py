#!/usr/bin/env python
"""Benchmark of live mel streams through the stand-alone vocoder (streaming.StreamingVocoder, vf_vocoder_chunks) on one GPU.

    python tools/bench_vocoder_stream.py [--steps K] [--warmup W] [--streams 1,8,64,256] [--out FILE]

For S streams and (W, M) = (window_frames, margin_frames) every stream pushes W frames per step (10 ms of audio per frame)
and the step vocodes what became ready.  Two arms, alternating step by step on contexts of their own:
  - stream: StreamingVocoder pushes from device-resident mels, then step(): one vf_vocoder_chunks call (gather from the
    rings, vocoder, crop, all on the device);
  - torch: each stream's resident history, torch slices of the same chunks, Vocoder.forward_batch and torch crops.
It checks that both arms give the same bits every step and reports ms/step, audio-s/s and whether a step stays within the
W x 10 ms of audio it adds (real time).  Then, for M in {0, 8, 32, 128, R} (R = arch.vocoder_receptive_field), the RMS and
largest deviation of the chunked stream (vocoder.vocode_chunked, W = 64) from Vocoder.forward on the whole mel, on the mel of
30 s of synthetic speech.  The weights are the seeded synthetic ones (weights.make_state), not a trained vocoder: the
deviations say how far a margin is from the whole-mel result for these weights only.  Prints one JSON line with the card's
name and power limit, read in the same run.
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

GEOMETRIES = [(16, 8), (64, 16)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--streams", default="1,8,64,256")
    ap.add_argument("--out", default="", help="also write the JSON line to this file")
    args = ap.parse_args()
    from voicefixer_main_b200.arch import VocoderConfig, vocoder_out_len, vocoder_receptive_field
    from voicefixer_main_b200.streaming import StreamingVocoder
    from voicefixer_main_b200.vocoder import Vocoder, vocode_chunked
    from voicefixer_main_b200.weights import make_state
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_vocoder_stream.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    cfg = VocoderConfig()
    voc_sd = {k: v for k, v in make_state(1234).items() if k.startswith("vocoder.")}
    card = card_info(0)

    def vocoder():
        return Vocoder().load_state_dict(voc_sd).eval().to(dev)

    # the mels of synthetic speech, long enough for every step; streams share a few sources at different offsets
    fe = vocoder()
    src = [fe._engine().frontend(synth_batch(1, 40 * SR, 900 + i).to(dev))[0][0] for i in range(4)]
    torch.cuda.synchronize()

    sampler = ClockSampler(0)
    sampler.start()
    table = []
    for W, M in GEOMETRIES:
        for S in [int(s) for s in args.streams.split(",")]:
            n_steps = args.warmup + args.steps
            assert (n_steps + 1) * W <= src[0].shape[0] - 64
            mels = [src[i % 4][(7 * i) % 64:][: (n_steps + 1) * W] for i in range(S)]
            v_stream, v_torch = vocoder(), vocoder()
            sv = StreamingVocoder(v_stream, W, M, max_streams=S)
            sids = [sv.open() for _ in range(S)]
            done = [0] * S                               # torch arm: chunks vocoded per stream

            def stream_step(k):
                for i, sid in enumerate(sids):
                    sv.push(sid, mels[i][k * W:(k + 1) * W])
                return sv.step()

            def torch_step(k):
                pushed = (k + 1) * W
                chunks, owners = [], []
                for i in range(S):
                    while pushed >= (done[i] + 1) * W + max(M, 1):
                        c = done[i]
                        s = max(0, c * W - M)
                        e = (c + 1) * W + M
                        chunks.append(mels[i][s:e])
                        owners.append((i, (c * W - s) * cfg.hop, vocoder_out_len(e - s, cfg) - ((c + 1) * W - s) * cfg.hop))
                        done[i] += 1
                if not chunks:
                    return {}
                outs = v_torch.forward_batch(chunks)
                res = {}
                for (i, left, right), o in zip(owners, outs):
                    res.setdefault(sids[i], []).append(o[left:o.numel() - right])
                return {sid: torch.cat(v) for sid, v in res.items()}

            ms = {"stream": [], "torch": []}
            same = True
            for k in range(n_steps):
                outs = {}
                for name, fn in (("stream", stream_step), ("torch", torch_step)):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize()
                    e0.record()
                    outs[name] = fn(k)
                    e1.record()
                    torch.cuda.synchronize()
                    if k >= args.warmup:
                        ms[name].append(e0.elapsed_time(e1))
                a, b = outs["stream"], outs["torch"]
                same = same and a.keys() == b.keys() and all(torch.equal(a[s], b[s]) for s in a)
            v_stream._engine().check_errors()
            v_torch._engine().check_errors()
            row = {"streams": S, "window_frames": W, "margin_frames": M, "bit_identical": same,
                   "budget_ms_per_step": W * 1000.0 * cfg.hop / SR}
            for name, v in ms.items():
                med = sorted(v)[len(v) // 2]
                row[name] = {"ms_per_step_median": med, "ms_min": min(v), "ms_max": max(v),
                             "audio_seconds_per_sec": S * W * cfg.hop / SR / (med * 1e-3),
                             "real_time": med <= row["budget_ms_per_step"]}
            table.append(row)
            print(json.dumps(row), file=sys.stderr)
            v_stream._engine().close()
            v_torch._engine().close()
    sampler.stop_flag = True

    # deviation of the chunked stream from the whole-mel forward, by margin
    R = vocoder_receptive_field(cfg)
    mel = src[0][:3000]
    whole = fe.forward(mel[None, None])[0, 0]
    dev_rows = []
    for M in (0, 8, 32, 128, R + R % 2):
        got = vocode_chunked(fe, mel, 64, M)
        d = (got - whole).double()
        dev_rows.append({"margin_frames": M, "rms_dev": float(d.pow(2).mean().sqrt()), "max_dev": float(d.abs().max()),
                         "bit_identical": bool(torch.equal(got.view(torch.int32), whole.view(torch.int32)))})
    fe._engine().check_errors()
    line = {"metric": "vocoder_stream_ms_per_step", "data": "synthetic (seeded weights and synthetic speech)",
            "steps": args.steps, "warmup": args.warmup, "table": table,
            "deviation_from_whole_mel": {"window_frames": 64, "frames": int(mel.shape[0]),
                                         "output_rms": float(whole.double().pow(2).mean().sqrt()),
                                         "receptive_field_frames": R, "rows": dev_rows},
            "card": card, "clocks": sampler.summary()}
    print(json.dumps(line))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
