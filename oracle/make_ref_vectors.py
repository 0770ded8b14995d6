"""Golden vectors for the tests that pin the oracle and the host-side mirrors against the reference's own modules.

Run where the reference tree exists:  python oracle/make_ref_vectors.py
Writes tests/golden/ref_oracle.npz (small model-level outputs), tests/golden/ref_unet.npz (UNet and handler outputs)
and tests/golden/ref_ola.npz (overlap-add outputs and call lists).  The tests then compare against these files and
need no reference tree.  Inputs come from the seeded helpers below (CPU torch generators), which the tests call too.

torch computes log10 (and tanh, exp, sqrt) through MKL's vector math, whose rounding differs between the code paths MKL
picks for the CPU (AVX512, AVX2, ...).  So the reference's to_log is also written once per path, each with a log10 probe
that tells the paths apart, to tests/golden/ref_log10_paths.npz; the test compares against the path its CPU runs.
"""
import importlib.util
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ref_import, vf_oracle as O            # noqa: E402
from voicefixer_main_b200.arch import UNET_PREFIX        # noqa: E402
from voicefixer_main_b200.weights import make_state      # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
MKL_PATHS = ("AVX512", "AVX2", "SSE4_2")                 # values of MKL_ENABLE_INSTRUCTIONS


def log10_probe():
    """torch.log10 on fixed inputs: its bits identify the MKL code path of the CPU that runs it."""
    return torch.log10(torch.linspace(1e-3, 30.0, 4096))


def log_helper_inputs():
    g = torch.Generator().manual_seed(21)
    x = torch.rand(3, 1, 7, 128, generator=g) * 3
    x[0, 0, 0, :4] = 0
    y = torch.randn(3, 1, 7, 128, generator=g) * 4
    return x, y


def unet_inputs():
    g = torch.Generator().manual_seed(3)
    return [10 ** (torch.randn(2, 1, t, 128, generator=g) - 1) for t in (64, 101, 130)]


def small_input():
    g = torch.Generator().manual_seed(4)
    return 10 ** (torch.randn(1, 1, 101, 128, generator=g) - 1)


def model_vectors(out):
    state = make_state(1234)
    model, _ = ref_import.build_reference_model(state)
    fb = model.mel.fb.numpy()
    nz = np.nonzero(fb)
    out["fb_shape"] = np.array(fb.shape)
    out["fb_rows"], out["fb_cols"], out["fb_vals"] = nz[0].astype(np.int32), nz[1].astype(np.int32), fb[nz]

    ref_import.install_shims()
    from tools.pytorch.pytorch_util import from_log, to_log
    x, y = log_helper_inputs()
    out["log_x"], out["log_to"] = x.numpy(), to_log(x).numpy()
    out["log_y"], out["log_from"] = y.numpy(), from_log(y).numpy()

    with torch.no_grad():
        for i, mel in enumerate(unet_inputs()):
            out[f"unet_out{i}"] = model(mel)["mel"].numpy()
        wav = O.synth_clips(2, 30000, seed=9)
        out["handler_out"] = ref_import.reference_handler_batch(model, wav, seg_samples=12000).numpy()

    from tools.utils import trim_center
    starts = []
    for le, lr in ((20, 14), (443646, 441000), (16, 16)):
        r = trim_center(torch.arange(float(le))[None, None], torch.zeros(1, 1, lr))[0].flatten()
        assert torch.equal(r, torch.arange(float(r[0]), float(r[0]) + lr)), "trim_center is not a slice"
        starts.append(int(r[0]))
    out["trim_cases"] = np.array([[20, 14], [443646, 441000], [16, 16]])
    out["trim_starts"] = np.array(starts)

    ssr = {k.replace(UNET_PREFIX, "generator.unet."): v for k, v in state.items() if k.startswith(UNET_PREFIX)}
    net = ref_import.build_reference_unet_v2(ssr)
    for n in (63 * 441, 70 * 441 + 17):
        wav = O.synth_clips(1, n, seed=n)[:, None, :]
        with torch.no_grad():
            sp, _, _ = O.wav_to_spectrogram_phase(wav)
            out[f"ssr_out{n}"] = net(sp, wav)["wav"].numpy()

    small = ref_import.build_reference_unet_small(state)
    mel = small_input()
    with torch.no_grad():
        a = small(O.to_log(mel))["mel"] + O.to_log(mel)
        b = model(mel)["mel"]
    assert torch.equal(a, b), "unet_small and unet differ"
    out["small_out"] = a.numpy()

    keys = [(k, tuple(v.shape)) for k, v in model.state_dict().items() if k.startswith(UNET_PREFIX)]
    out["sd_keys"] = np.array([k for k, _ in keys])
    out["sd_shapes"] = np.array([",".join(map(str, s)) for _, s in keys])


def ola_vectors(out):
    import test_longform_cpu as T
    ref_dir = ref_import.REFERENCE_ROOT
    for name, fname in (("boxcar", "overlapadd_boxcar.py"), ("ola", "overlapadd.py")):
        spec = importlib.util.spec_from_file_location("ref_" + name, os.path.join(ref_dir, "tools", "dsp", fname))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        cases = T.CASES if name == "boxcar" else T.OLA_CASES
        for n, w, m in cases:
            for windowed in (False, True):
                net = T.ToyNet()
                if name == "boxcar":
                    ref = mod.LambdaOverlapAdd(nnet=net, n_src=1, window_size=w, in_margin=m, window="hann", reorder_chunks=False)
                else:
                    ref = mod.LambdaOverlapAdd(nnet=net, n_src=1, window_size=w, hop_size=m, window="hann", reorder_chunks=False)
                ref.use_window = windowed
                key = T.ref_key(name, n, w, m, windowed)
                out[key + "_out"] = ref(T._signal(n)).numpy()
                out[key + "_calls"] = np.array(net.calls, dtype=np.int64)


def log10_paths(out):
    """The reference's to_log on log_helper_inputs() and log10_probe() under each of MKL_PATHS, one process per path."""
    with tempfile.TemporaryDirectory() as d:
        for isa in MKL_PATHS:
            f = os.path.join(d, isa + ".npz")
            subprocess.run([sys.executable, os.path.abspath(__file__), "--log10-path", f], check=True,
                           env={**os.environ, "MKL_ENABLE_INSTRUCTIONS": isa})
            g = np.load(f)
            out[isa + "_log_to"], out[isa + "_probe"] = g["log_to"], g["probe"]
    for p in MKL_PATHS:                # equal probes must mean equal outputs, or the probe cannot pick the path
        for q in MKL_PATHS:
            if np.array_equal(out[p + "_probe"], out[q + "_probe"]):
                assert np.array_equal(out[p + "_log_to"], out[q + "_log_to"]), (p, q)


def main():
    if not ref_import.available():
        raise SystemExit("reference tree not present at " + ref_import.REFERENCE_ROOT)
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    if "--log10-path" in sys.argv:
        ref_import.install_shims()
        from tools.pytorch.pytorch_util import to_log
        np.savez(sys.argv[sys.argv.index("--log10-path") + 1], log_to=to_log(log_helper_inputs()[0]).numpy(),
                 probe=log10_probe().numpy())
        return
    c = {}
    log10_paths(c)
    np.savez_compressed(os.path.join(GOLDEN, "ref_log10_paths.npz"), **c)
    a, b = {}, {}
    model_vectors(a)
    ola_vectors(b)
    big = {k: a.pop(k) for k in list(a) if k.startswith("unet_out") or k == "handler_out"}
    np.savez_compressed(os.path.join(GOLDEN, "ref_oracle.npz"), **a)
    np.savez_compressed(os.path.join(GOLDEN, "ref_unet.npz"), **big)
    np.savez_compressed(os.path.join(GOLDEN, "ref_ola.npz"), **b)
    for f in ("ref_oracle.npz", "ref_unet.npz", "ref_ola.npz", "ref_log10_paths.npz"):
        print(f, os.path.getsize(os.path.join(GOLDEN, f)), "bytes")


if __name__ == "__main__":
    main()
