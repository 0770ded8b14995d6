"""Write tests/golden/ref_lowpass.npz from the reference's own tools/dsp/lowpass.py (run under oracle.ref_import's shims).

    python oracle/make_golden_lowpass.py

Inputs are seeded float32 noise clips of N samples (0.05 s at 44.1 kHz).  Stored outputs, float64 as the reference returns
them (stft_hard: float32):
* lp/<type>/<order>/<cutoff>: lowpass(x, cutoff, 44100, order, type) for the six types
* bp/<type>/<order>: bandpass(x, 1000, 8000, 44100, order, type); lpf_cheby2 / bpf_cheby2: the *_filter entry points
* sr/<cutoff>: collate_fn_val's chain (data_module.py:144-146) - lowpass(.., order=8, "butter") then lowpass(.., "stft"),
  float32 as stack_convert converts it - called through the reference's lowpass exactly as collate_fn_val calls it
  (data_module.py itself does not import under the shims, so its loop is restated here)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_import  # noqa: E402

N = 2205
LP_CASES = [("butter", 8, 1000), ("butter", 3, 12000), ("cheby1", 8, 4000), ("cheby1", 2, 21000), ("ellip", 10, 1000),
            ("ellip", 5, 8000), ("bessel", 4, 2000), ("stft", 8, 1000), ("stft", 8, 12000), ("stft_hard", 8, 4000),
            ("b", 12, 4000.7), ("", 1, 8000)]
BP_CASES = [("butter", 5), ("cheby1", 10), ("ellip", 2), ("bessel", 3)]


def main():
    ref_import.install_shims()
    cwd = os.getcwd()
    os.chdir(ref_import.REPO_ROOT)
    try:
        from tools.dsp import lowpass as R
    finally:
        os.chdir(cwd)
    rng = np.random.default_rng(2024)
    x = (0.3 * rng.standard_normal(N)).astype(np.float32)
    out = {"x": x}
    for t, o, c in LP_CASES:
        out[f"lp/{t}/{o}/{c}"] = R.lowpass(x, c, 44100, o, _type=t)
    for t, o in BP_CASES:
        out[f"bp/{t}/{o}"] = R.bandpass(x, 1000, 8000, 44100, o, _type=t)
    out["lpf_cheby2"] = R.lowpass_filter(x, 4000, 44100, 6, "cheby2")
    out["bpf_cheby2"] = R.bandpass_filter(x, 500, 6000, 44100, 4, "cheby2")
    for c in (1000, 2000, 4000, 8000, 12000):
        data = R.lowpass(x, highcut=c, fs=44100, order=8, _type="butter")
        out[f"sr/{c}"] = R.lowpass(data, highcut=c, fs=44100, order=8, _type="stft").astype(np.float32)
    path = os.path.join(ref_import.REPO_ROOT, "tests", "golden", "ref_lowpass.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()
