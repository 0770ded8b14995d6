"""Golden scores: the reference's own AudioMetrics.evaluation (evaluation_proc/metrics.py, imported unmodified) on the seeded
PCM16 pairs of oracle.scoring.score_pairs().

Run where the reference tree exists:  python oracle/make_ref_scores.py   -> tests/golden/ref_scores.npz
The third-party calls are stubbed with the restatements of oracle/scoring.py (librosa.load / librosa.stft, skimage's
structural_similarity); speechmetrics' sisdr / stoi / pesq are stubbed with NaN and not stored.  What this pins is the
reference's glue: the keys, EPS, to_log, the mel, the transposes and the lsd / sispec arithmetic.
"""
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_import, scoring as S            # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def reference_metrics():
    ref_import.install_shims()
    librosa = sys.modules["librosa"]
    librosa.load = lambda path, sr=None, mono=True: S.load(path)
    librosa.stft = lambda wav, hop_length=None, n_fft=None: S.stft(wav, n_fft=n_fft, hop_length=hop_length)
    sys.modules["skimage.metrics"].structural_similarity = S.ssim
    nan = float("nan")
    sys.modules["speechmetrics"].load = lambda *a, **k: (lambda est, target, rate: {"sisdr": nan, "stoi": nan, "pesq": nan})
    cwd = os.getcwd()
    os.chdir(ROOT)                                      # metrics.py runs git.Repo("", search_parent_directories=True)
    try:
        from evaluation_proc import metrics
    finally:
        os.chdir(cwd)
    assert metrics.EPS == 1e-12
    return metrics.AudioMetrics(rate=44100)


def main():
    if not ref_import.available():
        raise SystemExit("reference tree not present at " + ref_import.REFERENCE_ROOT)
    am = reference_metrics()
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for i, (est, tgt) in enumerate(S.score_pairs()):
            pe, pt = os.path.join(d, f"est{i}.wav"), os.path.join(d, f"tgt{i}.wav")
            S.write_pcm16(est, pe)
            S.write_pcm16(tgt, pt)
            with torch.no_grad():
                res = am.evaluation(pe, pt)
            keys = [k for k in res if k not in ("sisdr", "stoi", "pesq")]
            out[f"keys{i}"] = np.array(keys)
            out[f"values{i}"] = np.array([res[k] for k in keys], dtype=np.float64)
    np.savez_compressed(os.path.join(GOLDEN, "ref_scores.npz"), **out)
    print("ref_scores.npz", os.path.getsize(os.path.join(GOLDEN, "ref_scores.npz")), "bytes")


if __name__ == "__main__":
    main()
