"""handler_batch host logic with a stub engine: the segments are restore_array's, they reach the engine longest first and
come back to their files in order, and a file handler() would reject fails the call before any restore or file write."""
import os
import wave

import numpy as np
import pytest
import torch
from scipy.signal import resample_poly

from voicefixer_main_b200 import handler as H
from voicefixer_main_b200._lib import EngineError

SEG = H.SEG_LENGTH


class StubEngine:
    device = torch.device("cpu")
    loaded = True

    def __init__(self):
        self.calls = []

    def restore_varlen(self, packed, lengths, unify_energy=False, mel_out=None, log_mel_out=None):
        self.calls.append(list(lengths))
        return packed.clone()

    def to_pcm16(self, x, saturate=False):
        return (x * 32768.0).to(torch.int32).to(torch.int16)        # exact on samples decoded from PCM16


class StubModel:
    """What handler() / handler_batch touch of the model: .to, .device, ._engine and restore_array's .restore."""
    device = torch.device("cpu")

    def __init__(self):
        self._eng = StubEngine()

    def to(self, device):
        return self

    def _engine(self):
        return self._eng

    def restore(self, seg, unify_energy=False):
        self._eng.calls.append([seg.shape[1]])
        return seg


@pytest.mark.parametrize("n", [1, 1025, SEG - 1, SEG, SEG + 1, SEG + 1025, 2 * SEG - 1, 2 * SEG, 2 * SEG + 5000])
def test_segment_plan_is_restore_arrays_loop(n):
    m = StubModel()
    wav = np.arange(n, dtype=np.float32)
    out = H.restore_array(m, wav, "cpu")
    bounds = H.segment_bounds(n)
    assert [c[0] for c in m._eng.calls] == [e - s for s, e in bounds]
    assert bounds[0][0] == 0 and bounds[-1][1] == n and all(a[1] == b[0] for a, b in zip(bounds, bounds[1:]))
    assert torch.equal(out[0], torch.from_numpy(wav))
    assert H.segment_bounds(0) == []


@pytest.mark.parametrize("rate", [8000, 16000, 22050, 48000])
def test_resampled_length_is_resample_polys(rate):
    for n in (1, 999, 16000 + 123, 48000):
        want = len(resample_poly(np.zeros(n), 44100 // np.gcd(44100, rate), rate // np.gcd(44100, rate)))
        assert H._rate_len(n, rate) == want


def _write(path, n, seed):
    pcm = np.random.default_rng(seed).integers(-20000, 20000, n).astype(np.int16)
    H.save_pcm16(pcm, str(path))
    return str(path)


def _frames(path):
    with wave.open(path, "rb") as w:
        return w.readframes(w.getnframes())


def test_segments_go_longest_first_and_return_to_their_files(tmp_path, monkeypatch):
    m = StubModel()
    monkeypatch.setattr(H, "model", m)
    lengths = [30000, SEG + 40000, 5000, 120000, 5000]
    items = [(_write(tmp_path / f"in{i}.wav", n, i), str(tmp_path / f"out{i}.wav"), None) for i, n in enumerate(lengths)]
    res = H.handler_batch(items, ckpt=None, device="cpu")
    assert res == [{}] * len(items)
    assert m._eng.calls == [[SEG], [120000, 40000, 30000, 5000, 5000]]       # full 60 s segments in a call of their own
    for inp, out, _ in items:
        assert _frames(out) == _frames(inp)          # the stub restores the identity: every sample back in place
    assert H.handler_batch([], ckpt=None, device="cpu") == []


@pytest.mark.parametrize("n, n_target, exc", [
    (SEG + 1000, None, EngineError),            # last segment of 1000 samples
    (1024, None, EngineError),
    (0, None, RuntimeError),                    # nothing to restore
    (5000, 1000, EngineError),                  # the target slice is too short for the front end
    (5000, 6000, AssertionError),               # the target slice has another frame count
    (SEG + 5000, SEG + 1000, EngineError),      # ... of the last segment only
])
def test_rejected_file_fails_before_any_restore_or_write(tmp_path, monkeypatch, n, n_target, exc):
    m = StubModel()
    monkeypatch.setattr(H, "model", m)
    good = (_write(tmp_path / "good.wav", 30000, 1), str(tmp_path / "good_out.wav"), None)
    tgt = _write(tmp_path / "tgt.wav", n_target, 3) if n_target is not None else None
    bad = (_write(tmp_path / "bad.wav", n, 2), str(tmp_path / "bad_out.wav"), tgt)
    with pytest.raises(exc, match="bad.wav"):
        H.handler_batch([good, bad, good], ckpt=None, device="cpu")
    assert m._eng.calls == []
    assert not os.path.exists(good[1]) and not os.path.exists(bad[1])
