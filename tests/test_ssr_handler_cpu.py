"""handler_unet host logic with a stub engine: handler() cuts handler.py's segments, handler_batch sends the same segments
longest first and puts them back in their files, a file handler() would reject fails the call before any restore or file
write, refresh_model picks the model class from hp, and the dict is the last segment's four metrics in the reference's
order."""
import json
import os
import wave

import numpy as np
import pytest
import torch

from voicefixer_main_b200 import handler_unet as HU
from voicefixer_main_b200._lib import EngineError
from voicefixer_main_b200.arch import frames_for

SEG = HU.SEG_LENGTH
KEYS = ["mel-lsd", "mel-sispec", "mel-non-log-sispec", "mel-ssim"]


def _stub_mel(x, n):
    """What the stubs give as the linear mel of an n-sample clip starting with sample x: T rows of x + n."""
    return torch.full((frames_for(n), 128), float(x) + n)


class StubEngine:
    device = torch.device("cpu")
    loaded = True

    def __init__(self):
        self.calls = []

    def ssr_restore_varlen(self, packed, lengths, out=None, mel_out=None, peak_normalise=False):
        assert peak_normalise
        self.calls.append(list(lengths))
        if mel_out is not None:
            rows, start = 0, 0
            for n in lengths:
                mel_out[rows:rows + frames_for(n)] = _stub_mel(packed[start], n)
                rows, start = rows + frames_for(n), start + n
        return packed.clone()

    def finalize(self, wav, n):
        assert wav.shape[1] == n
        return wav.clone()

    def to_pcm16(self, x, saturate=False):
        return (x * 32768.0).to(torch.int32).to(torch.int16)        # exact on samples decoded from PCM16


class StubModel:
    """What handler() / handler_batch touch of the model: .to, .device, ._engine, .restore and .pre."""
    device = torch.device("cpu")

    def __init__(self):
        self._eng = StubEngine()

    def to(self, device):
        return self

    def _engine(self):
        return self._eng

    def restore(self, seg):
        self._eng.calls.append([seg.shape[1]])
        return seg.clone()

    def pre(self, x):
        assert x.dim() == 3 and x.shape[:2] == (1, 1)
        n = x.shape[2]
        if n <= 1024:
            raise EngineError(-1, "reflect padding needs more than 1024 samples")
        return None, _stub_mel(x[0, 0, 0], n)[None, None]


class StubMetrics:
    """AudioMetrics with each value naming its inputs: lsd / ssim read the estimate / target mel, sispec its maps."""

    def __init__(self, owner):
        pass

    def lsd(self, est, target):
        assert est.shape == target.shape
        return est[0, 0, 0, 0]

    def sispec(self, est, target, est_map=0, target_map=0):
        return torch.tensor(10.0 * est_map + target_map)

    def ssim(self, est, target):
        if est.shape[2] < 7:
            raise ValueError("win_size exceeds image extent")
        return target[0, 0, 0, 0]


@pytest.fixture
def stub(monkeypatch):
    m = StubModel()
    monkeypatch.setattr(HU, "model", m)
    monkeypatch.setattr(HU, "AudioMetrics", StubMetrics)
    return m


def _write(path, n, seed):
    pcm = np.random.default_rng(seed).integers(-20000, 20000, n).astype(np.int16)
    HU.save_pcm16(pcm, str(path))
    return str(path), pcm


def _frames(path):
    with wave.open(path, "rb") as w:
        return w.readframes(w.getnframes())


def test_batch_sends_handlers_segments_longest_first_and_returns_them_in_order(tmp_path, stub):
    lengths = [30000, SEG + 40000, 5000, 120000, 2 * SEG + 3000]
    ins = [_write(tmp_path / f"in{i}.wav", n, i)[0] for i, n in enumerate(lengths)]
    tgts = [_write(tmp_path / f"tgt{i}.wav", n, 50 + i)[0] if i % 2 else None for i, n in enumerate(lengths)]
    one = [HU.handler(s, str(tmp_path / f"one{i}.wav"), t, None, "cpu") for i, (s, t) in enumerate(zip(ins, tgts))]
    per_file = [c[0] for c in stub._eng.calls]
    assert per_file == [e - s for n in lengths for s, e in HU.segment_bounds(n)]       # handler()'s break_point loop
    stub._eng.calls.clear()
    batch = HU.handler_batch([(s, str(tmp_path / f"batch{i}.wav"), t) for i, (s, t) in enumerate(zip(ins, tgts))], None, "cpu")
    assert stub._eng.calls == [[SEG, SEG, SEG], [120000, 40000, 30000, 5000, 3000]]
    assert batch == one
    for i, src in enumerate(ins):
        assert _frames(str(tmp_path / f"batch{i}.wav")) == _frames(src)                 # the stub restores the identity
        assert _frames(str(tmp_path / f"one{i}.wav")) == _frames(src)
    assert HU.handler_batch([], None, "cpu") == []


def test_dict_is_the_last_segments_with_the_reference_keys_in_order(tmp_path, stub):
    n = SEG + 5000
    src, x = _write(tmp_path / "in.wav", n, 1)
    tgt, t = _write(tmp_path / "tgt.wav", n, 2)
    for res in (HU.handler(src, str(tmp_path / "one.wav"), tgt, None, "cpu"),
                HU.handler_batch([(src, str(tmp_path / "batch.wav"), tgt)], None, "cpu")[0]):
        assert list(res) == KEYS
        assert res["mel-lsd"] == _stub_mel(x[SEG] / 32768.0, 5000)[0, 0]      # the restored last segment's mel
        assert res["mel-ssim"] == _stub_mel(t[SEG] / 32768.0, 5000)[0, 0]     # against the last target slice's mel
        assert res["mel-sispec"] == 11.0 and res["mel-non-log-sispec"] == 0.0   # to_log of both / neither
    assert HU.handler(src, str(tmp_path / "none.wav"), None, None, "cpu") == {}


@pytest.mark.parametrize("n, n_target, exc", [
    (SEG + 1000, None, EngineError),            # last segment of 1000 samples
    (0, None, RuntimeError),                    # nothing to restore
    (5000, 1000, EngineError),                  # the target slice is too short for the front end
    (5000, 6000, AssertionError),               # the target slice has another frame count
    (2000, 2000, ValueError),                   # 5 frames with a target: mel-ssim's 7x7 window
    (SEG + 2000, SEG + 2000, ValueError),       # ... in the last segment
])
def test_rejected_file_fails_like_handler_before_any_restore_or_write(tmp_path, stub, n, n_target, exc):
    tgt = _write(tmp_path / "tgt.wav", n_target, 3)[0] if n_target is not None else None
    bad = (_write(tmp_path / "bad.wav", n, 2)[0], str(tmp_path / "bad_out.wav"), tgt)
    with pytest.raises(exc):
        HU.handler(*bad, None, "cpu")
    stub._eng.calls.clear()
    good = (_write(tmp_path / "good.wav", 30000, 1)[0], str(tmp_path / "good_out.wav"), None)
    with pytest.raises(exc, match="bad.wav"):
        HU.handler_batch([good, bad, good], None, "cpu")
    assert stub._eng.calls == []
    assert not os.path.exists(good[1]) and not os.path.exists(bad[1])


def _hp(unet):
    from voicefixer_main_b200.model import HParams, default_hparams
    d = json.loads(json.dumps(default_hparams()))
    if unet is not None:
        d["task"]["ssr"] = {"ssr_task": {"denoising": True}, "ssr_model": {"unet": unet}}
    return HParams(**d)


@pytest.mark.parametrize("unet, cls", [(True, "SSR_UNet"), (False, "GSR_UNet"), (None, "GSR_UNet")])
def test_refresh_model_picks_the_class_from_hp(tmp_path, monkeypatch, unet, cls):
    import voicefixer_main_b200 as P
    ckpt = str(tmp_path / "m.ckpt")
    torch.save({"state_dict": {}}, ckpt)
    monkeypatch.setattr(HU, "model", None)
    monkeypatch.setattr(HU, "hp", _hp(unet))
    HU.refresh_model(ckpt)
    assert type(HU.model) is getattr(P, cls) and not HU.model.training
    monkeypatch.setattr(HU, "hp", None)                 # no hp: default_hparams(), which selects no SSR model
    HU.refresh_model(ckpt)
    assert type(HU.model) is P.GSR_UNet
