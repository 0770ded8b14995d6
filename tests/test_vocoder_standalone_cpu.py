"""The stand-alone Vocoder's host side without a GPU: packing arithmetic, argument checks (every refusal before any engine
call) and oracle's segmentation, against stub engines."""
import numpy as np
import pytest
import torch

from voicefixer_main_b200 import handler as H
from voicefixer_main_b200.arch import VocoderConfig, vocoder_out_len
from voicefixer_main_b200.vocoder import Vocoder, check_mels, length_groups, packing


class StubEngine:
    """Records the packed calls; the vocoder output of clip i is L_i copies of i, the resynthesis halves its input."""

    def __init__(self, device="cpu"):
        self.device = torch.device(device)
        self.loaded = True
        self.calls = []

    def vocoder_varlen(self, mel_packed, frames):
        self.calls.append(("vocoder_varlen", tuple(mel_packed.shape), list(frames)))
        return torch.cat([torch.full((vocoder_out_len(t, VocoderConfig()),), float(i)) for i, t in enumerate(frames)])

    def resynth_varlen(self, wav_packed, lengths):
        self.calls.append(("resynth_varlen", list(lengths)))
        return wav_packed * 0.5

    def to_pcm16(self, x, saturate=False):
        return torch.from_numpy((x.numpy() * np.float32(32768)).astype(np.int32).astype(np.int16))


def stub_vocoder(device="cpu"):
    v = Vocoder()
    v._eng = StubEngine(device)
    v.device = v._eng.device
    return v


def test_packing_arithmetic():
    frames = [1, 2, 3, 63, 64, 65, 101, 1001, 6001]
    f, s = packing(frames)
    assert f == [0, 1, 3, 6, 69, 133, 198, 299, 1300, 7301]
    # L = (T + T % 2 + tail_pad_base) * hop
    want = [(t + t % 2 + 4) * 441 for t in frames]
    assert [s[i + 1] - s[i] for i in range(len(frames))] == want
    assert want[:3] == [2646, 2646, 3528]
    assert s[-1] == sum(want)


def test_length_groups():
    # buckets 64, 6016, 128, 64, 1024, 3008, 3136, 576, 512: longest first, a clip joins the open group while its bucket
    # exceeds half of the bucket of the group's first clip
    assert length_groups([1, 6001, 65, 64, 1001, 3000, 3100, 513, 512]) == [[1, 6], [5], [4, 7], [8], [2], [3, 0]]
    assert length_groups([5]) == [[0]]
    assert sorted(i for g in length_groups(list(range(1, 400))) for i in g) == list(range(399))


def test_forward_batch_splits_at_the_clip_boundaries():
    v = stub_vocoder()
    frames = [3, 64, 1, 6001]
    outs = v.forward_batch([torch.zeros(t, 128) for t in frames])
    # one packed call per length group, longest first; the stub's clip i of a call is filled with i
    assert v._eng.calls == [("vocoder_varlen", (6001, 128), [6001]), ("vocoder_varlen", (68, 128), [64, 3, 1])]
    assert [o.numel() for o in outs] == [vocoder_out_len(t, VocoderConfig()) for t in frames]
    assert [set(o.tolist()) for o in outs] == [{1.0}, {0.0}, {2.0}, {0.0}]


def test_forward_packs_equal_lengths():
    v = stub_vocoder()
    y = v(torch.zeros(3, 1, 5, 128))
    assert v._eng.calls == [("vocoder_varlen", (15, 128), [5, 5, 5])]
    assert y.shape == (3, 1, vocoder_out_len(5, VocoderConfig()))


@pytest.mark.parametrize("mel, exc", [
    ("not a tensor", TypeError),
    (torch.zeros(1, 1, 5, 128, dtype=torch.float64), TypeError),
    (torch.zeros(1, 5, 128), ValueError),
    (torch.zeros(1, 2, 5, 128), ValueError),
    (torch.zeros(1, 1, 5, 80), ValueError),
    (torch.zeros(1, 1, 0, 128), ValueError),
])
def test_forward_refusals(mel, exc):
    v = stub_vocoder()
    with pytest.raises(exc):
        v.forward(mel)
    assert v._eng.calls == []


def test_forward_cuda_flag():
    """A mel that is not on the vocoder's device needs cuda=True (there is no CPU path)."""
    v = stub_vocoder("meta")
    with pytest.raises(RuntimeError, match="cuda=True"):
        v.forward(torch.zeros(1, 1, 5, 128), cuda=False)
    assert v._eng.calls == []


@pytest.mark.parametrize("mels, exc", [
    ([], ValueError),
    ("mels", ValueError),
    ([torch.zeros(5, 128), torch.zeros(5, 127)], ValueError),
    ([torch.zeros(1, 5, 128)], ValueError),
    ([torch.zeros(0, 128)], ValueError),
    ([torch.zeros(5, 128, dtype=torch.float16)], TypeError),
])
def test_forward_batch_refusals(mels, exc):
    v = stub_vocoder()
    with pytest.raises(exc):
        v.forward_batch(mels)
    assert v._eng.calls == []
    with pytest.raises(exc):
        check_mels(mels, torch.device("cpu"))


def test_resynth_batch_refusals():
    v = stub_vocoder()
    for wavs in ([], [torch.zeros(2000), torch.zeros(1024)], [torch.zeros(1, 2000)], [torch.zeros(2000, dtype=torch.float64)]):
        with pytest.raises((ValueError, TypeError)):
            v.resynth_batch(wavs)
    assert v._eng.calls == []


def test_not_on_a_device():
    v = Vocoder()
    for call in (lambda: v.forward(torch.zeros(1, 1, 5, 128)), lambda: v.forward_batch([torch.zeros(5, 128)]),
                 lambda: v.resynth_batch([torch.zeros(2000)]), lambda: v.oracle("in.wav", "out.wav")):
        with pytest.raises(RuntimeError, match="CUDA device|cuda"):
            call()
    with pytest.raises(RuntimeError, match="cuda=False"):
        stub_vocoder().oracle("in.wav", "out.wav", cuda=False)
    with pytest.raises(RuntimeError, match="cuda=False"):
        stub_vocoder().oracle_batch([("in.wav", "out.wav")], cuda=False)
    with pytest.raises(NotImplementedError):
        Vocoder(sample_rate=16000)


def test_load_state_dict_accepts_both_key_forms():
    from voicefixer_main_b200.weights import make_vocoder_state
    sd = make_vocoder_state()
    bare = {k[len("vocoder."):]: t for k, t in sd.items()}
    a = Vocoder().load_state_dict(sd)
    b = Vocoder().load_state_dict({**bare, "generator.x": torch.zeros(1)})
    assert a.state_dict().keys() == b.state_dict().keys() == sd.keys()
    with pytest.raises(NotImplementedError):
        Vocoder().load_state_dict(sd, strict=False)


def test_oracle_segments_as_handler(tmp_path):
    """oracle cuts a file into handler()'s 60 s segments and resynthesises them with resynth_batch."""
    n = 2 * H.SEG_LENGTH + 5000
    x = (np.sin(np.arange(n) * 0.01) * 0.5).astype(np.float32)
    src, dst = str(tmp_path / "in.wav"), str(tmp_path / "out.wav")
    H.save_wave(x, src)
    v = stub_vocoder()
    v.oracle(src, dst)
    bounds = H.segment_bounds(n)
    assert [e - s for s, e in bounds] == [H.SEG_LENGTH, H.SEG_LENGTH, 5000]
    assert v._eng.calls == [("resynth_varlen", [H.SEG_LENGTH, H.SEG_LENGTH]), ("resynth_varlen", [5000])]
    got, rate = H.read_pcm16(dst)
    assert rate == 44100 and got.shape == (n,)
    wav = H.load_wav(src)
    assert np.array_equal(got, (wav * np.float32(0.5) * np.float32(32768)).astype(np.short) / np.float32(32768))
    # a file with a segment of 1024 samples or fewer fails as handler() does, before any call
    H.save_wave(np.zeros(H.SEG_LENGTH + 1000, np.float32), src)
    v = stub_vocoder()
    with pytest.raises(Exception, match="reflect padding"):
        v.oracle(src, dst)
    assert v._eng.calls == []


def test_oracle_batch_groups_full_segments(tmp_path):
    lengths = [H.SEG_LENGTH + 3000, 4000, 2 * H.SEG_LENGTH]
    items = []
    for i, n in enumerate(lengths):
        src = str(tmp_path / f"in{i}.wav")
        H.save_wave(np.full(n, 0.25, np.float32), src)
        items.append((src, str(tmp_path / f"out{i}.wav")))
    v = stub_vocoder()
    v.oracle_batch(items)
    assert v._eng.calls == [("resynth_varlen", [H.SEG_LENGTH] * 3), ("resynth_varlen", [4000, 3000])]
    for (_, out), n in zip(items, lengths):
        assert H.read_pcm16(out)[0].shape == (n,)
