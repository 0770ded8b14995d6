"""The WAV parser (voicefixer_main_b200/wavfile.py) and the decode oracle (oracle/wavfile.py) on hand-built files: every
sample format and channel count against scipy.io.wavfile.read, the downmix against numpy's own mean, 16-bit files against
read_pcm16, and the files that must be rejected.  No GPU."""
import numpy as np
import pytest
import torch
from scipy.io import wavfile as scipy_wav

from oracle import wavfile as O
from voicefixer_main_b200 import wavfile as W
from voicefixer_main_b200.handler import decode_wavs, load_wav, read_pcm16

CHANNELS = (1, 2, 3, 6, 8, 9, 16)
FORMATS = (W.U8, W.S16, W.S24, W.S32, W.F32, W.F64)
EXTRA = ((b"LIST", b"INFOISFT\x05\x00\x00\x00vf1\x00\x00"), (b"bext", b"odd"))      # odd payloads: pad bytes


def _file(tmp_path, name, frames, channels, fmt, seed=0, **kw):
    x = O.random_data(np.random.default_rng(seed), frames, channels, fmt)
    path = tmp_path / name
    path.write_bytes(O.wav_bytes(O.encode(x, fmt), 48000, channels, fmt, **kw))
    return str(path), x


def _scaled(ref, fmt):
    """scipy's read scaled as libsndfile normalises it, in float64: u8 offset, integers left-justified in their dtype."""
    if fmt == W.U8:
        return (ref.astype(np.float64) - 128) / 128
    if fmt in (W.F32, W.F64):
        return ref.astype(np.float64)
    return ref.astype(np.float64) / -float(np.iinfo(ref.dtype).min)


def _same(a, b):
    """Bit-identical, NaN matching NaN."""
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b, equal_nan=True) and \
        np.array_equal(np.signbit(a), np.signbit(b))


@pytest.mark.filterwarnings("ignore::scipy.io.wavfile.WavFileWarning")      # scipy skips the LIST / bext chunks too
@pytest.mark.parametrize("fmt", FORMATS, ids=W.NAMES)
@pytest.mark.parametrize("channels", CHANNELS)
def test_parser_and_oracle_match_scipy(tmp_path, fmt, channels):
    for k, kw in enumerate(({}, {"before": EXTRA}, {"after": EXTRA, "extensible": True})):
        path, _ = _file(tmp_path, f"f{k}.wav", 301, channels, fmt, seed=channels, **kw)
        w = W.parse(path)
        rate, ref = scipy_wav.read(path)
        ref = ref.reshape(len(ref), -1)
        assert (w.rate, w.channels, w.format, w.frames) == (rate, channels, fmt, 301) == (48000, ref.shape[1], fmt, ref.shape[0])
        assert len(w.data) == 301 * channels * W.WIDTH[fmt]
        exact = _scaled(ref, fmt)
        x = O.samples(w.data, w.channels, w.format)
        assert x.dtype == np.float32 and np.array_equal(x, exact.astype(np.float32))
        if fmt not in (W.S32, W.F64):                 # the float32 value is the exact one
            assert np.array_equal(x.astype(np.float64), exact)
        assert _same(O.first64(w.data, w.channels, w.format), exact[:, 0])


@pytest.mark.parametrize("channels", list(CHANNELS) + [5, 7, 15, 17, 23, 24, 31, 33, 63, 64])
def test_downmix_is_numpys_mean(channels):
    rng = np.random.default_rng(channels)
    x = (rng.standard_normal((20000, channels)) * np.exp2(rng.integers(-40, 40, (20000, channels)))).astype(np.float32)
    x[::13] = -0.0
    want = x[:, 0] if channels == 1 else x.mean(axis=1)
    assert _same(O.downmix(x), want)


def test_one_channel_keeps_the_sign_of_zero():
    x = np.array([[-0.0], [0.0], [1.5]], np.float32)
    assert _same(O.downmix(x), x[:, 0])        # librosa leaves a 1-D signal alone; mean(axis=1) would give +0.0


@pytest.mark.parametrize("channels", CHANNELS)
def test_16_bit_oracle_is_read_pcm16(tmp_path, channels):
    path, _ = _file(tmp_path, "a.wav", 4410, channels, W.S16, seed=3)
    mono, rate, first = O.load(path)
    got, got_rate = read_pcm16(path)
    assert rate == got_rate == 48000 and _same(mono, got)
    (x, r, c), = decode_wavs([path], first=True)          # a 16-bit file needs no engine
    assert r == 48000 and _same(x, got) and _same(c, first.astype(np.float32))
    assert np.array_equal(c.astype(np.float64), first)


def test_data_chunk_past_the_end_and_partial_frames(tmp_path):
    x = O.random_data(np.random.default_rng(1), 100, 2, W.S24)
    data = O.encode(x, W.S24)
    path = tmp_path / "cut.wav"
    path.write_bytes(O.wav_bytes(data, 44100, 2, W.S24, data_size=len(data) + 1000))
    w = W.parse(str(path))
    assert w.frames == 100 and bytes(w.data) == data
    path.write_bytes(O.wav_bytes(data + b"\x01\x02\x03\x04", 44100, 2, W.S24))        # 4 bytes: not a whole frame
    w = W.parse(str(path))
    assert w.frames == 100 and bytes(w.data) == data


def test_extensible_valid_bits_read_at_container_width(tmp_path):
    x = O.random_data(np.random.default_rng(2), 50, 2, W.S24) & ~0xF          # 20 valid bits in 24
    path = tmp_path / "e.wav"
    path.write_bytes(O.wav_bytes(O.encode(x, W.S24), 96000, 2, W.S24, extensible=True, valid_bits=20))
    w = W.parse(str(path))
    assert (w.format, w.rate, w.frames) == (W.S24, 96000, 50)
    assert np.array_equal(O.samples(w.data, 2, W.S24), (x / 2.0 ** 23).astype(np.float32))


@pytest.mark.parametrize("case, match", [
    ({"tag": 7}, "compressed format tag 0x0007 \\(mu-law\\)"),
    ({"tag": 6}, "compressed format tag 0x0006 \\(A-law\\)"),
    ({"tag": 2}, "compressed format tag 0x0002 \\(MS ADPCM\\)"),
    ({"tag": 0x11}, "compressed format tag 0x0011 \\(IMA ADPCM\\)"),
    ({"block_align": 5}, "block align 5 is not 2 channels x 2 bytes"),
    ({"tag": 3}, "16-bit IEEE float is not supported"),
])
def test_rejected_headers(tmp_path, case, match):
    path = tmp_path / "bad.wav"
    path.write_bytes(O.wav_bytes(b"\x00" * 40, 44100, 2, W.S16, **case))
    with pytest.raises(ValueError, match=match) as e:
        W.parse(str(path))
    assert str(path) in str(e.value)


def test_rejected_containers(tmp_path):
    good = O.wav_bytes(b"\x00" * 40, 44100, 2, W.S16)
    cases = {
        "rf64.wav": (b"RF64" + good[4:], "RF64"),
        "rifx.wav": (b"RIFX" + good[4:], "RIFX"),
        "text.wav": (b"hello world, not a wav", "not a RIFF WAVE"),
        "nofmt.wav": (good.replace(b"fmt ", b"junk"), "no 'fmt ' chunk"),
        "nodata.wav": (good.replace(b"data", b"junk"), "no 'data' chunk"),
        "mp3.wav": (O.wav_bytes(b"\x00" * 40, 44100, 2, W.S16, extensible=True, tag=0x55), "compressed format tag 0x0055"),
        "guid.wav": (O.wav_bytes(b"\x00" * 40, 44100, 2, W.S16, extensible=True).replace(b"\x38\x9b\x71", b"\x38\x9b\x72"),
                     "subformat GUID"),
        "c65.wav": (O.wav_bytes(b"", 44100, 65, W.S16), "65 channels"),
        "c0.wav": (O.wav_bytes(b"", 44100, 0, W.S16), "0 channels"),
        "rate0.wav": (O.wav_bytes(b"\x00" * 4, 0, 2, W.S16), "sample rate 0"),
    }
    bits12 = bytearray(good)
    bits12[34:36] = (12).to_bytes(2, "little")
    cases["bits12.wav"] = (bytes(bits12), "12-bit PCM")
    for name, (raw, match) in cases.items():
        path = tmp_path / name
        path.write_bytes(raw)
        with pytest.raises(ValueError, match=match):
            W.parse(str(path))


def test_other_formats_need_an_engine(tmp_path):
    path, _ = _file(tmp_path, "a.wav", 2000, 2, W.S24)
    with pytest.raises(ValueError, match="engine="):
        load_wav(path, sample_rate=48000)
    with pytest.raises(ValueError, match="engine="):
        decode_wavs([path])
    with pytest.raises(ValueError, match="need 16-bit PCM"):
        read_pcm16(path)


@pytest.mark.parametrize("fmt", (W.S32, W.F64), ids=("s32", "f64"))
def test_time_domain_scoring_refuses_a_rounded_first_channel(tmp_path, fmt):
    from voicefixer_main_b200.edges import AudioMetrics
    path, _ = _file(tmp_path, "t.wav", 44100, 2, fmt)
    est, _ = _file(tmp_path, "e.wav", 44100, 1, W.S16)
    with pytest.raises(ValueError, match="do not fit float32 exactly"):
        AudioMetrics(object()).evaluation(est, path, time_domain=True)


def test_evaluation_batch_takes_any_iterable_of_pairs(tmp_path):
    from voicefixer_main_b200.edges import AudioMetrics

    class Scorer:             # stands in for the engine: the two scoring calls, recorded
        device = "cpu"

        def __init__(self):
            self.calls = []

        def score_varlen(self, est, est_lengths, target, target_lengths):
            self.calls.append((est.clone(), list(est_lengths), target.clone(), list(target_lengths)))
            return torch.arange(8 * len(est_lengths), dtype=torch.float64).view(-1, 8)

    ests = [_file(tmp_path, f"e{i}.wav", 44100 + 441 * i, 1, W.S16, seed=i)[0] for i in range(2)]
    tgts = [_file(tmp_path, f"t{i}.wav", 44100 + 441 * i, 2, W.S16, seed=9 + i)[0] for i in range(2)]
    for path in ests + tgts:         # AudioMetrics scores 44.1 kHz targets; _file writes 48 kHz
        raw = bytearray(open(path, "rb").read())
        raw[24:28] = (44100).to_bytes(4, "little")
        open(path, "wb").write(bytes(raw))
    eng = Scorer()
    from_list = AudioMetrics(eng).evaluation_batch(list(zip(ests, tgts)))
    from_iter = AudioMetrics(eng).evaluation_batch(zip(ests, tgts))
    assert len(from_list) == 2 and from_iter == from_list
    a, b = eng.calls
    assert all(torch.equal(x, y) if isinstance(x, torch.Tensor) else x == y for x, y in zip(a, b))
    assert a[1] == [44100, 44541] and a[3] == [44100, 44541]
