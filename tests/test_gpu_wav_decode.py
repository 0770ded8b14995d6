"""vf_decode_pcm_varlen (Engine.decode_pcm_varlen) against the decode oracle, bit for bit, and the file paths that use it:
24-bit and float stereo files through handler_batch, handler and restore_array."""
import numpy as np
import pytest
import torch

from oracle import vf_oracle as VO
from oracle import wavfile as O
from voicefixer_main_b200 import wavfile as W

pytestmark = pytest.mark.gpu

CHANNELS = (1, 2, 3, 6, 8, 9, 16)
FORMATS = (W.U8, W.S16, W.S24, W.S32, W.F32, W.F64)
LENGTHS = (1, 2, 1023, 3 * 48000 + 7)


@pytest.fixture(scope="module")
def eng():
    from voicefixer_main_b200.model import Engine
    e = Engine("cuda:0")
    yield e
    e.check_errors()
    e.close()


def _info(x, fmt, rate=48000):
    """An in-memory WavInfo of samples x [frames, C]."""
    return W.WavInfo("<memory>", rate, x.shape[1], fmt, x.shape[0], memoryview(O.encode(x, fmt)))


def _same(a, b):
    """Bit-identical, NaN matching NaN (whatever its payload)."""
    a, b = np.asarray(a), np.asarray(b)
    nan = np.isnan(a)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(nan, np.isnan(b)) and \
        np.array_equal(a[~nan].view(np.uint8), b[~nan].view(np.uint8))


def _oracle(w):
    return O.downmix(O.samples(w.data, w.channels, w.format)), O.first64(w.data, w.channels, w.format)


def _rows(eng, infos, first=True):
    mono, ch0 = eng.decode_pcm_varlen(infos, first=first)
    cut = np.cumsum([w.frames for w in infos])[:-1]
    return np.split(mono.cpu().numpy(), cut), (np.split(ch0.cpu().numpy(), cut) if first else None)


def test_every_format_and_channel_count_in_one_call(eng):
    rng = np.random.default_rng(0)
    infos = [_info(O.random_data(rng, n, c, f), f) for f in FORMATS for c in CHANNELS for n in LENGTHS]
    mono, first = _rows(eng, infos)
    for w, m, f in zip(infos, mono, first):
        want_m, want_f = _oracle(w)
        assert _same(m, want_m), (W.NAMES[w.format], w.channels, w.frames)
        assert _same(f, want_f), (W.NAMES[w.format], w.channels, w.frames)
    _, none = _rows(eng, infos[:3], first=False)
    assert none is None


def test_special_float_values(eng):
    special = [np.nan, np.inf, -np.inf, -0.0, 0.0, 1e-40, -1e-45, 3e38, 1e-300, -1e300, 1.0000000596046448]
    rng = np.random.default_rng(1)
    infos = []
    for fmt in (W.F32, W.F64):
        for c in (1, 2, 9):
            x = rng.choice(np.array(special), size=(4000, c))
            infos.append(_info(x.astype(np.float32 if fmt == W.F32 else np.float64), fmt))
    mono, first = _rows(eng, infos)
    for w, m, f in zip(infos, mono, first):
        with np.errstate(over="ignore", invalid="ignore"):           # Inf - Inf, float64 beyond float32's range
            want_m, want_f = _oracle(w)
        assert _same(m, want_m) and _same(f, want_f), (W.NAMES[w.format], w.channels)


def test_bits_do_not_depend_on_batch_slot_or_split(eng):
    rng = np.random.default_rng(2)
    probe = [_info(O.random_data(rng, 5000, c, f), f) for f, c in ((W.S24, 2), (W.F32, 9), (W.U8, 3))]
    alone = [_rows(eng, [w]) for w in probe]
    filler = [_info(O.random_data(rng, int(n), 2, W.S16), W.S16) for n in rng.integers(1, 50, 1500)]
    for slot in (0, 1, 1023, 1024, 1499):            # 1500 rows: two sub-batches, the split at row 1024
        infos = filler[:slot] + probe + filler[slot:]
        mono, first = _rows(eng, infos)
        for k, (m, f) in enumerate(alone):
            assert _same(mono[slot + k], m[0]) and _same(first[slot + k], f[0]), (slot, k)
    for k, w in enumerate(probe):
        want_m, _ = _oracle(w)
        assert _same(alone[k][0][0], want_m)


def test_16_bit_stereo_is_read_pcm16(eng, tmp_path):
    from voicefixer_main_b200.handler import read_pcm16
    path = tmp_path / "s.wav"
    x = O.random_data(np.random.default_rng(3), 44100, 2, W.S16)
    path.write_bytes(O.wav_bytes(O.encode(x, W.S16), 44100, 2, W.S16))
    mono, first = _rows(eng, [W.parse(str(path))])
    got, _ = read_pcm16(str(path))
    assert _same(mono[0], got)
    assert _same(first[0], x[:, 0] / 32768.0)


def _speech(n, seed, channels):
    """Seeded speech-like stereo samples in [-0.99, 0.99]: one synthetic clip per channel."""
    return np.stack([VO.synth_clips(1, n, seed=seed + c)[0].clamp(-0.99, 0.99).numpy().astype(np.float64)
                     for c in range(channels)], axis=1)


@pytest.fixture(scope="module")
def model(state):
    from voicefixer_main_b200 import VoiceFixer
    m = VoiceFixer().load_state_dict(state).eval().to("cuda:0")
    yield m
    m._engine().check_errors()
    m._eng.close()
    torch.cuda.empty_cache()


def test_handler_batch_on_24_bit_and_float_stereo(model, tmp_path, monkeypatch):
    from voicefixer_main_b200 import handler as H
    monkeypatch.setattr(H, "model", model)
    eng = model._engine()
    items = []
    for i, (fmt, n) in enumerate(((W.S24, 48000 + 311), (W.F32, 2 * 48000), (W.S24, 72000))):
        x = _speech(n, 40 + 3 * i, 2)
        data = O.encode(np.round(x * 2 ** 23).astype(np.int64) if fmt == W.S24 else x.astype(np.float32), fmt)
        src, tgt = tmp_path / f"in{i}.wav", tmp_path / f"tgt{i}.wav"
        src.write_bytes(O.wav_bytes(data, 48000, 2, fmt, extensible=i == 2))
        t = _speech(n, 90 + i, 2)
        tgt.write_bytes(O.wav_bytes(O.encode(t.astype(np.float32), W.F32), 48000, 2, W.F32))
        items.append((str(src), f"out{i}.wav", str(tgt) if i != 1 else None))
    (tmp_path / "one").mkdir()
    (tmp_path / "batch").mkdir()
    one = [H.handler(s, str(tmp_path / "one" / o), t, ckpt=None, device=model.device) for s, o, t in items]
    batch = H.handler_batch([(s, str(tmp_path / "batch" / o), t) for s, o, t in items], ckpt=None, device=model.device)
    eng.check_errors()
    assert one == batch and one[0] and not one[1]
    for src, out, _ in items:
        a, b = (tmp_path / "one" / out).read_bytes(), (tmp_path / "batch" / out).read_bytes()
        assert a == b, out
        mono, rate, _ = O.load(src)
        wav = H._to_rate(src, mono, rate, 44100, eng)
        pcm = eng.to_pcm16(H.restore_array(model, wav, model.device)[0]).cpu().numpy()
        w = W.parse(str(tmp_path / "one" / out))
        assert (w.rate, w.channels, w.format) == (44100, 1, W.S16)
        assert np.array_equal(np.frombuffer(w.data, "<i2"), pcm), out


def test_evaluation_scores_a_float_stereo_target_as_decoded(model, tmp_path):
    from voicefixer_main_b200.edges import SCORE_KEYS, TIME_KEYS, AudioMetrics
    from voicefixer_main_b200.handler import save_pcm16
    eng = model._engine()
    n = 44100 + 777
    est = tmp_path / "est.wav"
    save_pcm16((_speech(n, 7, 1)[:, 0] * 32767).astype(np.int16), str(est))
    tgt = tmp_path / "tgt.wav"
    tgt.write_bytes(O.wav_bytes(O.encode(_speech(n, 8, 2).astype(np.float32), W.F32), 44100, 2, W.F32))
    got = AudioMetrics(model).evaluation(str(est), str(tgt), time_domain=True)
    (e, _, e0), (t, _, t0) = O.load(str(est)), O.load(str(tgt))
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(eng.device)
    spectral = eng.score_varlen(dev(e), [n], dev(t), [n]).cpu().tolist()[0]
    td = eng.score_time_varlen(dev(e0), [n], dev(t0), [n]).cpu().tolist()[0]
    assert got == dict(zip(TIME_KEYS, td), **dict(zip(SCORE_KEYS, spectral)))
