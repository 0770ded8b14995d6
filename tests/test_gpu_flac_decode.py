"""vf_decode_flac_varlen (Engine.decode_flac_varlen) against the FLAC oracle and against the WAV path, bit for bit, and
the file paths that read FLAC: handler, handler_batch, evaluation_batch, oracle_batch, make_sr_testset, restore_file and
convert_flac_to_wav."""
import os

import numpy as np
import pytest
import torch

from oracle import flac as F
from oracle import vf_oracle as VO
from oracle import wavfile as OW
from voicefixer_main_b200 import flacfile as FF
from voicefixer_main_b200 import wavfile as W

pytestmark = pytest.mark.gpu

PCM_FORMAT = {8: W.U8, 16: W.S16, 24: W.S24}


@pytest.fixture(scope="module")
def eng():
    from voicefixer_main_b200.model import Engine
    e = Engine("cuda:0")
    yield e
    e.check_errors()
    e.close()


def _write(tmp_path, name, raw):
    p = tmp_path / name
    p.write_bytes(raw)
    return str(p)


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _split(mono, ch0, frames):
    cut = np.cumsum(frames)[:-1]
    return np.split(mono.cpu().numpy(), cut), np.split(ch0.cpu().numpy(), cut)


def test_feature_matrix_in_one_call_matches_the_oracle_and_the_wav_path(eng, tmp_path):
    streams = F.feature_matrix(seed=0)
    infos = [FF.parse(_write(tmp_path, f"{name}.flac", raw)) for name, raw, _, _, _ in streams]
    pcm = eng.decode_flac_pcm(infos)
    for (name, raw, x, bits, rate), w, b in zip(streams, infos, pcm):
        assert (w.rate, w.channels, w.bits, w.total) == (rate, x.shape[1], bits, x.shape[0]), name
        assert b.tobytes() == F.wav_bytes(x, bits), name
        assert FF.pcm_bytes_md5(b, bits) == w.md5 == F.md5_of(x, bits), name
    mono, ch0 = _split(*eng.decode_flac_varlen(infos, first=True), [w.total for w in infos])
    wavs = [W.WavInfo("<memory>", rate, x.shape[1], PCM_FORMAT[bits], x.shape[0], memoryview(F.wav_bytes(x, bits)))
            for _, _, x, bits, rate in streams]
    wmono, wch0 = _split(*eng.decode_pcm_varlen(wavs, first=True), [w.frames for w in wavs])
    for (name, raw, x, bits, rate), m, c, wm, wc, wv in zip(streams, mono, ch0, wmono, wch0, wavs):
        assert _same(m, wm) and _same(c, wc), name
        want = OW.downmix(OW.samples(wv.data, wv.channels, wv.format))
        assert _same(m, want) and _same(c, OW.first64(wv.data, wv.channels, wv.format)), name


def test_bits_do_not_depend_on_batch_slot_or_split(eng, tmp_path):
    streams = F.feature_matrix(seed=1)
    probe = [FF.parse(_write(tmp_path, f"p{i}.flac", s[1])) for i, s in enumerate(streams[::9])]
    alone = [eng.decode_flac_varlen([w], first=True) for w in probe]
    rng = np.random.default_rng(5)
    filler = []
    for i in range(600):                                  # 600 rows: two sub-batches, the split at row 512
        bits = (8, 16, 24)[i % 3]
        x = F.signal(rng, int(rng.integers(1, 300)), 1 + i % 3, bits)
        filler.append(FF.parse(_write(tmp_path, f"f{i}.flac", F.encode(x, 8000, bits, blocks=int(rng.integers(16, 200)),
                                                                       variable=bool(i % 2)))))
    for slot in (0, 511, 512, 600):
        infos = filler[:slot] + probe + filler[slot:]
        mono, ch0 = _split(*eng.decode_flac_varlen(infos, first=True), [w.total for w in infos])
        for k, (m, c) in enumerate(alone):
            assert _same(mono[slot + k], m.cpu().numpy()) and _same(ch0[slot + k], c.cpu().numpy()), (slot, k)


def test_a_header_inside_a_verbatim_frame_does_not_change_the_result(eng, tmp_path):
    bits, block = 16, 256
    x = F.signal(np.random.default_rng(2), 4 * block, 1, bits)
    fake = F.frame_bytes(x[block:2 * block], 1, bits)[:6]   # the next frame's complete header, valid CRC-8
    assert F.crc8(fake[:5]) == fake[5]
    words = np.frombuffer(fake, ">i2").astype(np.int64)
    x[100:103, 0] = words                                    # frame 0's samples 100 .. 102, big-endian on the wire
    raw = F.encode(x, 44100, bits, blocks=block, frame=lambda k, s, b: {"subframes": [{"type": "verbatim"}]})
    assert fake in raw[raw.index(b"\xff\xf8"):]
    w = FF.parse(_write(tmp_path, "fake.flac", raw))
    assert eng.decode_flac_pcm([w])[0].tobytes() == F.wav_bytes(x, bits)


def test_six_byte_sample_numbers(eng, tmp_path):
    frames, values, start = [], [], 0
    n_frames = 1030                                          # 1030 x 65535 > 2^26: the last frames' numbers take 6 bytes
    for k in range(n_frames):
        v = (k * 37) % 255 - 127
        frames.append(F.frame_bytes(np.full((65535, 1), v), start, 8, variable=True,
                                    subframes=[{"type": "constant"}]))
        values.append(v)
        start += 65535
    assert F.coded(start - 65535)[0] == 0xFC and len(F.coded(start - 65535)) == 6
    raw = F.container(frames, 44100, 1, 8, start, 65535, 65535, bytes(16))
    w = FF.parse(_write(tmp_path, "long.flac", raw))
    mono, ch0 = eng.decode_flac_varlen([w], first=True)
    want = np.repeat(np.array(values, np.float32) / np.float32(128), 65535)
    assert _same(mono.cpu().numpy(), want)
    assert _same(ch0.cpu().numpy(), want.astype(np.float64))


def test_a_flipped_bit_or_a_truncated_file_fails_the_call_naming_it(eng, tmp_path):
    x = F.signal(np.random.default_rng(3), 3000, 2, 16)
    raw = F.encode(x, 44100, 16, blocks=1000, frame=lambda k, s, b: {"subframes": [{"type": "verbatim"}] * 2})
    good = FF.parse(_write(tmp_path, "good.flac", raw))
    flipped = bytearray(raw)
    flipped[-1000] ^= 0x04                                  # a sample bit of the last frame
    bad = FF.parse(_write(tmp_path, "flipped.flac", bytes(flipped)))
    with pytest.raises(ValueError, match="flipped.flac: frame CRC-16 mismatch"):
        eng.decode_flac_varlen([good, bad])
    cut = FF.parse(_write(tmp_path, "cut.flac", raw[:-700]))
    with pytest.raises(ValueError, match="cut.flac: a frame runs past the end"):
        eng.decode_flac_varlen([cut, good])
    eng.check_errors()


# ----------------------------------------------------------------------------------------------- the callers
def _speech(n, seed, channels):
    return np.stack([VO.synth_clips(1, n, seed=seed + c)[0].clamp(-0.99, 0.99).numpy().astype(np.float64)
                     for c in range(channels)], axis=1)


def _pair(tmp_path, stem, x, rate, bits):
    """The same int samples as stem.flac and stem.wav -> (flac path, wav path)."""
    f = _write(tmp_path, f"{stem}.flac", F.encode(x, rate, bits, blocks=4096, frame=lambda k, s, b: {
        "assign": 10 if x.shape[1] == 2 else None, "subframes": [{"type": "lpc", "order": 8, "precision": 12, "shift": 11,
                                                                   "coefs": [1400, -300, 0, 0, 0, 0, 0, 0], "porder": 4 if b % 16 == 0 else 0}] *
        x.shape[1]}))
    w = _write(tmp_path, f"{stem}.wav", OW.wav_bytes(F.wav_bytes(x, bits), rate, x.shape[1], PCM_FORMAT[bits]))
    return f, w


def _ints(x, bits):
    return np.round(x * (2 ** (bits - 1) - 1)).astype(np.int64)


@pytest.fixture(scope="module")
def model(state):
    from voicefixer_main_b200 import VoiceFixer
    m = VoiceFixer().load_state_dict(state).eval().to("cuda:0")
    yield m
    m._engine().check_errors()
    m._eng.close()
    torch.cuda.empty_cache()


def test_handler_batch_and_handler_on_flac_are_the_wav_results(model, tmp_path, monkeypatch):
    from voicefixer_main_b200 import handler as H
    monkeypatch.setattr(H, "model", model)
    runs = {}
    for kind in ("flac", "wav"):
        (tmp_path / kind).mkdir()
    items = {"flac": [], "wav": []}
    for i, n in enumerate((48000 + 311, 72000)):
        src = _pair(tmp_path, f"in{i}", _ints(_speech(n, 40 + 3 * i, 2), 24), 48000, 24)
        tgt = _pair(tmp_path, f"tgt{i}", _ints(_speech(n, 90 + i, 2), 24), 48000, 24)
        for j, kind in enumerate(("flac", "wav")):
            items[kind].append((src[j], str(tmp_path / kind / f"out{i}.wav"), tgt[j]))
    for kind in ("flac", "wav"):
        batch = H.handler_batch(items[kind], ckpt=None, device=model.device)
        one = [H.handler(s, o + ".one.wav", t, ckpt=None, device=model.device) for s, o, t in items[kind]]
        runs[kind] = (batch, one, [open(o, "rb").read() for _, o, _ in items[kind]],
                      [open(o + ".one.wav", "rb").read() for _, o, _ in items[kind]])
    model._engine().check_errors()
    assert runs["flac"] == runs["wav"] and runs["flac"][0][0]


def test_evaluation_oracle_sr_testset_and_restore_file_on_flac(model, state, tmp_path):
    from voicefixer_main_b200.edges import AudioMetrics
    from voicefixer_main_b200.handler import restore_file
    from voicefixer_main_b200.lowpass import make_sr_testset
    from voicefixer_main_b200.vocoder import Vocoder
    n = 44100 + 777
    est = [_pair(tmp_path, f"est{i}", _ints(_speech(n, 7 + i, 1), 16), 44100, 16) for i in range(2)]
    tgt = [_pair(tmp_path, f"tgt{i}", _ints(_speech(n, 17 + i, 2), b), 44100, b) for i, b in enumerate((8, 24))]
    am = AudioMetrics(model)
    for td in (False, True):
        got = am.evaluation_batch([(e[0], t[0]) for e, t in zip(est, tgt)], time_domain=td)
        want = am.evaluation_batch([(e[1], t[1]) for e, t in zip(est, tgt)], time_domain=td)
        assert got == want and got
    voc = Vocoder(sample_rate=44100).load_state_dict({k[len("vocoder."):]: t for k, t in state.items()
                                                               if k.startswith("vocoder.")})
    voc = voc.eval().to("cuda:0")
    outs = {}
    for j, kind in enumerate(("flac", "wav")):
        d = tmp_path / f"o_{kind}"
        d.mkdir()
        voc.oracle_batch([(t[j], str(d / f"v{i}.wav")) for i, t in enumerate(tgt)])
        make_sr_testset(model._engine(), [t[j] for t in tgt], str(d / "sr"), cutoffs=(2000,))
        restore_file(model, tgt[0][j], str(d / "r.wav"))
        outs[kind] = sorted((os.path.relpath(os.path.join(r, f), d).replace(".flac", ".wav"),
                             open(os.path.join(r, f), "rb").read() if not f.endswith(".lst") else
                             open(os.path.join(r, f)).read().replace(".flac", ".wav").replace("o_flac", "o_wav"))
                            for r, _, fs in os.walk(d) for f in fs)
    voc._engine().check_errors()
    assert outs["flac"] == outs["wav"]


def test_convert_flac_to_wav(eng, tmp_path):
    rng = np.random.default_rng(4)
    root = tmp_path / "data"
    paths = []
    rels = ("a.flac", "s1/b.flac", "s1/s2/c.flac", "s1/s2/s3/d.flac", "t1/t2/t3/t4/e.flac", "t1/t2/t3/t4/f.flac")
    for i, rel in enumerate(rels):                        # the five depths the reference globs
        os.makedirs(os.path.dirname(root / rel), exist_ok=True)
        bits = (8, 16, 24)[i % 3]
        x = F.signal(rng, 5000 + i, i % 3 + 1, bits)
        (root / rel).write_bytes(F.encode(x, 22050, bits, blocks=1024))
        paths.append((str(root / rel), x, bits))
    os.makedirs(root / "t1/t2/t3/t4/t5")
    too_deep = root / "t1/t2/t3/t4/t5/g.flac"             # a sixth depth, which the reference does not glob
    too_deep.write_bytes(F.encode(F.signal(rng, 500, 1, 16), 22050, 16, blocks=256))
    written = FF.convert_flac_to_wav(str(root), eng, chunk_bytes=8000)   # several decode calls
    assert sorted(written) == sorted(p[:-5] + ".wav" for p, _, _ in paths)
    assert too_deep.exists()
    for p, x, bits in paths:
        assert not os.path.exists(p)
        w = W.parse(p[:-5] + ".wav")
        assert (w.rate, w.channels, w.format) == (22050, x.shape[1], PCM_FORMAT[bits])
        assert bytes(w.data) == F.wav_bytes(x, bits)
    bad = bytearray(F.encode(F.signal(rng, 3000, 1, 16), 22050, 16, blocks=1024))
    bad[-100] ^= 0x10
    (root / "bad.flac").write_bytes(bytes(bad))
    (root / "z.flac").write_bytes(F.encode(F.signal(rng, 3000, 1, 16), 22050, 16, blocks=1024))
    with pytest.raises(ValueError, match="bad.flac"):
        FF.convert_flac_to_wav(str(root), eng)
    assert (root / "bad.flac").exists() and not (root / "bad.wav").exists() and (root / "z.flac").exists()


def test_a_row_full_of_candidate_headers_fails_alone(eng, tmp_path):
    good = [FF.parse(_write(tmp_path, f"g{i}.flac", F.encode(F.signal(np.random.default_rng(i), 3000, 1, 8), 8000, 8,
                                                               blocks=256))) for i in range(2)]
    head = bytearray([0xFF, 0xF8, 0x80, 0x02, 0x00])       # 256 samples, STREAMINFO's rate, mono, 8 bits, frame 0
    head.append(F.crc8(head))
    dense = F.container([bytes(head) * 2000], 8000, 1, 8, 1000, 256, 256, bytes(16))   # a candidate every 6 bytes
    bad = FF.parse(_write(tmp_path, "dense.flac", dense))
    with pytest.raises(ValueError, match="dense.flac"):
        eng.decode_flac_varlen(good + [bad])
    mono, _ = eng.decode_flac_varlen(good)
    assert mono.numel() == 6000


def test_the_first_bad_frame_is_reported_when_a_later_frame_breaks_the_chain(eng, tmp_path):
    x = F.signal(np.random.default_rng(6), 64, 1, 8)
    frames = [F.frame_bytes(x[k * 16:(k + 1) * 16], k, 8) for k in range(4)]
    y = np.full((16, 1), 100)
    y[1] = 200                                             # FIXED-1 predicts 200, outside 8 bits: ERANGE in frame 1
    frames[1] = F.frame_bytes(y, 1, 8, subframes=[{"type": "fixed", "order": 1}])
    f3 = bytearray(frames[3])
    f3[-3] ^= 0x01                                         # frame 3: CRC-16 mismatch, which stops the chain there
    frames[3] = bytes(f3)
    raw = F.container(frames, 8000, 1, 8, 64, 16, 16, bytes(16))
    with pytest.raises(F.FlacError) as want:
        F.decode(raw, "t")
    assert want.value.code == F.ERANGE
    p = _write(tmp_path, "first.flac", raw)
    with pytest.raises(ValueError) as got:
        eng.decode_flac_varlen([FF.parse(p)])
    assert str(got.value) == f"{p}: {FF.ERRORS[F.ERANGE]} (frame at byte {want.value.at})"



def test_every_frame_rejection_names_the_file_and_the_oracles_reason(eng, tmp_path):
    for name, raw, code in F.rejections():
        p = _write(tmp_path, f"{name}.flac", raw)
        try:
            w = FF.parse(p)
        except ValueError as e:                               # caught on the host, at the first frame's header
            assert f"{name}.flac" in str(e)
            continue
        with pytest.raises(ValueError) as e:
            eng.decode_flac_varlen([w])
        assert str(e.value).startswith(f"{p}: {FF.ERRORS[code]}"), (name, str(e.value))
    eng.check_errors()
