"""sisdr and stoi on the GPU (vf_score_time_varlen, Engine.score_time_varlen, AudioMetrics.evaluation(_batch)(...,
time_domain=True)) against the float64 restatement of oracle/speech_metrics.py.

Bars (oracle/speech_metrics.py, sisdr_bar / stoi_bar): sisdr within 10 / ln 10 * (4 gamma_N + 4 u 10^(sisdr / 20)) dB for
a pair padded to N samples - four N-term float64 sums whose order differs, and the rounding of e - a r relative to |a r| -
and stoi within 1e4 * gamma_720 + gamma_(15 J): band values that end chains of at most 720 float64 operations, a 1e4
budget for the conditioning of the normalised correlations, and the final sum.  Both stay below about 5e-9 for a minute
of audio.  Every fixture keeps its frame energies at least 1e-6 dB from the silence threshold, so no rounding can flip a
frame of the mask."""
import os

import numpy as np
import pytest
import torch

from oracle import scoring as S
from oracle import speech_metrics as M
from oracle import vf_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    """An engine with only the mel filterbank: scoring needs no checkpoint."""
    from voicefixer_main_b200.model import Engine
    e = Engine("cuda:0")
    e.load_state({}, need=())
    yield e
    e.close()
    torch.cuda.empty_cache()


def _speech(n, seed, silences=()):
    x = O.synth_clips(1, n, seed=seed)[0].clamp(-0.9, 0.9).numpy().astype(np.float32)
    for a, b in silences:
        x[int(a * 44100):int(b * 44100)] = 0
    return x


def _noisy(x, seed, n=None):
    n = len(x) if n is None else n
    g = np.random.default_rng(seed)
    y = np.zeros(n, np.float32)
    m = min(n, len(x))
    y[:m] = x[:m]
    return (y + 0.05 * g.standard_normal(n) + 0.005).astype(np.float32)


def _cases():
    """(name, est, target) float32 pairs at 44.1 kHz."""
    s1, s37, s10, s61 = _speech(44100, 1), _speech(163170, 2), _speech(441000, 3), _speech(44100 * 61, 4)
    sil = _speech(44100 * 4, 5, silences=((1.0, 1.6), (2.5, 2.7)))
    few = _speech(44100 * 2, 6, silences=((0.0, 0.9), (1.1, 2.0)))
    s2, s3 = _speech(88200, 7), _speech(132300, 8)
    short = _speech(1129, 9)                       # 257 samples at 10 kHz: the shortest legal pair, one frame
    return [
        ("shortest", _noisy(short, 10), short),
        ("1s", _noisy(s1, 11), s1),
        ("3.7s", _noisy(s37, 12), s37),
        ("10s", _noisy(s10, 13), s10),
        ("est_shorter", _noisy(s3, 14, len(s3) - 5000), s3),
        ("est_longer", _noisy(s2, 15, len(s2) + 7000), s2),
        ("silences", _noisy(sil, 16), sil),
        ("identical", s2.copy(), s2),
        ("zero_est", np.zeros_like(s3), s3),
        ("below_30_frames", _noisy(few, 17), few),
        ("61s", _noisy(s61, 18), s61),
    ]


@pytest.fixture(scope="module")
def cases():
    cs = _cases()
    for name, e, t in cs:
        assert M.silence_margin(e.astype(np.float64), t.astype(np.float64)) >= 1e-6, name
    return cs


@pytest.fixture(scope="module")
def reference(cases):
    return [M.time_scores(e.astype(np.float64), t.astype(np.float64)) for _, e, t in cases]


def _score(eng, pairs):
    ests, tgts = [e for e, _ in pairs], [t for _, t in pairs]
    out = eng.score_time_varlen(torch.from_numpy(np.concatenate(ests)).cuda(), [len(e) for e in ests],
                                torch.from_numpy(np.concatenate(tgts)).cuda(), [len(t) for t in tgts])
    return out.cpu()


def test_matches_restatement(eng, cases, reference):
    got = _score(eng, [(e, t) for _, e, t in cases]).numpy()
    eng.check_errors()
    worst = {}
    for (name, e, t), want, row in zip(cases, reference, got):
        n = max(len(e), len(t))
        snr = 0.0 if name == "identical" else want["sisdr"]      # Snn is exactly 0 on both sides for identical signals
        bars = {"sisdr": M.sisdr_bar(n, snr), "stoi": M.stoi_bar(n)}
        for k, v in zip(M.KEYS, row):
            err = abs(v - want[k])
            assert err <= bars[k], (name, k, v, want[k], bars[k])
            worst[k] = max(worst.get(k, 0.0), err / bars[k])
    print(f"worst error / bar: {worst}")
    by = {name: row for (name, _, _), row in zip(cases, got)}
    assert by["shortest"][1] == 1e-5 and by["below_30_frames"][1] == 1e-5
    assert by["zero_est"][1] == 0.0 and by["zero_est"][0] == 0.0
    assert abs(by["identical"][1] - 1) < 1e-12


def test_pair_alone_in_batch_and_in_sub_batches_bit_identical(eng, cases):
    pairs = [(e, t) for _, e, t in cases]
    big = pairs + [pairs[-1], pairs[-1]]            # three 61 s pairs: more than one sub-batch of 16384 * 441 samples
    together = _score(eng, big)
    for i, p in enumerate(pairs):
        assert torch.equal(_score(eng, [p]), together[i:i + 1]), cases[i][0]
    assert torch.equal(together[-1], together[len(pairs) - 1])
    assert torch.equal(torch.cat([_score(eng, big[:4]), _score(eng, big[4:])]), together)


def test_rejected_pairs_raise_before_gpu_work(eng):
    from voicefixer_main_b200._lib import EngineError
    ok = _speech(44100, 20)
    before = eng.launch_count()
    with pytest.raises(EngineError, match="pair 1"):
        _score(eng, [(ok, ok), (ok[:1128], ok[:1000])])         # 256 samples at 10 kHz: no STOI frame
    assert eng.launch_count() == before


def _write(tmp, name, x, rate=44100, channels=1):
    path = os.path.join(tmp, name)
    pcm = O.to_int16(np.clip(x, -0.99, 0.99))
    if channels == 2:                                # the second channel differs: speechmetrics reads the first
        pcm = np.stack([pcm, (pcm // 2).astype(np.int16)], axis=1).reshape(-1)
        import wave
        with wave.open(path, "wb") as w:
            w.setnchannels(2)
            w.setsampwidth(2)
            w.setframerate(rate)
            w.writeframes(pcm.tobytes())
        return path
    S.write_pcm16(pcm, path, rate)
    return path


def test_evaluation_batch_time_domain(eng, tmp_path):
    from voicefixer_main_b200.edges import SCORE_KEYS, AudioMetrics
    d = str(tmp_path)
    pairs = []
    for i, (n, silences) in enumerate(((44100, ()), (163170, ((1.0, 1.5),)), (441000, ()), (88200 + 300, ()))):
        t = _speech(n, 30 + i, silences)
        e = _noisy(t, 40 + i, n - 200 if i == 3 else n)
        pairs.append((_write(d, f"e{i}.wav", e, channels=2 if i == 2 else 1), _write(d, f"t{i}.wav", t)))
    pairs.append((pairs[0][0], None))
    am = AudioMetrics(eng)
    batch = am.evaluation_batch(pairs, time_domain=True)
    assert batch == [am.evaluation(pe, pt, time_domain=True) for pe, pt in pairs]
    plain = am.evaluation_batch(pairs)
    assert batch[-1] == {} and plain[-1] == {}
    for (pe, pt), got, spectral in zip(pairs[:-1], batch, plain):
        assert list(got) == ["sisdr", "stoi", *SCORE_KEYS]
        assert {k: got[k] for k in SCORE_KEYS} == spectral
        e, t = M.load_first_channel(pe), M.load_first_channel(pt)
        want = M.time_scores(e, t)
        n = max(len(e), len(t))
        assert abs(got["sisdr"] - want["sisdr"]) <= M.sisdr_bar(n, want["sisdr"])
        assert abs(got["stoi"] - want["stoi"]) <= M.stoi_bar(n)


def test_evaluation_time_domain_rejects_other_rates_before_gpu_work(eng, tmp_path):
    from voicefixer_main_b200.edges import AudioMetrics
    d = str(tmp_path)
    t = _speech(44100, 50)
    good = (_write(d, "e.wav", _noisy(t, 51)), _write(d, "t.wav", t))
    slow = _write(d, "e22.wav", _noisy(t, 52)[::2].copy(), rate=22050)
    am = AudioMetrics(eng)
    before = eng.launch_count()
    with pytest.raises(ValueError, match="e22.wav"):
        am.evaluation_batch([good, (slow, good[1])], time_domain=True)
    assert eng.launch_count() == before
