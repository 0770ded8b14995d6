"""16 kHz scoring on the GPU (vf_metric_spectrogram_ex, vf_score_varlen_ex, vf_score_time_varlen_ex and
AudioMetrics(eng, rate=16000)) against the CPU restatement of tests/oracle_16k.py."""
import numpy as np
import pytest
import torch

import oracle_16k as R
from oracle import scoring as S
from oracle import speech_metrics as M
from oracle import vf_oracle as O
from test_gpu_scoring import _close, _ulp_ok

pytestmark = pytest.mark.gpu

SEG = 16000 * 61


@pytest.fixture(scope="module")
def eng():
    """A scoring-only engine: load_state({}) loads both rates' filterbanks."""
    from voicefixer_main_b200.model import Engine
    e = Engine("cuda:0")
    e.load_state({}, need=())
    yield e
    e.close()
    torch.cuda.empty_cache()


def _wav(n, seed, silence=0):
    x = O.synth_clips(1, n, seed=seed)[0].clamp(-0.99, 0.99).numpy().astype(np.float32)
    x[:silence] = 0
    return x


def _rows(lengths):
    return np.cumsum([0] + [R.frames(n) for n in lengths])


def test_metric_spectrogram_and_mel_match_restatement(eng):
    lengths = [961, 16000, 16001, 160000 - 1, 160000 + 1, SEG + 7]
    wavs = [_wav(n, 20 + i, silence=5000 if i == 1 else 0) for i, n in enumerate(lengths)]
    sp, mel = eng.metric_spectrogram(torch.from_numpy(np.concatenate(wavs)).cuda(), lengths, rate=16000)
    torch.cuda.synchronize()
    rows = _rows(lengths)
    assert sp.shape == (rows[-1], 372) and mel.shape == (rows[-1], 80)
    sp, mel = sp.cpu().numpy(), mel.cpu().numpy()
    for i, w in enumerate(wavs):
        want = R.spectrogram(w)
        got = sp[rows[i]:rows[i + 1]]
        assert got.shape == want.shape
        assert _ulp_ok(got, want).all(), i
        want_mel = R.mel(torch.from_numpy(want)).numpy()
        err = np.abs(mel[rows[i]:rows[i + 1]] - want_mel).max(axis=1)
        assert (err <= 1e-5 * np.maximum(want_mel.max(axis=1), 1e-30)).all(), i
    silent = sp[rows[1]:rows[1] + 3]            # frames 0-2 of the clip with 5000 silent samples read only silence
    assert (silent == 0).all()


def test_rates_and_lengths_are_checked(eng):
    from voicefixer_main_b200._lib import EngineError
    x = torch.from_numpy(_wav(2000, 1)).cuda()
    with pytest.raises(EngineError, match="rate 22050"):
        eng.metric_spectrogram(x, [2000], rate=22050)
    with pytest.raises(EngineError, match="need 372 "):
        eng.metric_spectrogram(x[:371], [371], rate=16000)
    sp, _ = eng.metric_spectrogram(x[:372], [372], rate=16000, want_mel=False)
    assert sp.shape == (3, 372)
    with pytest.raises(EngineError, match="fewer than SSIM's 7"):
        eng.score_varlen(x[:960], [960], x[:960], [960], rate=16000)
    with pytest.raises(EngineError, match="rate 8000"):
        eng.score_time_varlen(x, [2000], x, [2000], rate=8000)


def test_16k_filterbank_is_required():
    from voicefixer_main_b200 import _lib as L
    from voicefixer_main_b200.model import Engine, melscale_fbanks
    e = Engine("cuda:0")
    fb = melscale_fbanks().contiguous()
    descs = (L.VfTensorDesc * 1)()
    descs[0].name, descs[0].data, descs[0].ndim, descs[0].on_device = b"mel.fb", fb.data_ptr(), 2, 0
    descs[0].shape[0], descs[0].shape[1] = 1025, 128
    e._ck(e.lib.vf_load_weights(e.ctx, descs, 1))
    x = torch.from_numpy(_wav(2000, 1)).cuda()
    with pytest.raises(L.EngineError, match="metrics.mel_16k.fb"):
        e.metric_spectrogram(x, [2000], rate=16000)
    sp, _ = e.metric_spectrogram(x, [2000], rate=16000, want_mel=False)     # the spectrogram alone needs no filterbank
    assert sp.shape == (R.frames(2000), 372)
    e.close()


def _pairs(tmp_path, spec, est_rate=16000):
    from voicefixer_main_b200.handler import _rate_len
    out = []
    for i, (n_e, n_t, silence) in enumerate(spec):
        t = _wav(n_t, 500 + i, silence)
        e = (t[:n_e] if n_e <= n_t else np.pad(t, (0, n_e - n_t))) + 0.02 * _wav(n_e, 600 + i)
        if est_rate != 16000:        # the same signal at est_rate: linear interpolation is enough for a test input
            n = _rate_len(n_e, 16000, est_rate)
            e = np.interp(np.arange(n) * 16000 / est_rate, np.arange(n_e), e).astype(np.float32)
        pe, pt = str(tmp_path / f"e{i}.wav"), str(tmp_path / f"t{i}.wav")
        S.write_pcm16(np.round(np.clip(e, -1, 1) * 32767).astype(np.int16), pe, est_rate)
        S.write_pcm16(np.round(np.clip(t, -1, 1) * 32767).astype(np.int16), pt, 16000)
        out.append((pe, pt))
    return out


SPEC = [(961, 961, 0), (16000, 16000, 0), (16001, 16100, 0), (59999, 59999, 12000)]


def test_evaluation_matches_oracle(eng, tmp_path):
    from voicefixer_main_b200.edges import AudioMetrics
    am = AudioMetrics(eng, rate=16000)
    pairs = _pairs(tmp_path, SPEC)
    for pe, pt in pairs:
        got = am.evaluation(pe, pt)
        assert list(got) == list(S.KEYS)
        _close(got, R.evaluation(pe, pt))
    assert am.evaluation(pairs[0][0], None) == {}


def test_evaluation_batch_equals_evaluation_across_sub_batches(eng, tmp_path):
    from voicefixer_main_b200.edges import AudioMetrics
    am = AudioMetrics(eng, rate=16000)
    # three 61 s pairs hold 18303 frames per side, more than the 16384-frame sub-batch cap: two sub-batches at least
    pairs = _pairs(tmp_path, [(16000, 16000, 0), (SEG, SEG, 0), (5000, 5000, 0), (SEG, SEG, 0), (SEG, SEG, 40000),
                              (16001, 16100, 0)])
    pairs.insert(2, (pairs[0][0], None))
    n0 = eng.launch_count()
    batch = am.evaluation_batch(pairs)
    assert eng.launch_count() - n0 >= 20            # ten launches per sub-batch
    one = [am.evaluation(pe, pt) for pe, pt in pairs]
    assert batch == one
    assert batch[2] == {}


def test_est_at_44k_against_16k_targets(eng, tmp_path):
    from voicefixer_main_b200.edges import AudioMetrics
    from voicefixer_main_b200.handler import _to_rate, read_pcm16
    am = AudioMetrics(eng, rate=16000)
    pairs = _pairs(tmp_path, [(16000, 16000, 0), (48000, 48000, 0), (30001, 30001, 6000)], est_rate=44100)
    batch = am.evaluation_batch(pairs)
    for (pe, pt), got in zip(pairs, batch):
        e16 = _to_rate(pe, *read_pcm16(pe), 16000, eng)            # the GPU resampler's 16 kHz est
        _close(got, R.evaluation(pe, pt, est=e16))
        assert got == am.evaluation(pe, pt)
    with pytest.raises(ValueError, match="sisdr / stoi"):
        am.evaluation_batch(pairs, time_domain=True)


def test_time_domain_matches_restatement(eng, tmp_path):
    from voicefixer_main_b200.edges import AudioMetrics
    am = AudioMetrics(eng, rate=16000)
    pairs = _pairs(tmp_path, SPEC + [(SEG, SEG, 30000)])
    batch = am.evaluation_batch(pairs, time_domain=True)
    plain = am.evaluation_batch(pairs)
    for (pe, pt), got, spectral in zip(pairs, batch, plain):
        assert list(got) == ["sisdr", "stoi"] + list(S.KEYS)
        assert {k: got[k] for k in S.KEYS} == spectral
        e, t = M.load_first_channel(pe), M.load_first_channel(pt)
        want = R.time_scores(e, t)
        n = max(len(e), len(t))
        assert abs(got["sisdr"] - want["sisdr"]) <= M.sisdr_bar(n, want["sisdr"]), (pe, got["sisdr"], want["sisdr"])
        assert abs(got["stoi"] - want["stoi"]) <= R.stoi_bar(n), (pe, got["stoi"], want["stoi"])


def _packed(lengths, seed):
    return torch.from_numpy(np.concatenate([_wav(n, seed + i) for i, n in enumerate(lengths)])).cuda()


def test_pair_values_do_not_depend_on_batch_or_position(eng):
    lengths = [961, 16001, 40000, 7777]
    e, t = _packed(lengths, 70), _packed(lengths, 80)
    rows = np.cumsum([0] + lengths)
    for fn in (eng.score_varlen, eng.score_time_varlen):
        full = fn(e, lengths, t, lengths, rate=16000).cpu()
        order = [3, 1, 0, 2]
        pe = torch.cat([e[rows[i]:rows[i + 1]] for i in order])
        pt = torch.cat([t[rows[i]:rows[i + 1]] for i in order])
        perm = fn(pe, [lengths[i] for i in order], pt, [lengths[i] for i in order], rate=16000).cpu()
        for k, i in enumerate(order):
            assert torch.equal(perm[k], full[i]), (fn.__name__, i)
            one = fn(e[rows[i]:rows[i + 1]], [lengths[i]], t[rows[i]:rows[i + 1]], [lengths[i]], rate=16000).cpu()
            assert torch.equal(one[0], full[i]), (fn.__name__, i)


def _scores_44k(engine):
    lengths = [3000, 44100, 100000]
    e, t = _packed(lengths, 90), _packed(lengths, 95)
    sp, mel = engine.metric_spectrogram(e, lengths)
    return [sp, mel, engine.score_varlen(e, lengths, t, lengths), engine.score_time_varlen(e, lengths, t, lengths)]


def test_16k_calls_leave_44k_results_unchanged(eng):
    from voicefixer_main_b200.model import Engine
    lengths = [16000, 20000]
    e, t = _packed(lengths, 40), _packed(lengths, 45)
    eng.score_varlen(e, lengths, t, lengths, rate=16000)
    eng.score_time_varlen(e, lengths, t, lengths, rate=16000)
    eng.metric_spectrogram(e, lengths, rate=16000)
    after = _scores_44k(eng)
    fresh = Engine("cuda:0")
    fresh.load_state({}, need=())
    want = _scores_44k(fresh)
    torch.cuda.synchronize()
    for a, b in zip(after, want):
        assert torch.equal(a, b)
    fresh.close()
