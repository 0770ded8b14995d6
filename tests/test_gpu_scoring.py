"""Scoring on the GPU (vf_metric_spectrogram, vf_ssim, vf_score_varlen, AudioMetrics.evaluation / evaluation_batch, and
handler's meta["mel_ssim"]) against the CPU restatement of oracle/scoring.py."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import scoring as S
from oracle import vf_oracle as O

pytestmark = pytest.mark.gpu

SEG = 44100 * 60


@pytest.fixture(scope="module")
def eng():
    """An engine with only the mel filterbank: scoring needs no checkpoint."""
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


def _ulp_ok(got, want):
    """Every bin within 2 ulp of the restatement, or 1e-12 of its frame's largest bin."""
    ulp = np.spacing(np.abs(want).astype(np.float32))
    tol = np.maximum(2 * ulp, 1e-12 * want.max(axis=1, keepdims=True))
    return np.abs(got - want) <= tol


def test_metric_spectrogram_and_mel_match_restatement(eng):
    lengths = [6 * 441 + 5, 44100, 163170, 441000, SEG + 44100]
    wavs = [_wav(n, 10 + i, silence=5000 if i == 1 else 0) for i, n in enumerate(lengths)]
    sp, mel = eng.metric_spectrogram(torch.from_numpy(np.concatenate(wavs)).cuda(), lengths)
    torch.cuda.synchronize()
    rows = np.cumsum([0] + [1 + n // 441 for n in lengths])
    sp, mel = sp.cpu().numpy(), mel.cpu().numpy()
    for i, w in enumerate(wavs):
        want = S.spectrogram(w)
        got = sp[rows[i]:rows[i + 1]]
        assert got.shape == want.shape
        assert _ulp_ok(got, want).all(), i
        want_mel = S.mel(torch.from_numpy(want)).numpy()
        err = np.abs(mel[rows[i]:rows[i + 1]] - want_mel).max(axis=1)
        assert (err <= 1e-5 * np.maximum(want_mel.max(axis=1), 1e-30)).all(), i
    silent = sp[rows[1]:rows[1] + 2]            # frames 0 and 1 of the clip with 5000 silent samples: all zero
    assert (silent == 0).all()


def test_ssim_kernel_matches_restatement(eng):
    g = torch.Generator().manual_seed(3)
    x = torch.rand(5, 40, 131, generator=g) * 3
    y = x + 0.4 * torch.randn(5, 40, 131, generator=g)
    got = eng.ssim(x.cuda(), y.cuda()).cpu().numpy()
    same = eng.ssim(x.cuda(), x.cuda()).cpu().numpy()
    for i in range(5):
        assert abs(got[i] - S.ssim(x[i].numpy(), y[i].numpy())) < 1e-9
    assert (same == 1.0).all()
    t = torch.rand(2, 7, 7, generator=g)
    assert eng.ssim(t.cuda(), t.cuda()).cpu().tolist() == [1.0, 1.0]


def _pairs(tmp_path, spec):
    out = []
    for i, (n_e, n_t, silence) in enumerate(spec):
        t = _wav(n_t, 300 + i, silence)
        e = (t[:n_e] if n_e <= n_t else np.pad(t, (0, n_e - n_t))) + 0.02 * _wav(n_e, 400 + i)
        pe, pt = str(tmp_path / f"e{i}.wav"), str(tmp_path / f"t{i}.wav")
        S.write_pcm16(np.round(np.clip(e, -1, 1) * 32767).astype(np.int16), pe)
        S.write_pcm16(np.round(np.clip(t, -1, 1) * 32767).astype(np.int16), pt)
        out.append((pe, pt))
    return out


def _close(a, b):
    for k in S.KEYS:
        if k.endswith("ssim"):
            assert abs(a[k] - b[k]) < 1e-6, (k, a[k], b[k])
        else:
            assert abs(a[k] - b[k]) <= 1e-4 * max(1.0, abs(b[k])), (k, a[k], b[k])


def test_evaluation_matches_oracle(eng, tmp_path):
    from voicefixer_main_b200.edges import AudioMetrics
    am = AudioMetrics(eng)
    pairs = _pairs(tmp_path, [(3100, 3100, 0), (44100, 44100, 0), (20000, 20200, 0), (163170, 163170, 30000)])
    for pe, pt in pairs:
        got = am.evaluation(pe, pt)
        assert list(got) == list(S.KEYS)
        _close(got, S.evaluation(pe, pt))
    assert am.evaluation(pairs[0][0], None) == {}


def test_evaluation_batch_equals_evaluation_across_sub_batches(eng, tmp_path):
    from voicefixer_main_b200.edges import AudioMetrics
    am = AudioMetrics(eng)
    # three 61 s pairs exceed the 16384-frame sub-batch cap: the call runs in more than one sub-batch
    pairs = _pairs(tmp_path, [(44100, 44100, 0), (SEG + 44100, SEG + 44100, 0), (5000, 5000, 0), (SEG + 44100, SEG + 44100, 0),
                              (SEG + 44100, SEG + 44100, 100000), (20000, 20200, 0)])
    pairs.insert(2, (pairs[0][0], None))
    n0 = eng.launch_count()
    batch = am.evaluation_batch(pairs)
    assert eng.launch_count() - n0 >= 20            # ten launches per sub-batch, at least two sub-batches
    one = [am.evaluation(pe, pt) for pe, pt in pairs]
    assert batch == one
    assert batch[2] == {}


def test_varlen_lsd_sispec_bits_equal_single_image_calls(eng):
    from voicefixer_main_b200.arch import frames_for
    lengths = [3000, 44100, 9000, 100000]
    e = torch.from_numpy(np.concatenate([_wav(n, 50 + i) for i, n in enumerate(lengths)])).cuda()
    t = torch.from_numpy(np.concatenate([_wav(n, 60 + i) for i, n in enumerate(lengths)])).cuda()
    scores = eng.score_varlen(e, lengths, t, lengths).cpu()
    sp_e, mel_e = eng.metric_spectrogram(e, lengths)
    sp_t, mel_t = eng.metric_spectrogram(t, lengths)
    rows = np.cumsum([0] + [frames_for(n) for n in lengths])
    for i in range(len(lengths)):
        for col, (a, b) in ((0, (sp_e, sp_t)), (4, (mel_e, mel_t))):
            x, y = a[rows[i]:rows[i + 1]].contiguous(), b[rows[i]:rows[i + 1]].contiguous()
            out = torch.empty(3, device="cuda")
            st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            p = lambda z: ctypes.c_void_p(z.data_ptr())
            eng._ck(eng.lib.vf_lsd(eng.ctx, p(x), p(y), 1, x.shape[0], x.shape[1], p(out), st))
            eng._ck(eng.lib.vf_sispec(eng.ctx, p(x), p(y), 1, x.numel(), 0, 0, ctypes.c_void_p(out.data_ptr() + 4), st))
            eng._ck(eng.lib.vf_sispec(eng.ctx, p(x), p(y), 1, x.numel(), 1, 1, ctypes.c_void_p(out.data_ptr() + 8), st))
            want = out.cpu().double()
            assert torch.equal(scores[i, col:col + 3], want), (i, col)
            assert scores[i, col + 3].item() == eng.ssim(x[None], y[None]).item()


# ------------------------------------------------------------------ handler / handler_batch with meta["mel_ssim"]
TEST_SET = [(44100, 44100, False), (163170, 44100, True), (441000, 44100, False), (SEG + 44100, 44100, True),
            (55125, 22050, True)]


@pytest.fixture(scope="module")
def model(state):
    from voicefixer_main_b200 import VoiceFixer
    m = VoiceFixer().load_state_dict(state).eval().to("cuda:0")
    yield m
    m._engine().check_errors()
    m._eng.close()
    torch.cuda.empty_cache()


def _write_set(H, d, spec):
    os.makedirs(d / "one")
    os.makedirs(d / "batch")
    items = []
    for i, (n, rate, has_target) in enumerate(spec):
        src = str(d / f"in{i}.wav")
        H.save_pcm16(O.to_int16(O.synth_clips(1, n, seed=100 + i)[0].clamp(-0.99, 0.99).numpy()), src, sample_rate=rate)
        tgt = None
        if has_target:
            tgt = str(d / f"tgt{i}.wav")
            H.save_pcm16(O.to_int16(O.synth_clips(1, n, seed=200 + i)[0].clamp(-0.99, 0.99).numpy()), tgt, sample_rate=rate)
        items.append((src, f"in{i}.wav", tgt))
    return items


def test_handler_mel_ssim(model, tmp_path, monkeypatch):
    from voicefixer_main_b200 import handler as H
    from voicefixer_main_b200.edges import AudioMetrics
    monkeypatch.setattr(H, "model", model)
    items = _write_set(H, tmp_path, TEST_SET)
    meta = {"mel_ssim": True, "unify_energy": True}
    one = [H.handler(s, str(tmp_path / "one" / o), t, ckpt=None, device=model.device, meta=meta) for s, o, t in items]
    batch = H.handler_batch([(s, str(tmp_path / "batch" / o), t) for s, o, t in items], ckpt=None, device=model.device, meta=meta)
    for (_, o, t), a, b in zip(items, one, batch):
        with open(tmp_path / "one" / o, "rb") as f1, open(tmp_path / "batch" / o, "rb") as f2:
            assert f1.read() == f2.read()
        assert a == b
        assert set(a) == ({"mel-lsd", "mel-sispec", "mel-non-log-sispec", "mel-ssim"} if t else set())
    # "mel-ssim" is vf_ssim of the mels "mel-lsd" used: recompute them for the 3.7 s file (one segment)
    src, _, tgt = items[1]
    wav = torch.from_numpy(H.read_pcm16(src)[0])[None].cuda()
    model.restore(wav, unify_energy=True)
    mel_noisy, log_mel = model._engine().restore_stages(1, wav.shape[1])
    _, target_mel = model.pre(torch.from_numpy(H.read_pcm16(tgt)[0])[None, None].cuda())
    eng = model._engine()
    den = eng.amp_to_original_f(eng.from_log(log_mel[:, None])[:, 0].contiguous(), mel_noisy.contiguous())
    got = AudioMetrics(model).ssim(den[:, None].contiguous(), target_mel.contiguous())
    assert one[1]["mel-ssim"] == float(got)
    assert abs(one[1]["mel-ssim"] - S.ssim(den[0].cpu().numpy(), target_mel[0, 0].cpu().numpy())) < 1e-9
    assert H.handler(src, str(tmp_path / "plain.wav"), tgt, ckpt=None, device=model.device, meta={"unify_energy": True}) == \
        {k: v for k, v in one[1].items() if k != "mel-ssim"}


def test_handler_mel_ssim_rejects_short_segment(model, tmp_path, monkeypatch):
    from voicefixer_main_b200 import handler as H
    monkeypatch.setattr(H, "model", model)
    items = _write_set(H, tmp_path, [(30000, 44100, False), (1025, 44100, True)])
    with pytest.raises(ValueError, match="in1.wav"):
        H.handler_batch([(s, str(tmp_path / "batch" / o), t) for s, o, t in items], ckpt=None, device=model.device,
                        meta={"mel_ssim": True})
    assert os.listdir(tmp_path / "batch") == []
    with pytest.raises(ValueError):
        H.handler(items[1][0], str(tmp_path / "one" / "x.wav"), items[1][2], ckpt=None, device=model.device, meta={"mel_ssim": True})
    assert os.listdir(tmp_path / "one") == []
    torch.cuda.synchronize()
    model._engine().check_errors()
