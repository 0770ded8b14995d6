"""The SSR / GSR-UNet evaluation handler (handler_unet) and its batched call (vf_ssr_restore_varlen_mels): the output mel and
peak normalise of every clip must have the bits of the one-clip calls they replace, handler() must agree with the CPU
oracle's composition of eval_gsr_unet.py:49-74, and handler_batch must write handler()'s bytes and return its floats."""
import ctypes
import os
import wave

import numpy as np
import pytest
import torch

from oracle import scoring as S
from oracle import vf_oracle as O

pytestmark = pytest.mark.gpu

SEG = 44100 * 60
WAV_RMS_TOL = 1e-3          # the SSR waveform bar of test_gpu_round2.py


def _new_model(ssr_state):
    from voicefixer_main_b200 import SSR_UNet
    return SSR_UNet().load_state_dict(ssr_state).eval().to("cuda:0")


def _close(m):
    """Frees the context's plans now, so the device memory they hold does not shrink the plan budget of later modules."""
    m._engine().check_errors()
    m._eng.close()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def ssr_state():
    from voicefixer_main_b200.weights import make_ssr_state
    return make_ssr_state(1234)


@pytest.fixture(scope="module")
def model(ssr_state):
    m = _new_model(ssr_state)
    yield m
    _close(m)


@pytest.fixture
def fresh_model(ssr_state):
    m = _new_model(ssr_state)
    yield m
    _close(m)


@pytest.fixture
def HU(model, monkeypatch):
    from voicefixer_main_b200 import handler_unet
    monkeypatch.setattr(handler_unet, "model", model)
    return handler_unet


# ------------------------------------------------------------------ vf_ssr_restore_varlen_mels directly
# 1025: the shortest clip (T = 3); 5000: T = 12 (even); 70 * 441 + 17: T = 71 (odd); 27883 / 28229: T = 64 / 65; 10 s
LENGTHS = [1025, 5000, 70 * 441 + 17, 27883, 28229, 441000]


def _clips(lengths, seed):
    """Clips scaled to a peak of 0.4 or 1.0 in turn: the restored output of the synthetic network peaks at about 1.35x its
    input's (plus a floor near 0.3), so the set holds outputs on both sides of the normalise threshold."""
    out = []
    for i, n in enumerate(lengths):
        c = O.synth_clips(1, n, seed=seed + i)[0]
        out.append((c / c.abs().max() * (0.4 if i % 2 == 0 else 1.0)).cuda())
    return out


def _call(eng, clips, mels=True, peak=True):
    from voicefixer_main_b200.arch import frames_for
    rows = sum(frames_for(c.numel()) for c in clips)
    mel = torch.full((rows, 128), float("nan"), device="cuda") if mels else None
    out = eng.ssr_restore_varlen(torch.cat(clips), [c.numel() for c in clips], mel_out=mel, peak_normalise=peak)
    return out, mel


def test_mels_and_peak_normalise_equal_the_one_clip_calls(model):
    from voicefixer_main_b200.arch import frames_for
    eng = model._engine()
    clips = _clips(LENGTHS, seed=2300)
    out, mel = _call(eng, clips)
    plain = eng.ssr_restore_varlen(torch.cat(clips), LENGTHS)
    eng.check_errors()
    peaks = []
    for c, o, p, m in zip(clips, torch.split(out, LENGTHS), torch.split(plain, LENGTHS),
                          torch.split(mel, [frames_for(n) for n in LENGTHS])):
        raw = model.restore(c[None].contiguous())
        assert torch.equal(p, raw[0]), c.numel()
        assert torch.equal(m, model.pre(raw[:, None])[1][0, 0]), c.numel()          # mel of the un-normalised output
        assert torch.equal(o, eng.finalize(raw, c.numel())[0]), c.numel()
        peaks.append(float(raw.abs().max()))
    eng.check_errors()
    print("raw restored peaks", peaks)
    assert any(p > 1 for p in peaks) and any(p < 1 for p in peaks)


def _raw(eng, fn, clips, *extra):
    offs = np.concatenate([[0], np.cumsum([c.numel() for c in clips])])
    packed = torch.cat(clips)
    out = torch.empty_like(packed)
    with torch.cuda.device(eng.device):
        n0 = eng.launch_count()
        rc = getattr(eng.lib, fn)(eng.ctx, ctypes.c_void_p(packed.data_ptr()), (ctypes.c_int64 * len(offs))(*offs.tolist()),
                                  len(clips), ctypes.c_void_p(out.data_ptr()), *extra,
                                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        return rc, out, eng.launch_count() - n0


def test_null_and_zero_behave_as_ssr_restore_varlen(model):
    eng = model._engine()
    clips = _clips([5000, 20000, 1025], seed=2400)
    rc0, ref, n_ref = _raw(eng, "vf_ssr_restore_varlen", clips)
    rc1, got, n_got = _raw(eng, "vf_ssr_restore_varlen_mels", clips, 0, None)
    eng.check_errors()
    assert rc0 == rc1 == 0 and torch.equal(got, ref) and n_got == n_ref
    _, mel = _call(eng, clips, peak=False)
    mel_only = torch.empty_like(mel)
    _, got2, n_mel = _raw(eng, "vf_ssr_restore_varlen_mels", clips, 0, ctypes.c_void_p(mel_only.data_ptr()))
    _, _, n_peak = _raw(eng, "vf_ssr_restore_varlen_mels", clips, 1, None)
    eng.check_errors()
    assert torch.equal(got2, ref) and torch.equal(mel_only, mel)
    assert n_mel == n_ref + 2 and n_peak == n_ref + 2            # one sub-batch: front end + gather / peak + scale


def test_sub_batches_and_graph_replay_give_the_same_bits(fresh_model):
    eng = fresh_model._engine()
    clips = _clips([44100, 30000, 50000, 1025, 40000, 44100 + 441], seed=2500)
    calls = [[t.clone() for t in _call(eng, clips)] for _ in range(3)]     # eager, capture, replay
    one_plan = eng.plan_cache_info()["bytes"]
    cap_mb = (one_plan >> 20) * 2 // 3                                     # the 6-clip plan no longer fits
    eng.set_option("plan_cache_mb", cap_mb)
    split = _call(eng, clips)
    eng.check_errors()
    assert eng.plan_cache_info()["bytes"] <= cap_mb << 20 < one_plan
    for k in range(2):
        assert torch.equal(calls[0][k], calls[2][k]) and torch.equal(calls[0][k], calls[1][k])
        assert torch.equal(split[k], calls[0][k])


def test_unknown_flags_fail_and_leave_the_context_usable(model):
    from voicefixer_main_b200._lib import VF_EINVAL
    eng = model._engine()
    clips = _clips([5000, 20000], seed=2600)
    ref = [t.clone() for t in _call(eng, clips)]
    for flags in (2, 3, 0x80000000):
        assert _raw(eng, "vf_ssr_restore_varlen_mels", clips, flags, None)[0] == VF_EINVAL
    assert "unknown flag bits" in eng.lib.vf_last_error(eng.ctx).decode()
    again = _call(eng, clips)
    eng.check_errors()
    assert all(torch.equal(a, r) for a, r in zip(again, ref))


# ------------------------------------------------------------------ handler() and handler_batch()
def _pcm(n, seed):
    return O.to_int16(O.synth_clips(1, n, seed=seed)[0].clamp(-0.99, 0.99).numpy())


def _read(path):
    with wave.open(path, "rb") as w:
        return np.frombuffer(w.readframes(w.getnframes()), dtype=np.int16)


def test_handler_matches_the_cpu_oracle(HU, ssr_state, tmp_path):
    """eval_gsr_unet.py:49-74 on one 1 s segment (T = 101) composed from the CPU oracle: restore, the mel of the output, the
    four metrics against the target's mel, peak normalise, int16."""
    src, tgt, dst = str(tmp_path / "in.wav"), str(tmp_path / "tgt.wav"), str(tmp_path / "out.wav")
    x = _pcm(44100, 31)
    t = _pcm(44100, 32)
    HU.save_pcm16(x, src)
    HU.save_pcm16(t, tgt)
    got = HU.handler(src, dst, tgt, None, HU.model.device)
    HU.model._engine().check_errors()
    seg = torch.from_numpy(x.astype(np.float32) / 32768.0)[None, None]
    tseg = torch.from_numpy(t.astype(np.float32) / 32768.0)[None, None]
    with torch.no_grad():
        out = O.ssr_forward(ssr_state, seg, exact_stft=True)
        mel_out = O.pre(out, exact=True)[1].float()
        target_mel = O.pre(tseg, exact=True)[1].float()
    want = {
        "mel-lsd": float(S.lsd(mel_out, target_mel)),
        "mel-sispec": float(S.sispec(S.to_log(mel_out), S.to_log(target_mel))),
        "mel-non-log-sispec": float(S.sispec(mel_out, target_mel)),
        "mel-ssim": S.ssim(mel_out[0, 0].numpy(), target_mel[0, 0].numpy()),
    }
    assert list(got) == list(want)
    ref_pcm = O.to_int16(O.peak_normalize(out)[0, 0].numpy())
    wav_err = float(np.sqrt(np.mean(((_read(dst).astype(np.float64) - ref_pcm) / 32768.0) ** 2)))
    # Tolerances from the distance between the engine's output mel and the oracle's (the mel of a waveform within the
    # waveform bar), through bounds of each metric's sensitivity:
    # - lsd is a per-frame RMS over bins of 2 log10(target / est): it moves by at most 2 max|d log10 est|.
    # - sispec = 20 log10(|t_p| / |e - t_p|) with t_p the projection of the estimate e on the target: a change d of e
    #   changes both norms by at most |d|, so the value by at most 20 (log10(1 + |d| / |t_p|) - log10(1 - |d| / |e - t_p|)).
    # - ssim: the mels lie far above its constants (c1 = 4e-4, c2 = 3.6e-3 for data range 2), so each window's value is a
    #   ratio of local statistics, which a relative change rho of every value moves by O(rho): 10 rho, rho the largest
    #   relative mel change 10^max|d log10 mel| - 1.
    gpu_mel = HU.model.pre(HU.model.restore(seg[0].cuda()).contiguous()[:, None])[1].cpu()
    d_log = float((S.to_log(gpu_mel) - S.to_log(mel_out)).abs().max())

    def sispec_bound(e, tg, e2):
        dn = float((e2 - e).double().norm())
        e, tg = e.double().flatten(), tg.double().flatten()
        tp = (e @ tg) / (tg @ tg) * tg
        r1, r2 = dn / float(tp.norm()), dn / float((e - tp).norm())
        return 20 * (np.log10(1 + r1) - np.log10(1 - r2)) if r2 < 1 else float("inf")

    tol = {
        "mel-lsd": 2 * d_log + 1e-5,
        "mel-sispec": sispec_bound(S.to_log(mel_out), S.to_log(target_mel), S.to_log(gpu_mel)) + 1e-4,
        "mel-non-log-sispec": sispec_bound(mel_out, target_mel, gpu_mel) + 1e-4,
        "mel-ssim": 10 * (10 ** d_log - 1) + 1e-6,
    }
    diffs = {k: abs(got[k] - want[k]) for k in want}
    print("handler vs oracle: wav rms err", wav_err, "max |d log10 mel|", d_log)
    print("metrics", got, "oracle", want, "diffs", diffs, "tolerances", tol)
    assert wav_err < WAV_RMS_TOL
    for k in want:
        assert diffs[k] <= tol[k], (k, diffs[k], tol[k])


# (samples, rate, target): the shortest legal file, 1 s, 3.7 s, 10 s, 61 s (a 60 s segment and a 1 s one), 22.05 kHz.  Files
# with a target need SSIM's 7 frames, so the 1025-sample file has none.
TEST_SET = [(1025, 44100, False), (44100, 44100, True), (163170, 44100, True), (441000, 44100, False),
            (SEG + 44100, 44100, True), (55125, 22050, True), (77175, 22050, False)]


def _write_set(H, d, spec):
    os.makedirs(d / "one")
    os.makedirs(d / "batch")
    items = []
    for i, (n, rate, has_target) in enumerate(spec):
        src = str(d / f"in{i}.wav")
        H.save_pcm16(_pcm(n, 100 + i), src, sample_rate=rate)
        tgt = None
        if has_target:
            tgt = str(d / f"tgt{i}.wav")
            H.save_pcm16(_pcm(n, 200 + i), tgt, sample_rate=rate)
        items.append((src, f"in{i}.wav", tgt))
    return items


def _run_both(H, d, items, meta):
    dev = H.model.device
    one = [H.handler(src, str(d / "one" / out), tgt, ckpt=None, device=dev, meta=meta) for src, out, tgt in items]
    batch = H.handler_batch([(src, str(d / "batch" / out), tgt) for src, out, tgt in items], ckpt=None, device=dev, meta=meta)
    H.model._engine().check_errors()
    for (_, out, _), a, b in zip(items, one, batch):
        with open(d / "one" / out, "rb") as f1, open(d / "batch" / out, "rb") as f2:
            assert f1.read() == f2.read(), out
        assert a == b, (out, a, b)
    return one


def test_batch_matches_handler_per_file(HU, tmp_path):
    metrics = _run_both(HU, tmp_path, _write_set(HU, tmp_path, TEST_SET), {})
    assert [bool(m) for m in metrics] == [t for _, _, t in TEST_SET]
    assert all(list(m) == ["mel-lsd", "mel-sispec", "mel-non-log-sispec", "mel-ssim"] for m in metrics if m)


def test_saturate_matches_handler(HU, tmp_path):
    _run_both(HU, tmp_path, _write_set(HU, tmp_path, [(30000, 44100, False), (163170, 44100, True), (5000, 44100, False)]),
              {"saturate": True})


@pytest.mark.parametrize("n, n_target", [
    (SEG + 1000, None),      # a last segment of 1000 samples
    (5000, 6000),            # a target slice with another frame count
    (2000, 2000),            # a segment with a target and 5 frames: mel-ssim's 7x7 window
])
def test_rejected_file_fails_the_call_before_any_write(HU, tmp_path, n, n_target):
    items = _write_set(HU, tmp_path, [(30000, 44100, False), (n, 44100, n_target is not None)])
    if n_target is not None:
        HU.save_pcm16(_pcm(n_target, 300), items[1][2])
    with pytest.raises(Exception) as one:
        HU.handler(items[1][0], str(tmp_path / "one" / items[1][1]), items[1][2], ckpt=None, device=HU.model.device)
    with pytest.raises(Exception) as batch:
        HU.handler_batch([(s, str(tmp_path / "batch" / o), t) for s, o, t in items], ckpt=None, device=HU.model.device)
    assert type(batch.value) is type(one.value) and "in1.wav" in str(batch.value)
    assert os.listdir(tmp_path / "batch") == []
    assert HU.handler_batch([], ckpt=None, device=HU.model.device) == []
    torch.cuda.synchronize()
    HU.model._engine().check_errors()
