"""A test set restored in one batched call (handler_batch, vf_restore_varlen_mels): every output file must have the bytes, and
every metrics dict the floats, that handler() gives that file on its own."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import vf_oracle as O

pytestmark = pytest.mark.gpu

SEG = 44100 * 60

# (samples, rate, target): the shortest legal file, 1 s, 3.7 s, 10 s, 61 s (a 60 s segment and a 1 s one), 22.05 kHz
TEST_SET = [(1025, 44100, True), (44100, 44100, False), (163170, 44100, True), (441000, 44100, False),
            (SEG + 44100, 44100, True), (55125, 22050, True)]


def _new_model(state):
    from voicefixer_main_b200 import VoiceFixer
    return VoiceFixer().load_state_dict(state).eval().to("cuda:0")


def _close(m):
    """Frees the context's plans now: the model sits in reference cycles, so collection would come at an arbitrary later
    point, and until then the device memory it holds shrinks the plan budget of every model created after it."""
    m._engine().check_errors()
    m._eng.close()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def model(state):
    m = _new_model(state)
    yield m
    _close(m)


@pytest.fixture
def fresh_model(state):
    m = _new_model(state)
    yield m
    _close(m)


@pytest.fixture
def handler_module(model, monkeypatch):
    from voicefixer_main_b200 import handler as H
    monkeypatch.setattr(H, "model", model)
    return H


def _pcm(n, seed):
    return O.to_int16(O.synth_clips(1, n, seed=seed)[0].clamp(-0.99, 0.99).numpy())


def _write_set(H, d, spec):
    """Input (and target) files of `spec` under d; returns the items with outputs under d/one and d/batch."""
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


def _run_both(H, model, d, items, meta):
    one = [H.handler(src, str(d / "one" / out), tgt, ckpt=None, device=model.device, meta=meta) for src, out, tgt in items]
    batch = H.handler_batch([(src, str(d / "batch" / out), tgt) for src, out, tgt in items], ckpt=None, device=model.device,
                            meta=meta)
    model._engine().check_errors()
    for (_, out, _), a, b in zip(items, one, batch):
        with open(d / "one" / out, "rb") as f1, open(d / "batch" / out, "rb") as f2:
            assert f1.read() == f2.read(), out
        assert a == b, (out, a, b)
    return one


@pytest.mark.parametrize("unify_energy", [False, True])
def test_batch_matches_handler_per_file(handler_module, model, tmp_path, unify_energy):
    items = _write_set(handler_module, tmp_path, TEST_SET)
    metrics = _run_both(handler_module, model, tmp_path, items, {"unify_energy": unify_energy})
    assert [bool(m) for m in metrics] == [t for _, _, t in TEST_SET]
    assert all(set(m) == {"mel-lsd", "mel-sispec", "mel-non-log-sispec"} for m in metrics if m)


def test_saturate_matches_handler(handler_module, model, tmp_path):
    items = _write_set(handler_module, tmp_path, [(30000, 44100, False), (163170, 44100, True), (5000, 44100, False)])
    _run_both(handler_module, model, tmp_path, items, {"saturate": True})


def test_rejected_file_raises_handlers_exception_and_writes_nothing(handler_module, model, tmp_path):
    H = handler_module
    items = _write_set(H, tmp_path, [(30000, 44100, False), (SEG + 1000, 44100, False)])   # last segment: 1000 samples
    with pytest.raises(Exception) as one:
        H.handler(items[1][0], str(tmp_path / "one" / items[1][1]), None, ckpt=None, device=model.device)
    with pytest.raises(Exception) as batch:
        H.handler_batch([(s, str(tmp_path / "batch" / o), t) for s, o, t in items], ckpt=None, device=model.device)
    assert type(batch.value) is type(one.value) and "in1.wav" in str(batch.value)
    assert os.listdir(tmp_path / "batch") == []
    torch.cuda.synchronize()
    model._engine().check_errors()


# ------------------------------------------------------------------ vf_restore_varlen_mels directly
LENGTHS = [1025, 27883, 5000, 441000, 28229, 44113, 88700]


def _clips(lengths, seed):
    return [O.synth_clips(1, n, seed=seed + i)[0].cuda() for i, n in enumerate(lengths)]


def _mels_call(eng, clips, unify_energy=False):
    from voicefixer_main_b200.arch import frames_for
    rows = sum(frames_for(c.numel()) for c in clips)
    mel, log_mel = torch.full((rows, 128), float("nan"), device="cuda"), torch.full((rows, 128), float("nan"), device="cuda")
    out = eng.restore_varlen(torch.cat(clips), [c.numel() for c in clips], unify_energy=unify_energy, mel_out=mel,
                             log_mel_out=log_mel)
    return out, mel, log_mel


def _split_mels(m, clips):
    from voicefixer_main_b200.arch import frames_for
    return list(torch.split(m, [frames_for(c.numel()) for c in clips]))


def test_packed_mels_equal_restore_stages_of_each_clip(model):
    eng = model._engine()
    clips = _clips(LENGTHS, seed=1300)
    out, mel, log_mel = _mels_call(eng, clips, unify_energy=True)
    plain = eng.restore_varlen(torch.cat(clips), LENGTHS, unify_energy=True)
    eng.check_errors()
    assert torch.equal(out, plain)
    for c, m, lm, o in zip(clips, _split_mels(mel, clips), _split_mels(log_mel, clips), torch.split(out, LENGTHS)):
        w = model.restore(c[None].contiguous(), unify_energy=True)
        want_mel, want_log = eng.restore_stages(1, c.numel())
        assert torch.equal(o, w[0]), c.numel()
        assert torch.equal(m, want_mel[0]) and torch.equal(lm, want_log[0]), c.numel()


def test_split_sub_batches_write_every_clips_mels(fresh_model):
    eng = fresh_model._engine()
    clips = _clips([44100, 30000, 50000, 1025, 40000, 44100 + 441], seed=1700)
    full = [t.clone() for t in _mels_call(eng, clips)]
    one_plan = eng.plan_cache_info()["bytes"]
    cap_mb = (one_plan >> 20) * 2 // 3                    # the 6-clip plan no longer fits
    eng.set_option("plan_cache_mb", cap_mb)
    got = _mels_call(eng, clips)
    eng.check_errors()
    assert eng.plan_cache_info()["bytes"] <= cap_mb << 20 < one_plan
    for g, f in zip(got, full):
        assert torch.equal(g, f)


def _raw(eng, fn, clips, *mels):
    offs = np.concatenate([[0], np.cumsum([c.numel() for c in clips])])
    packed = torch.cat(clips)
    out = torch.empty_like(packed)
    args = [eng.ctx, ctypes.c_void_p(packed.data_ptr()), (ctypes.c_int64 * len(offs))(*offs.tolist()), len(clips),
            ctypes.c_void_p(out.data_ptr()), 0]
    with torch.cuda.device(eng.device):
        n0 = eng.launch_count()
        eng._ck(getattr(eng.lib, fn)(*args, *mels, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
        return out, eng.launch_count() - n0


def test_null_outputs_behave_as_restore_varlen(model):
    eng = model._engine()
    clips = _clips([5000, 20000, 1025], seed=1900)
    ref, n_ref = _raw(eng, "vf_restore_varlen", clips)
    got, n_got = _raw(eng, "vf_restore_varlen_mels", clips, None, None)
    assert torch.equal(got, ref) and n_got == n_ref
    _, mel, _ = _mels_call(eng, clips)
    mel_only = torch.empty_like(mel)
    got2, n_mels = _raw(eng, "vf_restore_varlen_mels", clips, ctypes.c_void_p(mel_only.data_ptr()), None)
    eng.check_errors()
    assert torch.equal(got2, ref) and n_mels == n_ref + 1          # one copy kernel for the one sub-batch
    assert torch.equal(mel_only, mel)


def test_graph_replay_gives_the_first_calls_bits(fresh_model):
    eng = fresh_model._engine()
    clips = _clips([3 * 44100, 5000, 20000, 1025], seed=2100)
    calls = [[t.clone() for t in _mels_call(eng, clips)] for _ in range(3)]     # eager, capture, replay
    eng.check_errors()
    for a, b in zip(calls[0], calls[2]):
        assert torch.equal(a, b)
