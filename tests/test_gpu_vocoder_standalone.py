"""The stand-alone vocoder: vf_vocoder_varlen, vf_resynth / vf_resynth_varlen on vocoder-only plans, and
voicefixer_main_b200.vocoder.Vocoder, the pip package's stand-alone class.

Every packed clip must carry the bits of its fixed-shape batch-1 call: vf_vocoder for a mel, vf_frontend -> vf_vocoder ->
vf_finalize for a resynthesised clip, on a context that also holds an analysis module.  A context with only the vocoder's
weights gives the same bytes, refuses the restores, and sizes its plans by what they hold."""
import ctypes
import dataclasses

import numpy as np
import pytest
import torch

import test_gpu_plan_replay as PR
from oracle import vf_oracle as O
from voicefixer_main_b200 import _lib as VL
from voicefixer_main_b200._lib import VF_EINVAL, VF_ESTATE, EngineError
from voicefixer_main_b200.arch import VocoderConfig, frames_for, vocoder_out_len
from voicefixer_main_b200.model import Engine, VoiceFixer
from voicefixer_main_b200.vocoder import Vocoder

pytestmark = pytest.mark.gpu

FRAMES = [1, 2, 3, 63, 64, 65, 101, 1001, 6001]
PLAN_VARLEN, PLAN_VOC, PLAN_VOC_VARLEN = 2, 4, 5
SR = 44100


def mels(frames, seed=7):
    """Seeded linear mels with the range of speech: |x| up to ~10, many small values."""
    g = torch.Generator().manual_seed(seed)
    return [((torch.rand(t, 128, generator=g) * 2.2) ** 4).cuda() for t in frames]


def clips(lengths, seed=21):
    return [O.synth_clips(1, n, seed=seed + i)[0].float().cuda() for i, n in enumerate(lengths)]


def bits(t):
    return t.contiguous().view(torch.int32)


def vocoder_state(state):
    return {k: v for k, v in state.items() if k.startswith("vocoder.")}


@pytest.fixture(scope="module")
def full(state):
    e = Engine("cuda:0")
    e.load_state(state, need=("unet", "vocoder"))
    yield e
    e.check_errors()
    e.close()


@pytest.fixture(scope="module")
def voc_only(state):
    e = Engine("cuda:0")
    e.load_state(vocoder_state(state), need=("vocoder",))
    yield e
    e.check_errors()
    e.close()


@pytest.fixture(scope="module")
def mel_ref(full):
    """Each mel of FRAMES through vf_vocoder at batch 1 on the full context."""
    ms = mels(FRAMES)
    refs = [full.vocoder(m[None])[0] for m in ms]
    torch.cuda.synchronize()
    return ms, refs


def check_packed(out, refs, frames, name):
    off = 0
    for t, r in zip(frames, refs):
        n = vocoder_out_len(t, VocoderConfig())
        assert r.numel() == n
        assert torch.equal(bits(out[off:off + n]), bits(r)), (name, "clip of", t, "frames differs from vf_vocoder")
        off += n
    assert off == out.numel()


# ------------------------------------------------------------------ 1. bit-identity of mels
def test_vocoder_varlen_equals_vf_vocoder_per_clip(full, mel_ref):
    ms, refs = mel_ref
    out = full.vocoder_varlen(torch.cat(ms), FRAMES)
    check_packed(out, refs, FRAMES, "one call")
    # another order: a clip's bits depend neither on its slot nor on its neighbours
    perm = [8, 0, 4, 7, 1, 6, 2, 5, 3]
    out = full.vocoder_varlen(torch.cat([ms[i] for i in perm]), [FRAMES[i] for i in perm])
    check_packed(out, [refs[i] for i in perm], [FRAMES[i] for i in perm], "permuted")
    # a small plan budget splits the call into sub-batches
    full.set_option("plan_cache_mb", 12 * 1024)
    try:
        assert full.selftest_sub_batch(PLAN_VOC_VARLEN, len(FRAMES), 6016) < len(FRAMES)
        out = full.vocoder_varlen(torch.cat(ms), FRAMES)
        check_packed(out, refs, FRAMES, "sub-batched")
    finally:
        full.set_option("plan_cache_mb", 0)
    full.check_errors()


def test_vocoder_varlen_refuses_bad_offsets(voc_only):
    """An empty or decreasing frame range fails with VF_EINVAL before anything is launched."""
    x = torch.cat(mels([5, 3]))
    out = torch.empty(100000, device="cuda")
    launches = voc_only.launch_count()
    for off in ([0, 5, 5, 8], [0, 5, 3, 8], [1, 5, 8]):
        table = (ctypes.c_int64 * len(off))(*off)
        rc = voc_only.lib.vf_vocoder_varlen(voc_only.ctx, ctypes.c_void_p(x.data_ptr()), table, len(off) - 1,
                                            ctypes.c_void_p(out.data_ptr()), None)
        assert rc == VF_EINVAL, (off, rc)
    assert voc_only.launch_count() == launches
    with pytest.raises(ValueError):
        voc_only.vocoder_varlen(x, [5, 4])
    with pytest.raises(ValueError):
        voc_only.vocoder_varlen(x, [])


# ------------------------------------------------------------------ 2. vocoder-only context
def test_vocoder_only_context(full, voc_only, mel_ref, state):
    ms, refs = mel_ref
    check_packed(voc_only.vocoder_varlen(torch.cat(ms), FRAMES), refs, FRAMES, "vocoder-only context")
    wav = clips([SR])[0][None].contiguous()
    for call in (lambda: voc_only.restore(wav), lambda: voc_only.restore_varlen(wav[0], [SR]),
                 lambda: voc_only.vocoder(ms[3][None])):
        with pytest.raises(EngineError) as e:
            call()
        assert e.value.code == VF_ESTATE
    # still usable, same bytes
    check_packed(voc_only.vocoder_varlen(torch.cat(ms[:4]), FRAMES[:4]), refs[:4], FRAMES[:4], "after refusals")
    voc_only.check_errors()
    # plans hold the vocoder only: at one budget, a 10 s bucket's sub-batch is at least the restore's
    for e in (full, voc_only):
        e.set_option("plan_cache_mb", 16 * 1024)
    try:
        voc = voc_only.selftest_sub_batch(PLAN_VOC_VARLEN, 256, 1024)
        gsr = full.selftest_sub_batch(PLAN_VARLEN, 256, 1024)
        print(f"sub-batch at a 10 s bucket under 16 GiB: vocoder-only {voc}, restore {gsr}")
        assert voc >= gsr and voc > 1
    finally:
        for e in (full, voc_only):
            e.set_option("plan_cache_mb", 0)


# ------------------------------------------------------------------ 3. resynthesis
LENGTHS = [1025, 1500, SR + 17, 3 * SR, 10 * SR + 7, 60 * SR]


def resynth_ref(full, x):
    mel = full.frontend(x[None])[0]
    return full.finalize(full.vocoder(mel), x.numel())[0]


def test_resynth_varlen_equals_the_composed_calls(full, voc_only):
    cs = clips(LENGTHS)
    refs = [resynth_ref(full, x) for x in cs]
    for e in (voc_only, full):
        out = e.resynth_varlen(torch.cat(cs), LENGTHS)
        for x, r, o in zip(cs, refs, torch.split(out, LENGTHS)):
            assert torch.equal(bits(o), bits(r)), ("resynth_varlen", x.numel())
    # the fixed-shape call equals the packed one
    for x, r in zip(cs[:3], refs[:3]):
        assert torch.equal(bits(voc_only.resynth(x[None])[0]), bits(r))
    voc_only.check_errors()


def test_resynth_against_the_oracle(voc_only, state):
    """The vocoder-only chain of oracle/vf_oracle.py: pre -> vocoder on the linear mel -> peak normalise -> trim_center."""
    n = SR // 2 + 3
    x = clips([n], seed=33)[0]
    got = voc_only.resynth_varlen(x, [n]).cpu().double()
    with torch.no_grad():
        _, mel = O.pre(x.cpu()[None, None, :])
        want = O.trim_center(O.peak_normalize(O.vocoder_forward(state, mel.float())), n)[0, 0].double()
    rms = float(torch.sqrt(torch.mean((got - want) ** 2)))
    print(f"resynth vs oracle: RMS {rms:.3e}")
    assert rms < 1e-3


def test_resynth_length_rules(state, voc_only):
    x = clips([5000])[0]
    with pytest.raises(EngineError) as e:
        voc_only.resynth_varlen(torch.cat([x, x[:1024]]), [5000, 1024])
    assert e.value.code == VF_EINVAL
    # trim_center's d == 1 case (no tail frames, T even, n = 441 (T - 1) + 440), as vf_restore_varlen refuses it
    e0 = Engine("cuda:0", dataclasses.replace(VocoderConfig(), tail_pad_base=0))
    try:
        e0.load_state(vocoder_state(state), need=("vocoder",))
        bad = clips([441 * 9 + 440], seed=990)[0]
        launches = e0.launch_count()
        with pytest.raises(EngineError) as err:
            e0.resynth_varlen(torch.cat([x, bad]), [5000, bad.numel()])
        assert err.value.code == VF_EINVAL and e0.launch_count() == launches
        e0.check_errors()
    finally:
        e0.close()
    voc_only.check_errors()


# ------------------------------------------------------------------ 4. float64 replay of the vocoder-only plans
VOC_PLANS = {"voc.voc3": (PLAN_VOC, 3), "voc_varlen.voc1": (PLAN_VOC_VARLEN, 1)}


@pytest.fixture(scope="module")
def replay_setup(state):
    e = Engine("cuda:0")
    e.load_state(vocoder_state(state), need=("vocoder",))
    cfg = VL.VfConfig()
    VL.load_library().vf_default_config(ctypes.byref(cfg))
    yield e, state, cfg
    e.check_errors()
    e.close()


@pytest.mark.parametrize("name", list(VOC_PLANS))
def test_vocoder_plans_replay_against_float64(replay_setup, name):
    """Every launch of a vocoder-only plan checked as test_gpu_plan_replay checks the restore plans'."""
    e, sd, cfg = replay_setup
    kind, terms = VOC_PLANS[name]
    e.set_option("vocoder_terms", terms)
    if kind == PLAN_VOC:
        wav, lengths = torch.stack([O.synth_clips(1, PR.N_LONG, seed=11)[0].float(), PR.wide_clip(PR.N_LONG, 12)]).cuda(), None
    else:
        wav, lengths = PR.inputs(PLAN_VARLEN)
    rp = PR.Replay(name, sd, cfg, lengths is not None)
    rp.lengths = lengths
    PR.PAIR_STAGE.clear()
    if terms == 1:
        PR.PAIR_STAGE[cfg.voc_num_stages - 1] = True
    try:
        got = e.selftest_plan_trace(kind, wav, lengths, rp.on_op, direct_steps=True)
        e.check_errors()
        for _ in range(2):          # eager, then from the plan's graph
            want = e.resynth(wav) if lengths is None else e.resynth_varlen(wav, lengths)
            torch.cuda.synchronize()
            assert torch.equal(bits(got), bits(want)), (name, "traced output differs from the product call")
        n = len(lengths) if lengths else wav.shape[0]
        T = (1 + max(lengths) // PR.HOP + 63) // 64 * 64 if lengths else 1 + wav.shape[1] // PR.HOP
        gemms = e.selftest_plan_gemms(kind, n, T)
        assert gemms and all(label.startswith("voc.") for label, _ in gemms), name
        assert {sg for _, sg in gemms} == rp.sigs, (name, "configurations not replayed")
        assert rp.kinds == PR.want_kinds("voc", terms, False), (name, rp.kinds)
        print(f"{name}: {rp.ops} ops, worst err / bound {rp.worst:.3e} at {rp.worst_op}; arena {rp.arena / 2 ** 20:.1f} MiB")
    finally:
        e.set_option("vocoder_terms", 1)


# ------------------------------------------------------------------ 5. the Python surface
@pytest.fixture(scope="module")
def voc(state):
    v = Vocoder(sample_rate=44100).load_state_dict({k[len("vocoder."):]: t for k, t in vocoder_state(state).items()})
    v = v.eval().to("cuda:0")
    yield v
    v._engine().check_errors()


def test_vocoder_class_matches_the_c_calls(voc, full, mel_ref):
    ms, refs = mel_ref
    # forward: equal lengths in one call
    x = torch.stack([ms[6], ms[6] * 0.5])[:, None]
    y = voc(x)
    assert y.shape == (2, 1, vocoder_out_len(101, VocoderConfig()))
    assert torch.equal(bits(y[:, 0]), bits(full.vocoder(x[:, 0].contiguous())))
    assert torch.equal(bits(voc.forward(x.cpu(), cuda=True)), bits(y))
    # forward_batch: one view per clip
    outs = voc.forward_batch(ms)
    for o, r in zip(outs, refs):
        assert torch.equal(bits(o), bits(r))
    # resynth_batch
    cs = clips([1025, SR, 2 * SR + 5])
    for x, o in zip(cs, voc.resynth_batch(cs)):
        assert torch.equal(bits(o), bits(resynth_ref(full, x)))


def test_oracle_batch_writes_the_oracle_bytes(voc, tmp_path):
    from voicefixer_main_b200.handler import save_wave
    lengths = [SR + 1000, 61 * SR + 123, 5 * SR]
    items = []
    for i, n in enumerate(lengths):
        src = str(tmp_path / f"in{i}.wav")
        save_wave(O.synth_clips(1, n, seed=50 + i)[0].numpy() * 0.5, src)
        items.append((src, str(tmp_path / f"batch{i}.wav")))
    voc.oracle_batch(items)
    for i, (src, dst) in enumerate(items):
        one = str(tmp_path / f"one{i}.wav")
        voc.oracle(src, one)
        with open(one, "rb") as a, open(dst, "rb") as b:
            assert a.read() == b.read(), src
    with pytest.raises(RuntimeError):
        voc.oracle(items[0][0], str(tmp_path / "x.wav"), cuda=False)


def test_restore_inmem_with_the_stand_alone_vocoder(state, voc):
    model = VoiceFixer().load_state_dict(state).eval().to("cuda:0")
    wav = O.synth_clips(1, 30 * SR + 3 * SR, seed=77)[0].numpy()
    want = model.restore_inmem(wav, cuda=True, mode=0, your_vocoder_func=model.vocoder.forward)
    got = model.restore_inmem(wav, cuda=True, mode=0, your_vocoder_func=voc.forward)
    assert got.shape == want.shape and np.array_equal(got.view(np.int32), want.view(np.int32))
    model._engine().check_errors()


# ------------------------------------------------------------------ 6. no regression of the restore plans
def voc_labels(cfg, terms):
    """The vocoder's launch list as plan.cu's build_vocoder makes it (trace labels: GEMMs and pairs by their label, the
    other ops by their kind's name)."""
    out = ["voc_condition"] + [f"voc.cond{i}" for i in range(cfg.voc_cond_layers)] + ["reflect_fill", "voc.stem"]
    for s in range(cfg.voc_num_stages):
        out.append(f"voc.up{s}")
        for i in range(cfg.voc_depth[s]):
            out += [f"voc.res{s}.{i}.pair"] if terms == 1 and s == cfg.voc_num_stages - 1 else [f"voc.res{s}.{i}.a", f"voc.res{s}.{i}.b"]
    return out + ["reflect_fill", "memset", "voc_tail"]


def trace_labels(e, kind, wav, lengths):
    got = []
    e.selftest_plan_trace(kind, wav, lengths, lambda after, t: got.append((t.list, t.label.decode(), t.op.is_log)) if not after else None)
    return got


def test_restore_plans_are_unchanged(full):
    """The restore plans' launch lists: the UNet list, then the vocoder list with its conditioning on the restored log-mel,
    then the finalize; the vocoder-only plans run the same vocoder list on the linear mel and nothing else."""
    cfg = VL.VfConfig()
    VL.load_library().vf_default_config(ctypes.byref(cfg))
    wav = clips([SR])[0]
    for fixed, varlen in ((0, PLAN_VARLEN), (PLAN_VOC, PLAN_VOC_VARLEN)):
        for kind in (fixed, varlen):
            lengths = [SR, 20000] if kind == varlen else None
            x = torch.cat([wav, wav[:20000]]) if lengths else wav[None].contiguous()
            got = trace_labels(full, kind, x, lengths)
            unet = [lb for li, lb, _ in got if li == 0]
            voc = [(lb, lg) for li, lb, lg in got if li == 1]
            assert [li for li, _, _ in got][-1] == 2 and [li for li, _, _ in got].count(2) == 1
            assert [lb for lb, _ in voc] == voc_labels(cfg, 1), kind
            assert voc[0][1] == (0 if fixed == PLAN_VOC else 1), kind
            gemms = [lb for lb, _ in full.selftest_plan_gemms(kind, len(lengths) if lengths else 1, 128 if lengths else frames_for(SR))]
            if fixed == PLAN_VOC:
                assert unet == [], kind
            else:
                assert unet[0] == "unet_first" and unet.count("pool") == 6, kind
                assert [lb for lb in unet if lb not in ("unet_first", "pool")] == [g for g in gemms if not g.startswith("voc.")]
    full.check_errors()
