"""Clips of different lengths in one call (vf_restore_varlen / VoiceFixer.restore_batch): every clip must come back with
exactly the bits a one-clip restore() gives it, whatever the other clips in the call are."""
import ctypes
import dataclasses

import pytest
import torch

from conftest import load_golden
from oracle import vf_oracle as O

pytestmark = pytest.mark.gpu

WAV_RMS_TOL = 1e-3

# 1025 samples: the shortest legal clip (T = 3, odd); 5000: T = 12 (even); 27883 / 28229: T = 64 / 65, either side of a
# 64-frame boundary of the UNet; 44113: T = 101; 88700: T = 202; 441000: 10 s, T = 1001 - alone in the 1024-frame bucket
LENGTHS = [1025, 27883, 5000, 441000, 28229, 44113, 88700]


def _clips(lengths, seed):
    return [O.synth_clips(1, n, seed=seed + i)[0].cuda() for i, n in enumerate(lengths)]


def _per_clip(model, clips, unify_energy=False):
    return [model.restore(c[None].contiguous(), unify_energy=unify_energy)[0].clone() for c in clips]


@pytest.fixture(scope="module")
def model(state):
    from voicefixer_main_b200 import VoiceFixer
    m = VoiceFixer().load_state_dict(state).eval().to("cuda:0")
    yield m
    m._engine().check_errors()


@pytest.mark.parametrize("unify_energy", [False, True])
def test_mixed_lengths_bit_identical_to_one_clip_restores(model, unify_energy):
    clips = _clips(LENGTHS, seed=300)
    got = model.restore_batch(clips, unify_energy=unify_energy)
    model._engine().check_errors()
    want = _per_clip(model, clips, unify_energy)
    assert [g.shape for g in got] == [c.shape for c in clips]
    for n, g, w in zip(LENGTHS, got, want):
        assert torch.equal(g, w), (n, float((g - w).abs().max()))


def test_one_plan_serves_changing_lengths_through_its_graph(model):
    """Same batch and bucket for every call: eager run, capture, replays.  Shorter clips follow longer ones in the same slots,
    so a row that is not rewritten as zero (a skipped tile that left stale data) would change the next clip's bits."""
    eng = model._engine()
    long_set = _clips([3 * 44100, 2 * 44100 + 3000, 2 * 44100], seed=400)           # T = 301, 208, 201: bucket 320
    short_set = _clips([3 * 44100 - 5, 5000, 20000], seed=500)                       # T = 300, 12, 46: bucket 320
    refs = {id(s): _per_clip(model, s) for s in (long_set, short_set)}
    plans_before = eng.plan_cache_info()["plans"]
    side = torch.cuda.Stream()
    for k, s in enumerate([long_set, short_set, long_set, short_set, long_set]):
        if k == 3:      # a use of the same plan on another stream is ordered after the previous one
            with torch.cuda.stream(side):
                got = model.restore_batch(s)
            torch.cuda.current_stream().wait_stream(side)
        else:
            got = model.restore_batch(s)
        for g, w in zip(got, refs[id(s)]):
            assert torch.equal(g, w), k
    eng.check_errors()
    assert eng.plan_cache_info()["plans"] == plans_before + 1      # one varlen plan for all five calls


def test_golden_clip_among_longer_clips(model, golden_fingerprint_ok):
    g = load_golden("e2e_1s.npz")
    gold = torch.from_numpy(g["wav"])[0].cuda()
    others = _clips([3 * 44100 + 77, 2 * 44100 + 11], seed=600)
    out = model.restore_batch([others[0], gold, others[1]])
    model._engine().check_errors()
    rms = float((out[1].cpu() - torch.from_numpy(g["out"])[0]).pow(2).mean().sqrt())
    print("golden 1 s clip inside a varlen batch: wav rms err", rms)
    assert rms < WAV_RMS_TOL


def test_sub_batches_give_the_same_bits(state):
    from voicefixer_main_b200 import VoiceFixer
    m = VoiceFixer().load_state_dict(state).eval().to("cuda:0")
    eng = m._engine()
    clips = _clips([44100, 30000, 50000, 1025, 40000, 44100 + 441], seed=700)
    full = [c.clone() for c in m.restore_batch(clips)]
    one_plan = eng.plan_cache_info()["bytes"]
    cap_mb = (one_plan >> 20) * 2 // 3                    # the 6-clip plan no longer fits
    eng.set_option("plan_cache_mb", cap_mb)
    got = m.restore_batch(clips)
    eng.check_errors()
    info = eng.plan_cache_info()
    print("varlen sub-batching: one plan", one_plan >> 20, "MB; capped", info)
    assert info["bytes"] <= cap_mb << 20 < one_plan
    for g, f in zip(got, full):
        assert torch.equal(g, f)


def test_simt_validation_path(model):
    eng = model._engine()
    clips = _clips([5000, 1025, 20000], seed=800)
    eng.set_option("validate_simt", 1)
    try:
        got = model.restore_batch(clips)
        want = _per_clip(model, clips)
        eng.check_errors()
    finally:
        eng.set_option("validate_simt", 0)
    for g, w in zip(got, want):
        assert torch.equal(g, w)


def _raw_call(eng, packed, offsets, flags=0):
    offs = (ctypes.c_int64 * len(offsets))(*offsets)
    out = torch.empty_like(packed)
    with torch.cuda.device(eng.device):
        return eng.lib.vf_restore_varlen(eng.ctx, ctypes.c_void_p(packed.data_ptr()), offs, len(offsets) - 1,
                                         ctypes.c_void_p(out.data_ptr()), flags, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


def test_bad_calls_fail_and_leave_the_context_usable(model, state):
    from voicefixer_main_b200 import VoiceFixer
    from voicefixer_main_b200._lib import VF_EINVAL
    from voicefixer_main_b200.arch import VocoderConfig
    eng = model._engine()
    clips = _clips([5000, 20000], seed=900)
    ref = [c.clone() for c in model.restore_batch(clips)]
    packed = torch.cat(clips + _clips([1024], seed=950))
    assert _raw_call(eng, packed, [0, 5000, 25000, 26024]) == VF_EINVAL            # a clip of 1024 samples
    assert _raw_call(eng, packed, [0, 5000, 5000, 25000]) == VF_EINVAL             # offsets not increasing
    assert _raw_call(eng, packed, [0, 25000, 5000]) == VF_EINVAL
    assert _raw_call(eng, packed, [7, 5000, 25000]) == VF_EINVAL                   # offsets[0] != 0
    assert _raw_call(eng, packed, [0, 5000, 25000], flags=2) == VF_EINVAL          # unknown flag bits
    with pytest.raises(ValueError):
        model.restore_batch([clips[0], clips[1][:1000]])
    # trim_center's d == 1 case: no tail frames and an even frame count T with n = 441 (T - 1) + 440 samples
    m0 = VoiceFixer(vocoder_config=dataclasses.replace(VocoderConfig(), tail_pad_base=0)).load_state_dict(state).eval().to("cuda:0")
    e0 = m0._engine()
    bad = _clips([441 * 9 + 440], seed=990)[0]                                     # T = 10, L = 4410, d = 1
    assert _raw_call(e0, torch.cat([clips[0], bad]), [0, 5000, 5000 + bad.numel()]) == VF_EINVAL
    with pytest.raises(Exception):
        m0.restore(bad[None].contiguous())
    torch.cuda.synchronize()
    e0.check_errors()
    # nothing was launched by the rejected calls: the next call restores the same bits
    again = model.restore_batch(clips)
    eng.check_errors()
    for a, r in zip(again, ref):
        assert torch.equal(a, r)
