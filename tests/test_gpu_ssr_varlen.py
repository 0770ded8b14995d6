"""Clips of different lengths through the SSR / GSR-UNet path in one call (vf_ssr_restore_varlen / SSR_UNet.restore_batch):
every clip must come back with exactly the bits a one-clip restore() gives it, whatever the other clips in the call are.
This is also what checks the varlen masking rule on the unet_v2 geometry (W0 = 1024 bins, row pitches 1025 ... 17,
both=True transposed-conv pruning)."""
import ctypes

import pytest
import torch

from conftest import load_golden
from oracle import vf_oracle as O

pytestmark = pytest.mark.gpu

WAV_RMS_TOL = 1e-3

# 1025 samples: the shortest legal clip (T = 3); 5000: T = 12 (even); 27883 / 28229: T = 64 / 65, either side of a 64-frame
# boundary of the UNet; 70 * 441 + 17: T = 71; 44113: T = 101; 132300: 3 s, the SSR config's segment; 441000: 10 s,
# T = 1001 - alone in the 1024-frame bucket
LENGTHS = [1025, 27883, 5000, 441000, 28229, 70 * 441 + 17, 44113, 132300]


def _clips(lengths, seed):
    return [O.synth_clips(1, n, seed=seed + i)[0].cuda() for i, n in enumerate(lengths)]


def _per_clip(model, clips):
    return [model.restore(c[None].contiguous())[0].clone() for c in clips]


def _new_model(ssr_state):
    from voicefixer_main_b200 import SSR_UNet
    return SSR_UNet().load_state_dict(ssr_state).eval().to("cuda:0")


@pytest.fixture(scope="module")
def ssr_state():
    from voicefixer_main_b200.weights import make_ssr_state
    return make_ssr_state(1234)


@pytest.fixture(scope="module")
def ssr_model(ssr_state):
    m = _new_model(ssr_state)
    yield m
    m._engine().check_errors()


def rms(x):
    return float(x.double().pow(2).mean().sqrt())


def test_mixed_lengths_bit_identical_to_one_clip_restores(ssr_model):
    clips = _clips(LENGTHS, seed=1300)
    got = ssr_model.restore_batch(clips)
    ssr_model._engine().check_errors()
    want = _per_clip(ssr_model, clips)
    assert [g.shape for g in got] == [c.shape for c in clips]
    for n, g, w in zip(LENGTHS, got, want):
        assert torch.isfinite(g).all(), n
        assert torch.equal(g, w), (n, float((g - w).abs().max()))


def test_one_plan_serves_changing_lengths_through_its_graph(ssr_state):
    """Same batch and bucket for every call: eager run, capture, replays.  Shorter clips follow longer ones in the same slots,
    so a stale row of d_sp / d_mag / d_frames that were read, or a row not rewritten as zero, would change the next clip's
    bits."""
    model = _new_model(ssr_state)
    eng = model._engine()
    long_set = _clips([3 * 44100, 2 * 44100 + 3000, 2 * 44100], seed=1400)          # T = 301, 208, 201: bucket 320
    short_set = _clips([3 * 44100 - 5, 5000, 20000], seed=1500)                      # T = 300, 12, 46: bucket 320
    refs = {id(s): _per_clip(model, s) for s in (long_set, short_set)}
    plans_before = eng.plan_cache_info()["plans"]
    side = torch.cuda.Stream()
    for k, s in enumerate([long_set, short_set, long_set, short_set, long_set]):
        if k == 3:      # a use of the same plan on another stream is ordered after the previous one
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                got = model.restore_batch(s)
            torch.cuda.current_stream().wait_stream(side)
        else:
            got = model.restore_batch(s)
        for g, w in zip(got, refs[id(s)]):
            assert torch.equal(g, w), k
    eng.check_errors()
    assert eng.plan_cache_info()["plans"] == plans_before + 1      # one varlen plan for all five calls


def test_golden_pair_among_longer_clips(ssr_model, golden_fingerprint_ok):
    g = load_golden("ssr_t64.npz")
    gold = torch.from_numpy(g["wav"]).cuda()                        # [2, N], T = 64
    ref = torch.from_numpy(g["out"])
    others = _clips([3 * 44100 + 77, 2 * 44100 + 11], seed=1600)
    out = ssr_model.restore_batch([others[0], gold[0], others[1], gold[1]])
    ssr_model._engine().check_errors()
    got = torch.stack([out[1], out[3]])
    e = rms(got.cpu() - ref)
    print("golden ssr_t64 pair inside a varlen batch: wav rms err", e, "ref rms", rms(ref))
    assert e < WAV_RMS_TOL
    for i in range(2):
        assert rms(got[i].cpu() - ref[i]) < WAV_RMS_TOL, i
    pair = ssr_model.restore(gold.contiguous())
    assert torch.equal(got, pair)


def test_sub_batches_give_the_same_bits(ssr_state):
    m = _new_model(ssr_state)
    eng = m._engine()
    clips = _clips([44100, 30000, 50000, 1025, 40000, 44100 + 441], seed=1700)
    full = [c.clone() for c in m.restore_batch(clips)]
    one_plan = eng.plan_cache_info()["bytes"]
    cap_mb = (one_plan >> 20) * 2 // 3                    # the 6-clip plan no longer fits
    eng.set_option("plan_cache_mb", cap_mb)
    got = m.restore_batch(clips)
    eng.check_errors()
    info = eng.plan_cache_info()
    print("ssr varlen sub-batching: one plan", one_plan >> 20, "MB; capped", info)
    assert info["bytes"] <= cap_mb << 20 < one_plan
    for g, f in zip(got, full):
        assert torch.equal(g, f)


def test_simt_validation_path(ssr_model):
    eng = ssr_model._engine()
    clips = _clips([5000, 1025, 20000], seed=1800)
    eng.set_option("validate_simt", 1)
    try:
        got = ssr_model.restore_batch(clips)
        want = _per_clip(ssr_model, clips)
        eng.check_errors()
    finally:
        eng.set_option("validate_simt", 0)
    for g, w in zip(got, want):
        assert torch.equal(g, w)


def _raw_call(eng, fn, packed, offsets, *flags):
    offs = (ctypes.c_int64 * len(offsets))(*offsets)
    out = torch.empty_like(packed)
    with torch.cuda.device(eng.device):
        return getattr(eng.lib, fn)(eng.ctx, ctypes.c_void_p(packed.data_ptr()), offs, len(offsets) - 1,
                                    ctypes.c_void_p(out.data_ptr()), *flags,
                                    ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


def test_bad_calls_fail_and_leave_the_context_usable(ssr_model, state):
    from voicefixer_main_b200 import VoiceFixer
    from voicefixer_main_b200._lib import VF_EINVAL, VF_ESTATE
    eng = ssr_model._engine()
    clips = _clips([5000, 20000], seed=1900)
    ref = [c.clone() for c in ssr_model.restore_batch(clips)]
    packed = torch.cat(clips + _clips([1024], seed=1950))
    fn = "vf_ssr_restore_varlen"
    assert _raw_call(eng, fn, packed, [0, 5000, 25000, 26024]) == VF_EINVAL       # a clip of 1024 samples
    assert _raw_call(eng, fn, packed, [0, 5000, 5000, 25000]) == VF_EINVAL        # offsets not increasing
    assert _raw_call(eng, fn, packed, [0, 25000, 5000]) == VF_EINVAL
    assert _raw_call(eng, fn, packed, [7, 5000, 25000]) == VF_EINVAL              # offsets[0] != 0
    with pytest.raises(ValueError):
        ssr_model.restore_batch([clips[0], clips[1][:1000]])
    # each entry point needs its own network: a VoiceFixer-only context has no unet_v2, an SSR-only one no vocoder
    vf = VoiceFixer().load_state_dict(state).eval().to("cuda:0")
    assert _raw_call(vf._engine(), fn, packed, [0, 5000, 25000]) == VF_ESTATE
    assert _raw_call(eng, "vf_restore_varlen", packed, [0, 5000, 25000], 0) == VF_ESTATE
    torch.cuda.synchronize()
    vf._engine().check_errors()
    # nothing was launched by the rejected calls: the next call restores the same bits
    again = ssr_model.restore_batch(clips)
    eng.check_errors()
    for a, r in zip(again, ref):
        assert torch.equal(a, r)
