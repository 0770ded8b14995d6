"""Live streams and long recordings through the SSR / GSR-UNet path (vf_ssr_restore_chunks / StreamingRestorer over SSR_UNet,
restore_longform over SSR_UNet): every stream's concatenated step outputs are BoxcarOverlapAdd(RestoreNet(ssr_model)) of the
whole stream bit for bit, the call itself is vf_ssr_restore_varlen of the gathered, zero-filled chunks, cropped, and the
stacked rows of restore_longform give the bits of one-chunk restores.  Sizes are small: unet_v2 costs about 8 times the
ResUNet per frame."""
import ctypes
import random

import pytest
import torch

from test_gpu_streaming import GEOMETRIES, L_RING, TABLE, _offline, _ring, _session, _signal, edge_lengths
from voicefixer_main_b200.longform import BoxcarOverlapAdd, restore_longform
from voicefixer_main_b200.streaming import OPEN, StreamingRestorer

pytestmark = pytest.mark.gpu


def _new_model(ssr_state, cls_name="SSR_UNet"):
    import voicefixer_main_b200 as V
    return getattr(V, cls_name)().load_state_dict(ssr_state).eval().to("cuda:0")


@pytest.fixture(scope="module")
def ssr_state():
    from voicefixer_main_b200.weights import make_ssr_state
    return make_ssr_state(1234)


@pytest.fixture(scope="module")
def ssr_model(ssr_state):
    m = _new_model(ssr_state)
    yield m
    m._engine().check_errors()


@pytest.mark.parametrize("W,M", GEOMETRIES)
def test_streams_bit_identical_to_boxcar_overlap_add(ssr_model, W, M):
    lengths = edge_lengths(W, M)
    xs = [_signal(n, 60 + i) for i, n in enumerate(lengths)]
    got = _session(ssr_model, W, M, xs, seed=W + 3)
    ssr_model._engine().check_errors()
    for n, x, g in zip(lengths, xs, got):
        want = _offline(ssr_model, W, M, x)
        assert g.shape == (n,)
        assert torch.equal(g, want), (n, float((g - want).abs().max()))


def test_a_stream_alone_and_among_31_others(ssr_model):
    W, M = GEOMETRIES[1]
    x = _signal(9 * W + 777, 6)
    alone = _session(ssr_model, W, M, [x], seed=1)[0]
    others = [_signal(random.Random(i).randrange(W // 2, 8 * W), 200 + i) for i in range(31)]
    crowd = _session(ssr_model, W, M, [x] + others, seed=2)
    ssr_model._engine().check_errors()
    assert torch.equal(alone, crowd[0])
    assert torch.equal(alone, _offline(ssr_model, W, M, x))


def _by_hand(eng, ring, table):
    """The chunks sliced out of the ring with torch, zero-filled past `valid`, restored by ssr_restore_varlen, then cropped."""
    L = ring.shape[1]
    xs = []
    for s, length, cl, cr, start, valid in table:
        p = torch.arange(start, start + length, device=ring.device)
        xs.append(torch.where(p < valid, ring[s, p % L], torch.zeros((), device=ring.device)))
    out = eng.ssr_restore_varlen(torch.cat(xs), [t[1] for t in table])
    outs = torch.split(out, [t[1] for t in table])
    return torch.cat([o[cl:o.numel() - cr] for o, (_, _, cl, cr, _, _) in zip(outs, table)])


def test_ssr_restore_chunks_is_ssr_restore_varlen_of_the_sliced_chunks(ssr_model):
    """TABLE: a ring wrap, a `valid` cut, an all-zero chunk, a whole-ring chunk and a 1025-sample chunk."""
    eng = ssr_model._engine()
    ring = _ring(1)
    got = eng.ssr_restore_chunks(ring, TABLE)
    want = _by_hand(eng, ring, TABLE)
    eng.check_errors()
    assert got.shape == want.shape == (sum(t[1] - t[2] - t[3] for t in TABLE),)
    assert torch.equal(got, want)
    # and a chunk is vf_ssr_restore (batch 1) of its samples: the first chunk of TABLE reads ring[0, :5000]
    one = ssr_model.restore(ring[0:1, :5000].contiguous())[0]
    assert torch.equal(got[:5000], one)


def test_sub_batches_and_padding_rows_give_the_same_bits(ssr_state):
    """11 chunks: one sub-batch on the 16-row plan; with the plan budget capped, sub-batches of 4 (the last padded from 3)."""
    m = _new_model(ssr_state)
    eng = m._engine()
    ring = _ring(2)
    table = [(i % 3, 2000 + 700 * i, i, 3 * i, 1000 * i, OPEN if i % 2 else 15000) for i in range(11)]
    full = eng.ssr_restore_chunks(ring, table).clone()
    one_plan = eng.plan_cache_info()["bytes"]
    eng.set_option("plan_cache_mb", max(1, (one_plan >> 20) * 9 // 16))     # 8 rows fit: shapes 1, 2, 4 (7 rows) together
    got = eng.ssr_restore_chunks(ring, table)
    eng.check_errors()
    info = eng.plan_cache_info()
    print("ssr_restore_chunks sub-batching: 16-row plan", one_plan >> 20, "MB; capped", info)
    assert info["bytes"] < one_plan
    assert torch.equal(got, full)
    assert torch.equal(got, _by_hand(eng, ring, table))


def _raw(eng, ring, rows, n, out, n_streams=3, ring_len=L_RING):
    with torch.cuda.device(eng.device):
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        return eng.lib.vf_ssr_restore_chunks(eng.ctx, ctypes.c_void_p(ring.data_ptr()), n_streams, ring_len, rows, n,
                                             ctypes.c_void_p(out.data_ptr()), st)


def test_bad_calls_fail_and_leave_the_context_usable(ssr_model, state):
    from voicefixer_main_b200 import VoiceFixer
    from voicefixer_main_b200._lib import VF_EINVAL, VF_ESTATE, EngineError, VfChunk
    eng = ssr_model._engine()
    ring = _ring(3)
    ref = eng.ssr_restore_chunks(ring, TABLE).clone()
    good = (0, 5000, 10, 10, 100, OPEN)
    bad = [(3, 5000, 0, 0, 0, OPEN),                 # stream out of range
           (-1, 5000, 0, 0, 0, OPEN),
           (0, L_RING + 1, 0, 0, 0, OPEN),           # longer than the ring
           (0, 1024, 0, 0, 0, OPEN),                 # too short for restore()
           (0, 5000, 2500, 2500, 0, OPEN),           # the crops leave nothing
           (0, 5000, -1, 0, 0, OPEN),
           (0, 5000, 0, 0, -1, OPEN)]                # start < 0
    for row in bad:
        with pytest.raises(EngineError) as e:
            eng.ssr_restore_chunks(ring, [good, row])
        assert e.value.code == VF_EINVAL, row
        assert torch.equal(eng.ssr_restore_chunks(ring, TABLE), ref), row
    rows = (VfChunk * 1)(VfChunk(*good))
    out = torch.empty(5000, device="cuda")
    assert _raw(eng, ring, rows, 0, out) == VF_EINVAL                     # no chunks
    assert _raw(eng, ring, rows, 1, out, n_streams=0) == VF_EINVAL
    # over 2^30 samples: refused before the ring is touched (length > ring_len is checked first, so the ring claims more)
    huge = (VfChunk * 1)(VfChunk(0, (1 << 30) + 1, 0, 0, 0, OPEN))
    assert _raw(eng, ring, huge, 1, out, ring_len=(1 << 30) + 2) == VF_EINVAL
    # a length vf_restore_chunks refuses only for trim_center (with a vocoder without tail frames) is valid here
    n = 441 * 9 + 440
    got = eng.ssr_restore_chunks(ring, [(0, n, 0, 0, 0, OPEN)])
    assert torch.equal(got, ssr_model.restore(ring[0:1, :n].contiguous())[0])
    # a VoiceFixer-only context has no unet_v2
    vf = VoiceFixer().load_state_dict(state).eval().to("cuda:0")
    assert _raw(vf._engine(), ring, rows, 1, out) == VF_ESTATE
    torch.cuda.synchronize()
    vf._engine().check_errors()
    eng.check_errors()
    assert torch.equal(eng.ssr_restore_chunks(ring, TABLE), ref)


def test_gsr_unet_streams_too(ssr_state):
    gsr = _new_model(ssr_state, "GSR_UNet")
    W, M = GEOMETRIES[0]
    lengths = [W // 2, 4 * W + 100, 7 * W + M + 3]
    xs = [_signal(n, 80 + i) for i, n in enumerate(lengths)]
    got = _session(gsr, W, M, xs, seed=5)
    gsr._engine().check_errors()
    for x, g in zip(xs, got):
        assert torch.equal(g, _offline(gsr, W, M, x))
    with pytest.raises(ValueError, match="unify_energy"):
        StreamingRestorer(gsr, W, M, unify_energy=True)


def test_restore_longform_equals_one_chunk_restores(ssr_model):
    """Middle chunks stacked 8 rows per call (2 clips x 4 chunks) against every chunk of every clip restored alone."""

    class OneRowNet:
        in_channels = 1                                   # not batch_invariant: one chunk per call

        def __call__(self, x):
            return {"wav": torch.cat([ssr_model.restore(x[b:b + 1, 0].contiguous()) for b in range(x.shape[0])])[:, None]}

    W, M = 22050, 4410
    n = 5 * W + 8837                                      # 6 chunks, ragged tail
    wav = torch.stack([_signal(n, 90), _signal(n, 91)]).cuda()
    got = restore_longform(ssr_model, wav, window_size=W, in_margin=M)
    want = BoxcarOverlapAdd(OneRowNet(), 1, W, M)(wav[:, None, :])[:, 0]
    ssr_model._engine().check_errors()
    assert got.shape == (2, n)
    assert torch.equal(got, want), float((got - want).abs().max())


def test_plans_stay_flat_while_the_stream_count_varies(ssr_model):
    """After the power-of-two shapes are warm, a session whose active chunk count changes every step builds and evicts no
    plan (every chunk of this geometry is under 64 frames: one bucket)."""
    W, M = GEOMETRIES[0]
    eng = ssr_model._engine()
    ring = _ring(4)
    for rows in (1, 2, 4, 8, 16):
        eng.ssr_restore_chunks(ring, [(r % 3, W + 2 * M, M, M, 100 * r, OPEN) for r in range(rows)])
    before = eng.plan_cache_info()
    rng = random.Random(7)
    n_streams = 16
    sr = StreamingRestorer(ssr_model, W, M, max_streams=n_streams)
    ids = [sr.open() for _ in range(n_streams)]
    counts = []
    for step in range(24):
        active = rng.sample(ids, rng.randrange(1, n_streams + 1))
        for sid in active:
            sr.push(sid, _signal(W + 2 * M if step == 0 else W, 1000 * step + sid))
        out = sr.step()
        counts.append(len(out))
    eng.check_errors()
    after = eng.plan_cache_info()
    print("chunks per step", counts, "plans", before, "->", after)
    assert len(set(counts)) >= 6
    assert after["plans"] == before["plans"] and after["evicted"] == before["evicted"]
