"""Live streams restored chunk by chunk (vf_restore_chunks / StreamingRestorer): every stream's concatenated step outputs are
BoxcarOverlapAdd(RestoreNet(model)) of the whole stream bit for bit, whatever the pushes and the other streams were, and
the call itself is the varlen restore of the gathered, zero-filled chunks, cropped."""
import random

import pytest
import torch

from oracle import vf_oracle as O
from voicefixer_main_b200.longform import BoxcarOverlapAdd, RestoreNet
from voicefixer_main_b200.streaming import OPEN, StreamingRestorer

pytestmark = pytest.mark.gpu

# (W, M): M > 1024 so a last chunk of 0 < last < M is restorable; 8820 / 2205 is 0.2 s with a quarter-window margin
GEOMETRIES = [(4096, 1536), (8820, 2205)]


def edge_lengths(W, M):
    return [W // 2,                  # n < W: one chunk, cut to n
            W + M // 2,              # W <= n < W + M: the first chunk leaves only after close
            3 * W,                   # last == 0
            4 * W + 100,             # 0 < last < M
            5 * W + M + 7,           # last > M
            13 * W + 5]              # the ring (2 (W + 2M)) wraps several times


def _signal(n, seed):
    return O.synth_clips(1, n, seed=seed)[0]


@pytest.fixture(scope="module")
def model(state):
    from voicefixer_main_b200 import VoiceFixer
    m = VoiceFixer().load_state_dict(state).eval().to("cuda:0")
    yield m
    m._engine().check_errors()


def _offline(model, W, M, x, unify_energy=False):
    return BoxcarOverlapAdd(RestoreNet(model, unify_energy=unify_energy), 1, W, M)(x.cuda()[None, None])[0, 0]


def _session(model, W, M, xs, seed, unify_energy=False, max_streams=None):
    """All streams of xs through one StreamingRestorer: staggered opens, random pushes of at most W + 2M samples (host and
    device tensors alternately), random skipped steps.  -> the concatenated outputs per stream."""
    rng = random.Random(seed)
    sr = StreamingRestorer(model, W, M, max_streams=max_streams or len(xs), unify_energy=unify_energy)
    opens = sorted(rng.randrange(0, 3) for _ in xs)
    sids, pos, outs = {}, {}, {}
    step = 0
    while len(sids) < len(xs) or sr._streams:
        for i, t in enumerate(opens):
            if t == step and i not in sids:
                sids[i], pos[i] = sr.open(), 0
        for i, sid in sids.items():
            if pos[i] is None or rng.random() < 0.2:
                continue
            k = min(rng.randrange(0, W + 2 * M + 1), xs[i].numel() - pos[i])
            piece = xs[i][pos[i]:pos[i] + k]
            sr.push(sid, piece.cuda() if step % 2 else piece)
            pos[i] += k
            if pos[i] == xs[i].numel():
                sr.close(sid)
                pos[i] = None
        for sid, o in sr.step().items():
            outs.setdefault(sid, []).append(o.clone())
        step += 1
    return [torch.cat(outs[sids[i]]) for i in range(len(xs))]


@pytest.mark.parametrize("W,M", GEOMETRIES)
@pytest.mark.parametrize("unify_energy", [False, True])
def test_streams_bit_identical_to_boxcar_overlap_add(model, W, M, unify_energy):
    lengths = edge_lengths(W, M)
    xs = [_signal(n, 40 + i) for i, n in enumerate(lengths)]
    got = _session(model, W, M, xs, seed=W + int(unify_energy), unify_energy=unify_energy)
    model._engine().check_errors()
    for n, x, g in zip(lengths, xs, got):
        want = _offline(model, W, M, x, unify_energy)
        assert g.shape == (n,)
        assert torch.equal(g, want), (n, float((g - want).abs().max()))


def test_a_stream_alone_and_among_31_others(model):
    W, M = GEOMETRIES[1]
    x = _signal(9 * W + 777, 5)
    alone = _session(model, W, M, [x], seed=1)[0]
    others = [_signal(random.Random(i).randrange(W // 2, 8 * W), 100 + i) for i in range(31)]
    crowd = _session(model, W, M, [x] + others, seed=2)
    model._engine().check_errors()
    assert torch.equal(alone, crowd[0])
    assert torch.equal(alone, _offline(model, W, M, x))


def _by_hand(eng, ring, table, unify_energy=False):
    """The chunks sliced out of the ring with torch, zero-filled past `valid`, restored by restore_varlen, then cropped."""
    L = ring.shape[1]
    xs = []
    for s, length, cl, cr, start, valid in table:
        p = torch.arange(start, start + length, device=ring.device)
        xs.append(torch.where(p < valid, ring[s, p % L], torch.zeros((), device=ring.device)))
    out = eng.restore_varlen(torch.cat(xs), [t[1] for t in table], unify_energy=unify_energy)
    outs = torch.split(out, [t[1] for t in table])
    return torch.cat([o[cl:o.numel() - cr] for o, (_, _, cl, cr, _, _) in zip(outs, table)])


L_RING = 20000
TABLE = [(0, 5000, 0, 0, 0, OPEN),
         (1, 6000, 100, 200, 17000, OPEN),                  # wraps round the ring
         (2, 4500, 0, 1000, 39000, 41000),                  # wraps, and zero from position 41000 on
         (0, 3000, 5, 5, 3 * L_RING + 100, 1500),           # all past `valid`: zeros
         (1, L_RING, 1, 2, 123456, OPEN),                   # the whole ring
         (2, 1025, 0, 1024, 7, OPEN)]                       # the shortest chunk, one sample kept


def _ring(seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(3, L_RING, generator=g) * 0.3).cuda()


@pytest.mark.parametrize("unify_energy", [False, True])
def test_restore_chunks_is_restore_varlen_of_the_sliced_chunks(model, unify_energy):
    eng = model._engine()
    ring = _ring(1)
    got = eng.restore_chunks(ring, TABLE, unify_energy=unify_energy)
    want = _by_hand(eng, ring, TABLE, unify_energy)
    eng.check_errors()
    assert got.shape == want.shape == (sum(t[1] - t[2] - t[3] for t in TABLE),)
    assert torch.equal(got, want)


def test_sub_batches_and_padding_rows_give_the_same_bits(state):
    """11 chunks: one sub-batch on the 16-row plan; with the plan budget capped, sub-batches of 4 (the last padded from 3)."""
    from voicefixer_main_b200 import VoiceFixer
    m = VoiceFixer().load_state_dict(state).eval().to("cuda:0")
    eng = m._engine()
    ring = _ring(2)
    table = [(i % 3, 2000 + 700 * i, i, 3 * i, 1000 * i, OPEN if i % 2 else 15000) for i in range(11)]
    full = eng.restore_chunks(ring, table).clone()
    one_plan = eng.plan_cache_info()["bytes"]
    eng.set_option("plan_cache_mb", max(1, (one_plan >> 20) * 9 // 16))     # 8 rows fit: shapes 1, 2, 4 (7 rows) together
    got = eng.restore_chunks(ring, table)
    eng.check_errors()
    info = eng.plan_cache_info()
    print("restore_chunks sub-batching: 16-row plan", one_plan >> 20, "MB; capped", info)
    assert info["bytes"] < one_plan
    assert torch.equal(got, full)
    assert torch.equal(got, _by_hand(eng, ring, table))


def test_bad_calls_fail_with_einval_and_leave_the_context_usable(model, state):
    import ctypes
    import dataclasses
    from voicefixer_main_b200 import VoiceFixer
    from voicefixer_main_b200._lib import VF_EINVAL, EngineError, VfChunk
    from voicefixer_main_b200.arch import VocoderConfig
    eng = model._engine()
    ring = _ring(3)
    ref = eng.restore_chunks(ring, TABLE).clone()
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
            eng.restore_chunks(ring, [good, row])
        assert e.value.code == VF_EINVAL, row
    rows = (VfChunk * 1)(VfChunk(*good))
    out = torch.empty(5000, device="cuda")
    with torch.cuda.device(eng.device):
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        assert eng.lib.vf_restore_chunks(eng.ctx, ctypes.c_void_p(ring.data_ptr()), 3, L_RING, rows, 1,
                                         ctypes.c_void_p(out.data_ptr()), 2, st) == VF_EINVAL      # unknown flag bits
        assert eng.lib.vf_restore_chunks(eng.ctx, ctypes.c_void_p(ring.data_ptr()), 3, L_RING, rows, 0,
                                         ctypes.c_void_p(out.data_ptr()), 0, st) == VF_EINVAL      # no chunks
    # a length trim_center refuses (no tail frames, T = 10 even, n = 441 (T - 1) + 440): VF_EINVAL, as restore() fails
    m0 = VoiceFixer(vocoder_config=dataclasses.replace(VocoderConfig(), tail_pad_base=0)).load_state_dict(state).eval().to("cuda:0")
    with pytest.raises(EngineError) as e:
        m0._engine().restore_chunks(ring, [(0, 441 * 9 + 440, 0, 0, 0, OPEN)])
    assert e.value.code == VF_EINVAL
    with pytest.raises(ValueError, match="trim_center"):
        StreamingRestorer(m0, 441 * 8, 440 + 441)        # W + M = 441 * 9 + 440
    eng.check_errors()
    again = eng.restore_chunks(ring, TABLE)
    eng.check_errors()
    assert torch.equal(again, ref)


def test_plans_stay_flat_while_the_stream_count_varies(model):
    """After the power-of-two shapes are warm, a session whose active chunk count changes every step builds and evicts no
    plan (every chunk of this geometry is under 64 frames: one bucket)."""
    W, M = GEOMETRIES[0]
    eng = model._engine()
    ring = _ring(4)
    for rows in (1, 2, 4, 8, 16):
        eng.restore_chunks(ring, [(r % 3, W + 2 * M, M, M, 100 * r, OPEN) for r in range(rows)])
    before = eng.plan_cache_info()
    rng = random.Random(7)
    n_streams = 16
    sr = StreamingRestorer(model, W, M, max_streams=n_streams)
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
