"""The stream scheduler of voicefixer_main_b200/streaming.py, CPU only: StreamingRestorer over a fake engine whose
restore_chunks does vf_restore_chunks' gather, zero fill, network and crop in torch with a toy network.  The chunk tables a
session emits must be BoxcarOverlapAdd.plan's, and the streams' outputs BoxcarOverlapAdd's with the same network, bit for
bit, however the pushes are split and whichever streams share a step."""
import random

import pytest
import torch

from voicefixer_main_b200.arch import VocoderConfig
from voicefixer_main_b200.longform import BoxcarOverlapAdd
from voicefixer_main_b200.streaming import OPEN, StreamingRestorer

# (W, M): M > 1024 so that a last chunk with 0 < last < M (M + last samples) is still a clip restore() accepts
GEOMETRIES = [(4096, 1536), (2400, 1100)]


def toy_net(x):
    """Row-wise and element-wise (the same bits at any batch), and dependent on the chunk's extent through the flip and the
    position ramp, so a chunk cut at the wrong place changes the output."""
    pos = torch.arange(x.shape[-1], dtype=x.dtype) * 2.0 ** -12
    return {"wav": 0.5 * x + 0.25 * x.flip(-1) + pos}


class ToyRestoreNet:
    batch_invariant = True
    in_channels = 1

    def __call__(self, x):
        return toy_net(x)


class FakeEngine:
    device = torch.device("cpu")
    voc_cfg = VocoderConfig()

    def __init__(self):
        self.calls = []

    def restore_chunks(self, ring, table, unify_energy=False):
        self.calls.append([tuple(t) for t in table])
        L = ring.shape[1]
        kept = []
        for s, length, cl, cr, start, valid in table:
            assert 0 <= s < ring.shape[0] and 1024 < length <= L and start >= 0 and cl + cr < length
            pos = torch.arange(start, start + length)
            x = ring[s, pos % L].clone()
            x[pos >= valid] = 0
            kept.append(toy_net(x[None, None])["wav"][0, 0, cl:length - cr])
        return torch.cat(kept)


class FakeModel:
    def __init__(self):
        self.engine = FakeEngine()

    def _engine(self):
        return self.engine


def expected_plan(W, M, n):
    """BoxcarOverlapAdd.plan(n) as (start, length, crop_left, crop_right), the single chunk cut to n as ola_forward does."""
    plan, _ = BoxcarOverlapAdd(None, 1, W, M).plan(n)
    return [(a, b - a, cl, (b - n) if len(plan) == 1 else cr) for a, b, cl, cr in plan]


def offline(W, M, x):
    return BoxcarOverlapAdd(ToyRestoreNet(), 1, W, M)(x[None, None])[0, 0]


def signal(n, seed):
    return torch.randn(n, generator=torch.Generator().manual_seed(seed))


def run_session(W, M, lengths, seed, max_streams=None):
    """Streams of the given lengths, opened at staggered steps, pushed in random pieces (each at most W + 2M, the size that
    always fits after a step) and closed when complete.  -> (signals, outputs, {sid: [(start, length, cl, cr)]}, engine)."""
    rng = random.Random(seed)
    model = FakeModel()
    sr = StreamingRestorer(model, W, M, max_streams=max_streams or len(lengths))
    xs = [signal(n, seed * 100 + i) for i, n in enumerate(lengths)]
    opens = sorted(rng.randrange(0, 4) for _ in lengths)
    sids, pos = {}, {}
    outs, tables = {}, {}
    step = 0
    while len(sids) < len(lengths) or sr._streams:
        for i, t in enumerate(opens):
            if t == step and i not in sids:
                sids[i] = sr.open()
                pos[i] = 0
        for i, sid in sids.items():
            if pos[i] is None or rng.random() < 0.2:        # some streams skip a step
                continue
            k = min(rng.randrange(0, W + 2 * M + 1), lengths[i] - pos[i])
            sr.push(sid, xs[i][pos[i]:pos[i] + k])
            pos[i] += k
            if pos[i] == lengths[i]:
                sr.close(sid)
                pos[i] = None
        slots = {st.slot: sid for sid, st in sr._streams.items()}
        before = len(model.engine.calls)
        for sid, o in sr.step().items():
            outs.setdefault(sid, []).append(o)
        assert len(model.engine.calls) - before <= 1                  # one restore_chunks call per step
        for call in model.engine.calls[before:]:
            for s, length, cl, cr, start, valid in call:
                tables.setdefault(slots[s], []).append((start, length, cl, cr))
        step += 1
        assert step < 10000
    return xs, {i: torch.cat(outs.get(sids[i], [torch.zeros(0)])) for i in sids}, {i: tables.get(sids[i], []) for i in sids}, model.engine


def edge_lengths(W, M):
    return [W // 2,                  # n < W: one chunk
            W + M // 2,              # W <= n < W + M: the first chunk only restored after close
            3 * W,                   # last == 0
            4 * W + 100,             # 0 < last < M
            5 * W + M + 7,           # last > M
            23 * W + 5]              # the ring (2 (W + 2M)) wraps many times


@pytest.mark.parametrize("W,M", GEOMETRIES)
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_tables_and_outputs_match_boxcar_overlap_add(W, M, seed):
    lengths = edge_lengths(W, M) + [random.Random(seed).randrange(W, 12 * W) for _ in range(4)]
    xs, outs, tables, eng = run_session(W, M, lengths, seed)
    for i, n in enumerate(lengths):
        assert tables[i] == expected_plan(W, M, n), (i, n)
        assert outs[i].shape == (n,)
        assert torch.equal(outs[i], offline(W, M, xs[i])), (i, n)
    valid = {row[5] for call in eng.calls for row in call}
    assert OPEN in valid and valid - {OPEN}                            # early middle chunks and after-close chunks both ran


def test_output_does_not_depend_on_push_split_or_neighbours():
    W, M = GEOMETRIES[0]
    n = 9 * W + 333
    x = signal(n, 77)
    alone = FakeModel()
    sr = StreamingRestorer(alone, W, M, max_streams=1)
    a = sr.open()
    got = []
    for k in range(0, n, W):
        sr.push(a, x[k:k + W])
        got += list(sr.step().values())
    sr.close(a)
    got += list(sr.step().values())
    one = torch.cat(got)
    xs, outs, _, _ = run_session(W, M, [n, 5 * W, 7 * W + 1, 2 * W - 3], seed=9)
    assert torch.equal(one, offline(W, M, x))
    assert torch.equal(outs[0], offline(W, M, xs[0]))


def test_readiness_rule():
    """Chunk i leaves as a middle chunk once (i + 1) W + M samples are in, not a sample earlier."""
    W, M = GEOMETRIES[1]
    m = FakeModel()
    sr = StreamingRestorer(m, W, M)
    a = sr.open()
    sr.push(a, signal(W + M - 1, 1))
    assert sr.step() == {} and not m.engine.calls
    sr.push(a, signal(1, 2))
    out = sr.step()
    assert list(out) == [a] and out[a].numel() == W
    assert m.engine.calls[-1] == [(0, W + M, 0, M, 0, OPEN)]
    sr.push(a, signal(W - 1, 3))
    assert sr.step() == {}
    sr.push(a, signal(1, 4))
    sr.step()
    assert m.engine.calls[-1] == [(0, W + 2 * M, M, M, W - M, OPEN)]


def test_ring_overflow_raises_and_names_the_stream():
    W, M = GEOMETRIES[0]
    sr = StreamingRestorer(FakeModel(), W, M, max_streams=2)
    a, b = sr.open(), sr.open()
    sr.push(a, signal(W + 2 * M, 1))
    sr.push(a, signal(W + 2 * M, 2))                 # the ring holds 2 (W + 2M)
    with pytest.raises(OverflowError, match=f"stream {a}"):
        sr.push(a, signal(1, 3))
    sr.push(b, signal(2 * (W + 2 * M), 4))           # the other stream's row is untouched
    sr.step()
    sr.push(a, signal(W + 2 * M, 5))                 # after a step a push of W + 2M always fits
    with pytest.raises(OverflowError):
        sr.push(b, signal(2 * (W + 2 * M), 6))


def test_bad_arguments():
    m = FakeModel()
    with pytest.raises(ValueError):
        StreamingRestorer(m, 4097, 1000)                     # odd window
    for M in (0, 4096, 5000, -1):
        with pytest.raises(ValueError):
            StreamingRestorer(m, 4096, M)
    with pytest.raises(ValueError, match="1024"):
        StreamingRestorer(m, 1000, 24)                       # W + M = 1024: restore() refuses the first chunk
    with pytest.raises(ValueError, match="2\\^30"):
        StreamingRestorer(m, 1 << 30, 1)                     # W + 2M over the per-clip limit
    sr = StreamingRestorer(m, 2400, 1100, max_streams=1)
    a = sr.open()
    with pytest.raises(RuntimeError):
        sr.open()                                            # max_streams
    with pytest.raises(TypeError):
        sr.push(a, torch.zeros(10, dtype=torch.float64))
    with pytest.raises(TypeError):
        sr.push(a, torch.zeros(2, 10))
    with pytest.raises(KeyError):
        sr.push(a + 1, torch.zeros(10))


def test_close_refuses_an_unusable_last_chunk_and_keeps_the_stream_open():
    W, M = 4096, 512                                         # last chunk = M + last samples
    m = FakeModel()
    sr = StreamingRestorer(m, W, M)
    a = sr.open()
    x = signal(3 * W + 400, 5)
    out = []
    for k in range(0, x.numel(), W):
        sr.push(a, x[k:k + W])
        out += list(sr.step().values())
    with pytest.raises(ValueError, match=f"stream {a}.*1024"):
        sr.close(a)                                          # 912 samples
    sr.push(a, signal(200, 6))
    sr.close(a)
    with pytest.raises(ValueError):
        sr.push(a, signal(1, 7))                             # closed
    out = torch.cat(out + list(sr.step().values()))
    x = torch.cat([x, signal(200, 6)])
    assert torch.equal(out, offline(W, M, x))
    assert sr.step() == {} and not sr._streams                # the stream is gone, its ring row free
    b = sr.open()
    assert b == a + 1                                         # ids are not reused
    sr.close(b)                                               # an empty stream restores nothing
    assert sr.step() == {}
