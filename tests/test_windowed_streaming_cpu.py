"""The windowed stream scheduler of voicefixer_main_b200/streaming.py, CPU only: WindowedStreamingRestorer over a fake engine
whose restore_windows does vf_restore_windows' gather (leading zeros before position 0, zeros past `valid`), network,
rounded synthesis products, ascending accumulation and emission in torch with a toy network.  The windows a session
restores must be F.unfold(padding=W)'s minus the two that contribute nothing, and the streams' outputs the ascending-order
fold of those windows, bit for bit, however the pushes are split and whichever streams share a step."""
import random

import pytest
import torch
import torch.nn.functional as F

from test_streaming_cpu import FakeEngine as _BoxcarFakeEngine
from test_streaming_cpu import ToyRestoreNet, signal, toy_net
from voicefixer_main_b200.longform import WindowedOverlapAdd
from voicefixer_main_b200.streaming import OPEN, WindowedStreamingRestorer

# (W, hop): W / hop = 2, 3, 4, 1 and a hop that divides nothing in sight
GEOMETRIES = [(4096, 2048), (2400, 800), (2400, 600), (1200, 1200), (2048, 1500)]


class FakeEngine(_BoxcarFakeEngine):
    def restore_windows(self, ring, windows, W, synthesis, acc, emits, unify_energy=False):
        self.calls.append(([tuple(w) for w in windows], [tuple(e) for e in emits]))
        R, A = ring.shape[1], acc.shape[1]
        last = {}
        for s, start, valid in windows:
            assert 0 <= s < ring.shape[0] and W <= R and -W <= start and start > last.get(s, -(1 << 62))
            last[s] = start
            pos = torch.arange(start, start + W)
            x = ring[s, pos % R].clone()
            x[(pos < 0) | (pos >= valid)] = 0
            y = toy_net(x[None, None])["wav"][0, 0]
            prod = y * synthesis                             # rounded fp32 products, then the adds
            keep = (pos >= 0) & (pos < valid)
            slots = pos[keep] % A
            acc[s, slots] = acc[s, slots] + prod[keep]
        out = []
        for s, start, count in emits:
            slots = torch.arange(start, start + count) % A
            out.append(acc[s, slots].clone())
            acc[s, slots] = 0
        return torch.cat(out) if out else torch.zeros(0)


class FakeModel:
    def __init__(self):
        self.engine = FakeEngine()

    def _engine(self):
        return self.engine


def synthesis(W, hop, window):
    ola = WindowedOverlapAdd(None, 1, W, hop, window=window, reorder_chunks=False)
    if ola.use_window:
        return ola.window
    return torch.full((W,), float(torch.tensor(1.0) / torch.tensor(W / hop, dtype=torch.float32)))


def ascending_fold(x, W, hop, window):
    """WindowedOverlapAdd's result with the fold written out: every window of F.unfold(padding=W) through the network, times
    the synthesis table, and each output sample summed from 0 over its windows in ascending order (CUDA col2im's order)."""
    n = x.numel()
    syn = synthesis(W, hop, window)
    xp = F.pad(x, (W, W))
    out = torch.zeros(n)
    for k in range((n + W) // hop + 1):
        y = toy_net(xp[k * hop:k * hop + W][None, None])["wav"][0, 0] * syn
        lo, hi = max(0, k * hop - W), min(n, k * hop)
        if lo < hi:
            out[lo:hi] = out[lo:hi] + y[lo - (k * hop - W):hi - (k * hop - W)]
    return out


def contributing_starts(W, hop, n):
    """Starts of the windows of a stream of n samples that contribute to its output: k = 1 .. while k hop - W < n."""
    return [k * hop - W for k in range(1, (n + W) // hop + 1) if k * hop - W < n]


def run_session(W, hop, lengths, seed, window="hanning", max_streams=None):
    """Streams of the given lengths, opened at staggered steps, pushed in random pieces of at most W (the size that always
    fits after a step) and closed when complete.  -> (signals, outputs, {i: window starts}, engine)."""
    rng = random.Random(seed)
    model = FakeModel()
    sr = WindowedStreamingRestorer(model, W, hop, window=window, max_streams=max_streams or len(lengths))
    xs = [signal(n, seed * 100 + i) for i, n in enumerate(lengths)]
    opens = sorted(rng.randrange(0, 4) for _ in lengths)
    sids, pos, outs, starts = {}, {}, {}, {}
    step = 0
    while len(sids) < len(lengths) or sr._streams:
        for i, t in enumerate(opens):
            if t == step and i not in sids:
                sids[i], pos[i] = sr.open(), 0
        for i, sid in sids.items():
            if pos[i] is None or rng.random() < 0.2:
                continue
            k = min(rng.randrange(0, W + 1), lengths[i] - pos[i])
            sr.push(sid, xs[i][pos[i]:pos[i] + k])
            pos[i] += k
            if pos[i] == lengths[i]:
                sr.close(sid)
                pos[i] = None
        slots = {st.slot: sid for sid, st in sr._streams.items()}
        before = len(model.engine.calls)
        for sid, o in sr.step().items():
            assert o.numel() > 0
            outs.setdefault(sid, []).append(o)
        assert len(model.engine.calls) - before <= 1                  # one restore_windows call per step
        for windows, _ in model.engine.calls[before:]:
            for s, start, valid in windows:
                starts.setdefault(slots[s], []).append(start)
        step += 1
        assert step < 10000
    assert not sr.acc.any()                                           # every released slot left zero
    return (xs, {i: torch.cat(outs.get(sids[i], [torch.zeros(0)])) for i in sids},
            {i: starts.get(sids[i], []) for i in sids}, model.engine)


def edge_lengths(W, hop):
    return [0,
            hop // 2,                # n < hop
            W - 7,                   # n < W
            5 * hop,                 # hop | n
            7 * hop - W if 7 * hop > W else 3 * hop,   # hop | n + W
            W + 1,
            29 * W + 5]              # the ring (2W) wraps many times


@pytest.mark.parametrize("W,hop", GEOMETRIES)
@pytest.mark.parametrize("seed", [1, 2])
def test_windows_and_outputs_match_the_ascending_fold(W, hop, seed):
    lengths = edge_lengths(W, hop) + [random.Random(seed).randrange(1, 9 * W) for _ in range(4)]
    window = "hanning" if seed == 1 else None
    xs, outs, starts, eng = run_session(W, hop, lengths, seed, window=window)
    for i, n in enumerate(lengths):
        assert starts[i] == contributing_starts(W, hop, n), (i, n)
        assert -W not in starts[i]                                         # window 0 is never restored
        assert outs[i].shape == (n,)
        assert torch.equal(outs[i], ascending_fold(xs[i], W, hop, window)), (i, n)
    valid = {w[2] for windows, _ in eng.calls for w in windows}
    assert OPEN in valid and valid - {OPEN}                                  # windows of open and of closed streams ran


def test_the_last_window_is_skipped_when_hop_divides_n_plus_w():
    W, hop = 2400, 800
    n = 6 * hop - W                                                          # (n + W) / hop = 6: window 6 reads only past n
    assert (n + W) % hop == 0
    xs, outs, starts, _ = run_session(W, hop, [n], seed=3)
    assert starts[0] == [k * hop - W for k in range(1, 6)]
    assert torch.equal(outs[0], ascending_fold(xs[0], W, hop, "hanning"))


@pytest.mark.parametrize("window", ["hanning", None])
@pytest.mark.parametrize("n", [4096 * 3 + 17, 1000, 8192])
def test_ascending_restatement_is_f_fold_at_half_window_hops(window, n):
    """With W / hop = 2 every output sample is a sum of two terms, so any order gives the same bits: the restatement must
    then be WindowedOverlapAdd itself."""
    W = 4096
    x = signal(n, 5)
    ref = WindowedOverlapAdd(ToyRestoreNet(), 1, W, W // 2, window=window, reorder_chunks=False)(x[None, None])[0, 0]
    assert torch.equal(ascending_fold(x, W, W // 2, window), ref)


def test_readiness_and_emission_rule():
    """Window k leaves once k hop samples are in; sample t once the windows up to floor((t + W) / hop) are added."""
    W, hop = 2400, 800
    m = FakeModel()
    sr = WindowedStreamingRestorer(m, W, hop)
    a = sr.open()
    sr.push(a, signal(hop - 1, 1))
    assert sr.step() == {} and not m.engine.calls
    sr.push(a, signal(1, 2))
    assert sr.step() == {}                                    # window 1 added, nothing final yet
    assert m.engine.calls[-1] == ([(0, hop - W, OPEN)], [(0, 0, 0)])
    sr.push(a, signal(2 * hop, 3))
    out = sr.step()                                           # windows 2, 3: samples below 4 hop - W = 800 are final
    assert m.engine.calls[-1] == ([(0, 2 * hop - W, OPEN), (0, 3 * hop - W, OPEN)], [(0, 0, 4 * hop - W)])
    assert list(out) == [a] and out[a].numel() == 4 * hop - W
    sr.close(a)                                               # n = 3 hop: windows 4 and 5 remain (5 hop - W < n)
    out = sr.step()
    assert m.engine.calls[-1] == ([(0, 4 * hop - W, 3 * hop), (0, 5 * hop - W, 3 * hop)], [(0, 4 * hop - W, 3 * hop - (4 * hop - W))])
    assert out[a].numel() == 3 * hop - (4 * hop - W) and not sr._streams


def test_output_does_not_depend_on_push_split_or_neighbours():
    W, hop = 2400, 600
    n = 11 * W + 333
    x = signal(n, 77)
    sr = WindowedStreamingRestorer(FakeModel(), W, hop, max_streams=1)
    a = sr.open()
    got = []
    for k in range(0, n, W):
        sr.push(a, x[k:k + W])
        got += list(sr.step().values())
    sr.close(a)
    got += list(sr.step().values())
    want = ascending_fold(x, W, hop, "hanning")
    assert torch.equal(torch.cat(got), want)
    xs, outs, _, _ = run_session(W, hop, [n, 5 * W, 7 * W + 1, 2 * W - 3], seed=9)
    assert torch.equal(outs[0], ascending_fold(xs[0], W, hop, "hanning"))


def test_a_reused_slot_starts_from_zero():
    W, hop = 2400, 800
    sr = WindowedStreamingRestorer(FakeModel(), W, hop, max_streams=1)
    for i, n in enumerate([5 * W + 11, 3 * W - 5, hop + 1]):
        x = signal(n, 30 + i)
        a = sr.open()
        assert sr._streams[a].slot == 0
        got = []
        for k in range(0, n, W):
            sr.push(a, x[k:k + W])
            got += list(sr.step().values())
        sr.close(a)
        got += list(sr.step().values())
        assert torch.equal(torch.cat(got), ascending_fold(x, W, hop, "hanning")), n
        assert not sr.acc.any() and not sr._streams


def test_ring_overflow_raises_and_names_the_stream():
    W, hop = 2400, 800
    sr = WindowedStreamingRestorer(FakeModel(), W, hop, max_streams=2)
    a, b = sr.open(), sr.open()
    sr.push(a, signal(2 * W, 1))                      # nothing read yet: the ring holds 2W from position 0
    with pytest.raises(OverflowError, match=f"stream {a}"):
        sr.push(a, signal(1, 2))
    sr.push(b, signal(W, 3))                          # the other stream's row is untouched
    sr.step()
    sr.push(a, signal(W, 4))                          # after a step a push of W always fits
    sr.push(b, signal(W, 5))
    sr.step()
    sr.push(b, signal(W, 6))
    with pytest.raises(OverflowError):
        sr.push(b, signal(W + 1, 7))


def test_bad_arguments():
    m = FakeModel()
    with pytest.raises(ValueError, match="even"):
        WindowedStreamingRestorer(m, 4097)
    for hop in (0, -1, 4097):
        with pytest.raises(ValueError, match="hop_size"):
            WindowedStreamingRestorer(m, 4096, hop)
    with pytest.raises(ValueError, match="1024"):
        WindowedStreamingRestorer(m, 1024)                   # restore() refuses windows of 1024 samples
    with pytest.raises(ValueError, match="2\\^30"):
        WindowedStreamingRestorer(m, (1 << 30) + 2)
    with pytest.raises(ValueError):
        WindowedStreamingRestorer(m, 4096, max_streams=0)
    sr = WindowedStreamingRestorer(m, 2400, 800, max_streams=1)
    a = sr.open()
    with pytest.raises(RuntimeError):
        sr.open()                                            # max_streams
    with pytest.raises(TypeError):
        sr.push(a, torch.zeros(10, dtype=torch.float64))
    with pytest.raises(TypeError):
        sr.push(a, torch.zeros(2, 10))
    with pytest.raises(KeyError):
        sr.push(a + 1, torch.zeros(10))
    with pytest.raises(KeyError):
        sr.close(a + 1)
    sr.push(a, signal(100, 1))
    sr.close(a)
    with pytest.raises(ValueError, match="closed"):
        sr.push(a, signal(1, 2))
    with pytest.raises(ValueError, match="closed"):
        sr.close(a)
    sr.step()
    b = sr.open()
    assert b == a + 1                                        # ids are not reused
    sr.close(b)                                              # an empty stream restores nothing
    assert sr.step() == {} and not sr._streams
