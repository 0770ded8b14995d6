"""Live streams restored with windowed overlap-add (vf_restore_windows / vf_ssr_restore_windows / WindowedStreamingRestorer):
every stream's concatenated step outputs are WindowedOverlapAdd(RestoreNet(model)) of the whole stream on the device bit for
bit, whatever the pushes and the other streams were, and the call itself is the varlen restore of the torch-gathered,
zero-led windows followed by ascending-order synthesis-weighted accumulation.  W / hop = 3 and 4 are included: with two
terms per sample the summation order could not show."""
import ctypes
import random

import pytest
import torch

from oracle import vf_oracle as O
from voicefixer_main_b200.longform import RestoreNet, WindowedOverlapAdd
from voicefixer_main_b200.streaming import OPEN, WindowedStreamingRestorer

pytestmark = pytest.mark.gpu

# (W, hop): W / hop = 2, 3 and 4; 8820 is 0.2 s
GEOMETRIES = [(4096, 2048), (8820, 2940), (8820, 2205)]


def edge_lengths(W, hop):
    return [hop // 2,                # n < hop
            W - 7,                   # n < W
            5 * hop,                 # hop | n
            7 * hop - W,             # hop | n + W: the last window contributes nothing
            6 * W + 5]               # the ring (2W) wraps several times


def _signal(n, seed):
    return O.synth_clips(1, n, seed=seed)[0]


@pytest.fixture(scope="module")
def model(state):
    from voicefixer_main_b200 import VoiceFixer
    m = VoiceFixer().load_state_dict(state).eval().to("cuda:0")
    yield m
    m._engine().check_errors()


@pytest.fixture(scope="module")
def ssr_state():
    from voicefixer_main_b200.weights import make_ssr_state
    return make_ssr_state(1234)


def _offline(model, W, hop, window, x, unify_energy=False):
    ola = WindowedOverlapAdd(RestoreNet(model, unify_energy), 1, W, hop, window=window, reorder_chunks=False)
    return ola(x.cuda()[None, None])[0, 0]


def _session(model, W, hop, xs, seed, window="hanning", unify_energy=False, max_streams=None):
    """All streams of xs through one WindowedStreamingRestorer: staggered opens, random pushes of at most W samples (host
    and device tensors alternately), random skipped steps.  -> the concatenated outputs per stream."""
    rng = random.Random(seed)
    sr = WindowedStreamingRestorer(model, W, hop, window=window, max_streams=max_streams or len(xs), unify_energy=unify_energy)
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
            k = min(rng.randrange(0, W + 1), xs[i].numel() - pos[i])
            piece = xs[i][pos[i]:pos[i] + k]
            sr.push(sid, piece.cuda() if step % 2 else piece)
            pos[i] += k
            if pos[i] == xs[i].numel():
                sr.close(sid)
                pos[i] = None
        for sid, o in sr.step().items():
            outs.setdefault(sid, []).append(o.clone())
        step += 1
    assert not sr.acc.any()
    return [torch.cat(outs[sids[i]]) for i in range(len(xs))]


def _check_streams(model, W, hop, window, unify_energy, seed, lengths=None):
    lengths = lengths or edge_lengths(W, hop)
    xs = [_signal(n, seed + i) for i, n in enumerate(lengths)]
    got = _session(model, W, hop, xs, seed=seed, window=window, unify_energy=unify_energy)
    model._engine().check_errors()
    for n, x, g in zip(lengths, xs, got):
        want = _offline(model, W, hop, window, x, unify_energy)
        assert g.shape == (n,)
        assert torch.equal(g, want), (n, float((g - want).abs().max()))


@pytest.mark.parametrize("W,hop", GEOMETRIES)
@pytest.mark.parametrize("window", ["hanning", None])
@pytest.mark.parametrize("unify_energy", [False, True])
def test_streams_bit_identical_to_windowed_overlap_add(model, W, hop, window, unify_energy):
    _check_streams(model, W, hop, window, unify_energy, seed=W + hop + int(unify_energy) + 7 * (window is None))


@pytest.mark.parametrize("cls_name", ["SSR_UNet", "GSR_UNet"])
@pytest.mark.parametrize("W,hop", GEOMETRIES[1:])
@pytest.mark.parametrize("window", ["hanning", None])
def test_ssr_streams_bit_identical_to_windowed_overlap_add(ssr_state, cls_name, W, hop, window):
    import voicefixer_main_b200 as V
    m = getattr(V, cls_name)().load_state_dict(ssr_state).eval().to("cuda:0")
    with pytest.raises(ValueError, match="unify_energy"):
        WindowedStreamingRestorer(m, W, hop, unify_energy=True)
    _check_streams(m, W, hop, window, False, seed=W + hop + 3, lengths=[hop // 2, 7 * hop - W, 3 * W + 5])
    m._engine().check_errors()
    m._engine().close()


def test_a_stream_alone_and_among_31_others(model):
    W, hop = GEOMETRIES[1]
    x = _signal(9 * W + 777, 5)
    alone = _session(model, W, hop, [x], seed=1)[0]
    others = [_signal(random.Random(i).randrange(hop // 2, 6 * W), 100 + i) for i in range(31)]
    crowd = _session(model, W, hop, [x] + others, seed=2)
    model._engine().check_errors()
    assert torch.equal(alone, crowd[0])
    assert torch.equal(alone, _offline(model, W, hop, "hanning", x))


W_CALL = 8820
R_RING = 20000
A_LEN = 3 * W_CALL
# (stream, start, valid), W / hop = 3: leading zeros, ring wrap, zeros past `valid`, and windows that overlap an emission range
WINDOWS = [(0, -W_CALL + 2940, OPEN), (0, -W_CALL + 5880, OPEN), (0, 0, OPEN), (0, 2940, OPEN),
           (1, 17000, OPEN), (1, 19940, OPEN), (1, 22880, 30000),
           (2, 39000 - W_CALL, 41000), (2, 39000, 41000)]
EMITS = [(0, 0, 2940), (1, 16000, 9000), (2, 39000 - W_CALL, 5000)]


def _ring(seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(3, R_RING, generator=g) * 0.3).cuda()


def _acc(seed, emits):
    """Accumulators with partial sums pending from earlier steps where the emission ranges begin."""
    g = torch.Generator().manual_seed(seed)
    acc = torch.zeros(3, A_LEN)
    for s, start, _ in emits:
        slots = torch.arange(start, start + 1500) % A_LEN
        acc[s, slots] = torch.randn(1500, generator=g) * 0.1
    return acc.cuda()


def _synthesis(W, hop, window):
    ola = WindowedOverlapAdd(None, 1, W, hop, window=window, reorder_chunks=False)
    if ola.use_window:
        return ola.window.cuda()
    return torch.full((W,), float(torch.tensor(1.0) / torch.tensor(W / hop, dtype=torch.float32)), device="cuda")


def _by_hand(eng, ring, windows, W, syn, acc, emits, unify_energy=False, ssr=False):
    """The windows sliced out of the ring with torch (zero before 0 and past `valid`), restored by restore_varlen, weighted,
    added into acc window after window in table order, then the emission ranges copied out and zeroed."""
    R, A = ring.shape[1], acc.shape[1]
    xs = []
    for s, start, valid in windows:
        p = torch.arange(start, start + W, device=ring.device)
        xs.append(torch.where((p >= 0) & (p < valid), ring[s, p % R], torch.zeros((), device=ring.device)))
    lengths = [W] * len(windows)
    out = eng.ssr_restore_varlen(torch.cat(xs), lengths) if ssr else eng.restore_varlen(torch.cat(xs), lengths,
                                                                                        unify_energy=unify_energy)
    for (s, start, valid), y in zip(windows, torch.split(out, lengths)):
        p = torch.arange(start, start + W, device=ring.device)
        keep = (p >= 0) & (p < valid)
        slots = p[keep] % A
        acc[s, slots] = acc[s, slots] + (y * syn)[keep]
    got = []
    for s, start, count in emits:
        slots = torch.arange(start, start + count, device=ring.device) % A
        got.append(acc[s, slots].clone())
        acc[s, slots] = 0
    return torch.cat(got)


@pytest.mark.parametrize("window", ["hanning", None])
@pytest.mark.parametrize("unify_energy", [False, True])
def test_restore_windows_is_restore_varlen_then_ascending_accumulation(model, window, unify_energy):
    eng = model._engine()
    ring, syn = _ring(1), _synthesis(W_CALL, 2940, window)
    acc = _acc(2, EMITS)
    acc_ref = acc.clone()
    got = eng.restore_windows(ring, WINDOWS, W_CALL, syn, acc, EMITS, unify_energy=unify_energy)
    want = _by_hand(eng, ring, WINDOWS, W_CALL, syn, acc_ref, EMITS, unify_energy)
    eng.check_errors()
    assert got.shape == want.shape == (sum(e[2] for e in EMITS),)
    assert torch.equal(got, want)
    assert torch.equal(acc, acc_ref)                                   # the pending partial sums too


def test_ssr_restore_windows_is_ssr_restore_varlen_then_ascending_accumulation(ssr_state):
    from voicefixer_main_b200 import SSR_UNet
    m = SSR_UNet().load_state_dict(ssr_state).eval().to("cuda:0")
    eng = m._engine()
    ring, syn = _ring(3), _synthesis(W_CALL, 2940, "hanning")
    acc = _acc(4, EMITS)
    acc_ref = acc.clone()
    got = eng.ssr_restore_windows(ring, WINDOWS, W_CALL, syn, acc, EMITS)
    want = _by_hand(eng, ring, WINDOWS, W_CALL, syn, acc_ref, EMITS, ssr=True)
    eng.check_errors()
    assert torch.equal(got, want) and torch.equal(acc, acc_ref)
    eng.close()


def _as_chunks(windows, W):
    """The same rows as restore_chunks would run them (same lengths, streams and count: the same sub-batches and plans)."""
    return [(s, W, 0, 0, max(0, start), OPEN) for s, start, _ in windows]


def test_sub_batches_padding_rows_and_launch_count(state):
    """11 windows: one sub-batch on the 16-row plan; with the plan budget capped, sub-batches of 4 (the last padded from 3).
    Either way the bits are the same, and a call launches what restore_chunks launches on the same rows (a gather, the
    chain and one output kernel per sub-batch) plus one emission."""
    from voicefixer_main_b200 import VoiceFixer
    m = VoiceFixer().load_state_dict(state).eval().to("cuda:0")
    eng = m._engine()
    W, hop = 4096, 1024
    ring, syn = _ring(5), _synthesis(W, hop, "hanning")
    windows = [(i % 3, (i // 3) * hop - W + hop, OPEN if i % 2 else 15000) for i in range(11)]
    emits = [(s, 0, 2 * hop) for s in range(3)]

    def launches(fn):
        fn()
        fn()                                   # the chain's graph is captured on a plan's second use
        before = eng.launch_count()
        fn()
        return eng.launch_count() - before

    def windows_call():
        return eng.restore_windows(ring, windows, W, syn, torch.zeros(3, 2 * W, device="cuda"), emits)

    full = windows_call().clone()
    assert launches(windows_call) == launches(lambda: eng.restore_chunks(ring, _as_chunks(windows, W))) + 1
    one_plan = eng.plan_cache_info()["bytes"]
    eng.set_option("plan_cache_mb", max(1, (one_plan >> 20) * 9 // 16))     # 8 rows fit: shapes 1, 2, 4 (7 rows) together
    got = windows_call()
    assert launches(windows_call) == launches(lambda: eng.restore_chunks(ring, _as_chunks(windows, W))) + 1
    eng.check_errors()
    info = eng.plan_cache_info()
    print("restore_windows sub-batching: 16-row plan", one_plan >> 20, "MB; capped", info)
    assert info["bytes"] < one_plan
    assert torch.equal(got, full)
    assert torch.equal(got, _by_hand(eng, ring, windows, W, syn, torch.zeros(3, 2 * W, device="cuda"), emits))
    eng.close()


def test_bad_calls_fail_with_einval_and_leave_the_context_usable(model, state):
    import dataclasses
    from voicefixer_main_b200 import VoiceFixer
    from voicefixer_main_b200._lib import VF_EINVAL, EngineError, VfEmit, VfWindow
    from voicefixer_main_b200.arch import VocoderConfig
    eng = model._engine()
    ring, syn = _ring(6), _synthesis(W_CALL, 2940, "hanning")
    acc0 = _acc(7, EMITS)
    ref = eng.restore_windows(ring, WINDOWS, W_CALL, syn, acc0.clone(), EMITS).clone()

    def einval(windows, emits, W=W_CALL, synthesis=syn, ring=ring, m=eng):
        acc = acc0.clone()
        with pytest.raises(EngineError) as e:
            m.restore_windows(ring, windows, W, synthesis, acc, emits)
        assert e.value.code == VF_EINVAL, (windows, emits)
        assert torch.equal(acc, acc0)                                  # nothing was queued

    good_w, good_e = [(0, 0, OPEN)], [(0, 0, 100)]
    einval([(3, 0, OPEN)], good_e)                                     # stream out of range
    einval([(-1, 0, OPEN)], good_e)
    einval(good_w, [(3, 0, 100)])
    einval(good_w, good_e, W=R_RING + 2, synthesis=torch.zeros(R_RING + 2, device="cuda"))    # W over the ring
    einval(good_w, good_e, W=1024, synthesis=torch.zeros(1024, device="cuda"))                # W restore() refuses
    einval(good_w, good_e, synthesis=None)                             # no synthesis table
    einval([(0, 2940, OPEN), (0, 0, OPEN)], good_e)                    # not in ascending start
    einval([(0, 0, OPEN), (0, 0, OPEN)], good_e)
    einval([(0, -W_CALL - 1, OPEN)], good_e)                           # starts before the leading padding
    einval([(1, 0, OPEN)], good_e)                                     # no emission range for its stream
    einval([(0, 0, OPEN)], [(0, 1, 100)])                              # writes before the pending span
    einval([(0, 2 * A_LEN, OPEN)], good_e)                             # writes past it
    einval(good_w, [(0, 0, 100), (0, 100, 100)])                       # a second emission range
    einval(good_w, [(0, -1, 100)])
    einval(good_w, [(0, 0, A_LEN + 1)])                                # reads past the pending span
    einval(good_w, [(0, 0, -1)])
    rows = (VfWindow * 1)(VfWindow(*good_w[0]))
    ems = (VfEmit * 1)(VfEmit(*good_e[0]))
    acc, out = acc0.clone(), torch.empty(100, device="cuda")
    P = ctypes.c_void_p
    with torch.cuda.device(eng.device):
        st = P(torch.cuda.current_stream().cuda_stream)
        args = (P(ring.data_ptr()), 3, R_RING)
        tail = (W_CALL, P(syn.data_ptr()), P(acc.data_ptr()), A_LEN)
        assert eng.lib.vf_restore_windows(eng.ctx, *args, rows, 1, *tail, ems, 1, P(out.data_ptr()), 2, st) == VF_EINVAL  # flags
        assert eng.lib.vf_restore_windows(eng.ctx, *args, rows, 0, *tail, ems, 1, P(out.data_ptr()), 0, st) == VF_EINVAL  # no windows
        assert eng.lib.vf_restore_windows(eng.ctx, *args, rows, 1, *tail, ems, 0, P(out.data_ptr()), 0, st) == VF_EINVAL  # no emits
    assert torch.equal(acc, acc0)
    # a W trim_center refuses (no tail frames, T = 10 even, n = 441 (T - 1) + 440): VF_EINVAL, as restore() fails.  Every such
    # length is odd, so WindowedStreamingRestorer refuses it as odd first.
    m0 = VoiceFixer(vocoder_config=dataclasses.replace(VocoderConfig(), tail_pad_base=0)).load_state_dict(state).eval().to("cuda:0")
    W0 = 441 * 9 + 440
    einval([(0, 0, OPEN)], good_e, W=W0, synthesis=torch.zeros(W0, device="cuda"), m=m0._engine())
    m0._engine().close()
    eng.check_errors()
    again = eng.restore_windows(ring, WINDOWS, W_CALL, syn, acc0.clone(), EMITS)
    eng.check_errors()
    assert torch.equal(again, ref)


def test_plans_stay_flat_while_the_window_count_varies(model):
    """After the power-of-two shapes are warm, a session whose window count changes every step builds and evicts no plan
    (every window of this geometry is under 64 frames: one bucket)."""
    W, hop = 8820, 2940
    eng = model._engine()
    ring = _ring(8)
    for rows in (1, 2, 4, 8, 16, 32, 64):
        eng.restore_chunks(ring, [(r % 3, W, 0, 0, 100 * r, OPEN) for r in range(rows)])
    before = eng.plan_cache_info()
    rng = random.Random(7)
    n_streams = 16
    sr = WindowedStreamingRestorer(model, W, hop, max_streams=n_streams)
    ids = [sr.open() for _ in range(n_streams)]
    counts = []
    for step in range(24):
        active = rng.sample(ids, rng.randrange(1, n_streams + 1))
        for sid in active:
            k = rng.choice([hop, 2 * hop, W])
            sr.push(sid, _signal(k, 1000 * step + sid))
        n_windows = sum(len(sr._windows(st)) for st in sr._streams.values())
        sr.step()
        counts.append(n_windows)
    eng.check_errors()
    after = eng.plan_cache_info()
    print("windows per step", counts, "plans", before, "->", after)
    assert len(set(counts)) >= 6
    assert after["plans"] == before["plans"] and after["evicted"] == before["evicted"]
