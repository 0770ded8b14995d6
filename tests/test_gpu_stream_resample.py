"""Live streams at their own sample rate (vf_resample_rings): StreamingResampler's concatenated outputs are the whole-signal
resample_to / resample bit for bit at the same length, however the pushes and steps fall and whichever streams share them;
the restorers' 8, 16 and 48 kHz streams are BoxcarOverlapAdd / WindowedOverlapAdd of the resampled whole stream bit for bit,
and their 44.1 kHz streams are untouched by the other-rate streams beside them; one launch per filter family per step; bad
calls fail with VF_EINVAL and leave the context usable."""
import ctypes
import random

import pytest
import torch

from oracle import vf_oracle as O
from voicefixer_main_b200 import _lib as VL
from voicefixer_main_b200.edges import resample_to, stream_filter
from voicefixer_main_b200.longform import BoxcarOverlapAdd, RestoreNet, WindowedOverlapAdd
from voicefixer_main_b200.streaming import StreamingResampler, StreamingRestorer, WindowedStreamingRestorer

pytestmark = pytest.mark.gpu

PAIRS = [(r, 44100) for r in (8000, 11025, 16000, 22050, 24000, 32000, 48000)] + [(44100, 16000), (44100, 48000)]
RES = [None, "kaiser_best", "kaiser_fast"]


def _signal(n, seed):
    return O.synth_clips(1, n, seed=seed)[0] if n >= 2 else torch.randn(n, generator=torch.Generator().manual_seed(seed))


@pytest.fixture(scope="module")
def model(state):
    from voicefixer_main_b200 import VoiceFixer
    m = VoiceFixer().load_state_dict(state).eval().to("cuda:0")
    yield m
    m._engine().check_errors()


@pytest.fixture(scope="module")
def ssr_model():
    from voicefixer_main_b200 import SSR_UNet
    from voicefixer_main_b200.weights import make_ssr_state
    m = SSR_UNet().load_state_dict(make_ssr_state(1234)).eval().to("cuda:0")
    yield m
    m._engine().check_errors()


def _whole(eng, x, rate, rate_out, res_type):
    return resample_to(eng, x.cuda()[None], rate, rate_out, res_type)[0]


def _run(sr, specs, seed, pattern="random", limit=None):
    """Streams (rate, x) through one streaming object: staggered opens, pushes by `pattern` ("ones": one sample, "long":
    longer than any filter span, "random": 0 .. limit), host and device tensors alternately, steps after every push
    ("every"), only once all are closed ("close") or at random.  -> the concatenated outputs per stream."""
    rng = random.Random(seed)
    opens = sorted(rng.randrange(0, 3) for _ in specs)
    sids, pos, outs = {}, {}, {}
    step = 0
    while len(sids) < len(specs) or sr._streams:
        for i, t in enumerate(opens):
            if t == step and i not in sids:
                sids[i], pos[i] = sr.open(specs[i][0]), 0
        for i, sid in sids.items():
            rate, x = specs[i]
            if pos[i] is None or (pattern == "random" and rng.random() < 0.2):
                continue
            cap = limit(rate) if limit else 1 << 30
            k = {"ones": 1, "long": rng.randrange(600, 3000)}.get(pattern, rng.randrange(0, cap + 1))
            k = min(k, cap, x.numel() - pos[i])
            piece = x[pos[i]:pos[i] + k]
            sr.push(sid, piece.cuda() if step % 2 else piece)
            pos[i] += k
            if pos[i] == x.numel():
                sr.close(sid)
                pos[i] = None
        all_in = all(p is None for p in pos.values()) and len(sids) == len(specs)
        if pattern != "close" or all_in:
            for sid, o in sr.step().items():
                outs.setdefault(sid, []).append(o.clone())
        step += 1
    empty = torch.zeros(0, device=sr.engine.device)
    return [torch.cat(outs.get(sids[i], [empty])) for i in range(len(specs))]


def _check_resampler(eng, specs, rate_out, res_type, seed, pattern="random", max_streams=None):
    rs = StreamingResampler(eng, rate_out=rate_out, res_type=res_type, max_streams=max_streams or len(specs))
    got = _run(rs, specs, seed, pattern, limit=lambda r: rs.max_input_rate)
    eng.check_errors()
    for (rate, x), g in zip(specs, got):
        want = _whole(eng, x, rate, rate_out, res_type)
        assert g.shape == want.shape, (rate, x.numel(), pattern)
        assert torch.equal(g, want), (rate, x.numel(), pattern, float((g - want).abs().max()))
    return got


@pytest.mark.parametrize("res_type", RES)
@pytest.mark.parametrize("rate,rate_out", PAIRS)
def test_resampler_equals_the_whole_signal_under_every_split(model, rate, rate_out, res_type):
    eng = model._engine()
    x = _signal(1500, rate)
    for pattern in ("ones", "long", "every", "close", "random"):
        _check_resampler(eng, [(rate, x), (rate, _signal(5000, rate + 1))], rate_out, res_type, seed=rate, pattern=pattern)


@pytest.mark.parametrize("res_type", RES)
def test_32_streams_of_mixed_rates_share_each_step(model, res_type):
    rates = [8000, 11025, 16000, 22050, 24000, 32000, 48000, 44100]
    rng = random.Random(3)
    specs = [(rates[i % len(rates)], _signal(rng.randrange(2000, 9000), 70 + i)) for i in range(32)]
    _check_resampler(model._engine(), specs, 44100, res_type, seed=11)


@pytest.mark.parametrize("res_type", RES)
@pytest.mark.parametrize("rate,rate_out", [(16000, 44100), (48000, 44100), (44100, 16000)])
def test_streams_of_1_to_40_samples(model, rate, rate_out, res_type):
    ratio = float(rate_out) / rate
    specs = [(rate, _signal(n, 300 + n)) for n in range(1, 41) if res_type is None or int(n * ratio) >= 1]
    _check_resampler(model._engine(), specs, rate_out, res_type, seed=5, pattern="ones")
    _check_resampler(model._engine(), specs, rate_out, res_type, seed=6, pattern="close")


def test_a_stream_alone_and_among_31_others(model):
    eng = model._engine()
    x = _signal(20000, 9)
    for res_type in RES:
        alone = _check_resampler(eng, [(16000, x)], 44100, res_type, seed=1)[0]
        others = [(random.Random(i).choice([8000, 16000, 48000, 44100]), _signal(random.Random(i).randrange(100, 20000), 900 + i))
                  for i in range(31)]
        crowd = _check_resampler(eng, [(16000, x)] + others, 44100, res_type, seed=2)
        assert torch.equal(alone, crowd[0])


# ---- the restorers
W, M = 8820, 2205                 # chunked: 0.2 s windows with a quarter-window margin
WW, HOP = 8820, 2940              # windowed
# (rate, samples): every length leaves a last chunk restore() accepts at both geometries
MIXED = [(8000, 5000), (16000, 11000), (48000, 30000), (44100, 26561), (44100, 9000)]


def _specs(lengths, seed):
    return [(rate, _signal(n, seed + i)) for i, (rate, n) in enumerate(lengths)]


def _restorer_session(sr, specs, seed):
    return _run(sr, specs, seed, limit=sr.max_push)


def _offline_chunked(model, x44, unify_energy=False, W=W, M=M):
    return BoxcarOverlapAdd(RestoreNet(model, unify_energy=unify_energy), 1, W, M)(x44[None, None])[0, 0]


def _offline_windowed(model, x44, unify_energy=False):
    ola = WindowedOverlapAdd(RestoreNet(model, unify_energy), 1, WW, HOP, window="hanning", reorder_chunks=False)
    return ola(x44[None, None])[0, 0]


def _check_restorer(model, make, offline, specs, seed, res_type=None, unify_energy=False):
    eng = model._engine()
    got = _restorer_session(make(res_type), specs, seed)
    eng.check_errors()
    for (rate, x), g in zip(specs, got):
        want = offline(model, _whole(eng, x, rate, 44100, res_type), unify_energy)
        assert g.shape == want.shape, (rate, x.numel())
        assert torch.equal(g, want), (rate, x.numel(), float((g - want).abs().max()))
    return got


@pytest.fixture(params=[1, 3], ids=["terms1", "terms3"])
def voc_terms(model, request):
    e = model._engine()
    e.set_option("vocoder_terms", request.param)
    yield model
    e.set_option("vocoder_terms", 1)


@pytest.mark.parametrize("unify_energy", [False, True])
def test_streaming_restorer_mixed_rates(voc_terms, unify_energy):
    specs = _specs(MIXED, 10)
    make = lambda res: StreamingRestorer(voc_terms, W, M, max_streams=len(specs), unify_energy=unify_energy, res_type=res)
    got = _check_restorer(voc_terms, make, _offline_chunked, specs, seed=21, unify_energy=unify_energy)
    # the 44.1 kHz streams alone give the same bits
    at44 = [i for i, (r, _) in enumerate(specs) if r == 44100]
    alone = _restorer_session(make(None), [specs[i] for i in at44], seed=22)
    for i, a in zip(at44, alone):
        assert torch.equal(a, got[i])


@pytest.mark.parametrize("unify_energy", [False, True])
def test_windowed_streaming_restorer_mixed_rates(voc_terms, unify_energy):
    specs = _specs(MIXED, 30)
    make = lambda res: WindowedStreamingRestorer(voc_terms, WW, HOP, max_streams=len(specs), unify_energy=unify_energy,
                                                 res_type=res)
    got = _check_restorer(voc_terms, make, _offline_windowed, specs, seed=31, unify_energy=unify_energy)
    at44 = [i for i, (r, _) in enumerate(specs) if r == 44100]
    alone = _restorer_session(make(None), [specs[i] for i in at44], seed=32)
    for i, a in zip(at44, alone):
        assert torch.equal(a, got[i])


def test_ssr_restorers_mixed_rates(ssr_model):
    specs = _specs(MIXED[:4], 50)
    _check_restorer(ssr_model, lambda res: StreamingRestorer(ssr_model, W, M, max_streams=4, res_type=res),
                    _offline_chunked, specs, seed=51)
    _check_restorer(ssr_model, lambda res: WindowedStreamingRestorer(ssr_model, WW, HOP, max_streams=4, res_type=res),
                    _offline_windowed, specs, seed=52)


def test_kaiser_best_once_per_restorer_class(model):
    specs = _specs(MIXED[:4], 60)
    _check_restorer(model, lambda res: StreamingRestorer(model, W, M, max_streams=4, res_type=res), _offline_chunked, specs,
                    seed=61, res_type="kaiser_best")
    _check_restorer(model, lambda res: WindowedStreamingRestorer(model, WW, HOP, max_streams=4, res_type=res),
                    _offline_windowed, specs, seed=62, res_type="kaiser_best")


def test_a_step_adds_one_launch_per_filter_family(model):
    """Per vf_launch_count, a step with resampled streams is the same step's restore launches plus one."""
    eng = model._engine()
    for cls, geom, call in ((StreamingRestorer, (W, M), "restore_chunks"),
                            (WindowedStreamingRestorer, (WW, HOP), "restore_windows")):
        sr = cls(model, *geom, max_streams=3)
        inner = getattr(eng, call)
        counted = []

        def restore(*a, **k):
            before = eng.launch_count()
            out = inner(*a, **k)
            counted.append(eng.launch_count() - before)
            return out
        setattr(eng, call, restore)
        try:
            a, b, c = sr.open(16000), sr.open(8000), sr.open(44100)
            for step in range(6):
                counted.clear()
                for sid, rate in ((a, 16000), (b, 8000), (c, 44100)):
                    sr.push(sid, _signal(sr.max_push(rate) // 2, 100 * step + sid))
                before = eng.launch_count()
                sr.step()
                total = eng.launch_count() - before
                assert total == sum(counted) + 1, (cls.__name__, step, total, counted)
            for sid in (a, b):                         # only the 44.1 kHz stream left: no resample launch
                sr.close(sid)
            sr.step()
            counted.clear()
            sr.push(c, _signal(sr.max_push(), 7))
            before = eng.launch_count()
            sr.step()
            assert eng.launch_count() - before == sum(counted)
        finally:
            delattr(eng, call)
    eng.check_errors()


def _rows(spec):
    table = (VL.VfResampleRow * len(spec))()
    for t, kw in zip(table, spec):
        for k, v in kw.items():
            setattr(t, k, v)
    return table


def test_bad_calls_fail_with_einval_and_leave_the_context_usable(model):
    eng = model._engine()
    ring = (torch.randn(3, 4000, generator=torch.Generator().manual_seed(4)) * 0.3).cuda()
    out = torch.zeros(2, 3000, device="cuda")
    poly = stream_filter(eng, 16000, 44100)
    sinc = stream_filter(eng, 16000, 44100, "kaiser_fast")
    P = dict(family=VL.VF_RESAMPLE_POLY, up=poly.up, down=poly.down, taps=poly.taps.data_ptr())
    S = dict(family=VL.VF_RESAMPLE_SINC, table=sinc.table.data_ptr(), nwin=sinc.table.shape[0], ratio=sinc.ratio,
             num_table=sinc.num_table)
    OPEN = VL.VF_RESAMPLE_OPEN
    good = [dict(stream=0, m0=0, m1=2000, n=OPEN, avail=1000, out_stream=0, **P),
            dict(stream=2, m0=9000, m1=9500, n=OPEN, avail=4000, out_stream=1, **S)]

    def call(spec):
        with torch.cuda.device(eng.device):
            return eng.lib.vf_resample_rings(eng.ctx, ctypes.c_void_p(ring.data_ptr()), 3, 4000, _rows(spec), len(spec),
                                             ctypes.c_void_p(out.data_ptr()), 2, 3000,
                                             ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert call(good) == VL.VF_OK
    want = out.clone()
    bad = [dict(good[0], stream=3), dict(good[0], stream=-1),                 # stream out of range
           dict(good[0], m0=-1), dict(good[0], m0=10, m1=9),                  # m0 < 0, m1 < m0
           dict(good[0], m1=2770),                                            # reads input 1000: not pushed yet
           dict(good[1], m1=11100),                                           # the sinc window past avail
           dict(good[0], m0=0, avail=4100),                                   # input 0 is no longer in the ring
           dict(good[1], m0=4000, m1=4100, avail=5500),                       # the sinc left wing below the ring
           dict(good[0], n=1000, m1=2758),                                    # past ceil(n up / down) of a closed row
           dict(good[0], n=999, avail=1000),                                  # more inputs than the count
           dict(good[0], out_stream=2), dict(good[0], m1=3001, avail=1200),   # no such output row; more than out_len
           dict(good[0], family=2),                                           # unknown family
           dict(good[0], taps=None), dict(good[0], table=sinc.table.data_ptr()),   # a poly row with no taps / a table
           dict(good[1], table=None), dict(good[1], taps=poly.taps.data_ptr()),    # a sinc row with no table / taps
           dict(good[1], num_table=0), dict(good[1], nwin=sinc.num_table), dict(good[1], ratio=0.0)]
    for b in bad:
        out.fill_(7.0)
        assert call([good[0], b]) == VL.VF_EINVAL, b
        assert bool((out == 7.0).all()), b                                    # nothing was queued
    assert call(good) == VL.VF_OK
    eng.check_errors()
    assert torch.equal(out[0, :2000], want[0, :2000]) and torch.equal(out[1, 0:500], want[1, 0:500])


def test_overflowing_push_and_bad_arguments(model):
    for sr in (StreamingRestorer(model, W, M, max_streams=2), WindowedStreamingRestorer(model, WW, HOP, max_streams=2)):
        sid = sr.open(16000)
        st = sr._streams[sid]
        sr.push(sid, _signal(sr.max_push(16000), 1))
        ring, in_ring, before = sr.ring.clone(), sr.in_ring.clone(), (st.pushed, st.src_pushed)
        with pytest.raises(OverflowError, match=f"stream {sid}"):
            sr.push(sid, _signal(sr.in_len, 2))
        assert (st.pushed, st.src_pushed) == before
        assert torch.equal(ring, sr.ring) and torch.equal(in_ring, sr.in_ring)
        for rate in (0, 48001):
            with pytest.raises(ValueError, match="rate"):
                sr.open(rate)
    with pytest.raises(ValueError, match="res_type"):
        StreamingRestorer(model, W, M, res_type="soxr_hq")
    rs = StreamingResampler(model, max_streams=1, max_input_rate=16000)
    a = rs.open(16000)
    rs.push(a, _signal(16000, 3))
    with pytest.raises(OverflowError, match=f"stream {a}"):
        rs.push(a, _signal(rs.ring_len, 4))
    model._engine().check_errors()


def test_nan_sample_in_a_16_khz_stream(model):
    """The contract of test_gpu_nonfinite_inputs.py on a 16 kHz stream: the restoring step raises VF_EDEVICE or returns
    only finite samples, and a clean run afterwards gives the fresh context's bits."""
    from test_gpu_nonfinite_inputs import check_entry
    eng = model._engine()
    x = _signal(11000, 77)

    def one_stream(v):
        sr = StreamingRestorer(model, W, M, max_streams=1)
        a = sr.open(16000)
        outs = []
        for i in range(0, v.numel(), 4000):
            sr.push(a, v[i:i + 4000])
            outs += [o.clone() for o in sr.step().values()]
        sr.close(a)
        outs += [o.clone() for o in sr.step().values()]
        return [torch.cat(outs)]
    bad = x.clone()
    bad[5000] = float("nan")
    check_entry(eng, "StreamingRestorer at 16 kHz", one_stream, x, [("one NaN sample", bad)])
