"""The host bookkeeping of resampling live streams (stream_resample.py), CPU only: the finality rule against brute force over
the whole-signal kernels' windows, the lengths at close, a float64 streaming restatement driven by StreamingResampler's own
bookkeeping through a fake engine, and the push capacity of the restorers' other-rate streams."""
import random
from fractions import Fraction

import numpy as np
import pytest
import scipy.signal
import torch

from oracle import resampy as R
from voicefixer_main_b200 import _lib as VL
from voicefixer_main_b200.edges import RES_TYPES, design_filter_f64
from voicefixer_main_b200.stream_resample import StreamResampling
from voicefixer_main_b200.streaming import StreamingResampler, StreamingRestorer, WindowedStreamingRestorer

PAIRS = [(r, 44100) for r in (8000, 11025, 16000, 22050, 24000, 32000, 48000)] + [(44100, 16000), (44100, 48000)]
RES = [None, "kaiser_best", "kaiser_fast"]
BIG = 10 ** 12                    # an n past every window: the unclamped window


def kernel_windows(rate, rate_out, res_type, m, n):
    """(first, last, in_range) of outputs m (int64 array) of an n-input signal, restated from the kernels (edges.cu
    resample_poly_kernel, sinc.cu / oracle/resampy.py's loop bounds); in_range: m is an output the kernel computes (poly:
    m < ceil(n up / down); sinc: m < int(n ratio), not a fix_length zero)."""
    if res_type is None:
        fr = Fraction(rate_out, rate)
        up, down = fr.numerator, fr.denominator
        half = 10 * max(up, down)
        c = m * down
        first = np.where(c - half < 0, 0, (c - half + up - 1) // up)
        return first, np.minimum((c + half) // up, n - 1), m < -(-(n * up) // down)
    num_zeros, precision = RES_TYPES[res_type][:2]
    num_table = 2 ** precision
    nwin = num_table * num_zeros + 1
    ratio = float(rate_out) / rate
    scale = min(1.0, ratio)
    step = int(scale * num_table)
    t_out = m / ratio
    nt = t_out.astype(np.int64)
    frac = scale * (t_out - nt)
    kl = np.minimum(nt + 1, (nwin - (frac * num_table).astype(np.int64)) // step)
    kr = np.minimum(n - nt - 1, (nwin - ((scale - frac) * num_table).astype(np.int64)) // step)
    first = np.where(kl > 0, nt - kl + 1, nt + 1)
    last = np.where(kr > 0, nt + kr, np.where(kl > 0, nt, nt - 1))
    return first, last, m < int(n * ratio)


def reach(g):
    return (g.half // g.up + 2) if g.poly else g.k_max + 2


@pytest.mark.parametrize("res_type", RES)
@pytest.mark.parametrize("rate,rate_out", PAIRS)
def test_finality_rule_against_brute_force(rate, rate_out, res_type):
    """For every p up to 300 and every m: final exactly when, for every n >= p, m is an output the kernel computes, its
    window is the same as for any longer signal and ends before p.  final_count(p) is the first m that is not final."""
    g = StreamResampling(rate, rate_out, res_type)
    P = 300
    m = np.arange(int(np.ceil((P + reach(g) + 2) * rate_out / rate)) + 8, dtype=np.int64)
    f_inf, l_inf, _ = kernel_windows(rate, rate_out, res_type, m, BIG)
    for p in range(0, P + 1):
        brute = np.ones(m.shape, bool)
        for n in list(range(max(p, 1), p + reach(g) + 2)) + [BIG]:
            f, l, ok = kernel_windows(rate, rate_out, res_type, m, n)
            brute &= ok & (f == f_inf) & (l == l_inf) & (l <= p - 1)
        if p == 0:
            brute[:] = False
        rule = np.array([g.is_final(int(x), p) for x in m])
        assert np.array_equal(rule, brute), (p, np.flatnonzero(rule != brute)[:5])
        first_not = int(np.flatnonzero(~brute)[0])
        assert g.final_count(p) == first_not, p
        # what the ring must keep, and the bounds the restorers size their rings with
        M = first_not
        assert g.keep_from(M) <= max(0, int(f_inf[M:].min())), p
        assert p - g.keep_from(M) <= g.history, p
        if p:
            assert g.due(p) - M <= g.tail, p


@pytest.mark.parametrize("res_type", RES)
@pytest.mark.parametrize("rate,rate_out", PAIRS)
def test_lengths_at_close(rate, rate_out, res_type):
    g = StreamResampling(rate, rate_out, res_type)
    for n in list(range(1, 60)) + [441, 4410, 12345, 44100 * 3 + 7]:
        if res_type is None:
            fr = Fraction(rate_out, rate)
            want = scipy.signal.resample_poly(np.zeros(n), fr.numerator, fr.denominator).shape[0]
        elif int(n * (float(rate_out) / rate)) == 0:
            with pytest.raises(ValueError, match="too small"):
                g.out_len(n)
            continue
        else:
            want = R.out_len(n, rate, rate_out)
        assert g.out_len(n) == g.due(n) == want, n
    assert g.out_len(0) == 0


class F64Engine:
    """vf_resample_rings restated in float64 over the same table: each row's outputs from the ring, every read checked to
    lie in what the ring holds; the values are recorded per (ring slot, step) at float64."""
    device = torch.device("cpu")

    def __init__(self):
        self.records = {}

    def resample_rings(self, in_ring, rows, out):
        L = in_ring.shape[1]
        for s, f, m0, m1, n, avail, out_stream, out_offset in rows:
            assert 0 <= m0 < m1 and out_stream == -1 and avail >= 0
            ys = []
            for m in range(m0, m1):
                ys.append(f(m, n, lambda i: _read(in_ring, s, L, i, avail)))
            y = np.array(ys)
            out[out_offset:out_offset + m1 - m0] = torch.from_numpy(y.astype(np.float32))
            self.records[s] = y
        return out


def _read(ring, s, L, i, avail):
    assert avail - L <= i < avail, (i, avail, L)
    return float(ring[s, i % L])


class PolyF64:
    """resample_poly's output m in float64 with resample_poly's own float64 taps."""

    def __init__(self, up, down):
        self.up, self.down, self.half = up, down, 10 * max(up, down)
        self.h = design_filter_f64(up, down)

    def __call__(self, m, n, x):
        c = m * self.down
        lo = max(0, -(-(c - self.half) // self.up))
        hi = min((c + self.half) // self.up, n - 1)
        return sum(self.h[c - i * self.up + self.half] * x(i) for i in range(lo, hi + 1))


class SincF64:
    """resampy's output t in float64 (oracle/resampy.py's loop, accumulated in float64)."""

    def __init__(self, res_type, ratio):
        self.win, self.delta, self.num_table, self.scale = R.tables(res_type, ratio)
        self.ratio, self.step = ratio, int(self.scale * self.num_table)
        self.nwin = self.win.shape[0]

    def __call__(self, t, n, x):
        if n != VL.VF_RESAMPLE_OPEN and t >= int(n * self.ratio):
            return 0.0
        tr = t / self.ratio
        nt = int(tr)
        frac = self.scale * (tr - nt)
        y = 0.0
        for f, count, src in ((frac, nt + 1, lambda i: nt - i), (self.scale - frac, n - nt - 1, lambda k: nt + 1 + k)):
            index_frac = f * self.num_table
            off = int(index_frac)
            eta = index_frac - off
            for i in range(min(count, (self.nwin - off) // self.step)):
                y += (self.win[off + i * self.step] + eta * self.delta[off + i * self.step]) * x(src(i))
        return y


class F64Resampler(StreamingResampler):
    """StreamingResampler whose rows carry the float64 restatements instead of device filters."""

    def step(self):
        import voicefixer_main_b200.streaming as S
        keep = S.stream_filter
        S.stream_filter = lambda eng, r_in, r_out, res: (PolyF64(*_reduced(r_in, r_out)) if res is None
                                                         else SincF64(res, float(r_out) / r_in))
        try:
            return super().step()
        finally:
            S.stream_filter = keep


def _reduced(r_in, r_out):
    fr = Fraction(r_out, r_in)
    return fr.numerator, fr.denominator


@pytest.mark.parametrize("rate,rate_out,res_type", [(16000, 44100, None), (44100, 16000, None), (48000, 44100, None),
                                                    (8000, 44100, "kaiser_fast"), (44100, 16000, "kaiser_fast")])
def test_f64_streaming_restatement_matches_the_whole_signal(rate, rate_out, res_type):
    """Streams pushed in seeded random splits with random skipped steps: the float64 outputs the bookkeeping asks for,
    concatenated, are resample_poly of the whole signal within 1e-9 of max|x|; for a sinc res_type, the same float64 loop
    over the whole signal at librosa's length."""
    rng = random.Random(rate + rate_out)
    eng = F64Engine()
    rs = F64Resampler(eng, rate_out=rate_out, res_type=res_type, max_streams=3, max_input_rate=48000)
    for n in (1, 37, 700, 5000):
        x = np.random.default_rng(n).standard_normal(n).astype(np.float32)
        if res_type is not None and int(n * (float(rate_out) / rate)) == 0:
            continue
        sid = rs.open(rate)
        slot = rs._streams[sid].slot
        got, pos = [], 0
        while True:
            if pos < n and rng.random() < 0.8:
                k = min(n - pos, rng.choice([1, 3, rng.randrange(1, 400)]))
                rs.push(sid, torch.from_numpy(x[pos:pos + k]))
                pos += k
                if pos == n:
                    rs.close(sid)
            if rng.random() < 0.7 or pos == n:
                if sid in rs.step():
                    got.append(eng.records[slot])
            if sid not in rs._streams:
                break
        got = np.concatenate(got)
        if res_type is None:
            want = scipy.signal.resample_poly(x.astype(np.float64), *_reduced(rate, rate_out))
        else:
            f = SincF64(res_type, float(rate_out) / rate)
            want = np.array([f(t, n, lambda i: float(x[i])) for t in range(R.out_len(n, rate, rate_out))])
        assert got.shape == want.shape, n
        assert np.abs(got - want).max() <= 1e-9 * np.abs(x).max(), n


class RingEngine:
    """A restorer's engine for the capacity accounting: resample_rings checks the reads against what the input ring holds
    and the writes against the ring of 44.1 kHz samples still needed; the restore calls return zeros of the kept length."""
    device = torch.device("cpu")

    def __init__(self):
        from voicefixer_main_b200.arch import VocoderConfig
        self.voc_cfg = VocoderConfig()

    def resample_rings(self, in_ring, rows, out):
        for s, f, m0, m1, n, avail, out_stream, _ in rows:
            assert out_stream == s and 0 <= m0 < m1 and m1 - m0 <= out.shape[1]
        return out

    def restore_chunks(self, ring, table, unify_energy=False):
        return torch.zeros(sum(length - cl - cr for _, length, cl, cr, _, _ in table))

    def restore_windows(self, ring, windows, W, synthesis, acc, emits, unify_energy=False):
        return torch.zeros(sum(c for _, _, c in emits))


class RingModel:
    def __init__(self):
        self.e = RingEngine()

    def _engine(self):
        return self.e


def _restorers(res_type):
    return [StreamingRestorer(RingModel(), 8820, 2205, max_streams=3, res_type=res_type),
            WindowedStreamingRestorer(RingModel(), 8820, 2940, max_streams=3, res_type=res_type)]


@pytest.mark.parametrize("res_type", RES)
def test_push_capacity_guarantee_and_overflow(res_type):
    """Pushes of max_push(rate) after every step never raise, in the restore ring (checked by the 44.1 kHz count the
    restorer holds) or the input ring; one larger than the free space raises OverflowError naming the stream, with nothing
    copied and the stream unchanged; a push of max_push(rate) still fits afterwards."""
    for sr in _restorers(res_type):
        for rate in (8000, 16000, 48000, 44100):
            k = sr.max_push(rate)
            assert k > 0
            sid = sr.open(rate)
            st = sr._streams[sid]
            for step in range(12):
                sr.push(sid, torch.ones(k))
                sr.step()
                held44 = st.pushed - sr._keep_from(st)
                assert 0 <= held44 <= sr.ring_len
                if st.rs is not None:
                    assert st.src_pushed - st.rs.keep_from(st.pushed) <= st.rs.history
            ring, in_ring = sr.ring.clone(), sr.in_ring.clone()
            before = (st.pushed, st.src_pushed, st.next)
            with pytest.raises(OverflowError, match=f"stream {sid}"):
                sr.push(sid, torch.full((3 * sr.ring_len,), 2.0))
            assert (st.pushed, st.src_pushed, st.next) == before
            assert torch.equal(ring, sr.ring) and torch.equal(in_ring, sr.in_ring)
            sr.push(sid, torch.ones(k))
            sr.close(sid)
            sr.step()
            assert sid not in sr._streams


def test_bad_rates_and_res_types():
    for sr in _restorers(None):
        for rate in (0, -8000, 48001, 96000, 16000.5):
            with pytest.raises(ValueError, match="rate"):
                sr.open(rate)
    with pytest.raises(ValueError, match="res_type"):
        StreamingRestorer(RingModel(), 8820, 2205, res_type="soxr_hq")
    with pytest.raises(ValueError, match="res_type"):
        WindowedStreamingRestorer(RingModel(), 8820, res_type="linear")
    with pytest.raises(ValueError, match="res_type"):
        StreamingResampler(F64Engine(), res_type="sinc_best")
    rs = StreamingResampler(F64Engine(), rate_out=16000, max_input_rate=44100)
    with pytest.raises(ValueError, match="rate"):
        rs.open(48000)
    with pytest.raises(ValueError, match="rate"):
        rs.open(0)


def test_a_sinc_stream_too_short_to_resample_raises_at_close_and_stays_open():
    rs = StreamingResampler(F64Engine(), rate_out=16000, res_type="kaiser_best", max_input_rate=44100)
    sid = rs.open(44100)
    rs.push(sid, torch.ones(2))                          # int(2 * 16000 / 44100) == 0
    with pytest.raises(ValueError, match="too small"):
        rs.close(sid)
    assert rs._streams[sid].n is None
    rs.push(sid, torch.ones(1))
    rs.close(sid)
