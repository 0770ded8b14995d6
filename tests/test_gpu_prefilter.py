"""vf_remove_higher_frequency_varlen, the pip package's mode-1 pre-filter, on the GPU against the float64 oracle
(oracle/prefilter.py): cutoffs, output lengths and samples for a mixed call of seeded signals, row bits independent of
batch, slot and sub-batch, the non-finite flag, the VoiceFixer methods, and the mode-1 recipe of restore_inmem."""
import numpy as np
import pytest
import scipy.signal
import torch

from oracle import lowpass as LP
from oracle import prefilter as P
from oracle import vf_oracle as O
from voicefixer_main_b200 import _lib as VL

pytestmark = pytest.mark.gpu

SR = 44100
LENGTHS = [100, 511, 512, 1000, 1025, 44100 + 7, 1323000, 2646000]
KINDS = ["lp2k", "lp4k", "lp8k", "lp16k", "sweep", "speech", "silence"]


def signal(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind.startswith("lp"):
        x = LP.lowpass(0.3 * rng.standard_normal(n), int(kind[2:-1]) * 1000, SR)
    elif kind == "sweep":
        t = np.arange(n) / SR
        x = 0.5 * scipy.signal.chirp(t, 50, max(t[-1], 1 / SR), 20000, method="logarithmic")
    elif kind == "speech":
        x = O.synth_clips(1, n, seed=seed)[0].numpy()
    else:
        x = np.zeros(n)
    return np.asarray(x, np.float32)


def rows():
    """Two passes over LENGTHS, each length with a different signal kind: 16 rows, every kind at several lengths."""
    out = []
    for p in range(2):
        for i, n in enumerate(LENGTHS):
            kind = KINDS[(i + 3 * p) % len(KINDS)]
            out.append((f"{kind}/{n}", signal(kind, n, 100 * p + i)))
    return out


@pytest.fixture(scope="module")
def case():
    rs = rows()
    want = [P.remove_higher_frequency(x) for _, x in rs]
    return rs, want


@pytest.fixture(scope="module")
def eng():
    from voicefixer_main_b200.model import Engine
    e = Engine("cuda:0")
    yield e
    e.close()


def run(eng, xs, ratio=0.95):
    """-> (list of float32 numpy outputs, numpy cutoffs) of one call on the clips xs."""
    packed = torch.from_numpy(np.concatenate(xs)).cuda()
    out, lengths, cutoff = eng.remove_higher_frequency_varlen(packed, [len(x) for x in xs], ratio)
    eng.check_errors()
    return [o.cpu().numpy() for o in torch.split(out, lengths)], cutoff.cpu().numpy()


def test_mixed_call_against_float64_oracle(eng, case):
    rs, want = case
    got, cut = run(eng, [x for _, x in rs])
    for (name, x), g, c, (y, c_ref, margin) in zip(rs, got, cut, want):
        assert c == c_ref, (name, int(c), c_ref)
        assert g.shape == (512 * (len(x) // 512),), (name, g.shape)
        err = np.abs(g.astype(np.float64) - y)
        assert _within_tolerance(g, y, x), (name, float(err.max()))
        print(f"{name}: cutoff {int(c)}, margin {margin:.3e}, largest error {err.max() if err.size else 0:.3e}")


def test_oracle_margins(case):
    """Every row's cutoff is decided by a margin far above float64 rounding (silence: all energies exactly 0)."""
    rs, want = case
    for (name, x), (_, c, margin) in zip(rs, want):
        threshold = _features(x).sum() * 0.95
        assert (threshold == 0 and c == 0) or margin > 1e-9 * threshold, (name, c, margin, threshold)


def _features(x):
    X = np.fft.rfft(P._frames(x) * P._window(), axis=1)
    return np.maximum(np.log10(np.hypot(X.real, X.imag) + P.EPS), 0)


def _within_tolerance(g, y, x):
    """1 float32 ulp of the oracle, plus the float64 FFT's rounding (about 2^-52 x 4500) of the clip's scale."""
    tol = np.spacing(np.abs(y).astype(np.float32)).astype(np.float64) + 1e-12 * max(np.abs(x).max(), 1e-30)
    return (np.abs(g.astype(np.float64) - y) <= tol).all()


@pytest.mark.parametrize("ratio", [0.5, 1.0])
def test_other_ratios_against_float64_oracle(eng, case, ratio):
    """The ratio reaches the scan: the mixed call at 0.5 and at 1.0 gives the oracle's cutoffs and samples.  At 0.5 every
    row's margin is far above rounding.  At 1.0 the last running sum meets the threshold exactly (trailing bins of zero
    energy add exact zeros), so the cutoff is decided by which frames' features are positive: every positive feature is
    checked to be far from 0, so |X| + 1e-8 is never within rounding of 1."""
    rs, _ = case
    got, cut = run(eng, [x for _, x in rs], ratio)
    for (name, x), g, c in zip(rs, got, cut):
        y, c_ref, margin = P.remove_higher_frequency(x, ratio)
        f = _features(x)
        threshold = f.sum() * ratio
        if ratio < 1:
            assert (threshold == 0 and c_ref == 0) or margin > 1e-9 * threshold, (name, ratio, margin, threshold)
        else:
            assert (f[f > 0] > 1e-9).all(), (name, float(f[f > 0].min()))
        assert c == c_ref, (name, ratio, int(c), c_ref)
        assert _within_tolerance(g, y, x), (name, ratio)


def test_small_kept_bins_are_rescaled(eng):
    """The kept bins are scaled by |X| / (|X| + 1e-8), which matters where |X| is small: loud wideband noise then a tail at
    1e-7 (its bins near 3e-6, a change of about 0.3 %).  The GPU matches the oracle, and in the tail differs by thousands
    of float32 ulps from the oracle without the scaling (EPS = 0 at the same cutoff)."""
    rng = np.random.default_rng(5)
    x = np.concatenate([0.5 * rng.standard_normal(3 * SR), 1e-7 * rng.standard_normal(2 * SR)]).astype(np.float32)
    y, c_ref, margin = P.remove_higher_frequency(x)
    assert margin > 1e-9 * _features(x).sum() * 0.95
    (g,), (c,) = run(eng, [x])
    assert c == c_ref and 0 < c < P.BINS, (int(c), c_ref)
    assert _within_tolerance(g, y, x)
    unscaled, _, _ = P.remove_higher_frequency(x, eps=0.0, cutoff=c_ref)
    tail = slice(3 * SR + P.N_FFT, g.shape[0])               # samples whose frames hold only the tail
    ulps = np.abs(g[tail].astype(np.float64) - unscaled[tail]) / np.spacing(np.abs(g[tail]))
    print(f"tail: median {np.median(ulps):.0f} float32 ulps from the unscaled output")
    assert np.median(ulps) > 1000


def test_row_bits_do_not_depend_on_batch_slot_or_sub_batch(eng, case):
    rs, _ = case
    xs = [x for _, x in rs]
    mixed, mixed_cut = run(eng, xs)
    rev, rev_cut = run(eng, xs[::-1])
    # 260 one-frame rows first: the first sub-batch ends at 256 rows; three 60 s rows first: the frame cap splits the rest
    tiny = [signal("lp8k", 100, 900 + i) for i in range(260)]
    by_rows, by_rows_cut = run(eng, tiny + xs)
    long = [signal("speech", 2646000, 950 + i) for i in range(3)]
    by_frames, by_frames_cut = run(eng, long + xs)
    for i, x in enumerate(xs):
        alone, alone_cut = run(eng, [x])
        for what, y, c in (("mixed", mixed[i], mixed_cut[i]), ("reversed", rev[-1 - i], rev_cut[-1 - i]),
                           ("after 260 rows", by_rows[260 + i], by_rows_cut[260 + i]),
                           ("after three 60 s rows", by_frames[3 + i], by_frames_cut[3 + i])):
            assert c == alone_cut[0] and np.array_equal(y.view(np.int32), alone[0].view(np.int32)), (rs[i][0], what)


def test_nonfinite_rows_raise_and_the_context_recovers(eng):
    clean = [signal("speech", 30000, 5), signal("lp4k", 20000, 6)]
    want, want_cut = run(eng, clean)
    for v in (float("nan"), float("inf")):
        bad = [c.copy() for c in clean]
        bad[1][12345] = v
        packed = torch.from_numpy(np.concatenate(bad)).cuda()
        eng.remove_higher_frequency_varlen(packed, [len(b) for b in bad], 0.95)
        with pytest.raises(VL.EngineError) as e:
            eng.check_errors()
        assert e.value.code == VL.VF_EDEVICE, (v, e.value)
    got, got_cut = run(eng, clean)
    assert np.array_equal(got_cut, want_cut)
    for g, w in zip(got, want):
        assert np.array_equal(g.view(np.int32), w.view(np.int32))


def test_argument_checks_name_the_row(eng):
    x = torch.zeros(3000, device="cuda")
    for lengths, ratio, what in (([1000, 2000], 0.0, "ratio"), ([1000, 2000], 1.0000001, "ratio"),
                                 ([1000, 0, 2000], 0.95, "row 1")):
        with pytest.raises(VL.EngineError) as e:
            eng.remove_higher_frequency_varlen(x, lengths, ratio)
        assert e.value.code == VL.VF_EINVAL and what in str(e.value), (lengths, ratio, e.value)


@pytest.fixture(scope="module")
def model():
    from voicefixer_main_b200 import VoiceFixer
    from voicefixer_main_b200.weights import make_state
    m = VoiceFixer().load_state_dict(make_state(1234)).eval().to("cuda:0")
    yield m
    m._eng.close()


def test_voicefixer_methods(model):
    x = signal("speech", 3 * SR + 17, 41)
    one = model.remove_higher_frequency(x)
    outs, cut = model.remove_higher_frequency_batch([signal("lp2k", 5000, 42), torch.from_numpy(x).cuda(), x[:300]])
    assert isinstance(one, np.ndarray) and one.dtype == np.float32 and one.shape == (512 * (len(x) // 512),)
    assert np.array_equal(one.view(np.int32), outs[1].cpu().numpy().view(np.int32))
    assert outs[2].numel() == 0 and cut.shape == (3,) and cut.dtype == torch.int32
    assert all(o.is_cuda and o.dtype == torch.float32 for o in outs)


def test_mode1_recipe(model):
    """restore_inmem(wav, mode=1) as the package runs it: 30 s segments, each pre-filtered, restored and trimmed to the
    filtered length.  One pre-filter call for all segments, one restore_batch call for all filtered segments."""
    seg = 30 * SR
    wav = O.synth_clips(1, 70 * SR, seed=77)[0].numpy()
    segments = [wav[s:s + seg] for s in range(0, len(wav), seg)]
    filtered, _ = model.remove_higher_frequency_batch(segments)
    restored = model.restore_batch(filtered, unify_energy=True)
    out = torch.cat(restored)
    assert out.numel() == 2 * 1322496 + 512 * ((10 * SR) // 512)
    for f, r in zip(filtered, restored):
        alone = model.restore(f[None], unify_energy=True)[0]
        assert torch.equal(alone, r)
    model._engine().check_errors()
