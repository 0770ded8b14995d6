"""Long-form overlap-add with context margins (voicefixer_main_b200/longform.py) - host logic, CPU only.

The mirror is checked (a) against the outputs of the reference's own LambdaOverlapAdd (tools/dsp/overlapadd_boxcar.py:338-534)
with identical toy networks, stored in tests/golden/ref_ola.npz by oracle/make_ref_vectors.py, and (b) through properties
that need no reference: the batched schedule equals the sequential one, and with a margin at least as long as the
network's receptive field the chunking is invisible."""
import os
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from voicefixer_main_b200.longform import BoxcarOverlapAdd, WindowedOverlapAdd

GOLDEN_OLA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_ola.npz")
CASES = [(1000, 256, 32), (1024, 256, 32), (200, 256, 32), (256, 256, 64), (513, 256, 255), (2049, 512, 100)]


class ToyNet(torch.nn.Module):
    """Deterministic non-linear FIR network with the nnet protocol: [B, C, L] -> {"wav": [B, 1, L]}."""

    def __init__(self, taps=9, batch_invariant=False):
        super().__init__()
        g = torch.Generator().manual_seed(5)
        self.k = torch.randn(1, 1, taps, generator=g) * 0.3
        self.batch_invariant = batch_invariant
        # the reference constructor reads nnet.f_helper.stft.conv_real.weight for its dtype (:411)
        self.f_helper = types.SimpleNamespace(stft=types.SimpleNamespace(conv_real=types.SimpleNamespace(weight=torch.zeros(1))))
        self.calls = []

    def forward(self, x):
        self.calls.append(tuple(x.shape))
        y = F.conv1d(x[:, :1, :], self.k, padding=self.k.shape[-1] // 2)
        return {"wav": torch.tanh(y) + 0.1 * y}


def _signal(n, batch=2):
    g = torch.Generator().manual_seed(n)
    return torch.randn(batch, 1, n, generator=g)


def ref_key(kind, n, w, m, windowed):
    return f"{kind}_{n}_{w}_{m}_{int(windowed)}"


def _reference(kind, n, w, m, windowed):
    """Output and network calls of the reference's LambdaOverlapAdd on _signal(n) with a ToyNet (oracle/make_ref_vectors.py)."""
    g = np.load(GOLDEN_OLA)
    key = ref_key(kind, n, w, m, windowed)
    return torch.from_numpy(g[key + "_out"]), [tuple(int(v) for v in c) for c in g[key + "_calls"]]


@pytest.mark.parametrize("n,w,m", CASES)
@pytest.mark.parametrize("windowed", [False, True])
def test_matches_reference_lambda_overlap_add(n, w, m, windowed):
    x = _signal(n)
    our_net = ToyNet()
    # the reference ran with window="hann" and its boxcar path selected through use_window, as its own ola_forward does
    a, ref_calls = _reference("boxcar", n, w, m, windowed)
    ours = BoxcarOverlapAdd(our_net, n_src=1, window_size=w, in_margin=m, window="hann" if windowed else None)
    b = ours(x)
    assert a.shape == b.shape == (2, 1, n)
    assert torch.equal(a, b)
    assert sorted(ref_calls) == sorted(our_net.calls)              # same chunks reach the network


@pytest.mark.parametrize("n,w,m", CASES)
def test_batched_schedule_equals_sequential(n, w, m):
    x = _signal(n, batch=3)
    seq, bat = ToyNet(batch_invariant=False), ToyNet(batch_invariant=True)
    a = BoxcarOverlapAdd(seq, 1, w, m)(x)
    b = BoxcarOverlapAdd(bat, 1, w, m, max_batch=None)(x)
    assert torch.allclose(a, b, atol=1e-6)
    n_chunks = -(-n // w)
    assert len(seq.calls) == n_chunks
    assert len(bat.calls) == min(n_chunks, 3)                      # first, last, one stacked call for the middle
    if n_chunks > 3:
        assert bat.calls[0][0] == 3 * (n_chunks - 2)


@pytest.mark.parametrize("n,w,m", CASES)
def test_margin_hides_the_chunking(n, w, m):
    net = ToyNet(taps=9)                                           # receptive field 4 <= every margin above
    x = _signal(n, batch=1)
    whole = net(x)["wav"]
    chunked = BoxcarOverlapAdd(ToyNet(taps=9), 1, w, m)(x)
    assert torch.allclose(whole, chunked, atol=1e-6)


def test_plan_and_argument_checks():
    ola = BoxcarOverlapAdd(ToyNet(), 1, 256, 32)
    chunks, last = ola.plan(1000)
    assert last == 1000 - 3 * 256
    assert chunks == [(0, 288, 0, 32), (224, 544, 32, 32), (480, 800, 32, 32), (736, 1000, 32, 0)]
    assert ola.plan(512)[0] == [(0, 288, 0, 32), (224, 512, 32, 0)]
    with pytest.raises(AssertionError):
        BoxcarOverlapAdd(ToyNet(), 1, 255, 32)
    with pytest.raises(ValueError):
        BoxcarOverlapAdd(ToyNet(), 1, 256, 256)
    with pytest.raises(NotImplementedError):
        BoxcarOverlapAdd(ToyNet(), 2, 256, 32, reorder_chunks=True)


# ------------------------------------------------------------------ windowed overlap-add (tools/dsp/overlapadd.py)
OLA_CASES = [(1000, 256, None), (1024, 256, 128), (300, 256, 64), (2049, 512, 256), (777, 128, 32)]


@pytest.mark.parametrize("n,w,hop", OLA_CASES)
@pytest.mark.parametrize("windowed", [True, False])
def test_windowed_ola_matches_reference(n, w, hop, windowed):
    """Against the reference's tools/dsp/overlapadd.py LambdaOverlapAdd (window="hann", use_window = windowed)."""
    x = _signal(n)
    our_net = ToyNet()
    a, ref_calls = _reference("ola", n, w, hop, windowed)
    ours = WindowedOverlapAdd(our_net, n_src=1, window_size=w, hop_size=hop, window="hann" if windowed else None,
                              reorder_chunks=False)
    b = ours(x)
    assert a.shape == b.shape == (2, 1, n)
    assert torch.equal(a, b)
    assert ref_calls == our_net.calls


@pytest.mark.parametrize("n,w,hop", OLA_CASES)
def test_windowed_ola_batched_equals_sequential_and_cola(n, w, hop):
    x = _signal(n, batch=2)
    seq, bat = ToyNet(batch_invariant=False), ToyNet(batch_invariant=True)
    a = WindowedOverlapAdd(seq, 1, w, hop, window="hanning", reorder_chunks=False)(x)
    b = WindowedOverlapAdd(bat, 1, w, hop, window="hanning", reorder_chunks=False, max_batch=None)(x)
    assert torch.allclose(a, b, atol=1e-6)
    assert len(bat.calls) == 1 and bat.calls[0][0] == 2 * len(seq.calls)   # the whole file in one call

    class Identity:
        batch_invariant = True

        def __call__(self, t):
            return {"wav": t[:, :1, :]}

    if hop is None or 2 * hop == w:                 # periodic hann at 50 % overlap sums to one: identity in, identity out
        y = WindowedOverlapAdd(Identity(), 1, w, hop, window="hann", reorder_chunks=False)(x)
        assert torch.allclose(y, x, atol=1e-6)


def test_max_batch_bounds_the_rows_per_call():
    """ADVICE r1: the stacked schedules run `max_batch` rows per nnet call (workspace grows with batch x length), with
    results identical to the unbounded stack; an n_src > 1 network with reorder_chunks is refused, not silently skipped."""
    x = _signal(20 * 256 + 17, batch=2)
    full, capped = ToyNet(batch_invariant=True), ToyNet(batch_invariant=True)
    a = BoxcarOverlapAdd(full, 1, 256, 32, max_batch=None)(x)
    b = BoxcarOverlapAdd(capped, 1, 256, 32, max_batch=6)(x)
    assert torch.equal(a, b)
    assert max(c[0] for c in capped.calls) <= 6 and max(c[0] for c in full.calls) == 2 * 19
    fullw, cappedw = ToyNet(batch_invariant=True), ToyNet(batch_invariant=True)
    aw = WindowedOverlapAdd(fullw, 1, 256, 128, reorder_chunks=False, max_batch=None)(x)
    bw = WindowedOverlapAdd(cappedw, 1, 256, 128, reorder_chunks=False, max_batch=8)(x)
    assert torch.equal(aw, bw)
    assert max(c[0] for c in cappedw.calls) <= 8 and len(fullw.calls) == 1

    class TwoSrc:
        batch_invariant = True

        def __call__(self, t):
            return {"wav": torch.cat([t, t], dim=1)}

    with pytest.raises(NotImplementedError):
        WindowedOverlapAdd(TwoSrc(), None, 256, 128)(x)                       # reorder_chunks defaults to True
    with pytest.raises(NotImplementedError):
        BoxcarOverlapAdd(TwoSrc(), None, 256, 32, reorder_chunks=True)(x)
