"""The stream scheduler of voicefixer_main_b200/streaming.py with an SSR / GSR-UNet model, CPU only: StreamingRestorer over a
fake SSR engine whose ssr_restore_chunks does vf_ssr_restore_chunks' gather, zero fill, network and crop in torch with a
toy network.  The chunk tables must be BoxcarOverlapAdd.plan's and the outputs BoxcarOverlapAdd(RestoreNet(model))'s bit
for bit; each step is one ssr_restore_chunks call; the refusals are the SSR restore's, with no vocoder in them."""
import dataclasses
import random
import re

import pytest
import torch

from test_streaming_cpu import GEOMETRIES, edge_lengths, expected_plan, signal, toy_net
from voicefixer_main_b200 import GSR_UNet, SSR_UNet
from voicefixer_main_b200.arch import VocoderConfig
from voicefixer_main_b200.longform import BoxcarOverlapAdd, RestoreNet, restore_longform
from voicefixer_main_b200.streaming import OPEN, StreamingRestorer, restore_rejects


class FakeSSREngine:
    """No voc_cfg and no restore_chunks: an SSR stream must neither ask about the vocoder nor take the VoiceFixer call."""
    device = torch.device("cpu")

    def __init__(self):
        self.calls = []

    def ssr_restore_chunks(self, ring, table):
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


class FakeSSR(SSR_UNet):
    """An SSR_UNet whose engine is the fake and whose restore() is the toy network; records restore()'s keyword arguments."""

    def __init__(self):             # no hparams, no device: nothing of SSR_UNet.__init__ is needed here
        self.engine = FakeSSREngine()
        self.restore_kwargs = []

    def _engine(self):
        return self.engine

    def restore(self, wav, **kw):
        self.restore_kwargs.append(kw)
        return toy_net(wav[:, None])["wav"][:, 0]


class FakeGSR(GSR_UNet, FakeSSR):
    pass


class VFEngine:
    """A VoiceFixer engine whose vocoder has no tail frames, so that trim_center refuses some lengths."""
    device = torch.device("cpu")
    voc_cfg = dataclasses.replace(VocoderConfig(), tail_pad_base=0)


class VFModel:
    def _engine(self):
        return VFEngine()


def offline(model, W, M, x):
    return BoxcarOverlapAdd(RestoreNet(model), 1, W, M)(x[None, None])[0, 0]


def run_session(model, W, M, lengths, seed):
    """As test_streaming_cpu.run_session, on `model`: staggered opens, random pushes of at most W + 2M, skipped steps, each
    stream closed once complete.  -> (signals, outputs, {i: [(start, length, cl, cr)]})."""
    rng = random.Random(seed)
    eng = model._engine()
    sr = StreamingRestorer(model, W, M, max_streams=len(lengths))
    xs = [signal(n, seed * 100 + i) for i, n in enumerate(lengths)]
    opens = sorted(rng.randrange(0, 4) for _ in lengths)
    sids, pos, outs, tables = {}, {}, {}, {}
    step = 0
    while len(sids) < len(lengths) or sr._streams:
        for i, t in enumerate(opens):
            if t == step and i not in sids:
                sids[i], pos[i] = sr.open(), 0
        for i, sid in sids.items():
            if pos[i] is None or rng.random() < 0.2:
                continue
            k = min(rng.randrange(0, W + 2 * M + 1), lengths[i] - pos[i])
            sr.push(sid, xs[i][pos[i]:pos[i] + k])
            pos[i] += k
            if pos[i] == lengths[i]:
                sr.close(sid)
                pos[i] = None
        slots = {st.slot: sid for sid, st in sr._streams.items()}
        before = len(eng.calls)
        for sid, o in sr.step().items():
            outs.setdefault(sid, []).append(o)
        assert len(eng.calls) - before <= 1                      # one ssr_restore_chunks call per step
        for call in eng.calls[before:]:
            for s, length, cl, cr, start, valid in call:
                tables.setdefault(slots[s], []).append((start, length, cl, cr))
        step += 1
        assert step < 10000
    return xs, {i: torch.cat(outs.get(sids[i], [torch.zeros(0)])) for i in sids}, {i: tables.get(sids[i], []) for i in sids}


@pytest.mark.parametrize("W,M", GEOMETRIES)
@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("cls", [FakeSSR, FakeGSR])
def test_tables_and_outputs_match_boxcar_overlap_add(cls, W, M, seed):
    lengths = edge_lengths(W, M) + [random.Random(seed).randrange(W, 12 * W) for _ in range(3)]
    model = cls()
    xs, outs, tables = run_session(model, W, M, lengths, seed)
    for i, n in enumerate(lengths):
        assert tables[i] == expected_plan(W, M, n), (i, n)
        assert outs[i].shape == (n,)
        assert torch.equal(outs[i], offline(model, W, M, xs[i])), (i, n)
    valid = {row[5] for call in model.engine.calls for row in call}
    assert OPEN in valid and valid - {OPEN}


def test_one_ssr_restore_chunks_call_per_step():
    W, M = GEOMETRIES[0]
    model = FakeSSR()
    sr = StreamingRestorer(model, W, M, max_streams=3)
    ids = [sr.open() for _ in range(3)]
    for step in range(4):
        for sid in ids:
            sr.push(sid, signal(W + M if step == 0 else W, 10 * step + sid))
        out = sr.step()
        assert sorted(out) == ids and len(model.engine.calls) == step + 1
        assert len(model.engine.calls[-1]) == 3                   # every stream's chunk in the one call
    assert sr.step() == {} and len(model.engine.calls) == 4       # nothing ready: no call


def test_restore_rejects_for_ssr():
    n = 441 * 9 + 440                    # T = 10: a vocoder output of 441 (T + T % 2) = n + 1 samples, which trim_center refuses
    assert "trim_center" in restore_rejects(VFEngine(), n)
    assert restore_rejects(VFEngine(), n, ssr=True) is None
    assert restore_rejects(FakeSSREngine(), n, ssr=True) is None   # the SSR rule never reads a vocoder config
    for bad, why in ((1024, "1024"), (5, "1024"), ((1 << 30) + 1, "2\\^30")):
        assert re.search(why, restore_rejects(FakeSSREngine(), bad, ssr=True)), bad
        assert restore_rejects(FakeSSREngine(), bad, ssr=True) == restore_rejects(VFEngine(), bad)   # the same words
    assert restore_rejects(FakeSSREngine(), 1025, ssr=True) is None
    assert restore_rejects(FakeSSREngine(), 1 << 30, ssr=True) is None


def test_ssr_stream_accepts_what_only_trim_center_refuses():
    """A window whose chunks VoiceFixer's vocoder could not trim (with that vocoder config) streams through an SSR model."""
    W, M = 441 * 8, 440 + 441                                     # W + M = 441 * 9 + 440
    with pytest.raises(ValueError, match="trim_center"):
        StreamingRestorer(VFModel(), W, M)
    model = FakeSSR()
    sr = StreamingRestorer(model, W, M)
    a = sr.open()
    x = signal(3 * W + 500, 3)                                    # last chunk: M + 500 samples
    got = []
    for k in range(0, x.numel(), W):
        sr.push(a, x[k:k + W])
        got += list(sr.step().values())
    sr.close(a)
    got += list(sr.step().values())
    assert torch.equal(torch.cat(got), offline(model, W, M, x))
    assert (0, W + M, 0, M, 0, OPEN) in model.engine.calls[0]
    with pytest.raises(ValueError, match="1024"):
        StreamingRestorer(model, 1000, 24)                        # W + M = 1024
    with pytest.raises(ValueError, match="2\\^30"):
        StreamingRestorer(model, 1 << 30, 1)


def test_close_refuses_a_last_chunk_of_1024_samples_or_fewer():
    W, M = 4096, 512
    model = FakeSSR()
    sr = StreamingRestorer(model, W, M)
    a = sr.open()
    x = signal(3 * W + 400, 5)                                    # last chunk: M + 400 = 912 samples
    for k in range(0, x.numel(), W):
        sr.push(a, x[k:k + W])
        sr.step()
    with pytest.raises(ValueError, match=f"stream {a}.*1024"):
        sr.close(a)
    sr.push(a, signal(200, 6))
    sr.close(a)
    assert sr.step() and not sr._streams


@pytest.mark.parametrize("cls", [FakeSSR, FakeGSR])
def test_unify_energy_with_an_ssr_model_raises(cls):
    model = cls()
    with pytest.raises(ValueError, match="unify_energy"):
        StreamingRestorer(model, 4096, 1536, unify_energy=True)
    with pytest.raises(ValueError, match="unify_energy"):
        RestoreNet(model, unify_energy=True)
    with pytest.raises(ValueError, match="unify_energy"):
        restore_longform(model, torch.zeros(1, 10000), window_size=4096, in_margin=1536, unify_energy=True)
    assert not model.engine.calls and not model.restore_kwargs


def test_restore_net_passes_no_unify_energy_to_an_ssr_model():
    model = FakeSSR()
    x = signal(3000, 1)[None, None].repeat(2, 1, 1)
    out = RestoreNet(model)(x)["wav"]
    assert model.restore_kwargs == [{}]
    assert out.shape == (2, 1, 3000) and torch.equal(out, toy_net(x)["wav"])
    W, M = 4096, 1536
    wav = torch.stack([signal(5 * W + 77, 2), signal(5 * W + 77, 3)])
    got = restore_longform(model, wav, window_size=W, in_margin=M, max_batch=4)
    assert all(kw == {} for kw in model.restore_kwargs)
    assert torch.equal(got, BoxcarOverlapAdd(RestoreNet(model), 1, W, M)(wav[:, None])[:, 0])
