"""The mel-stream vocoder of voicefixer_main_b200/streaming.py, CPU only: vocoder.chunk_plan against a brute-force mapping of
every output sample, StreamingVocoder over a fake engine whose vocoder_chunks does vf_vocoder_chunks' gather, zero fill,
vocoder and crop in torch with a toy vocoder, and arch.vocoder_receptive_field against a probe of the float64 oracle
vocoder.  A stream's outputs must be vocode_chunked's with the same vocoder, bit for bit, however the pushes are split and
whichever streams share a step."""
import random

import pytest
import torch

from oracle import vf_oracle as O
from voicefixer_main_b200.arch import VocoderConfig, vocoder_out_len, vocoder_receptive_field
from voicefixer_main_b200.streaming import OPEN, StreamingVocoder
from voicefixer_main_b200.vocoder import chunk_plan, vocode_chunked
from voicefixer_main_b200.weights import make_vocoder_state

CFG = VocoderConfig()
HOP = CFG.hop
GEOMETRIES = [(16, 8), (64, 16), (16, 0), (4, 10), (2, 2)]


def lengths_for(W, M):
    k = 5
    return sorted({1, W - 1, W, W + 1, W + M, W + M + 1, k * W, k * W + 1, 7 * W + 3 * M + 5} - {0})


# ------------------------------------------------------------------ chunk_plan
def brute_force_map(T, W, M):
    """For every sample n of a stream of T frames (vocoder_out_len(T) samples): the chunk that keeps it and the frame of
    the whole mel it belongs to, from the definition alone (chunk i keeps frames [i W, (i + 1) W) and the last chunk the
    tail padding)."""
    n_chunks = -(-T // W)
    out = []
    for n in range(vocoder_out_len(T, CFG)):
        t = n // HOP
        out.append((min(t // W, n_chunks - 1), t))
    return out


@pytest.mark.parametrize("W,M", GEOMETRIES)
def test_chunk_plan_matches_brute_force(W, M):
    for T in lengths_for(W, M) + [0]:
        plan = chunk_plan(T, W, M)
        assert len(plan) == -(-T // W)
        if T == 0:
            assert plan == []
            continue
        got = []
        for i, (s, length, cl, cr) in enumerate(plan):
            assert s == max(0, i * W - M) and s + length == min(T, (i + 1) * W + M), (T, i)
            assert 0 <= s and s + length <= T                                # no chunk reads outside the mel
            # W and M even: a chunk that ends before T has even length, one that ends at T the parity of T
            assert length % 2 == (T % 2 if s + length == T else 0)
            n_out = vocoder_out_len(length, CFG)
            assert 0 <= cl and 0 <= cr and cl + cr < n_out
            assert cl % HOP == 0 and cr % HOP == 0
            for j in range(cl, n_out - cr):                                  # chunk output sample j: frame s + j // hop
                got.append((i, s + j // HOP))
        assert len(got) == vocoder_out_len(T, CFG), (T, W, M)
        assert got == brute_force_map(T, W, M), (T, W, M)
        # a stream of at most W frames is one chunk: the whole output
        if T <= W:
            assert plan == [(0, T, 0, 0)]


def test_chunk_plan_refuses_bad_geometry():
    for W, M in ((3, 2), (0, 2), (4, 3), (4, -2), (-2, 0)):
        with pytest.raises(ValueError):
            chunk_plan(10, W, M)


# ------------------------------------------------------------------ the scheduler over a fake engine
def toy_vocoder(mel):
    """mel [T, 128] -> vocoder_out_len(T) samples.  Each frame's hop samples depend on its own values, its mirror in the chunk
    and its position in the chunk, and the tail padding holds its own ramp, so a chunk cut or cropped one position off
    changes the output."""
    T = mel.shape[0]
    x = mel.mean(dim=1)
    f = torch.cat([x + 0.25 * x.flip(0) + torch.arange(T, dtype=x.dtype) * 2.0 ** -10,
                   torch.full((T % 2 + CFG.tail_pad_base,), -4.0) + torch.arange(T % 2 + CFG.tail_pad_base) * 0.5])
    return f.repeat_interleave(HOP) + torch.arange(HOP, dtype=x.dtype).repeat(f.numel()) * 2.0 ** -14


class FakeEngine:
    device = torch.device("cpu")
    voc_cfg = CFG

    def __init__(self):
        self.calls = []

    def vocoder_chunks(self, ring, table):
        self.calls.append([tuple(t) for t in table])
        L = ring.shape[1]
        assert ring.shape[2] == 128
        kept = []
        for s, length, cl, cr, start, valid in table:
            n_out = vocoder_out_len(length, CFG)
            assert 0 <= s < ring.shape[0] and 1 <= length <= L and start >= 0 and cl + cr < n_out
            pos = torch.arange(start, start + length)
            x = ring[s, pos % L].clone()
            x[pos >= valid] = 0
            kept.append(toy_vocoder(x)[cl:n_out - cr])
        return torch.cat(kept)


class FakeVocoder:
    voc_cfg = CFG

    def __init__(self):
        self.engine = FakeEngine()

    def _engine(self):
        return self.engine

    def forward(self, mel):
        assert mel.dim() == 4 and mel.shape[:2] == (1, 1)
        return toy_vocoder(mel[0, 0])[None, None]


def mel_of(T, seed):
    return torch.rand(T, 128, generator=torch.Generator().manual_seed(seed)) ** 4 * 10


def run_session(W, M, lengths, seed, max_streams=None):
    """Streams of the given lengths, opened at staggered steps, pushed in random pieces (each at most W + 2M, the size that
    always fits after a step) and closed when complete.  -> (mels, outputs, {i: [(start, length, cl, cr)]}, vocoder)."""
    rng = random.Random(seed)
    voc = FakeVocoder()
    sv = StreamingVocoder(voc, W, M, max_streams=max_streams or len(lengths))
    mels = [mel_of(n, seed * 100 + i) for i, n in enumerate(lengths)]
    opens = sorted(rng.randrange(0, 4) for _ in lengths)
    sids, pos, outs, tables = {}, {}, {}, {}
    step = 0
    while len(sids) < len(lengths) or sv._streams:
        for i, t in enumerate(opens):
            if t == step and i not in sids:
                sids[i] = sv.open()
                pos[i] = 0
        for i, sid in sids.items():
            if pos[i] is None or rng.random() < 0.2:
                continue
            k = min(rng.randrange(0, W + 2 * M + 1), lengths[i] - pos[i])
            sv.push(sid, mels[i][pos[i]:pos[i] + k])
            pos[i] += k
            if pos[i] == lengths[i]:
                sv.close(sid)
                pos[i] = None
        slots = {st.slot: sid for sid, st in sv._streams.items()}
        before = len(voc.engine.calls)
        for sid, o in sv.step().items():
            outs.setdefault(sid, []).append(o)
        assert len(voc.engine.calls) - before <= 1                    # one vocoder_chunks call per step
        for call in voc.engine.calls[before:]:
            for s, length, cl, cr, start, valid in call:
                tables.setdefault(slots[s], []).append((start, length, cl, cr))
        # the overflow rule: after a step, fewer than W + 2M needed frames (at most W when M = 0) are held
        for st in sv._streams.values():
            assert st.pushed - sv._keep_from(st) < W + 2 * M + (M == 0)
        step += 1
        assert step < 10000
    outs = {i: torch.cat(outs.get(sids[i], [torch.zeros(0)])) for i in sids}
    return mels, outs, {i: tables.get(sids[i], []) for i in sids}, voc


@pytest.mark.parametrize("W,M", GEOMETRIES)
def test_streams_equal_vocode_chunked(W, M):
    lengths = lengths_for(W, M)
    for seed in (1, 2):
        mels, outs, tables, voc = run_session(W, M, lengths, seed)
        for i, T in enumerate(lengths):
            assert tables[i] == chunk_plan(T, W, M), (W, M, T)
            ref = vocode_chunked(voc, mels[i], W, M)
            assert outs[i].numel() == vocoder_out_len(T, CFG)
            assert torch.equal(outs[i], ref), (W, M, T, seed)


def test_long_streams_wrap_the_ring_many_times():
    W, M = 16, 8
    lengths = [45 * W + 3, 41 * W, 55 * W + 1]
    mels, outs, _, voc = run_session(W, M, lengths, seed=5)
    for i, T in enumerate(lengths):
        assert T > 10 * 2 * (W + 2 * M)
        assert torch.equal(outs[i], vocode_chunked(voc, mels[i], W, M))


def test_single_chunk_stream_is_forward():
    W, M = 64, 16
    voc = FakeVocoder()
    sv = StreamingVocoder(voc, W, M)
    for T in (1, 2, 33, W):
        mel = mel_of(T, T)
        a = sv.open()
        sv.push(a, mel)
        assert sv.step() == {}                  # nothing is final while the stream could still grow
        sv.close(a)
        out = sv.step()[a]
        assert torch.equal(out, voc.forward(mel[None, None])[0, 0])
        assert a not in sv._streams


def test_readiness_and_latency():
    """Chunk i leaves the step after (i + 1) W + M frames are in (one more when M = 0), and not before."""
    for W, M in ((16, 8), (16, 0)):
        voc = FakeVocoder()
        sv = StreamingVocoder(voc, W, M, max_streams=1)
        a = sv.open()
        mel = mel_of(10 * W, 3)
        pushed, emitted = 0, 0
        for t in range(10 * W):
            sv.push(a, mel[t:t + 1])
            pushed += 1
            out = sv.step()
            need = (emitted + 1) * W + max(M, 1)
            if pushed >= need:
                assert a in out and out[a].numel() == W * HOP
                emitted += 1
            else:
                assert out == {}
        assert emitted == 9


def test_reused_slot_and_empty_stream():
    W, M = 16, 8
    voc = FakeVocoder()
    sv = StreamingVocoder(voc, W, M, max_streams=1)
    a = sv.open()
    sv.close(a)                                  # T = 0: nothing to vocode, the slot is free again at once
    assert sv.step() == {} and a not in sv._streams
    outs = []
    for T in (3 * W + 5, 2 * W):
        b = sv.open()
        assert b != a                            # ids are never reused, slots are
        mel = mel_of(T, T)
        got = []
        for k in range(0, T, 7):
            sv.push(b, mel[k:k + 7])
            got += list(sv.step().values())
        sv.close(b)
        got += list(sv.step().values())
        assert torch.equal(torch.cat(got), vocode_chunked(voc, mel, W, M))
        outs.append(b)
    assert sv._free == [0]


def test_refusals():
    voc = FakeVocoder()
    for W, M in ((15, 8), (16, 7), (0, 0), (16, -2)):
        with pytest.raises(ValueError):
            StreamingVocoder(voc, W, M)
    with pytest.raises(ValueError):
        StreamingVocoder(voc, 16, 8, max_streams=0)
    sv = StreamingVocoder(voc, 16, 8, max_streams=2)
    a, b = sv.open(), sv.open()
    with pytest.raises(RuntimeError):
        sv.open()                                # too many streams
    for bad in (torch.zeros(4, 127), torch.zeros(128), torch.zeros(4, 128, dtype=torch.float64), [[0.0] * 128]):
        with pytest.raises(TypeError):
            sv.push(a, bad)
    sv.push(a, torch.zeros(2 * (16 + 16), 128))  # the whole ring
    with pytest.raises(OverflowError, match=f"stream {a}"):
        sv.push(a, torch.zeros(1, 128))
    sv.close(b)                                  # nothing pushed: gone at once
    with pytest.raises(KeyError):
        sv.push(b, torch.zeros(1, 128))
    sv.step()
    sv.push(a, torch.zeros(1, 128))              # fits again after the step
    sv.close(a)
    with pytest.raises(ValueError, match="closed"):
        sv.push(a, torch.zeros(1, 128))
    with pytest.raises(ValueError, match="closed"):
        sv.close(a)
    sv.step()
    with pytest.raises(KeyError):
        sv.push(a, torch.zeros(1, 128))


def test_table_rows():
    """A step's table rows: (slot, length, crop_left, crop_right, start, valid), valid OPEN while the stream is open."""
    W, M = 16, 8
    voc = FakeVocoder()
    sv = StreamingVocoder(voc, W, M)
    a = sv.open()
    sv.push(a, mel_of(3 * W + M, 1))
    sv.step()
    assert voc.engine.calls[-1] == [(0, W + M, 0, vocoder_out_len(W + M, CFG) - W * HOP, 0, OPEN),
                                    (0, W + 2 * M, M * HOP, vocoder_out_len(W + 2 * M, CFG) - (W + M) * HOP, W - M, OPEN),
                                    (0, W + 2 * M, M * HOP, vocoder_out_len(W + 2 * M, CFG) - (W + M) * HOP, 2 * W - M, OPEN)]
    sv.close(a)
    sv.step()
    T = 3 * W + M
    assert voc.engine.calls[-1] == [(0, T - (3 * W - M), M * HOP, 0, 3 * W - M, T)]


# ------------------------------------------------------------------ the receptive field
SMALL = [VocoderConfig(cond_channels=8, cond_layers=2, channels=16, upsample_scales=[2, 3], resstack_depth=[2, 2], hop=6),
         VocoderConfig(cond_channels=8, cond_layers=3, channels=16, upsample_scales=[3, 2, 2], resstack_depth=[3, 1, 2],
                       hop=12),
         VocoderConfig(cond_channels=4, cond_layers=1, channels=8, upsample_scales=[7, 3], resstack_depth=[4, 3], hop=21)]


@pytest.mark.parametrize("k", range(len(SMALL)))
def test_receptive_field_is_tight(k):
    """Perturb one frame of a float64 oracle run and find the frames whose samples change: the farthest is R frames away."""
    cfg = SMALL[k]
    R = vocoder_receptive_field(cfg)
    sd = {n: v.double() for n, v in make_vocoder_state(cfg, seed=11 + k).items()}
    T = 4 * R + 9
    g = torch.Generator().manual_seed(k)
    w = O.mel_weight(cfg).double()
    mel = w * 10.0 ** (-3 * torch.rand(T, cfg.num_mels, generator=g, dtype=torch.float64))     # inside the dB clip
    p = T // 2
    mel2 = mel.clone()
    mel2[p] *= 1.5
    with torch.no_grad():
        a = O.vocoder_forward(sd, mel[None, None], cfg)[0, 0]
        b = O.vocoder_forward(sd, mel2[None, None], cfg)[0, 0]
    changed = (a != b).nonzero()[:, 0]
    first, last = int(changed.min()) // cfg.hop, int(changed.max()) // cfg.hop
    assert max(p - first, last - p) == R, (cfg, R, p - first, last - p)


def test_receptive_field_of_the_default_config():
    """Cond-net 5 + stem 3 frames, then per stage 3288 samples of residual reach (sum 3^i + 1, i < 8) and the upsampler's
    taps, then the tail's 3 samples: 576 frames, about 5.8 s."""
    assert vocoder_receptive_field(CFG) == 576
    assert vocoder_receptive_field() == 576
