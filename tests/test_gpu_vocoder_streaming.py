"""Live mel streams through the stand-alone vocoder: vf_vocoder_chunks and streaming.StreamingVocoder.

A stream's concatenated step() outputs must be vocoder.vocode_chunked's bits - the chunks of vocoder.chunk_plan through
Vocoder.forward on torch slices, cropped - whatever the push splits and whichever streams share the steps; with a margin of
at least the vocoder's receptive field they must be forward on the whole mel, length included.  vf_vocoder_chunks itself is
checked against forward_batch on torch-gathered, zero-filled chunks, for its launches, its plan shapes and every refusal."""
import ctypes
import random

import pytest
import torch

from voicefixer_main_b200 import _lib as VL
from voicefixer_main_b200._lib import VF_EINVAL, VF_ESTATE, EngineError
from voicefixer_main_b200.arch import VocoderConfig, vocoder_out_len, vocoder_receptive_field
from voicefixer_main_b200.model import Engine, VoiceFixer
from voicefixer_main_b200.streaming import OPEN, StreamingVocoder
from voicefixer_main_b200.vocoder import Vocoder, chunk_plan, vocode_chunked
from voicefixer_main_b200.weights import make_ssr_state

pytestmark = pytest.mark.gpu

CFG = VocoderConfig()
HOP = CFG.hop


def bits(t):
    return t.contiguous().view(torch.int32)


def mel_of(T, seed):
    """A seeded linear mel with the range of speech: |x| up to ~10, many small values."""
    g = torch.Generator().manual_seed(seed)
    return ((torch.rand(T, 128, generator=g) * 2.2) ** 4).cuda()


@pytest.fixture(scope="module")
def voc(state):
    v = Vocoder().load_state_dict({k: t for k, t in state.items() if k.startswith("vocoder.")}).eval().to("cuda:0")
    yield v
    v._engine().check_errors()


@pytest.fixture(params=[1, 3], ids=["1term", "3term"])
def voc_terms(voc, request):
    e = voc._engine()
    e.set_option("vocoder_terms", request.param)
    yield voc
    e.set_option("vocoder_terms", 1)


def stream_all(sv, mels, seed, max_push=None):
    """Every mel of `mels` through one session of sv: streams opened at staggered steps, pushed in random pieces of at most
    W + 2M frames (host or device), closed when complete.  -> one concatenated output per mel."""
    rng = random.Random(seed)
    W, M = sv.window_frames, sv.margin_frames
    max_push = max_push or W + 2 * M
    opens = sorted(rng.randrange(0, 3) for _ in mels)
    sids, pos, outs = {}, {}, {}
    step = 0
    while len(sids) < len(mels) or sv._streams:
        for i, t in enumerate(opens):
            if t == step and i not in sids:
                sids[i] = sv.open()
                pos[i] = 0
        for i, sid in sids.items():
            if pos[i] is None:
                continue
            k = min(rng.randrange(0, max_push + 1), mels[i].shape[0] - pos[i])
            piece = mels[i][pos[i]:pos[i] + k]
            sv.push(sid, piece.cpu() if rng.random() < 0.3 else piece)
            pos[i] += k
            if pos[i] == mels[i].shape[0]:
                sv.close(sid)
                pos[i] = None
        for sid, o in sv.step().items():
            outs.setdefault(sid, []).append(o.clone())
        step += 1
        assert step < 10000
    torch.cuda.synchronize()
    return [torch.cat(outs[sids[i]]) for i in range(len(mels))]


# ------------------------------------------------------------------ 1. the stream is vocode_chunked
@pytest.mark.parametrize("W,M", [(32, 8), (64, 16), (16, 0)])
def test_stream_equals_vocode_chunked(voc_terms, W, M):
    lengths = [301, 250, W, 3 * W + M + 1]
    mels = [mel_of(T, 10 + i) for i, T in enumerate(lengths)]
    outs = stream_all(StreamingVocoder(voc_terms, W, M, max_streams=4), mels, seed=W + M)
    for T, m, o in zip(lengths, mels, outs):
        ref = vocode_chunked(voc_terms, m, W, M)
        assert o.numel() == ref.numel() == vocoder_out_len(T, CFG)
        assert torch.equal(bits(o), bits(ref)), (W, M, T)
    voc_terms._engine().check_errors()


# ------------------------------------------------------------------ 2. full context and single chunks are forward
def test_full_context_equals_forward(voc):
    """With M >= R (the receptive field) every kept frame sees what it sees in the whole mel: the stream is forward on the
    whole mel, length included."""
    R = vocoder_receptive_field(CFG)
    M = R + R % 2
    W = 128
    lengths = [1201, 3 * W + 2 * M + 2, 2 * M + 5]
    mels = [mel_of(T, 40 + i) for i, T in enumerate(lengths)]
    outs = stream_all(StreamingVocoder(voc, W, M, max_streams=3), mels, seed=3)
    for T, m, o in zip(lengths, mels, outs):
        ref = voc.forward(m[None, None])[0, 0]
        assert o.numel() == ref.numel() == vocoder_out_len(T, CFG)
        assert len(chunk_plan(T, W, M)) > 1
        assert torch.equal(bits(o), bits(ref)), T
    # a stream of at most W frames is one chunk: forward on it
    for T in (1, 2, 77, W):
        m = mel_of(T, T)
        o = stream_all(StreamingVocoder(voc, W, 8, max_streams=1), [m], seed=T)[0]
        assert torch.equal(bits(o), bits(voc.forward(m[None, None])[0, 0])), T


# ------------------------------------------------------------------ 3. neighbours and engines change no bit
def test_alone_equals_among_31_streams(voc):
    W, M = 32, 8
    mels = [mel_of(200 + 13 * i, 70 + i) for i in range(32)]
    among = stream_all(StreamingVocoder(voc, W, M, max_streams=32), mels, seed=8)
    alone = stream_all(StreamingVocoder(voc, W, M, max_streams=1), mels[5:6], seed=9)[0]
    assert torch.equal(bits(among[5]), bits(alone))
    assert torch.equal(bits(alone), bits(vocode_chunked(voc, mels[5], W, M)))


def test_voicefixer_engine_equals_stand_alone_vocoder(state, voc):
    model = VoiceFixer().load_state_dict(state).eval().to("cuda:0")
    W, M = 64, 16
    mels = [mel_of(333, 5), mel_of(128, 6)]
    a = stream_all(StreamingVocoder(model, W, M, max_streams=2), mels, seed=1)
    b = stream_all(StreamingVocoder(voc, W, M, max_streams=2), mels, seed=2)
    for x, y in zip(a, b):
        assert torch.equal(bits(x), bits(y))
    model._engine().check_errors()


# ------------------------------------------------------------------ 4. vf_vocoder_chunks against forward_batch
def gathered(ring, stream, start, length, valid):
    L = ring.shape[1]
    pos = torch.arange(start, start + length, device=ring.device)
    x = ring[stream, pos % L].clone()
    x[pos >= valid] = 0
    return x


def test_vocoder_chunks_ring_wrap_and_valid_cut(voc):
    e = voc._engine()
    ring = torch.stack([mel_of(50, 90 + s) for s in range(3)]).contiguous()           # [3, 50, 128]
    table = [(0, 40, 0, 0, 0, OPEN),                                 # no crop
             (1, 50, 3 * HOP, 17, 37, OPEN),                         # wraps the ring
             (2, 33, 5, 2 * HOP + 1, 120, 140),                      # wraps, and frames >= 140 are zeros
             (0, 21, 0, 0, 5, 5),                                    # all zeros
             (2, 9, HOP, HOP, 200, 205)]                             # odd length, zeros from frame 5
    kept = e.vocoder_chunks(ring, table)
    xs = [gathered(ring, s, start, n, valid) for s, n, _, _, start, valid in table]
    refs = voc.forward_batch(xs)
    off = 0
    for (s, n, cl, cr, start, valid), r in zip(table, refs):
        want = r[cl:r.numel() - cr]
        assert torch.equal(bits(kept[off:off + want.numel()]), bits(want)), (s, start, n)
        off += want.numel()
    assert off == kept.numel()
    e.check_errors()


def chain_launches(e, T):
    """Launches of one vf_vocoder_varlen sub-batch: the lengths table, the scatter, the chain and the pack."""
    before = e.launch_count()
    e.vocoder_varlen(mel_of(T, 1), [T])
    return e.launch_count() - before


def test_launches_sub_batches_and_flat_plans(voc):
    """Per sub-batch exactly the lengths table, one gather, the chain and one crop; a capped budget splits the call into
    power-of-two plans with padding rows, the bits unchanged; plans and evictions stay flat as the chunk count varies."""
    e = voc._engine()
    per_sub = chain_launches(e, 96)          # lengths table + copy + chain + copy: vf_vocoder_chunks has the same count
    ring = torch.stack([mel_of(96, 200 + s) for s in range(11)]).contiguous()
    table = [(s, 80 + (s % 3) * 8, 0, 0, s * 3, OPEN) for s in range(11)]
    kept = e.vocoder_chunks(ring, table)                            # warm the plans and graphs
    before = e.launch_count()
    assert torch.equal(bits(e.vocoder_chunks(ring, table)), bits(kept))
    assert e.launch_count() - before == per_sub
    refs = voc.forward_batch([gathered(ring, *t[:1], t[4], t[1], t[5]) for t in table])
    assert torch.equal(bits(kept), bits(torch.cat(refs)))
    e.set_option("plan_cache_mb", 1024)
    try:
        n_sub = None
        for _ in range(2):
            before = e.launch_count()
            got = e.vocoder_chunks(ring, table)
            n = (e.launch_count() - before) // per_sub
            assert (e.launch_count() - before) % per_sub == 0 and 1 < n < 11
            n_sub = n_sub or n
            assert n == n_sub
            assert torch.equal(bits(got), bits(kept))
        # chunk counts 1 .. 11 (each padded to a power of two within the cap): the plans stop growing after one round
        info = None
        for rnd in range(2):
            for k in list(range(1, 12)) + [7, 3, 11, 1]:
                got = e.vocoder_chunks(ring, table[:k])
                assert torch.equal(bits(got), bits(kept[:sum(vocoder_out_len(t[1], CFG) for t in table[:k])]))
            if rnd == 0:
                info = e.plan_cache_info()
        assert e.plan_cache_info()["plans"] == info["plans"] and e.plan_cache_info()["evicted"] == info["evicted"]
    finally:
        e.set_option("plan_cache_mb", 0)
    e.check_errors()


# ------------------------------------------------------------------ 5. refusals
def call(e, ring, n_streams, ring_frames, table, out):
    rows = (VL.VfChunk * max(1, len(table)))(*[VL.VfChunk(*t) for t in table])
    return e.lib.vf_vocoder_chunks(e.ctx, ctypes.c_void_p(ring.data_ptr()), n_streams, ring_frames, rows, len(table),
                                   ctypes.c_void_p(out.data_ptr()), None)


def test_refusals_leave_the_context_usable(voc):
    e = voc._engine()
    ring = torch.stack([mel_of(40, s) for s in range(2)]).contiguous()
    out = torch.empty(10 ** 6, device="cuda")
    good = (1, 30, 0, 0, 3, OPEN)
    n_out = vocoder_out_len(30, CFG)
    bad = [(2, 30, 0, 0, 0, OPEN), (-1, 30, 0, 0, 0, OPEN),           # stream out of range
           (0, 0, 0, 0, 0, OPEN), (0, -3, 0, 0, 0, OPEN), (0, 41, 0, 0, 0, OPEN),     # length < 1, > ring_frames
           (0, 30, n_out - 5, 5, 0, OPEN), (0, 30, -1, 0, 0, OPEN), (0, 30, 0, -1, 0, OPEN),   # crops
           (0, 30, 0, 0, -1, OPEN)]                                    # start < 0
    launches = e.launch_count()
    for b in bad:
        assert call(e, ring, 2, 40, [good, b], out) == VF_EINVAL, b
    assert e.launch_count() == launches                              # nothing was queued
    # length over vf_vocoder_varlen's maximum (checked with a ring that claims to be that long; nothing is read)
    big = (1 << 30) // HOP + 2
    assert call(e, ring, 1, big, [(0, big, 0, 0, 0, OPEN)], out) == VF_EINVAL
    assert e.launch_count() == launches
    kept = e.vocoder_chunks(ring, [good])                              # still usable
    ref = voc.forward(gathered(ring, 1, 3, 30, OPEN)[None, None])[0, 0]
    assert torch.equal(bits(kept), bits(ref))
    with pytest.raises(ValueError):
        e.vocoder_chunks(ring[0], [good])                             # not a frame ring
    e.check_errors()


def test_a_context_without_the_vocoder_refuses(state):
    e = Engine("cuda:0")
    try:
        e.load_state(make_ssr_state(1234), need=("ssr",))
        ring = mel_of(40, 1)[None].contiguous()
        launches = e.launch_count()
        with pytest.raises(EngineError) as ei:
            e.vocoder_chunks(ring, [(0, 30, 0, 0, 0, OPEN)])
        assert ei.value.code == VF_ESTATE
        assert e.launch_count() == launches
        wav = torch.randn(1, 44100, device="cuda")
        e.ssr_restore_varlen(wav[0], [44100])                      # the context is still usable
        e.check_errors()
    finally:
        e.close()
