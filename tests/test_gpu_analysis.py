"""The bi_gru and dnn analysis modules on the GPU: stage B against the reference goldens, the GRU kernel against a float64
reference of one layer, restore() against the oracle, restore_batch / handler_batch against their one-clip forms, and a
context reloaded with a different module."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import analysis as A
from oracle import vf_oracle as O

pytestmark = pytest.mark.gpu

STAGE_B_TOL = 1e-4          # absolute log-mel, the project's stage-B bar
WAV_RMS_TOL = 1e-3          # as smoke()
# One GRU layer: |h| < 1, and the kernel is fp32 FMA with a fixed K order and precise expf / tanhf; its output planes hold
# hi + lo to ~2^-22 relative.  fp32 rounding of ~260 terms per step, damped by the recurrence: 2e-5 absolute leaves a
# margin of well over 10x on the measured error (printed) and sits 100x below what any known-wrong variant differs by
# (tests/test_analysis_cpu.py::test_gru_mutations_break_the_gpu_bar).
GRU_TOL = 2e-5

KINDS = {"bigru": "bi_gru", "dnn": "dnn"}


def _hp(kind):
    from voicefixer_main_b200 import default_hparams
    hp = default_hparams()
    sel = hp["task"]["gsr"]["gsr_model"]["voicefixer"]
    for k in ("unet", "unet_small", "bi_gru", "dnn"):
        sel[k] = k == kind
    return hp


def _state(kind):
    from voicefixer_main_b200.weights import make_bigru_state, make_dnn_state, make_vocoder_state
    sd = (make_bigru_state if kind == "bi_gru" else make_dnn_state)(1234)
    sd.update(make_vocoder_state(seed=1235))
    return sd


def _model(kind):
    from voicefixer_main_b200 import VoiceFixer
    return VoiceFixer(_hp(kind)).load_state_dict(_state(kind)).eval().to("cuda:0")


def _close(m):
    m._engine().check_errors()
    m._eng.close()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", params=sorted(KINDS.values()))
def model(request):
    m = _model(request.param)
    yield m
    _close(m)


@pytest.fixture(scope="module")
def bigru_model():
    m = _model("bi_gru")
    yield m
    _close(m)


@pytest.mark.parametrize("t", [101, 1001])
def test_stage_b_matches_reference(model, t):
    tag = {v: k for k, v in KINDS.items()}[model.analysis_module_name]
    g = load_golden(f"stage_b_{tag}_t{t}.npz")
    mel = torch.from_numpy(g["mel_orig"]).float().cuda()
    got = model(mel)["mel"].double().cpu()
    err = float((got - torch.from_numpy(g["log_mel"])).abs().max())
    print(f"{tag} T={t}: stage-B max |err| {err:.3e}")
    assert err < STAGE_B_TOL


# ------------------------------------------------------------------------------------------------------- one GRU layer
def _run_gru(eng, G, w, b, lengths, relu, T):
    from voicefixer_main_b200 import _lib as L
    B = G.shape[0]
    Gf, wf, bf = (x.float().contiguous() for x in (G, w, b))
    out = np.full((2, B, T, 512), 0x7e00, dtype=np.uint16)            # NaN sentinels: every element must be written
    lens = (ctypes.c_int * B)(*lengths) if lengths is not None else None
    case = L.VfGruCase(batch=B, T=T, G=Gf.data_ptr(), w_hh=wf.data_ptr(), b_hn=bf.data_ptr(),
                       lengths=ctypes.addressof(lens) if lens is not None else None, relu=int(relu),
                       out=out.ctypes.data)
    eng.selftest_gru(case)
    planes = out.view(np.float16).astype(np.float64)
    return torch.from_numpy(planes[0] + planes[1]), Gf.double(), wf.double(), bf.double()


def _gru_inputs(B, T, seed, cin=256):
    g = torch.Generator().manual_seed(seed)
    gru = torch.nn.GRU(cin, 256, bidirectional=True, batch_first=True).double()
    with torch.no_grad():
        for p in gru.parameters():
            p.copy_((torch.rand(p.shape, generator=g, dtype=torch.float64) * 2 - 1) / 16)
    x = torch.randn(B, T, cin, generator=g, dtype=torch.float64)
    return A.gru_input(x, gru, 0)


def _check_gru(got, want, lengths, T):
    lengths = lengths or [T] * got.shape[0]
    assert not bool(torch.isnan(got).any()), "an output element was never written"
    for i, n in enumerate(lengths):
        for half, name in ((slice(0, 256), "forward"), (slice(256, 512), "reverse")):
            err = float((got[i, :n, half] - want[i, :n, half]).abs().max())
            print(f"clip {i} ({n} of {T} frames) {name}: max |err| {err:.3e}")
            assert err < GRU_TOL, (i, name, err)
        assert bool((got[i, n:] == 0).all()), f"clip {i}: frames past its end are not zero"


def test_gru_6001_frames_batch_4(bigru_model):
    B, T = 4, 6001
    G, w, b = _gru_inputs(B, T, seed=11)
    got, G, w, b = _run_gru(bigru_model._engine(), G, w, b, None, False, T)
    _check_gru(got, A.gru_layer(G, w, b), None, T)


def test_gru_mixed_lengths_with_relu(bigru_model):
    """Clips one frame short of the 64-frame bucket, of 3 frames and of the full bucket, across two clusters' clip groups;
    the layer-1 input width (512) and the module's ReLU."""
    T, lengths = 64, [63, 3, 64, 40, 17, 1]
    G, w, b = _gru_inputs(len(lengths), T, seed=12, cin=512)
    got, G, w, b = _run_gru(bigru_model._engine(), G, w, b, lengths, True, T)
    _check_gru(got, A.gru_layer(G, w, b, lengths, relu=True), lengths, T)


# The recurrence's edges: a last clip group holding 1 of GRU_CLIPS = 4 clips (B = 5), one-frame sequences, gates driven far
# past saturation (expf(-x) overflows to inf for x < -88.7, tanhf reaches +-1), and 35 clusters x 2 directions of 8 CTAs: 560
# CTAs of one per SM, more than 132 SMs run at once.
GRU_EDGES = {
    "last_group_1_of_4": dict(B=5, T=64, lengths=[64, 17, 64, 3, 50], cin=256, relu=False),
    "T1": dict(B=6, T=1, lengths=None, cin=512, relu=True),
    "all_lengths_1": dict(B=5, T=16, lengths=[1] * 5, cin=256, relu=False),
    "saturated_gates": dict(B=4, T=96, lengths=[96, 80, 1, 33], cin=256, relu=False, saturate=True),
    "B140_T64": dict(B=140, T=64, lengths="mixed", cin=512, relu=True),
}


@pytest.mark.parametrize("name", list(GRU_EDGES))
def test_gru_edges(bigru_model, name):
    spec = GRU_EDGES[name]
    B, T = spec["B"], spec["T"]
    lengths = spec["lengths"]
    if lengths == "mixed":
        lengths = [int(v) for v in np.random.default_rng(140).integers(1, T + 1, B)]
        lengths[::7] = [T] * len(lengths[::7])
    G, w, b = _gru_inputs(B, T, seed=len(name) * 31 + B, cin=spec["cin"])
    if spec.get("saturate"):
        g = torch.Generator().manual_seed(77)
        big = torch.rand(G.shape, generator=g, dtype=torch.float64) < 0.4
        mag = 100 + 200 * torch.rand(G.shape, generator=g, dtype=torch.float64)
        sign = torch.where(torch.rand(G.shape, generator=g, dtype=torch.float64) < 0.5, -1.0, 1.0)
        G = torch.where(big, sign * mag, G)
        assert float(G.abs().max()) > 89                    # expf(-x) of a gate overflows
    got, G, w, b = _run_gru(bigru_model._engine(), G, w, b, lengths, spec["relu"], T)
    _check_gru(got, A.gru_layer(G, w, b, lengths, relu=spec["relu"]), lengths, T)


# ------------------------------------------------------------------------------------------------------ whole restores
def test_restore_matches_oracle(model):
    wav = O.synth_clips(2, 44100, seed=31)
    out = model.restore(wav.cuda()).cpu()
    model._engine().check_errors()
    with torch.no_grad():
        ref = A.restore(_state(model.analysis_module_name), wav, model.analysis_module_name, exact_stft=True)
    rms = float((out - ref).pow(2).mean().sqrt())
    print(f"{model.analysis_module_name}: waveform RMS err {rms:.3e}")
    assert torch.isfinite(out).all() and rms < WAV_RMS_TOL


def test_restore_batch_bit_identical_to_one_clip_restores(model):
    lengths = [1025, 27883, 5000, 441000, 28229, 44113]
    clips = [O.synth_clips(1, n, seed=300 + i)[0].cuda() for i, n in enumerate(lengths)]
    got = model.restore_batch(clips)
    want = [model.restore(c[None])[0] for c in clips]
    model._engine().check_errors()
    for n, g, w in zip(lengths, got, want):
        assert torch.equal(g, w), (n, float((g - w).abs().max()))


def test_clip_bits_do_not_depend_on_batch(model):
    """The same clip alone and at position 21 of a 32-clip batch of one length: bit-identical."""
    n = 44100
    clips = O.synth_clips(32, n, seed=41).cuda()
    alone = model.restore(clips[21:22].contiguous())
    together = model.restore(clips)
    model._engine().check_errors()
    assert torch.equal(alone[0], together[21])


def test_handler_batch_matches_handler(bigru_model, tmp_path, monkeypatch):
    from voicefixer_main_b200 import handler as H
    monkeypatch.setattr(H, "model", bigru_model)
    spec = [(1025, True), (44100, False), (163170, True), (441000, True)]
    os.makedirs(tmp_path / "one")
    os.makedirs(tmp_path / "batch")
    items = []
    for i, (n, has_target) in enumerate(spec):
        src = str(tmp_path / f"in{i}.wav")
        H.save_pcm16(O.to_int16(O.synth_clips(1, n, seed=100 + i)[0].clamp(-0.99, 0.99).numpy()), src, sample_rate=44100)
        tgt = None
        if has_target:
            tgt = str(tmp_path / f"tgt{i}.wav")
            H.save_pcm16(O.to_int16(O.synth_clips(1, n, seed=200 + i)[0].clamp(-0.99, 0.99).numpy()), tgt, sample_rate=44100)
        items.append((src, f"in{i}.wav", tgt))
    dev = bigru_model.device
    one = [H.handler(s, str(tmp_path / "one" / o), t, ckpt=None, device=dev, meta={}) for s, o, t in items]
    batch = H.handler_batch([(s, str(tmp_path / "batch" / o), t) for s, o, t in items], ckpt=None, device=dev, meta={})
    bigru_model._engine().check_errors()
    for (_, o, _), a, b in zip(items, one, batch):
        with open(tmp_path / "one" / o, "rb") as f1, open(tmp_path / "batch" / o, "rb") as f2:
            assert f1.read() == f2.read(), o
        assert a == b, (o, a, b)


def test_context_reloaded_with_bigru_returns_bigru_results(state, bigru_model):
    """A context that has built UNet plans and is then loaded with bi_gru weights runs the bi_gru module."""
    from voicefixer_main_b200 import VoiceFixer
    g = load_golden("stage_b_bigru_t101.npz")
    mel = torch.from_numpy(g["mel_orig"]).float().cuda()
    m = VoiceFixer().load_state_dict(state).eval().to("cuda:0")
    try:
        eng = m._engine()
        unet_out = eng.unet_mel(mel[:, 0].contiguous())
        assert eng.plan_cache_info()["plans"] > 0
        eng.load_state(_state("bi_gru"), need=("bi_gru", "vocoder"))
        assert eng.plan_cache_info()["plans"] == 0
        got = eng.unet_mel(mel[:, 0].contiguous())
        eng.check_errors()
        assert torch.equal(got, bigru_model._engine().unet_mel(mel[:, 0].contiguous()))
        assert not torch.equal(got, unet_out)
        assert float((got[:, None].double().cpu() - torch.from_numpy(g["log_mel"])).abs().max()) < STAGE_B_TOL
    finally:
        _close(m)
