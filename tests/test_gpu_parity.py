"""GPU parity tests (run with -m gpu on an H100).  Everything goes through the C ABI
(libb200vf.so via ctypes); the oracle and the golden files are only the checker."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import vf_oracle as O

pytestmark = pytest.mark.gpu

MEL_TOL = 1e-4      # north star: mel mask within 1e-4 (log10 mel, max abs)
WAV_RMS_TOL = 1e-3  # north star: waveform within 1e-3 RMS


@pytest.fixture(scope="module")
def model(state):
    from voicefixer_main_b200 import VoiceFixer
    m = VoiceFixer().load_state_dict(state).eval().to("cuda:0")
    yield m
    m._engine().check_errors()


# ------------------------------------------------------------------ stage A
@pytest.mark.parametrize("name", ["stage_a_n4410.npz", "stage_a_n30001.npz"])
def test_frontend_matches_reference_golden(model, name):
    g = load_golden(name)
    wav = torch.from_numpy(g["wav"]).cuda()
    sp, cos, sin = model.f_helper.wav_to_spectrogram_phase(wav[:, None, :])
    mel = model.mel(sp.permute(0, 1, 3, 2)).permute(0, 1, 3, 2)
    assert sp.shape == g["sp"].shape and mel.shape == g["mel"].shape
    sp_ref, _, _ = O.wav_to_spectrogram_phase(torch.from_numpy(g["wav"])[:, None, :], exact=True)
    scale = float(sp_ref.max())
    # against the exact (fp64) transform: fp32 FFT rounding only
    assert float((sp.cpu().double() - sp_ref).abs().max()) < 2e-6 * scale
    # against the reference's own fp32 conv-DFT output (golden): its rounding is the larger one
    assert float((sp.cpu() - torch.from_numpy(g["sp"])).abs().max()) < 5e-6 * scale
    assert float((mel.cpu() - torch.from_numpy(g["mel"])).abs().max()) < 5e-6 * float(g["mel"].max())
    assert float((cos ** 2 + sin ** 2 - 1).abs().max()) < 1e-3 or float(sp.min()) <= 1.1e-4


def test_frontend_rejects_short_input(model):
    from voicefixer_main_b200._lib import EngineError
    with pytest.raises(EngineError):
        model.pre(torch.zeros(1, 1, 1000, device="cuda"))


# ------------------------------------------------------------------ stage B
@pytest.mark.parametrize("name", ["stage_b_t101.npz", "stage_b_t1001.npz"])
def test_unet_matches_reference_golden(model, name, golden_fingerprint_ok):
    g = load_golden(name)
    out = model(torch.from_numpy(g["mel_orig"]).cuda())["mel"].cpu()
    ref = torch.from_numpy(g["log_mel"])
    err = (out - ref).abs()
    print(name, "log-mel max err", float(err.max()), "rms", float(err.pow(2).mean().sqrt()))
    assert out.shape == ref.shape
    assert float(err.max()) < MEL_TOL
    lm = O.to_log(torch.from_numpy(g["mel_orig"]))
    assert float((out[..., 127] - lm[..., 127]).abs().max()) < 1e-6      # last bin is a pass-through


@pytest.mark.parametrize("t", [64, 130])
def test_unet_ragged_lengths_vs_oracle(model, state, t):
    gen = torch.Generator().manual_seed(t)
    mel = 10 ** (torch.randn(3, 1, t, 128, generator=gen) - 1)
    with torch.no_grad():
        ref = O.generator_forward(state, mel)
    out = model(mel.cuda())["mel"].cpu()
    assert float((out - ref).abs().max()) < MEL_TOL


def test_to_log_assertion_behaviour(model):
    mel = torch.rand(1, 1, 64, 128, device="cuda")
    mel[0, 0, 3, 5] = -0.5
    with pytest.raises(AssertionError):
        model(mel)
    model(mel.abs())      # flag is cleared; the next call works


# ------------------------------------------------------------------ stage C (oracle = restatement, parity unpinned)
def test_vocoder_vs_oracle(model, state):
    gen = torch.Generator().manual_seed(17)
    mel = 10 ** (torch.randn(2, 1, 37, 128, generator=gen) * 0.7 - 1.5)
    with torch.no_grad():
        ref = O.vocoder_forward(state, mel)
    out = model.vocoder(mel.cuda()).cpu()
    assert out.shape == ref.shape == (2, 1, (37 + 1 + 4) * 441)
    rms = float((out - ref).pow(2).mean().sqrt())
    print("vocoder rms err", rms, "max", float((out - ref).abs().max()), "ref rms", float(ref.pow(2).mean().sqrt()))
    assert rms < WAV_RMS_TOL * 0.2


# ------------------------------------------------------------------ end to end
def test_restore_matches_reference_golden_1s(model, golden_fingerprint_ok):
    g = load_golden("e2e_1s.npz")
    wav = torch.from_numpy(g["wav"])
    out = model.restore(wav.cuda()).cpu()
    eng = model._engine()
    eng.check_errors()
    _, log_mel = eng.restore_stages(*wav.shape)
    mel_err = float((log_mel.cpu()[:, None] - torch.from_numpy(g["log_mel"])).abs().max())
    rms = float((out - torch.from_numpy(g["out"])).pow(2).mean().sqrt())
    print("e2e 1s: log-mel max err", mel_err, "wav rms err", rms)
    assert out.shape == wav.shape
    assert rms < WAV_RMS_TOL
    assert mel_err < 5e-3      # includes the reference's own fp32 conv-DFT noise in quiet bins


def test_restore_10s_golden_and_batch_invariance(model, golden_fingerprint_ok):
    g = load_golden("e2e_10s.npz")
    wav = torch.from_numpy(g["wav"])
    other = O.synth_clips(2, wav.shape[1], seed=77)
    batch = torch.cat([other[:1], wav, other[1:]]).cuda()
    out = model.restore(batch)
    model._engine().check_errors()
    rms = float((out[1].cpu() - torch.from_numpy(g["out"])[0]).pow(2).mean().sqrt())
    print("e2e 10s wav rms err", rms)
    assert rms < WAV_RMS_TOL
    single = model.restore(batch[1:2].contiguous())
    assert torch.equal(single[0], out[1])         # clips are independent: batching must not change a bit
    again = model.restore(batch)
    assert torch.equal(again, out)                # deterministic


def test_vocoder_three_term_mode(model, golden_fingerprint_ok):
    """Stage C defaults to hi-only fp16 operands (the waveform bar, 1e-3 RMS, is far looser than the mel bar);
    the fp32-grade 3-term mode stays available and must agree even more closely."""
    g = load_golden("e2e_1s.npz")
    eng = model._engine()
    ref = torch.from_numpy(g["out"])
    out1 = model.restore(torch.from_numpy(g["wav"]).cuda()).cpu()
    eng.set_option("vocoder_terms", 3)
    try:
        out3 = model.restore(torch.from_numpy(g["wav"]).cuda()).cpu()
        eng.check_errors()
    finally:
        eng.set_option("vocoder_terms", 1)
    r1, r3 = float((out1 - ref).pow(2).mean().sqrt()), float((out3 - ref).pow(2).mean().sqrt())
    print("e2e 1s wav rms err: vocoder_terms=1", r1, " vocoder_terms=3", r3)
    assert r1 < WAV_RMS_TOL and r3 < 1e-5


def test_handler_protocol_drop_in(model, state):
    """The exact call sequence of eval_gsr_voicefixer.py:51-72 on the mirror objects."""
    wav = O.synth_clips(1, 22050, seed=5)
    segment = wav[0]
    inp = segment[None, None, ...].cuda()
    sp, _, _ = model.f_helper.wav_to_spectrogram_phase(inp)
    mel_noisy = model.mel(sp.permute(0, 1, 3, 2)).permute(0, 1, 3, 2)
    out_model = model(mel_noisy)
    denoised_mel = model._engine().from_log(out_model["mel"])
    out = model.vocoder(denoised_mel)
    if torch.max(torch.abs(out)) > 1.0:
        out = out / torch.max(torch.abs(out))
    out = O.trim_center(out, segment.shape[-1])
    with torch.no_grad():
        ref = O.restore(state, wav, exact_stft=True)
    assert out.shape == (1, 1, 22050)
    assert float((out[0].cpu() - ref).pow(2).mean().sqrt()) < WAV_RMS_TOL
    fused = model.restore(wav.cuda())
    assert float((fused.cpu() - out[0].cpu()).abs().max()) < 1e-5


def test_long_form_segment_loop(model, state, monkeypatch):
    """BASELINE config 5 path: handler()'s independent-segment loop (eval_gsr_voicefixer.py:47-75), checked
    against the oracle with a short segment length (ragged tail), then one real 60 s segment for size."""
    from voicefixer_main_b200 import handler as H
    wav = O.synth_clips(1, 4 * 44100 + 777, seed=31)[0]
    monkeypatch.setattr(H, "SEG_LENGTH", 66150)
    out = H.restore_array(model, wav.numpy(), model.device).cpu()
    with torch.no_grad():
        ref = O.restore(state, wav[None], exact_stft=True, seg_samples=66150)
    assert out.shape == ref.shape == (1, wav.numel())
    assert float((out - ref).pow(2).mean().sqrt()) < WAV_RMS_TOL
    monkeypatch.setattr(H, "SEG_LENGTH", 44100 * 60)
    long = O.synth_clips(1, 44100 * 61, seed=32)[0]
    out = H.restore_array(model, long.numpy(), model.device)
    model._engine().check_errors()
    assert out.shape == (1, 44100 * 61) and bool(torch.isfinite(out).all())
    tail = model.restore(long[None, 44100 * 60:].cuda())
    assert torch.equal(out[:, 44100 * 60:], tail)      # segments are independent: the tail is its own restore


@pytest.mark.parametrize("batch,n", [(1, 1025), (5, 28224), (3, 2 * 44100 + 123)])
def test_restore_edge_shapes_vs_oracle(model, state, batch, n):
    """Minimum length the reflect pad allows (T = 3 -> T' = 64), T an exact multiple of 64 (28224 / 441 = 64 -> T = 65),
    odd batch, ragged length: stage B log-mel and final waveform against the oracle."""
    wav = O.synth_clips(batch, n, seed=100 + batch)
    st = {}
    with torch.no_grad():
        ref = O.restore(state, wav, exact_stft=True, stages=st)
    out = model.restore(wav.cuda()).cpu()
    eng = model._engine()
    eng.check_errors()
    mel, log_mel = eng.restore_stages(batch, n)
    assert out.shape == (batch, n) and log_mel.shape == (batch, 1 + n // 441, 128)
    ref_mel = st["mel_noisy"][0][:, 0].float()
    assert float((mel.cpu() - ref_mel).abs().max()) < 5e-6 * float(ref_mel.max())
    assert float((out - ref).pow(2).mean().sqrt()) < WAV_RMS_TOL
    # stage B on the *same* mel input (the e2e log-mel also carries the front ends' fp32 noise in quiet bins)
    with torch.no_grad():
        ref_lm = O.generator_forward(state, mel.cpu()[:, None])
    assert float((log_mel.cpu() - ref_lm[:, 0]).abs().max()) < MEL_TOL


def test_host_entry_point_and_launch_count(model):
    wav = O.synth_clips(2, 8820, seed=8)
    pin_in, pin_out = wav.pin_memory(), torch.empty_like(wav).pin_memory()
    eng = model._engine()
    dev = model.restore(wav.cuda()).cpu()
    n0 = eng.launch_count()
    model.restore_host(pin_in, pin_out)
    torch.cuda.synchronize()
    assert eng.launch_count() - n0 > 100          # our kernels ran, not a library fallback
    assert torch.equal(pin_out, dev)
    assert eng.workspace_bytes(2, 8820) > 0


def test_pcm16_matches_save_wave_cast(model):
    """SURVEY.md 8(f) row 3: the int16 conversion of tools/file/wav.py:22-24 on the GPU, bit for bit."""
    g = torch.Generator().manual_seed(9)
    x = torch.rand(3, 70001, generator=g) * 2 - 1
    x = x * (x.abs() < 0.99997)                                    # keep |x * 2^15| < 32767 in the random part
    edge = torch.tensor([0.0, 1e-6, -1e-6, 0.5, -0.5, 1 - 2.0 ** -15, -(1 - 2.0 ** -15), 32767.5 / 32768, -32767.5 / 32768,
                         -1.0, 3.0517578125e-05, -3.0517578125e-05, 4.57763671875e-05, -4.57763671875e-05])
    x[0, :edge.numel()] = edge
    def expect(v):      # x * 2^15, truncate toward zero through a wide integer, keep the low 16 bits
        t = np.trunc(v.astype(np.float32) * np.float32(32768)).astype(np.int64)
        return (t & 0xffff).astype(np.uint16).view(np.int16)

    got = model._engine().to_pcm16(x.cuda()).cpu().numpy()
    assert got.dtype == np.int16 and got.shape == (3, 70001)
    assert np.array_equal(got, O.to_int16(x.numpy()))              # in range: numpy's own truncating cast
    assert np.array_equal(got, expect(x.numpy()))
    # +1.0 (a peak-normalised maximum) overflows: x86 numpy goes through int32 and keeps the low 16 bits
    one = model._engine().to_pcm16(torch.ones(4, device="cuda")).cpu().numpy()
    assert np.array_equal(one, np.full(4, -32768, dtype=np.int16))
    wav = O.synth_clips(2, 8820, seed=4).cuda()
    pcm = model.restore_pcm16(wav)
    assert pcm.dtype == torch.int16 and pcm.shape == (2, 8820)
    assert np.array_equal(pcm.cpu().numpy(), expect(model.restore(wav).cpu().numpy()))


def test_longform_margins_vs_oracle(model, state):
    """SURVEY.md 8(f) row 2: boxcar overlap-add with context margins (tools/dsp/overlapadd_boxcar.py:416-518) over
    the engine, middle chunks batched, against the same schedule over the oracle."""
    from voicefixer_main_b200.longform import BoxcarOverlapAdd, RestoreNet, restore_longform
    W, M = 22050, 4410
    n = 3 * W + 8837                                               # 4 chunks, ragged tail
    wav = O.synth_clips(2, n, seed=41)

    class OracleNet:
        def __call__(self, x):
            with torch.no_grad():
                return {"wav": O.restore(state, x[:, 0, :], exact_stft=True)[:, None, :]}

    ours = BoxcarOverlapAdd(RestoreNet(model), 1, W, M)(wav.cuda()[:, None, :])[:, 0].cpu()
    ref = BoxcarOverlapAdd(OracleNet(), 1, W, M)(wav[:, None, :])[:, 0]
    assert ours.shape == ref.shape == (2, n)
    assert float((ours - ref).pow(2).mean().sqrt()) < WAV_RMS_TOL
    again = restore_longform(model, wav.cuda(), window_size=W, in_margin=M).cpu()
    assert torch.equal(again, ours)


def test_handler_file_to_file(model, state, tmp_path, monkeypatch):
    """handler() end to end (eval_gsr_voicefixer.py:37-77): PCM16 wav in -> restored PCM16 wav out, int16 conversion on
    the GPU; checked against the oracle run on the decoded input."""
    from voicefixer_main_b200 import handler as H
    n = 44100 + 321
    pcm_in = O.to_int16(O.synth_clips(1, n, seed=77)[0].clamp(-0.99, 0.99).numpy())
    src, dst = str(tmp_path / "in.wav"), str(tmp_path / "out.wav")
    H.save_pcm16(pcm_in, src)
    monkeypatch.setattr(H, "model", model)
    metrics = H.handler(src, dst, None, ckpt=None, device=model.device, needrefresh=False, meta={})
    assert metrics == {}
    got = H.load_wav(dst)
    assert got.shape == (n,)
    x = torch.from_numpy(pcm_in.astype(np.float32) / 32768.0)[None]
    with torch.no_grad():
        ref = O.restore(state, x, exact_stft=True)[0].numpy()
    ref_pcm = O.to_int16(np.clip(ref, -1.0, 32767.0 / 32768.0)).astype(np.float64) / 32768.0
    keep = np.abs(ref) < 0.999                                    # the +1.0 peak sample wraps in int16 (tested above)
    d = got.astype(np.float64)[keep] - ref_pcm[keep]
    assert float(np.sqrt(np.mean(d * d))) < WAV_RMS_TOL


def test_vocoder_separate_planes_without_ar_inverse(model, state):
    """A residual slope with no fp16 inverse (0: ReLU) cannot use the (a, r) stream: the stacks keep x as separate hi/lo
    planes, added in the epilogue at every width, and the C = 64 stacks take two launches per residual pair."""
    from voicefixer_main_b200 import VocoderConfig, VoiceFixer
    cfg = VocoderConfig(res_slope=0.0)
    gen = torch.Generator().manual_seed(17)
    mel = 10 ** (torch.randn(2, 1, 37, 128, generator=gen) * 0.7 - 1.5)
    with torch.no_grad():
        ref = O.vocoder_forward(state, mel, cfg)
    m = VoiceFixer(vocoder_config=cfg).load_state_dict(state).eval().to("cuda:0")
    eng, eng_ar = m._engine(), model._engine()
    n0 = eng_ar.launch_count()
    model.vocoder(mel.cuda())
    n_ar = eng_ar.launch_count() - n0
    n1 = eng.launch_count()
    out = m.vocoder(mel.cuda()).cpu()
    eng.check_errors()
    assert eng.launch_count() - n1 > n_ar                         # no fused pair ran
    assert out.shape == ref.shape
    rms = float((out - ref).pow(2).mean().sqrt())
    print("separate-planes vocoder rms err", rms, "ref rms", float(ref.pow(2).mean().sqrt()))
    assert rms < WAV_RMS_TOL * 0.2
