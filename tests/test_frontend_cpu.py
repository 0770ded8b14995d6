"""The float64 references of tests/test_gpu_frontend.py, checked without a GPU: frontend64 restates the oracle's front end
(and the reference's own fp32 output), and the checks the GPU tests apply, fed a numpy-made kernel output, pass it and fail
for each plausibly broken front end or ISTFT, at a case the GPU tests run."""
import numpy as np
import pytest
import torch

import test_gpu_frontend as F
from conftest import load_golden
from oracle import layers as R
from oracle import vf_oracle as O

FB = O.mel_filterbank().numpy()


# ------------------------------------------------------------------ the references restate the reference
def test_frontend64_matches_the_oracle():
    g = torch.Generator().manual_seed(11)
    for n in (1025, 4410, 30001):
        wav = torch.randn(2, 1, n, generator=g, dtype=torch.float64) * 0.3
        wav[1, 0, 2000:9000] = 0
        sp, cos, sin = O.wav_to_spectrogram_phase(wav, exact=True)
        mel = O.mel_project(sp, O.mel_filterbank().double())
        for b in range(2):
            r = R.frontend64(wav[b, 0].numpy(), 1 + n // 441, FB)
            for k, want in (("mag", sp), ("cos", cos), ("sin", sin), ("mel", mel)):
                assert np.abs(r[k] - want[b, 0].numpy()).max() <= 1e-12 * max(1.0, float(want.abs().max())), (n, b, k)
            assert np.abs(r["logmel"] - O.to_log(mel[b, 0]).numpy()).max() <= 1e-12


@pytest.mark.parametrize("name", ["stage_a_n4410.npz", "stage_a_n30001.npz"])
def test_frontend64_matches_the_reference_fp32_output(name):
    """The reference's own sp and mel (fp32 conv-DFT) within the rounding test_frontend_matches_reference_golden allows."""
    g = load_golden(name)
    for b, x in enumerate(g["wav"]):
        r = R.frontend64(x, g["sp"].shape[2], FB)
        assert np.abs(r["mag"] - g["sp"][b, 0]).max() < 5e-6 * g["sp"].max()
        assert np.abs(r["mel"] - g["mel"][b, 0]).max() < 5e-6 * g["mel"].max()


# ------------------------------------------------------------------ a numpy front end, correct or broken
def emulate(clips, T, fb=FB, pad=("reflect", "reflect"), window=None, late=0, conj=False, clamp_mag=False, packed=False,
            round8=False):
    """The five outputs as the kernel writes them ([B][T][width] bits, sentinels past each clip's frames): float64 STFT
    rounded to fp32, the magnitude as sqrtf(max(fp32 power, 1e-8f)).  Mutations: pad mode per end, the window, frames `late`
    samples late, sin negated, the clamp on |X| instead of |X|^2, a varlen clip padded with its packed neighbours' samples
    (zeros past the buffer), magnitudes rounded to 8 mantissa bits in frames 60 dB or more below the clip's peak."""
    win = R.hann() if window is None else window
    outs = {k: np.full((len(clips), T, F.WIDTH[k]), F.SENT32, np.uint32) for k in F.OUTS}
    buf = np.concatenate([np.zeros(1024), np.concatenate(clips).astype(np.float64), np.zeros(1024 + late)])
    start = 0
    for b, x in enumerate(clips):
        n, Tb = len(x), 1 + len(x) // 441
        if packed:
            xp = buf[start:start + n + 2048 + late]
        else:
            xp = np.pad(np.pad(x.astype(np.float64), (1024, 0), mode=pad[0]), (0, 1024 + late), mode=pad[1])
        start += n
        X = np.fft.rfft(np.stack([xp[t * 441 + late:t * 441 + late + 2048] for t in range(Tb)]) * win, axis=-1)
        if clamp_mag:
            m = np.maximum(np.abs(X), 1e-8).astype(np.float32)
        else:
            m = np.sqrt(np.maximum((X.real ** 2 + X.imag ** 2).astype(np.float32), np.float32(1e-8)))
        if round8:
            quiet = np.abs(X).max(axis=1) <= 1e-3 * np.abs(X).max()
            mant, ex = np.frexp(m[quiet].astype(np.float64))
            m[quiet] = np.ldexp(np.round(mant * 512) / 512, ex)
        m64 = m.astype(np.float64)
        mel = m64 @ np.asarray(fb, np.float32).astype(np.float64)
        vals = {"sp_out": m64, "cos_out": X.real / m64, "sin_out": (-1 if conj else 1) * X.imag / m64, "mel_out": mel,
                "logmel_out": np.log10(np.maximum(mel, 1e-8))}
        for k, v in vals.items():
            outs[k][b, :Tb] = v.astype(np.float32).view(np.uint32)
    return outs


def _check(name, **mutation):
    clips = F.clips_of(name)
    varlen = name == "varlen"
    T = F.bucket(clips) if varlen else 1 + len(clips[0]) // 441
    return F.check_frontend(name, clips, emulate(clips, T, **mutation), FB)


@pytest.mark.parametrize("name", ["n1025.impulses", "n4409.tones.b5", "n4410.b3", "n4411.impulses", "n60s.dynamic", "varlen"])
def test_frontend_check_passes_an_fp32_rounded_reference(name):
    _check(name)


MUTATIONS = {
    "symmetric_pad_start": ("n1025.impulses", dict(pad=("symmetric", "reflect"))),
    "symmetric_pad_end": ("n1025.impulses", dict(pad=("reflect", "symmetric"))),
    "symmetric_hann": ("n4410.b3", dict(window=np.hanning(2048))),
    "frames_one_sample_late": ("n4410.b3", dict(late=1)),
    "conjugated_spectrum": ("n4409.tones.b5", dict(conj=True)),
    "clamp_on_magnitude": ("n4411.impulses", dict(clamp_mag=True)),
    "varlen_reads_its_neighbour": ("varlen", dict(packed=True)),
}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_frontend_check_catches(mutation):
    name, kw = MUTATIONS[mutation]
    with pytest.raises(AssertionError):
        _check(name, **kw)


def test_quiet_frames_rounded_to_8_bits_pass_the_global_tolerance_and_fail_the_per_frame_bound():
    """The per-clip tolerance of test_frontend_matches_reference_golden (2e-6 of the clip's largest magnitude, 5e-6 of its
    largest mel) cannot see magnitudes with 8 mantissa bits in frames 60 dB below the peak; the per-frame bound does."""
    name = "n60s.dynamic"
    clips = F.clips_of(name)
    T = 1 + len(clips[0]) // 441
    outs = emulate(clips, T, round8=True)
    r = R.frontend64(clips[0], T, FB)
    sp = outs["sp_out"][0].view(np.float32).astype(np.float64)
    mel = outs["mel_out"][0].view(np.float32).astype(np.float64)
    assert np.abs(sp - r["mag"]).max() < 2e-6 * r["mag"].max()
    assert np.abs(mel - r["mel"]).max() < 5e-6 * r["mel"].max()
    quiet = np.abs(r["X"]).max(axis=1) <= 1e-3 * np.abs(r["X"]).max()
    assert quiet.sum() > 1000 and (~quiet).sum() > 1000
    with pytest.raises(AssertionError):
        F.check_frontend(name, clips, outs, FB)


def test_istft_check_passes_the_reference_and_catches_kept_dc_imaginary_parts():
    B, T = 3, 20
    length = F.istft_lengths(T)["longest"]
    re, im = F.istft_inputs(B, T)
    Y = re.astype(np.float64) + 1j * im.astype(np.float64)
    out = lambda keep: np.stack([R.overlap_add(R.inverse_frames(Y[b], keep), length)[0] for b in range(B)]).astype(np.float32)
    F.check_istft("istft.ok", re, im, length, out(False))
    with pytest.raises(AssertionError):
        F.check_istft("istft.dc_imag", re, im, length, out(True))
