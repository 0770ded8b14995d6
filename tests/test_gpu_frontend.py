"""The STFT + mel front end (frontend.cu + fft.cuh), the stand-alone mel (vf_mel) and ISTFT (vf_istft) against float64
references (oracle/layers.py), frame by frame and bin by bin.

vf_selftest_op's VF_OP_FRONTEND case calls run_frontend, the function every restore and vf_frontend call, with the outputs
a call site asks for (uniform, or clips of different lengths with the product's lengths table).  Bounds, per frame t and
bin k (u = 2^-24, gamma_k = k u / (1 - k u), S_t = sum |x w| of the frame, as test_gpu_aux.py):

  X    windowed load v = fl(x fl(w)): |dv| <= gamma_2 |x w|.  The packed 1024-point FFT of z_j = v_2j + i v_2j+1 (sum |z_j|
       <= S_t): a radix-4 pass adds 4 inputs in two fp32 adds per component, 2u sum |in| by Minkowski; passes 2-5 first
       multiply by an fp32 twiddle (|dtw| <= u) in complex fp32, (sqrt(2) gamma_2 + u) |in|.  With the load,
       |dZ| <= (2 + 2 + 4 (2 + 3.83)) u S_t = 27.3 u S_t.  The split: dX_k = dZ_k (1 - i w) / 2 + conj(dZ_r) (1 + i w) / 2,
       at most sqrt(2) 27.3 u S_t, plus its own rounding (e, o, the fp32 twiddle product, the last add: 7.8 u S_t since
       |E_k| + |O_k| <= S_t).  So |dX_k| <= E_t = 48 u S_t (46.4 u to first order).
  sp   m = sqrtf(fmaxf(re^2 + im^2, 1e-8f)) is 1-Lipschitz in X (the clamp is max(|X|, 1e-4)), and the power, sqrtf and the
       fp32 clamp constant add 2u m: |dm_k| <= E_t + 2u m_k.
  cos, sin   X / max(|X|, r) moves by at most |dX| / max(|X| - |dX|, r) (r = 1e-4; two unit vectors differ by at most 2):
       phi_k = min(2, E_t / max(|X_k| - E_t, 1e-4)), plus 3u for the computed m and the IEEE division.
  mel  an fp32 fmaf chain of the filter's len_m stored values from 0: sum_f fb |dm_f| + gamma_len sum_f fb m_f.
  log-mel   dmel / (ln 10 max(mel - dmel, 1e-8)) + log10f's 2 ulp (2^-22 |log10|).
FLOOR = 2^-24 is the absolute floor of every bound.  Exact: frames of digital silence have sp = sqrtf(1e-8f) and
cos = sin = 0; outputs the call did not ask for, and rows t >= T_b of a varlen clip, keep their sentinels; a clip's rows are
the same bits in a batch of 3, in a varlen launch and alone.

Where ratios are small: a bin far below its frame's S_t (the noise floor of a tone, the silent bins around an impulse) gets
a bound of the frame's whole FFT rounding, which its few-ulp error does not approach; the phase bound is 2 (vacuous) where
|X_k| <= E_t, since there the phase is rounding noise in the kernel and the reference alike."""
import numpy as np
import pytest
import torch

import test_gpu_aux as A
import test_gpu_layers as G
from oracle import layers as R
from oracle import vf_oracle as O
from voicefixer_main_b200 import _lib as VL

pytestmark = pytest.mark.gpu

FRONTEND = 8                       # VF_OP_FRONTEND (include/b200vf.h)
U, FLOOR, SENT32, HOP = A.U, A.FLOOR, A.SENT32, A.HOP
gamma = A.gamma
C_X = 48 * U
OUTS = ("mel_out", "logmel_out", "sp_out", "cos_out", "sin_out")
WIDTH = {"mel_out": 128, "logmel_out": 128, "sp_out": 1025, "cos_out": 1025, "sin_out": 1025}
SP_SILENT = np.sqrt(np.float32(1e-8)).view(np.uint32)
report = A.report


# ------------------------------------------------------------------ signals and cases
def signal(kind, n, g):
    i = np.arange(n)
    if kind == "impulses":      # the reflect index math at both ends: each edge sample appears once in its frame
        x = np.zeros(n)
        pos = sorted({p for p in (0, 1, 1023, 1024, 1025, n - 1025, n - 1024, n - 2, n - 1) if 0 <= p < n})
        for j, p in enumerate(pos):
            x[p] = (1 + j / 8) * (-1) ** j
    elif kind == "dc":
        x = np.full(n, 0.75)
    elif kind == "nyquist":
        x = 0.5 * (-1.0) ** i
    elif kind.startswith("tone"):  # bin-centred: cycles of 2048 samples
        x = 0.6 * np.cos(2 * np.pi * int(kind[4:]) * i / 2048 + 0.3)
    elif kind == "noise":
        x = g.standard_normal(n) * 0.3
    elif kind == "int16":        # full scale, mostly positive: |X_0| near 32767 * 1024, its power near 1e15
        x = np.where(g.random(n) < 0.8, 32767.0, -32767.0)
    elif kind == "dynamic":      # > 100 dB across frames: loud, then noise at 1e-5, then exact zeros
        x = g.standard_normal(n)
        x[n // 2:] *= 1e-5
        x[4 * n // 5:] = 0
    else:
        raise ValueError(kind)
    return x.astype(np.float32)


CASES = {
    "n1025.impulses": dict(n=1025, kinds=["impulses"]),
    "n1026.b3": dict(n=1026, kinds=["impulses", "noise", "nyquist"]),
    "n2047.impulses": dict(n=2047, kinds=["impulses"]),
    "n2048.b3": dict(n=2048, kinds=["impulses", "dc", "int16"]),
    "n2049.int16": dict(n=2049, kinds=["int16"]),
    "n4409.tones.b5": dict(n=10 * HOP - 1, kinds=["dc", "nyquist", "tone1", "tone512", "tone1023"]),
    "n4410.b3": dict(n=10 * HOP, kinds=["impulses", "noise", "tone512"]),
    "n4411.impulses": dict(n=10 * HOP + 1, kinds=["impulses"]),
    "n30001.b3": dict(n=30001, kinds=["noise", "int16", "impulses"]),
    "n60s.dynamic": dict(n=44100 * 60, kinds=["dynamic"]),
    # clips of very different content side by side: reading a neighbour instead of reflecting breaks a bound
    "varlen": dict(ns=[1025, 63 * HOP + 100, 64 * HOP, 30001, 1025], kinds=["int16", "impulses", "noise", "impulses", "int16"]),
}


def clips_of(name):
    spec = CASES[name]
    g = A._rng(name)
    ns = spec.get("ns") or [spec["n"]] * len(spec["kinds"])
    return [signal(k, n, g) for k, n in zip(spec["kinds"], ns)]


def bucket(clips):
    return (max(1 + len(x) // HOP for x in clips) + 63) // 64 * 64


def filter_lengths(fb):
    """len_m of the packed filterbank (pack.cu load_all): first to last non-zero bin of filter m, 0 for an all-zero one."""
    nz = np.asarray(fb, np.float32) != 0
    lo, hi = nz.argmax(0), nz.shape[0] - 1 - nz[::-1].argmax(0)
    return np.where(nz.any(0), hi - lo + 1, 0)


def run_frontend(eng, name, clips, want=OUTS, varlen=False, T=None):
    """One VF_OP_FRONTEND launch; -> the five output arrays [B][T][width] (uint32 bits, sentinel-filled) and T."""
    B = len(clips)
    ns = [len(x) for x in clips]
    if varlen:
        T = bucket(clips) if T is None else T
    else:
        assert len(set(ns)) == 1
        T = 1 + ns[0] // HOP
    outs = {k: np.full((B, T, WIDTH[k]), SENT32, np.uint32) for k in OUTS}
    sel = {k: outs[k] for k in want}
    if varlen:
        c = A.Case(FRONTEND, B, A.offsets(ns), T=T, n=max(ns), in_wav=np.concatenate(clips), **sel)
    else:
        c = A.Case(FRONTEND, B, n=ns[0], in_wav=np.stack(clips), **sel)
    c.run(eng, name)
    assert c.oc.T == T
    return outs, T


class PerOutput(G.Checker):
    """A Checker that also keeps the worst err / bound of each output."""

    def __init__(self, name):
        super().__init__(name)
        self.per = {}

    def values(self, what, *args):
        c = G.Checker(self.name)
        c.values(what, *args)
        self.per[what] = max(self.per.get(what, 0.0), c.worst)
        self.worst = max(self.worst, c.worst)


def report_outputs(name, ck):
    report(name, ck)
    print("    " + ", ".join(f"{k} {v:.3e}" for k, v in ck.per.items()))


def check_frontend(name, clips, outs, fb, want=OUTS):
    """Every requested output of every clip against frontend64 with the bounds of the module docstring; exact silence;
    sentinels in rows t >= T_b and in the outputs that were not requested."""
    fb64 = np.asarray(fb, np.float32).astype(np.float64)
    afb = np.abs(fb64)
    glen = gamma(filter_lengths(fb))[None]
    ck = PerOutput(name)
    for k in OUTS:
        if k not in want:
            assert (outs[k] == SENT32).all(), (name, k, "written but not requested")
    for b, x in enumerate(clips):
        Tb = 1 + len(x) // HOP
        r = R.frontend64(x, Tb, fb)
        E = C_X * r["S"][:, None]
        silent = (r["S"] == 0)[:, None]
        got = {k: outs[k][b, :Tb].view(np.float32).astype(np.float64) for k in want}
        for k in want:
            assert (outs[k][b, Tb:] == SENT32).all(), (name, b, k, "rows past the clip written")
        if "sp_out" in want:
            ck.values("sp", got["sp_out"], r["mag"], E + 2 * U * r["mag"] + FLOOR, np.zeros(1, bool))
            assert (outs["sp_out"][b, :Tb][silent[:, 0]] == SP_SILENT).all(), (name, b, "sp of a silent frame")
        if "cos_out" in want:
            phi = np.minimum(2.0, E / np.maximum(np.abs(r["X"]) - E, 1e-4)) + 3 * U + FLOOR
            ck.values("cos", got["cos_out"], r["cos"], phi, silent)
            ck.values("sin", got["sin_out"], r["sin"], phi, silent)
        dmel = E * afb.sum(0)[None] + (2 * U + glen) * (r["mag"] @ afb)
        if "mel_out" in want:
            ck.values("mel", got["mel_out"], r["mel"], dmel + FLOOR, np.zeros(1, bool))
        if "logmel_out" in want:
            dl = dmel / (np.log(10.0) * np.maximum(r["mel"] - dmel, 1e-8)) + 2.0 ** -22 * np.abs(r["logmel"]) + FLOOR
            ck.values("logmel", got["logmel_out"], r["logmel"], dl, np.zeros(1, bool))
    return ck


@pytest.fixture(scope="module")
def eng():
    from voicefixer_main_b200.model import Engine
    e = Engine("cuda:0")
    e.load_state({"mel.fb": O.mel_filterbank()}, need=())
    yield e
    e.check_errors()
    e.close()


def custom_fb():
    """The built-in filterbank with a gap inside filter 100, an all-zero filter 64, and non-zeros at bin 0 (filter 0) and
    bin 1024 (filter 127)."""
    fb = O.mel_filterbank().numpy().copy()
    fb[0, 0] = 0.25
    fb[1024, 127] = 0.7
    fb[:, 64] = 0
    nz = np.flatnonzero(fb[:, 100])
    fb[nz[len(nz) // 2], 100] = 0
    return fb


@pytest.fixture(scope="module")
def eng_fb():
    from voicefixer_main_b200.model import Engine
    e = Engine("cuda:0")
    e.load_state({"mel.fb": torch.from_numpy(custom_fb())}, need=())
    yield e
    e.check_errors()
    e.close()


# ------------------------------------------------------------------ the front end
@pytest.mark.parametrize("name", [k for k in CASES if k != "varlen"])
def test_frontend_matches_float64(eng, name):
    clips = clips_of(name)
    outs, _ = run_frontend(eng, name, clips)
    report_outputs(name, check_frontend(name, clips, outs, O.mel_filterbank().numpy()))
    if len(clips) > 1:               # a clip's rows are the bits of a batch-1 launch on it
        for b, x in enumerate(clips):
            one, _ = run_frontend(eng, f"{name}.clip{b}", [x])
            for k in OUTS:
                assert np.array_equal(outs[k][b], one[k][0]), (name, b, k)


def test_frontend_varlen_matches_float64_and_each_clip_alone(eng):
    name = "varlen"
    clips = clips_of(name)
    outs, T = run_frontend(eng, name, clips, varlen=True)
    assert T == 128
    report_outputs(name, check_frontend(name, clips, outs, O.mel_filterbank().numpy()))
    for b, x in enumerate(clips):
        one, _ = run_frontend(eng, f"{name}.clip{b}", [x])
        Tb = 1 + len(x) // HOP
        for k in OUTS:
            assert np.array_equal(outs[k][b, :Tb], one[k][0]), (name, b, k)


SUBSETS = {
    "restore": ("mel_out", "logmel_out"),                   # restore_impl (uniform and varlen)
    "ssr": ("sp_out",),                                     # ssr_impl (uniform and varlen)
    "mel": ("mel_out",),                                    # ssr_restore_varlen's mel_out; Engine.frontend()
    "pre": ("mel_out", "sp_out", "cos_out", "sin_out"),     # vf_frontend for VoiceFixer.pre; frontend(want_phase=True)
    "mel_sp": ("mel_out", "sp_out"),                        # frontend(want_sp=True)
    "sp_phase": ("sp_out", "cos_out", "sin_out"),           # FDomainHelper.wav_to_spectrogram_phase (want_mel=False)
}


@pytest.mark.parametrize("varlen", [False, True])
@pytest.mark.parametrize("subset", list(SUBSETS))
def test_frontend_output_subsets(eng, subset, varlen):
    """Each call site's outputs are the bits of a launch that writes all five; the others keep their sentinels."""
    name = "varlen" if varlen else "n4410.b3"
    clips = clips_of(name)
    full, _ = run_frontend(eng, name, clips, varlen=varlen)
    want = SUBSETS[subset]
    part, _ = run_frontend(eng, f"{name}.{subset}", clips, want, varlen=varlen)
    for k in OUTS:
        assert np.array_equal(part[k], full[k] if k in want else np.full_like(full[k], SENT32)), (subset, k)


def test_frontend_custom_filterbank(eng_fb):
    """mel.fb loaded through Engine.load_state: the sparse packing (pack.cu) as the front end consumes it."""
    name = "n4410.b3"
    clips = clips_of(name)
    outs, _ = run_frontend(eng_fb, f"{name}.custom_fb", clips)
    report_outputs(f"{name}.custom_fb", check_frontend(f"{name}.custom_fb", clips, outs, custom_fb()))
    assert (outs["mel_out"][..., 64].view(np.float32) == 0).all()


def test_frontend_varlen_rows_must_cover_every_clip(eng):
    clips = clips_of("varlen")
    for T in (64, 68):           # the 30001-sample clip has 69 frames
        with pytest.raises(VL.EngineError) as ei:
            run_frontend(eng, "varlen.short_T", clips, varlen=True, T=T)
        assert ei.value.code == VL.VF_EINVAL


def test_batch_past_grid_y_is_refused_up_front(eng):
    """vf_frontend and vf_istft launch grid(T, batch): a batch above 65535 fails with VF_EINVAL before any launch."""
    dev = eng.device
    n0 = eng.launch_count()
    with pytest.raises(VL.EngineError) as ei:
        eng.frontend(torch.zeros(65536, 1025, device=dev))
    assert ei.value.code == VL.VF_EINVAL
    re = torch.zeros(65536, 3, 1025, device=dev)
    with pytest.raises(VL.EngineError) as ei:
        eng.istft(re, re, 1025)
    assert ei.value.code == VL.VF_EINVAL
    assert eng.launch_count() == n0


# ------------------------------------------------------------------ vf_mel: mel_kernel
def check_mel(name, x, got, fb):
    """x [n, 1025, T], got [n, 128, T]: an fp32 fmaf chain of len_m terms, gamma_len sum_f fb |x|."""
    x64 = np.asarray(x, np.float64)
    fb64 = np.asarray(fb, np.float32).astype(np.float64)
    want = np.einsum("oft,fm->omt", x64, fb64)
    bnd = gamma(filter_lengths(fb))[None, :, None] * np.einsum("oft,fm->omt", np.abs(x64), np.abs(fb64)) + FLOOR
    ck = G.Checker(name)
    ck.values("mel", got, want, bnd, np.zeros(1, bool))
    return ck


@pytest.mark.parametrize("which", ["builtin", "custom"])
@pytest.mark.parametrize("layout", ["time_fastest", "freq_fastest"])
def test_mel_of_identity_is_the_filterbank(eng, eng_fb, which, layout):
    """Every fma chain has one non-zero term: out[m, t] = fb[t, m] exactly, through both load paths of mel_kernel."""
    e, fb = (eng, O.mel_filterbank().numpy()) if which == "builtin" else (eng_fb, custom_fb())
    eye = torch.eye(1025, device=e.device)
    x = eye if layout == "time_fastest" else eye.t()
    assert (x.stride(-1) == 1) == (layout == "time_fastest")
    got = e.mel(x).cpu().numpy()                      # [128, 1025 frames]
    assert np.array_equal(got.T, np.asarray(fb, np.float32))


@pytest.mark.parametrize("T", [1, 7, 8, 9, 1025])
@pytest.mark.parametrize("layout", ["time_fastest", "freq_fastest"])
def test_mel_matches_float64(eng, layout, T):
    """Both load paths; frames in and past one MEL_TT = 8 tile; one clip, and three taken every other one from a larger
    tensor (a non-contiguous outer stride)."""
    name = f"mel.{layout}.T{T}"
    g = torch.Generator().manual_seed(T * 2 + (layout == "freq_fastest"))
    fb = O.mel_filterbank().numpy()
    for n_outer, step in ((1, 1), (3, 2)):
        shape = (n_outer * step, 1025, T) if layout == "time_fastest" else (n_outer * step, T, 1025)
        big = (torch.randn(*shape, generator=g) * 3).to(eng.device)
        x = big[::step] if layout == "time_fastest" else big[::step].transpose(1, 2)
        assert (x.stride(-1) == 1) == (layout == "time_fastest") and (step == 1 or not x.is_contiguous())
        got = eng.mel(x).cpu().numpy()
        report(f"{name}.outer{n_outer}", check_mel(name, x.cpu().numpy(), got, fb))


# ------------------------------------------------------------------ vf_istft: istft_frames_kernel (real / imag) + istft_ola_kernel
def istft_lengths(T):
    """A length with T = 1 + n / hop frames, five fewer, the longest with T frames, and the longest vf_istft accepts."""
    n = (T - 1) * HOP + 100
    return {"n": n, "n-5": n - 5, "last_of_T": (T - 1) * HOP + 440, "longest": (T - 1) * HOP + 1024}


def istft_inputs(B, T):
    """real / imag [B, T, 1025] with non-zero imaginary parts at DC and Nyquist (a real signal has none: they are dropped)."""
    g = A._rng(f"istft.{B}.{T}")
    re = (g.standard_normal((B, T, 1025)) * 2).astype(np.float32)
    im = (g.standard_normal((B, T, 1025)) * 2).astype(np.float32)
    im[:, :, 0], im[:, :, 1024] = 3.0, -2.5
    return re, im


def check_istft(name, re, im, length, out):
    """dY = 0 (the spectrum is given): frames as test_gpu_aux.istft_frame_error with phi = 0; overlap-add over the window sum
    (test_gpu_aux.ola_bound), which at the last samples of the longest length is a small Hann tail."""
    ck = G.Checker(name)
    for b in range(re.shape[0]):
        Y = re[b].astype(np.float64) + 1j * im[b].astype(np.float64)
        f64 = R.inverse_frames(Y)
        E = A.istft_frame_error(np.abs(Y), np.zeros(Y.shape))
        y, bnd = A.ola_bound(f64, E, length)
        ck.values("out", np.asarray(out[b], np.float64), y, bnd, np.zeros(1, bool))
    return ck


@pytest.mark.parametrize("which", ["n", "n-5", "last_of_T", "longest"])
@pytest.mark.parametrize("B,T", [(1, 3), (3, 20)])
def test_istft_matches_float64(eng, B, T, which):
    name = f"istft.b{B}.T{T}.{which}"
    length = istft_lengths(T)[which]
    re, im = istft_inputs(B, T)
    dre, dim = torch.from_numpy(re).to(eng.device), torch.from_numpy(im).to(eng.device)
    out = eng.istft(dre, dim, length).cpu().numpy()
    report(name, check_istft(name, re, im, length, out))
    if which == "longest":
        n0 = eng.launch_count()
        with pytest.raises(VL.EngineError) as ei:
            eng.istft(dre, dim, length + 1)
        assert ei.value.code == VL.VF_EINVAL and eng.launch_count() == n0
