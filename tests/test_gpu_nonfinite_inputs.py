"""Out-of-range and non-finite inputs at the public entry points: a call either raises VF_EDEVICE at check_errors, or
every sample it returns is finite.  It never returns a NaN or an infinity with VF_OK.

The restore and vocoder calls never synchronise, so the fp16 range flag (DESIGN.md §3) is how a caller learns that a call's
output is garbage.  The inputs are synthetic: clips scaled to the int16 range (x 32768) and by 1e6, one NaN sample, one +Inf
sample; for the vocoder entry points a mel holding one NaN or one 1e30.  After the failed calls, a clean call on the same
context gives the bits it gave on the fresh context.  Where a kernel clamps instead of flagging (DESIGN.md §3), the call is
VF_OK with finite output, which the property allows, and the test pins it: the STFT front end's power clamp maps a frame
holding a NaN or infinite sample to a finite magnitude, so the mel entry points (GSR restore, resynth, restore_chunks)
return finite audio; the fused SSR back end recomputes that frame's phase, which stays NaN, and raises the flag."""
import pytest
import torch

from oracle import vf_oracle as O
from voicefixer_main_b200 import _lib as VL

pytestmark = pytest.mark.gpu

N = 22050                     # 0.5 s clips
LENGTHS = [N, 13000]          # restore_varlen / restore_batch: two clips of different lengths


def flag(eng):
    try:
        eng.check_errors()
    except VL.EngineError as e:
        return e.code
    return VL.VF_OK


def holds(eng, what, call):
    """Runs call(); -> the check_errors code, after asserting the property."""
    out = call()
    outs = out if isinstance(out, (list, tuple)) else [out]
    code = flag(eng)
    assert code in (VL.VF_OK, VL.VF_EDEVICE), (what, "check_errors", code)
    if code == VL.VF_OK:
        for o in outs:
            assert bool(torch.isfinite(o).all()), (what, "non-finite output with VF_OK", int((~torch.isfinite(o)).sum()))
    return code


def wav_variants(base):
    """(what, wav) of the bad inputs, built from the clean clips `base` [B, n]."""
    out = [("x 32768", base * 32768), ("x 1e6", base * 1e6)]
    x = base.clone()
    x[0, x.shape[1] // 3] = float("nan")
    out.append(("one NaN sample", x))
    x = base.clone()
    x[-1, x.shape[1] // 2] = float("inf")
    out.append(("one +Inf sample", x))
    return out


def mel_variants(base):
    out = []
    for what, v in (("one NaN mel bin", float("nan")), ("one 1e30 mel bin", 1e30)):
        m = base.clone()
        m.view(-1, 128)[5, 40] = v
        out.append((what, m))
    return out


def check_entry(eng, name, call, clean_in, bad_ins):
    """The clean call first (the fresh context's bits), then every bad input, then the clean call again: same bits."""
    want = call(clean_in)
    want = [w.clone() for w in want] if isinstance(want, (list, tuple)) else want.clone()
    assert flag(eng) == VL.VF_OK, (name, "the clean call raised the flag")
    codes = {}
    for what, x in bad_ins:
        codes[what] = holds(eng, f"{name}: {what}", lambda: call(x))
    got = call(clean_in)
    assert flag(eng) == VL.VF_OK, (name, "the clean call after the bad ones raised the flag")
    pairs = zip(want, got) if isinstance(want, list) else [(want, got)]
    for w, g in pairs:
        assert torch.equal(w, g), (name, "clean call after a failed one differs from the fresh context's")
    print(f"{name}: " + ", ".join(f"{k} -> {'VF_EDEVICE' if v else 'VF_OK (finite)'}" for k, v in codes.items()))
    return codes


def _hp(module):
    from voicefixer_main_b200 import default_hparams
    hp = default_hparams()
    sel = hp["task"]["gsr"]["gsr_model"]["voicefixer"]
    for k in ("unet", "unet_small", "bi_gru", "dnn"):
        sel[k] = k == module
    return hp


def _gsr_model(module):
    from voicefixer_main_b200 import VoiceFixer
    from voicefixer_main_b200.weights import make_bigru_state, make_dnn_state, make_state, make_vocoder_state
    if module == "unet":
        sd = make_state(1234)
    else:
        sd = (make_bigru_state if module == "bi_gru" else make_dnn_state)(1234)
        sd.update(make_vocoder_state(seed=1235))
    return VoiceFixer(_hp(module)).load_state_dict(sd).eval().to("cuda:0")


@pytest.mark.parametrize("terms", [1, 3])
@pytest.mark.parametrize("module", ["unet", "bi_gru", "dnn"])
def test_gsr_restore_and_restore_varlen(module, terms):
    model = _gsr_model(module)
    eng = model._engine()
    eng.set_option("vocoder_terms", terms)
    try:
        base = O.synth_clips(2, N, seed=31).cuda()
        codes = check_entry(eng, f"{module}.voc{terms}.restore", lambda x: model.restore(x), base, wav_variants(base))
        assert codes["one NaN sample"] == codes["one +Inf sample"] == VL.VF_OK      # the front end's power clamp
        packed = torch.cat([base[0], base[1, :LENGTHS[1]]])
        bad = [(w, torch.cat([x[0], x[1, :LENGTHS[1]]])) for w, x in wav_variants(base)]
        check_entry(eng, f"{module}.voc{terms}.restore_varlen", lambda x: eng.restore_varlen(x, LENGTHS), packed, bad)
    finally:
        eng.set_option("vocoder_terms", 1)
        model._eng.close()


def test_ssr_restore():
    from voicefixer_main_b200 import SSR_UNet
    from voicefixer_main_b200.weights import make_ssr_state
    model = SSR_UNet().load_state_dict(make_ssr_state(1234)).eval().to("cuda:0")
    try:
        base = O.synth_clips(2, N, seed=32).cuda()
        codes = check_entry(model._engine(), "ssr.restore", lambda x: model.restore(x), base, wav_variants(base))
        assert codes["one NaN sample"] == codes["one +Inf sample"] == VL.VF_EDEVICE    # the ISTFT's NaN phase
    finally:
        model._eng.close()


@pytest.fixture(scope="module")
def vocoder():
    from voicefixer_main_b200.vocoder import Vocoder
    from voicefixer_main_b200.weights import make_vocoder_state
    v = Vocoder().load_state_dict(make_vocoder_state(seed=1235)).eval().to("cuda:0")
    yield v
    v._eng.close()


def _mels(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(B, 1, T, 128, generator=g) ** 4 * 3).cuda()     # linear mel magnitudes


@pytest.mark.parametrize("terms", [1, 3])
def test_vocoder_forward_forward_batch_and_resynth(vocoder, terms):
    eng = vocoder._engine()
    eng.set_option("vocoder_terms", terms)
    try:
        mel = _mels(2, 40, 33)
        codes = check_entry(eng, f"vocoder.voc{terms}.forward", lambda m: vocoder(m), mel, mel_variants(mel))
        assert codes["one NaN mel bin"] == VL.VF_OK          # voc_condition_kernel's clamp
        mels = [mel[0, 0], mel[1, 0, :23]]
        bad = [(w, [m[0, 0], m[1, 0, :23]]) for w, m in mel_variants(mel)]
        check_entry(eng, f"vocoder.voc{terms}.forward_batch", lambda ms: vocoder.forward_batch(ms), mels, bad)
        base = O.synth_clips(2, N, seed=34).cuda()
        check_entry(eng, f"vocoder.voc{terms}.resynth", lambda x: eng.resynth(x), base, wav_variants(base))
    finally:
        eng.set_option("vocoder_terms", 1)


def test_streaming_vocoder_step(vocoder):
    from voicefixer_main_b200.streaming import StreamingVocoder
    eng = vocoder._engine()

    def one_stream(mel):
        sv = StreamingVocoder(vocoder, 16, 4, max_streams=2)
        a = sv.open()
        sv.push(a, mel[0, 0])
        sv.close(a)
        return [o.clone() for o in sv.step().values()]
    mel = _mels(1, 24, 35)          # at most W + 2M frames in one push
    check_entry(eng, "StreamingVocoder.step", one_stream, mel, mel_variants(mel))


def test_restore_chunks():
    model = _gsr_model("unet")
    eng = model._engine()
    try:
        ring = (O.synth_clips(2, 20000, seed=36)).cuda()
        table = [(0, 8000, 0, 0, 0, 20000), (1, 6000, 100, 200, 17000, 20000)]

        def bad(v):
            r = ring.clone()
            r[1, 18000] = v
            return r
        check_entry(eng, "restore_chunks", lambda r: eng.restore_chunks(r, table), ring,
                    [("x 1e6", ring * 1e6), ("one NaN sample", bad(float("nan"))), ("one +Inf sample", bad(float("inf")))])
    finally:
        model._eng.close()
