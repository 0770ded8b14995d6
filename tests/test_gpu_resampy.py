"""librosa 0.8's resample(res_type="kaiser_best" / "kaiser_fast") on the GPU (vf_resample_sinc_varlen, edges.resample and the
res_type of the handlers and AudioMetrics) against the CPU restatement of oracle/resampy.py, bit for bit."""
import numpy as np
import pytest
import torch

import oracle_16k as R16
from oracle import resampy as R
from oracle import vf_oracle as O
from test_gpu_scoring import _close
from test_gpu_scoring16k import _pairs
from voicefixer_main_b200 import _lib as L

pytestmark = pytest.mark.gpu

RATE_PAIRS = [(16000, 44100), (44100, 16000), (8000, 44100), (22050, 44100), (48000, 44100), (44100, 48000)]
# 3 and 40 samples: shorter than the filter's half, both wing bounds bind; 147: 44.1 -> 48 kHz pads a zero tail
LENGTHS = [3, 40, 147, 1000, 16001, 44100 * 3 + 7]


@pytest.fixture(scope="module")
def eng():
    from voicefixer_main_b200.model import Engine
    e = Engine("cuda:0")
    yield e
    e.close()
    torch.cuda.empty_cache()


def _sig(n, seed):
    return (0.3 * np.random.default_rng(seed).standard_normal(n)).astype(np.float32)


def _bits(a):
    return np.asarray(a, np.float32).view(np.int32)


def _launches(eng, call):
    n0 = eng.launch_count()
    out = call()
    torch.cuda.synchronize()
    return eng.launch_count() - n0, out


@pytest.mark.parametrize("res_type", list(R.FILTERS))
@pytest.mark.parametrize("orig_sr, target_sr", RATE_PAIRS)
def test_rows_equal_the_restatement_bit_for_bit(eng, res_type, orig_sr, target_sr):
    from voicefixer_main_b200.edges import resample
    xs = [_sig(n, 10 + i) for i, n in enumerate(LENGTHS) if int(n * target_sr / orig_sr) >= 1]
    launches, ys = _launches(eng, lambda: resample(eng, xs, orig_sr, target_sr, res_type))
    assert launches == 1
    for x, y in zip(xs, ys):
        want = R.resample(x, orig_sr, target_sr, res_type)
        got = y.cpu().numpy()
        assert got.shape == want.shape and np.array_equal(_bits(got), _bits(want)), (len(x), res_type)
    eng.check_errors()


def test_row_bits_do_not_depend_on_batch_or_position(eng):
    from voicefixer_main_b200.edges import resample
    xs = [_sig(n, 40 + i) for i, n in enumerate([40, 5000, 16001, 777])]
    rates = [16000, 22050, 48000, 8000]
    full = resample(eng, xs, rates, 44100, "kaiser_best")
    order = [3, 1, 0, 2]
    perm = resample(eng, [xs[i] for i in order], [rates[i] for i in order], 44100, "kaiser_best")
    for k, i in enumerate(order):
        assert torch.equal(perm[k], full[i])
        assert torch.equal(resample(eng, [xs[i]], rates[i], 44100, "kaiser_best")[0], full[i])
    same = resample(eng, [xs[0]], 44100, 44100, "kaiser_best")[0]           # equal rates: librosa returns y unchanged
    assert torch.equal(same.cpu(), torch.from_numpy(xs[0]))


def _einval(call):
    with pytest.raises(L.EngineError) as e:
        call()
    assert e.value.code == L.VF_EINVAL


def test_abi_rejections(eng):
    from voicefixer_main_b200.edges import _sinc_filter
    x = torch.from_numpy(_sig(1000, 1)).cuda()
    tab, ratio, num_table = _sinc_filter(eng, "kaiser_fast", 16000, 44100)
    good = (tab, ratio, num_table)
    call = eng.resample_sinc_varlen
    n0 = eng.launch_count()
    _einval(lambda: call(x, [1000], [good], [1], [2757]))                        # no filter 1
    _einval(lambda: call(x, [1000], [(tab, 0.0, num_table)], [0], [10]))         # ratio 0
    _einval(lambda: call(x, [1000], [(tab, float("nan"), num_table)], [0], [10]))
    _einval(lambda: call(x, [1000], [(tab, ratio, 0)], [0], [10]))               # num_table 0
    _einval(lambda: call(x, [1000], [(tab, 1e-4, num_table)], [0], [10]))        # index step int(1e-4 * 128) = 0
    _einval(lambda: call(x, [1000], [(tab[:num_table], ratio, num_table)], [0], [10]))   # table of num_table entries
    _einval(lambda: call(x[:1], [1], [(tab, 0.5, num_table)], [0], [1]))         # int(1 * 0.5) = 0 samples
    _einval(lambda: call(x, [1000, 0], [good, good], [0, 0], [10, 10]))          # an empty row
    lib = eng.lib
    off = (L.c_int64 * 2)(0, 1000)
    out = torch.empty(2757, device="cuda")
    r = (L.c_double * 1)(ratio)
    k = (L.c_int * 1)(num_table)
    rows = (L.c_int * 1)(0)
    t_off = (L.c_int64 * 2)(0, tab.shape[0] - 1)
    rc = lib.vf_resample_sinc_varlen(eng.ctx, x.data_ptr(), off, 1, tab.data_ptr() + 8, t_off, r, k, 1, rows, out.data_ptr(),
                                     (L.c_int64 * 2)(0, 2757), None)
    assert rc == L.VF_EINVAL                                                       # tables not 16-byte aligned
    rc = lib.vf_resample_sinc_varlen(eng.ctx, x.data_ptr(), off, 1, tab.data_ptr(), t_off, r, k, 1, rows, out.data_ptr(),
                                     (L.c_int64 * 2)(0, 2757), None)
    assert rc == L.VF_OK
    torch.cuda.synchronize()
    assert eng.launch_count() - n0 == 1                                            # only the good call launched
    eng.check_errors()


def test_one_launch_per_512_rows(eng):
    from voicefixer_main_b200.edges import resample
    xs = [_sig(50 + i, i) for i in range(513)]
    launches, ys = _launches(eng, lambda: resample(eng, xs, 16000, 44100, "kaiser_fast"))
    assert launches == 2
    for i in (0, 511, 512):
        assert np.array_equal(_bits(ys[i].cpu().numpy()), _bits(R.resample(xs[i], 16000, 44100, "kaiser_fast")))


# ------------------------------------------------------------------------------------------------------- the handlers
def _pcm(n, seed):
    return O.to_int16(O.synth_clips(1, n, seed=seed)[0].clamp(-0.99, 0.99).numpy())


def _read(path):
    with open(path, "rb") as f:
        return f.read()


def _on_restatement(H, monkeypatch, res_type):
    """H.load_wav replaced by the restatement's resampling of the decoded file."""
    from voicefixer_main_b200.handler import read_pcm16

    def load(path, sample_rate=44100, engine=None, res_type_=None, **kw):
        x, rate = read_pcm16(path)
        return R.resample(x, rate, sample_rate, res_type)
    monkeypatch.setattr(H, "load_wav", load)


def _handler_on_restatement(H, model, tmp_path, monkeypatch, res_type):
    src, tgt = str(tmp_path / "in.wav"), str(tmp_path / "tgt.wav")
    H.save_pcm16(_pcm(40000, 7), src, sample_rate=16000)
    H.save_pcm16(_pcm(40000, 8), tgt, sample_rate=16000)
    got = H.handler(src, str(tmp_path / "got.wav"), tgt, ckpt=None, device=model.device, meta={"res_type": res_type})
    with monkeypatch.context() as mp:
        _on_restatement(H, mp, res_type)
        want = H.handler(src, str(tmp_path / "want.wav"), tgt, ckpt=None, device=model.device, meta={})
    model._engine().check_errors()
    assert got and got == want
    assert _read(tmp_path / "got.wav") == _read(tmp_path / "want.wav")
    poly = H.handler(src, str(tmp_path / "poly.wav"), tgt, ckpt=None, device=model.device, meta={})
    assert _read(tmp_path / "poly.wav") != _read(tmp_path / "got.wav")       # the default path is resample_poly's


MIXED = [(16000, 16000, True), (22050, 22050, False), (44100, 30000, True), (48000, 50000, True), (16000, 7000, False)]


def _batch_equals_handler(H, model, tmp_path, monkeypatch, res_type):
    import os
    os.makedirs(tmp_path / "one")
    os.makedirs(tmp_path / "batch")
    items = []
    for i, (rate, n, has_target) in enumerate(MIXED):
        src = str(tmp_path / f"in{i}.wav")
        H.save_pcm16(_pcm(n, 300 + i), src, sample_rate=rate)
        tgt = None
        if has_target:
            tgt = str(tmp_path / f"tgt{i}.wav")
            H.save_pcm16(_pcm(n, 400 + i), tgt, sample_rate=rate)
        items.append((src, f"o{i}.wav", tgt))
    meta = {"res_type": res_type}
    one = [H.handler(s, str(tmp_path / "one" / o), t, ckpt=None, device=model.device, meta=meta) for s, o, t in items]
    eng = model._engine()
    calls = []
    inner = eng.resample_sinc_varlen
    monkeypatch.setattr(eng, "resample_sinc_varlen", lambda *a: calls.append(len(a[1])) or inner(*a))
    batch = H.handler_batch([(s, str(tmp_path / "batch" / o), t) for s, o, t in items], ckpt=None, device=model.device,
                            meta=meta)
    eng.check_errors()
    assert calls == [6]                    # 4 inputs and 2 targets not at 44.1 kHz, in one call
    for (_, o, _), a, b in zip(items, one, batch):
        assert _read(tmp_path / "one" / o) == _read(tmp_path / "batch" / o), o
        assert a == b, o
    assert [bool(m) for m in one] == [t for _, _, t in MIXED]


@pytest.fixture(scope="module")
def vf_model(state):
    from voicefixer_main_b200 import VoiceFixer
    m = VoiceFixer().load_state_dict(state).eval().to("cuda:0")
    yield m
    m._engine().check_errors()
    m._eng.close()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def ssr_model():
    from voicefixer_main_b200 import SSR_UNet
    from voicefixer_main_b200.weights import make_ssr_state
    m = SSR_UNet().load_state_dict(make_ssr_state(1234)).eval().to("cuda:0")
    yield m
    m._engine().check_errors()
    m._eng.close()
    torch.cuda.empty_cache()


def test_handler_is_the_segment_loop_on_the_restatement(vf_model, tmp_path, monkeypatch):
    from voicefixer_main_b200 import handler as H
    monkeypatch.setattr(H, "model", vf_model)
    _handler_on_restatement(H, vf_model, tmp_path, monkeypatch, "kaiser_best")


def test_handler_batch_equals_handler_with_one_resample_call(vf_model, tmp_path, monkeypatch):
    from voicefixer_main_b200 import handler as H
    monkeypatch.setattr(H, "model", vf_model)
    _batch_equals_handler(H, vf_model, tmp_path, monkeypatch, "kaiser_best")


def test_unet_handler_is_the_segment_loop_on_the_restatement(ssr_model, tmp_path, monkeypatch):
    from voicefixer_main_b200 import handler_unet as HU
    monkeypatch.setattr(HU, "model", ssr_model)
    _handler_on_restatement(HU, ssr_model, tmp_path, monkeypatch, "kaiser_fast")


def test_unet_handler_batch_equals_handler_with_one_resample_call(ssr_model, tmp_path, monkeypatch):
    from voicefixer_main_b200 import handler_unet as HU
    monkeypatch.setattr(HU, "model", ssr_model)
    _batch_equals_handler(HU, ssr_model, tmp_path, monkeypatch, "kaiser_fast")


# ------------------------------------------------------------------------------------------------------ AudioMetrics
def test_16k_scores_of_44k_ests_use_the_restatements_est(tmp_path):
    from voicefixer_main_b200.edges import AudioMetrics
    from voicefixer_main_b200.handler import read_pcm16
    from voicefixer_main_b200.model import Engine
    e = Engine("cuda:0")
    e.load_state({}, need=())
    am = AudioMetrics(e, rate=16000, res_type="kaiser_best")
    pairs = _pairs(tmp_path, [(16000, 16000, 0), (48000, 48000, 0), (30001, 30001, 6000)], est_rate=44100)
    batch = am.evaluation_batch(pairs)
    for (pe, pt), got in zip(pairs, batch):
        e16 = R.resample(read_pcm16(pe)[0], 44100, 16000, "kaiser_best")
        _close(got, R16.evaluation(pe, pt, est=e16))
        assert got == am.evaluation(pe, pt)
    assert batch != AudioMetrics(e, rate=16000).evaluation_batch(pairs)          # resample_poly's est scores differently
    e.check_errors()
    e.close()
    torch.cuda.empty_cache()
