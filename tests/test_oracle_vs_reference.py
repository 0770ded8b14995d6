"""Pin the restatement in oracle/vf_oracle.py against the reference's own modules: their outputs on seeded inputs are
stored in tests/golden/ref_oracle.npz and ref_unet.npz (oracle/make_ref_vectors.py, run where the reference exists)."""
import numpy as np
import pytest
import torch

from oracle import vf_oracle as O
from oracle.make_ref_vectors import log_helper_inputs, small_input, unet_inputs
from conftest import load_golden


@pytest.fixture(scope="module")
def ref():
    return load_golden("ref_oracle.npz")


@pytest.fixture(scope="module")
def ref_unet():
    return load_golden("ref_unet.npz")


def test_mel_filterbank_bit_identical(ref):
    fb = O.mel_filterbank()
    ref_fb = torch.zeros(tuple(int(s) for s in ref["fb_shape"]))
    ref_fb[torch.from_numpy(ref["fb_rows"]).long(), torch.from_numpy(ref["fb_cols"]).long()] = torch.from_numpy(ref["fb_vals"])
    assert torch.equal(ref_fb, fb)
    assert int((fb != 0).sum()) == 2018            # SURVEY.md 8(a) a5 probe


def test_log_helpers_match_reference(ref):
    x, y = log_helper_inputs()
    assert torch.equal(torch.from_numpy(ref["log_x"]), x) and torch.equal(torch.from_numpy(ref["log_y"]), y)
    assert torch.equal(torch.from_numpy(ref["log_to"]), O.to_log(x))
    assert torch.equal(torch.from_numpy(ref["log_from"]), O.from_log(y))
    with pytest.raises(AssertionError):             # the reference's to_log asserts on negative input as well
        O.to_log(-x - 1)


def test_unet_restatement_matches_reference(ref_unet, state):
    for i, mel in enumerate(unet_inputs()):         # T = 64 (multiple of 64), 101 (the reference smoke shape), 130 (ragged)
        t = mel.shape[2]
        with torch.no_grad():
            mine = O.generator_forward(state, mel)
        want = torch.from_numpy(ref_unet[f"unet_out{i}"])
        assert want.shape == mine.shape == (2, 1, t, 128)
        assert float((want - mine).abs().max()) < 2e-5


def test_handler_restatement_matches_reference(ref_unet, state):
    wav = O.synth_clips(2, 30000, seed=9)
    with torch.no_grad():
        mine = O.restore(state, wav, seg_samples=12000)                 # 3 segments, last ragged
    want = torch.from_numpy(ref_unet["handler_out"])
    assert want.shape == mine.shape == wav.shape
    assert float((want - mine).abs().max()) < 1e-5


def test_trim_center_matches_reference(ref):
    for (le, lr), start in zip(ref["trim_cases"], ref["trim_starts"]):
        est = torch.arange(float(le))[None, None]
        assert torch.equal(torch.arange(float(start), float(start) + lr)[None, None], O.trim_center(est, int(lr)))


def test_unet_v2_ssr_restatement_matches_reference(ref, state):
    """Next path (SURVEY.md 8(f) row 1): models/components/unet_v2.py vs the restatement."""
    from voicefixer_main_b200.arch import UNET_PREFIX
    ssr = {k.replace(UNET_PREFIX, "generator.unet."): v for k, v in state.items() if k.startswith(UNET_PREFIX)}
    for n in (63 * 441, 70 * 441 + 17):                   # T = 64 (no time padding) and T = 71 -> T' = 128
        wav = O.synth_clips(1, n, seed=n)[:, None, :]
        with torch.no_grad():
            mine = O.ssr_forward(ssr, wav)
        want = torch.from_numpy(ref[f"ssr_out{n}"])
        assert want.shape == mine.shape == (1, 1, n)
        assert float((want - mine).abs().max()) < 1e-5


def test_unet_small_is_the_same_network(ref, state):
    """SURVEY.md 8(f) row 4: in this reference the *Res1B blocks of models/components/unet_small.py hold four ConvBlockRes
    each (modules.py:112-165), i.e. the layers and keys of unet.py - the generator checked bit for bit that its output
    equals unet.py's on this input before storing it; the product maps `unet_small: true` onto the same plan."""
    mel = small_input()
    with torch.no_grad():
        c = O.generator_forward(state, mel)
    a = torch.from_numpy(ref["small_out"])
    assert float((a - c).abs().max()) < 2e-5
