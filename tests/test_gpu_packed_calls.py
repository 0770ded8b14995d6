"""The packed-set entry points' sub-batch split and their context-owned scratch (csrc/standalone.cu): each call launches
exactly the kernels of the sub-batches its split rule gives, and calls on two streams that share one scratch, the second
growing it with no host synchronisation in between, give the bits of the same calls run alone."""
import math

import numpy as np
import pytest
import torch
from scipy import signal

from voicefixer_main_b200 import lowpass as LP

pytestmark = pytest.mark.gpu

MIN61 = 44100 * 61                  # 6101 frames: three such pairs pass the 16384-frame cap of a scoring sub-batch
SCORE_ROWS, IIR_ROWS = 128, 64      # SCORE_MAX_IMAGES, IIR_MAX_ROWS
SCORE_CAP_FRAMES, IIR_CAP = 16384, 1 << 24


def _engine():
    from voicefixer_main_b200.model import Engine
    e = Engine("cuda:0")
    e.load_state({}, need=())
    return e


@pytest.fixture(scope="module")
def eng():
    e = _engine()
    yield e
    e.close()
    torch.cuda.empty_cache()


def split(sizes, max_rows, cap=math.inf):
    """The split rule: a sub-batch takes items until it holds max_rows, or until the next item would take its size past
    cap (an item larger than cap runs alone) -> the items of each sub-batch."""
    subs, size = [[]], 0
    for i, n in enumerate(sizes):
        if len(subs[-1]) == max_rows or (subs[-1] and size + n > cap):
            subs.append([])
            size = 0
        subs[-1].append(i)
        size += n
    return subs


def stoi_tiles(n):
    """Correlation tiles of a pair padded to n samples (kernels.cuh: stoi_len10, stoi_frames, stoi_tiles)."""
    n10 = (n * 100 + 440) // 441
    frames = (n10 - 256 + 127) // 128 if n10 > 256 else 0
    return ((frames - 30) * 15 + 255) // 256 if frames > 30 else 0


def _noise(n, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return (0.1 * torch.randn(n, generator=g, dtype=torch.float64)).to(dtype).cuda()


def _launches(eng, call):
    n0 = eng.launch_count()
    out = call()
    torch.cuda.synchronize()
    return eng.launch_count() - n0, out


def _filters(k):
    sos = [signal.butter(4, 0.05 + 0.04 * f, output="sos") for f in range(k)]
    return sos, [signal.sosfilt_zi(s) for s in sos]


# ------------------------------------------------------------------------------------------------ exact launch counts
def test_score_varlen_launches_ten_per_sub_batch(eng):
    lengths = [3000] * 129 + [MIN61] * 3 + [5000]        # the row cap, then the frame cap
    subs = split([1 + n // 441 for n in lengths], SCORE_ROWS, SCORE_CAP_FRAMES)
    assert [len(s) for s in subs] == [128, 3, 2]
    x, y = _noise(sum(lengths), 1), _noise(sum(lengths), 2)
    n, _ = _launches(eng, lambda: eng.score_varlen(x, lengths, y, lengths))
    assert n == 10 * len(subs)


def test_score_time_varlen_launches_eight_per_sub_batch_seven_without_tiles(eng):
    lengths = [2000] * 129 + [MIN61] * 3 + [2000]         # 2000 samples: 2 STOI frames, no correlation tile
    subs = split(lengths, SCORE_ROWS, SCORE_CAP_FRAMES * 441)
    assert [len(s) for s in subs] == [128, 3, 2]
    x, y = _noise(sum(lengths), 3), _noise(sum(lengths), 4)
    n, _ = _launches(eng, lambda: eng.score_time_varlen(x, lengths, y, lengths))
    assert n == sum(8 if sum(stoi_tiles(lengths[i]) for i in s) else 7 for s in subs) == 7 + 8 + 8


def test_sosfiltfilt_varlen_launches_six_per_sub_batch_and_one_per_six_filters(eng):
    sos, zi = _filters(7)
    lengths = [300] * 65 + [5_000_000] * 4 + [300]        # the row cap, then the 2^24 extended-sample cap
    rows = [i % 7 for i in range(len(lengths))]
    subs = split([n + 2 * LP.padlen(sos[f]) for n, f in zip(lengths, rows)], IIR_ROWS, IIR_CAP)
    assert [len(s) for s in subs] == [64, 4, 2]
    x = _noise(sum(lengths), 5, torch.float64)
    n, _ = _launches(eng, lambda: eng.sosfiltfilt_varlen(x, lengths, sos, zi, rows))
    assert n == 6 * len(subs) + 2


def test_resample_poly_f64_varlen_launches_one_per_64_rows(eng):
    taps = torch.ones(5, dtype=torch.float64, device="cuda")
    x = _noise(130 * 100, 6, torch.float64)
    n, _ = _launches(eng, lambda: eng.resample_poly_f64_varlen(x, [100] * 130, [(1, 2, taps)], [0] * 130, [50] * 130))
    assert n == len(split([0] * 130, IIR_ROWS)) == 3


def test_ssim_launches_two_per_128_images(eng):
    x = _noise(130 * 7 * 7, 7).view(130, 7, 7)
    n, _ = _launches(eng, lambda: eng.ssim(x, x))
    assert n == 2 * len(split([0] * 130, SCORE_ROWS)) == 4


def test_metric_spectrogram_launches_one_per_128_clips_and_one_for_the_mel(eng):
    x = _noise(130 * 2000, 8)
    for want_mel in (False, True):
        n, _ = _launches(eng, lambda: eng.metric_spectrogram(x, [2000] * 130, want_mel=want_mel))
        assert n == len(split([0] * 130, SCORE_ROWS)) + want_mel == 2 + want_mel


# ----------------------------------------------------------------------------------- one scratch shared across streams
def _scratch_call(name):
    """(run(engine, lengths), small lengths, large lengths) of a scratch user: the large call needs more scratch."""
    small, large = [44100, 30000], [441000] * 3 + [100000]
    if name == "iir":
        sos, zi = _filters(1)
        x = {k: _noise(sum(v), 9, torch.float64) for k, v in (("small", small), ("large", large))}
        return lambda e, k, n: e.sosfiltfilt_varlen(x[k], n, sos, zi, [0] * len(n)), small, large
    est = {k: _noise(sum(v), 10) for k, v in (("small", small), ("large", large))}
    tgt = {k: _noise(sum(v), 11) for k, v in (("small", small), ("large", large))}
    fn = "score_varlen" if name == "score" else "score_time_varlen"
    return lambda e, k, n: getattr(e, fn)(est[k], n, tgt[k], n), small, large


@pytest.mark.parametrize("name", ["score", "time_score", "iir"])
def test_two_streams_share_one_scratch(eng, name):
    run, small, large = _scratch_call(name)
    alone = [run(eng, "small", small), run(eng, "large", large)]
    torch.cuda.synchronize()
    for same_stream in (False, True):
        e = _engine()                                     # an empty scratch: the large call grows it
        a, b = torch.cuda.Stream(), torch.cuda.Stream()
        a.wait_stream(torch.cuda.current_stream())
        b.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(a):
            got_small = run(e, "small", small)
        with torch.cuda.stream(a if same_stream else b):
            got_large = run(e, "large", large)
        torch.cuda.synchronize()
        assert torch.equal(got_small, alone[0]), same_stream
        assert torch.equal(got_large, alone[1]), same_stream
        e.close()
