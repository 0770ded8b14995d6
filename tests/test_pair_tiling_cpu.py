"""Design check for the fused residual-pair kernel (voicefixer_main_b200/csrc/pair_tc.cu), CPU only.

What can be checked here is its tiling arithmetic: tiles of 126
output rows with m0 = t0 - 1, conv_a evaluated on 128 rows m0 .. m0+127 from zero-filled out-of-range input rows,
h forced to zero outside the clip, conv_b evaluated on the 128-row tile with one undefined row on either side (only
rows 1..126 kept), the row masks of the two epilogues.  The emulation below follows the kernel's index expressions
line by line and must reproduce the plain conv pair of the oracle (vocoder_generator's `res.s.i` body)."""
import pytest
import torch
import torch.nn.functional as F

ROWS = 126


def direct_pair(x, wa, ba, wb, bb, dil, slope_h):
    """x [C, L] (one clip): x + conv_b(lrelu(conv_a(lrelu(x)) + ba)) + bb, zero padding - oracle/vf_oracle.py:241-247."""
    h = F.conv1d(F.leaky_relu(x, slope_h)[None], wa, ba, dilation=dil, padding=dil)
    h = F.conv1d(F.leaky_relu(h, slope_h), wb, bb, padding=1)
    return x + h[0]


def tiled_pair(x, wa, ba, wb, bb, dil, slope_h):
    C, L = x.shape
    xa = F.leaky_relu(x, slope_h)                       # the activated plane the previous epilogue stored
    out = torch.full_like(x, float("nan"))
    tiles = (L + ROWS - 1) // ROWS                      # engine.cu: tiles_per_img
    for ti in range(tiles):
        m0 = ti * ROWS - 1                              # pair_tc.cu: m0
        # phase 1: accumulator row j <-> t = m0 + j, taps read rows t + (tap - 1) * dil, out-of-range rows are zero (TMA fill)
        acc1 = torch.zeros(C, 128, dtype=x.dtype)
        for tap in range(3):
            rows = torch.arange(128) + m0 + (tap - 1) * dil
            a = torch.zeros(C, 128, dtype=x.dtype)
            ok = (rows >= 0) & (rows < L)
            a[:, ok] = xa[:, rows[ok]]
            acc1 += wa[:, :, tap] @ a
        # epilogue 1: bias, LeakyReLU, zero outside the clip; h row j sits at buffer row j + 1 of a 130-row tile
        t = torch.arange(128) + m0
        h = F.leaky_relu(acc1 + ba[:, None], slope_h)
        h[:, (t < 0) | (t >= L)] = 0.0
        buf = torch.full((C, 130), float("nan"), dtype=x.dtype)   # buffer rows 0 and 129 are never written
        buf[:, 1:129] = h
        # phase 2: tap view starts at buffer row `tap`
        acc2 = torch.zeros(C, 128, dtype=x.dtype)
        for tap in range(3):
            acc2 += wb[:, :, tap] @ buf[:, tap:tap + 128]
        # epilogue 2: rows 1..126 with t < L are stored
        res = acc2 + bb[:, None]
        for j in range(1, ROWS + 1):
            tt = m0 + j
            if tt < L:
                assert not torch.isnan(res[:, j]).any()   # the undefined edge rows must not leak into kept rows
                out[:, tt] = x[:, tt] + res[:, j]
    return out


@pytest.mark.parametrize("L,dil", [(126, 1), (127, 3), (500, 9), (1000, 27), (253, 243), (64, 1)])
def test_tiled_pair_equals_direct_pair(L, dil):
    g = torch.Generator().manual_seed(L + dil)
    C = 8
    x = torch.randn(C, L, generator=g, dtype=torch.float64)
    wa, wb = (torch.randn(C, C, 3, generator=g, dtype=torch.float64) * 0.3 for _ in range(2))
    ba, bb = (torch.randn(C, generator=g, dtype=torch.float64) for _ in range(2))
    ref = direct_pair(x, wa, ba, wb, bb, dil, 0.1)
    got = tiled_pair(x, wa, ba, wb, bb, dil, 0.1)
    assert not torch.isnan(got).any()
    assert float((ref - got).abs().max()) < 1e-10
