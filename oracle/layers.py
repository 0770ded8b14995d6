"""Float64 references of the conv layers the GEMM kernels run (gemm.cuh, pair_tc.cu), one layer at a time.

Plain torch.float64 functional ops on PyTorch-layout tensors, the layout conversions between them and the kernels'
"rows x channels" planes, the fp16 operand encodings (hi/lo split, the (a, r) residual stream) and the set of output
elements each layer writes.  Used by tests/test_gpu_layers.py (kernel vs reference) and tests/test_layers_cpu.py (the
references against vf_oracle, and the bars against mutated references)."""
import numpy as np
import torch
import torch.nn.functional as F

D = torch.float64


# ------------------------------------------------------------------ layouts
def nchw_to_rows(x):
    """[n, C, H, W] -> [n, H * (W + 1), C]: (h, w) pixels flattened with one zero pad column per image row (gemm.cuh)."""
    n, c, h, w = x.shape
    r = torch.zeros(n, h, w + 1, c, dtype=x.dtype)
    r[:, :, :w] = x.permute(0, 2, 3, 1)
    return r.reshape(n, h * (w + 1), c)


def rows_to_nchw(r, h, w, c_off=0, c=None):
    """Inverse of nchw_to_rows (the pad column is dropped); channels [c_off, c_off + c) of a concat buffer."""
    n, _, ld = r.shape
    c = ld - c_off if c is None else c
    return r[:, :h * (w + 1), c_off:c_off + c].reshape(n, h, w + 1, c)[:, :, :w].permute(0, 3, 1, 2)


def ncl_to_rows(x):
    """[n, C, L] -> [n, L, C]."""
    return x.permute(0, 2, 1)


def rows_to_ncl(r, c_off=0, c=None):
    c = r.shape[2] - c_off if c is None else c
    return r[:, :, c_off:c_off + c].permute(0, 2, 1)


# ------------------------------------------------------------------ fp16 operand encodings
def fp16(x):
    """Round to fp16 (nearest even) and back to float64."""
    return torch.as_tensor(x, dtype=D).to(torch.float32).to(torch.float16).to(D)


def split_hi_lo(x):
    """hi = fp16_rn(x), lo = fp16_rn(x - hi) (x is an fp32 value: the difference is exact)."""
    x = torch.as_tensor(x, dtype=D)
    hi = fp16(x)
    return hi, fp16(x - hi)


def ar_unact(a, s):
    """U(a) = min(a, a * fp16(1 / s)) evaluated in fp16 (ptx.cuh ar_unact)."""
    inv = np.float16(1.0 / s)
    a16 = np.asarray(a, np.float16)
    with np.errstate(over="ignore"):
        return np.minimum(a16, (a16 * inv).astype(np.float16))


def ar_encode(x, s):
    """The (a, r) pair of an fp32 residual stream x (gemm.cuh): a = fp16(lrelu_s(x)), r = fp16(x - U(a))."""
    x = np.asarray(x, np.float32)
    a = np.maximum(x, x * np.float32(s)).astype(np.float16)
    r = (x - ar_unact(a, s).astype(np.float32)).astype(np.float16)
    return a, r


def ar_decode(a, r, s):
    """x = U(a) + r."""
    return ar_unact(a, s).astype(np.float64) + np.asarray(r, np.float16).astype(np.float64)


def to_bits(h):
    """fp16 values -> their uint16 bit patterns (numpy)."""
    return np.asarray(torch.as_tensor(h).to(torch.float16).numpy()).view(np.uint16)


def from_bits(b):
    """uint16 bit patterns -> float64 (numpy)."""
    return np.asarray(b, np.uint16).view(np.float16).astype(np.float64)


# ------------------------------------------------------------------ the layers (PyTorch layouts, float64)
def conv2d(x, w, sc_x=None, sc_w=None, sc_b=None):
    """Conv2d 3x3 pad 1 no bias (modules.py:235-243), plus the 1x1 shortcut with bias (modules.py:245-247)."""
    y = F.conv2d(x.to(D), w.to(D), padding=1)
    if sc_w is not None:
        y = y + F.conv2d(sc_x.to(D), sc_w.to(D)[:, :, None, None], sc_b.to(D))
    return y


def conv_transpose2d(x, w, both):
    """ConvTranspose2d k3 s2 no bias, then the decoder's prune (modules.py:205-209): the last time row, and with
    both=True the last frequency column too."""
    y = F.conv_transpose2d(x.to(D), w.to(D), stride=2)
    return y[:, :, :-1, :-1] if both else y[:, :, :-1, :]


def conv1d(x, w, b, dilation=1, centered=True):
    """Conv1d, tap i at row offset (i - (k - 1) // 2) * dilation with zero padding when centred (an even k reaches one
    tap further right), at offset i otherwise (the caller padded the input)."""
    k = w.shape[2]
    x = x.to(D)
    if centered:
        x = F.pad(x, ((k - 1) // 2 * dilation, (k - 1 - (k - 1) // 2) * dilation))
    return F.conv1d(x, w.to(D), None if b is None else b.to(D), dilation=dilation)


def conv_transpose1d(x, w, b, s):
    """ConvTranspose1d kernel 2 s, stride s, padding s // 2 + s % 2, output_padding s % 2 (the vocoder's up-sampler)."""
    return F.conv_transpose1d(x.to(D), w.to(D), None if b is None else b.to(D), stride=s, padding=s // 2 + s % 2,
                              output_padding=s % 2)


def lrelu(x, s):
    return torch.where(x > 0, x, x * s)


def activate(x, act, slope):
    """gemm.cuh: 0 none, 1 LeakyReLU(slope), 2 ELU."""
    if act == 1:
        return lrelu(x, slope)
    if act == 2:
        return torch.where(x > 0, x, torch.expm1(x))
    return x


def pair(xa, x, wa, ba, wb, bb, dil, slope_h, fp16_h=False):
    """Fused pair (pair_tc.cu) on conv_a's input xa (the activated plane) and the stream x:
    y = x + conv_b(h) + bb, h = lrelu(conv_a(xa) + ba, slope_h) (fp16-rounded with fp16_h).  Returns (y, h)."""
    h = lrelu(conv1d(xa, wa, ba, dil), slope_h)
    if fp16_h:
        h = fp16(h)
    return x.to(D) + conv1d(h, wb, bb, 1), h


# ------------------------------------------------------------------ write sets
def write_rows_plain(n_img, out_img_rows, ld, out_row0, rows, c_off, cout):
    """MAP_PLAIN: GEMM row r of every image -> output row out_row0 + r, channels [c_off, c_off + cout)."""
    m = np.zeros((n_img, out_img_rows, ld), bool)
    m[:, out_row0:out_row0 + rows, c_off:c_off + cout] = True
    return m


def write_rows_convt2d(n_img, out_img_rows, ld, H, Wp, ct_out_wp, c_off, cout):
    """MAP_CONVT2D: every (2h + ph, 2w + pw) with 2w + pw < ct_out_wp; the column past the pitch is dropped."""
    m = np.zeros((n_img, out_img_rows, ld), bool)
    for ph in range(2):
        for pw in range(2):
            cols = 2 * np.arange(Wp) + pw
            cols = cols[cols < ct_out_wp]
            rr = ((2 * np.arange(H)[:, None] + ph) * ct_out_wp + cols[None, :]).ravel()
            m[:, rr, c_off:c_off + cout] = True
    return m


def write_rows_convt1d(n_img, out_img_rows, ld, out_row0, rows_in, s, out_rows_valid, c_off, cout):
    """MAP_CONVT1D: t = s * r + phase - pad for GEMM rows r < rows_in, kept when 0 <= t < out_rows_valid."""
    m = np.zeros((n_img, out_img_rows, ld), bool)
    pad = s // 2 + s % 2
    t = (s * np.arange(rows_in)[:, None] + np.arange(s)[None, :] - pad).ravel()
    t = t[(t >= 0) & (t < out_rows_valid)]
    m[:, out_row0 + t, c_off:c_off + cout] = True
    return m
