"""Float64 references of the kernels on the hot path, one launch at a time.

- The conv layers the GEMM kernels run (gemm.cuh, pair_tc.cu): plain torch.float64 functional ops on PyTorch-layout
  tensors, the layout conversions between them and the kernels' "rows x channels" planes, the fp16 operand encodings
  (hi/lo split, the (a, r) residual stream) and the set of output elements each layer writes.  Used by
  tests/test_gpu_layers.py (kernel vs reference) and tests/test_layers_cpu.py (the references against vf_oracle, and the
  bars against mutated references).
- The non-GEMM kernels of the same launch chains (aux.cu, istft.cu): the UNet's first layer with its input padding,
  pooling, the vocoder conditioning and its low-band sums, reflection padding, the tail conv, peak normalise + trim and the
  fused ISTFT of the SSR back end.  Used by tests/test_gpu_aux.py and tests/test_aux_cpu.py in the same two ways.
- The STFT + mel front end (frontend.cu) and the stand-alone mel and ISTFT: used by tests/test_gpu_frontend.py and
  tests/test_frontend_cpu.py."""
import numpy as np
import torch
import torch.nn.functional as F

D = torch.float64


# ------------------------------------------------------------------ layouts
def nchw_to_rows(x):
    """[n, C, H, W] -> [n, H * (W + 1), C]: (h, w) pixels flattened with one zero pad column per image row (gemm.cuh)."""
    n, c, h, w = x.shape
    r = torch.zeros(n, h, w + 1, c, dtype=x.dtype, device=x.device)
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


BN_EPS = 1e-5


def linear(x, w, b):
    """nn.Linear on the last axis in float64: x [..., K], w [N, K], b [N]."""
    return torch.as_tensor(x, dtype=D) @ torch.as_tensor(w, dtype=D).T + torch.as_tensor(b, dtype=D)


def bn_scalar(bn):
    """Eval-mode BatchNorm2d(1) of (weight, bias, running_mean, running_var) as (s, t) in float64: bn(x) = s x + t."""
    w, b, m, v = (float(q) for q in np.asarray(bn, np.float64))
    s = w / np.sqrt(v + BN_EPS)
    return s, b - m * s


def bn_fold(w, b, bn, shift_sum=True):
    """Linear(bn(x)) = x W'^T + b' with W' = s W, b' = b + t * sum_k W[:, k], in float64 (the loader's pack_linear with its
    input affine).  shift_sum=False is a known-wrong fold (b' = b + t), for tests of the GPU test's bar."""
    s, t = bn_scalar(bn)
    w, b = torch.as_tensor(w, dtype=D), torch.as_tensor(b, dtype=D)
    return s * w, b + t * (w.sum(1) if shift_sum else 1.0)


def gru_ih_bias(b_ih, b_hh, hidden=256, merge_n=False):
    """The input projection's bias of a bidirectional GRU layer, [2 * 3 H] (forward, reverse): b_ih + (b_hr, b_hz, 0).
    merge_n=True also adds b_hn (known-wrong: torch.nn.GRU applies it inside r * (W_hn h + b_hn))."""
    b = torch.as_tensor(b_ih, dtype=D).reshape(2, 3 * hidden).clone()
    bh = torch.as_tensor(b_hh, dtype=D).reshape(2, 3 * hidden)
    n = 3 * hidden if merge_n else 2 * hidden
    b[:, :n] += bh[:, :n]
    return b.reshape(-1)


def fma32(x, s, t):
    """fmaf(x, s, t) for float32 arrays: x s + t rounded once to float32.  x s is exact in float64; the float64 sum is
    corrected with its exact error (two-sum), which decides the float32 rounding when the sum sits on a float32 midpoint."""
    x, s, t = (np.asarray(q, np.float32).astype(np.float64) for q in (x, s, t))
    p = x * s
    hi = p + t
    bp = hi - t
    err = (p - bp) + (t - (hi - bp))
    y = hi.astype(np.float32)
    # hi on a float32 midpoint: the nearer neighbour on err's side, not the tie-to-even astype picked
    lo_n = np.nextafter(y, np.float32(-np.inf)).astype(np.float64)
    hi_n = np.nextafter(y, np.float32(np.inf)).astype(np.float64)
    y64 = y.astype(np.float64)
    below = (hi == (y64 + lo_n) / 2) & (err < 0)
    above = (hi == (y64 + hi_n) / 2) & (err > 0)
    y = np.where(below, np.nextafter(y, np.float32(-np.inf)), y)
    y = np.where(above, np.nextafter(y, np.float32(np.inf)), y)
    return y.astype(np.float32)


def affine_planes(x, scale, shift, valid_rows=None, fused=True):
    """The bi_gru / dnn input planes (gru_tc.cu affine_planes_kernel) of x [n, T, C] float32: y = fmaf(x, scale, shift),
    hi = fp16(y), lo = fp16(y - hi) as uint16 bits [2, n, T, C]; rows t >= valid_rows[b] are zeros.  fused=False rounds the
    product before the add (known-wrong, for tests of the GPU test's bar)."""
    x = np.asarray(x, np.float32)
    if fused:
        y = fma32(x, np.float32(scale), np.float32(shift))
    else:
        y = (x * np.float32(scale)).astype(np.float32) + np.float32(shift)
    if valid_rows is not None:
        for b, v in enumerate(valid_rows):
            y[b, int(v):] = 0
    hi = y.astype(np.float16)
    lo = (y - hi.astype(np.float32)).astype(np.float16)
    return np.stack([hi.view(np.uint16), lo.view(np.uint16)])


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


# ------------------------------------------------------------------ the non-GEMM kernels (aux.cu, istft.cu)
def unet_first(x, Tp, bn1_scale, bn1_shift, w1, bn2_scale, bn2_shift, w_sc, b_sc, slope=0.01):
    """encoder_block1.conv_block1 up to its second BN (unet.py:75-78, modules.py:263-271): x [n, T, W + 1] (the last bin is
    dropped) padded with zero input rows to Tp, then h = lrelu(bn1(x)), y = conv3x3(h), a = lrelu(bn2(y)) and the 1x1
    shortcut r = w_sc x + b_sc.  Returns (h, y, a, r) as [n, C, Tp, W] (h: [n, 1, Tp, W])."""
    x = torch.as_tensor(x, dtype=D)[:, None, :, :-1]
    x = F.pad(x, (0, 0, 0, Tp - x.shape[2]))
    h = lrelu(x * float(bn1_scale) + float(bn1_shift), slope)
    y = F.conv2d(h, torch.as_tensor(w1, dtype=D).reshape(-1, 1, 3, 3), padding=1)
    c = lambda v: torch.as_tensor(v, dtype=D)[None, :, None, None]
    a = lrelu(y * c(bn2_scale) + c(bn2_shift), slope)
    r = F.conv2d(x, torch.as_tensor(w_sc, dtype=D).reshape(-1, 1, 1, 1), torch.as_tensor(b_sc, dtype=D))
    return h, y, a, r


def pool(x, scale, shift, slope=0.01):
    """F.avg_pool2d(x, 2) (floor: an odd last row / column is dropped, modules.py:183) and the next block's bn1 + LeakyReLU.
    x [n, C, H, W] -> (v, a)."""
    v = F.avg_pool2d(torch.as_tensor(x, dtype=D), kernel_size=(2, 2))
    c = lambda t: torch.as_tensor(t, dtype=D)[None, :, None, None]
    return v, lrelu(v * c(scale) + c(shift), slope)


BAND = (5, int(128 * 0.2))       # amp_to_original_f's low band (tools/utils.py:50-55): mel bins [5, 25)


def band_sums(mel_lin, logmel_est, T_b=None):
    """Per clip (sum of the target's low band, sum of from_log(estimate)'s low band) over its first T_b[b] frames."""
    mel_lin, logmel_est = np.asarray(mel_lin, np.float64), np.asarray(logmel_est, np.float64)
    n, T = mel_lin.shape[:2]
    out = np.zeros((n, 2))
    for b in range(n):
        t = T if T_b is None else int(T_b[b])
        out[b, 0] = mel_lin[b, :t, BAND[0]:BAND[1]].sum()
        out[b, 1] = (10.0 ** np.minimum(logmel_est[b, :t, BAND[0]:BAND[1]], 5.0)).sum()
    return out


def voc_frames(T, tail_base=4):
    """Vocoder frames of a T-frame mel: the conditioning's tail pad is T % 2 + tail_base frames (vf_oracle.vocoder_condition)."""
    return T + T % 2 + tail_base


def voc_condition(mel, is_log, weight, Tv, amp_floor=1e-5, ref_db=20.0, min_db=-115.0, tail_value=-4.0, sums=None):
    """Vocoder conditioning of mel [n, T, 128] (linear, or log10 with is_log: from_log first), optionally scaled by
    amp_to_original_f's ratio sums[:, 0] / sums[:, 1]; -> [n, Tv, 128] with rows T.. Tv - 1 = tail_value."""
    m = np.asarray(mel, np.float64)
    if is_log:
        m = 10.0 ** np.minimum(m, 5.0)
    if sums is not None:
        m = m * (sums[:, 0] / sums[:, 1])[:, None, None]
    v = np.abs(m) / np.asarray(weight, np.float64)
    s = 20.0 * np.log10(np.maximum(v, amp_floor)) - ref_db
    c = np.clip((s - min_db) / -min_db, 0.0, 1.0)
    n, T, _ = c.shape
    return np.concatenate([c, np.full((n, Tv - T, 128), tail_value)], axis=1)


def reflect_pad(x, pad=3):
    """nn.ReflectionPad1d(pad) on rows: x [n, L, C] -> [n, L + 2 pad, C]."""
    x = torch.as_tensor(np.asarray(x))
    return F.pad(x.permute(0, 2, 1), (pad, pad), mode="reflect").permute(0, 2, 1).numpy()


def voc_tail(xpad, w, b, tanh):
    """The generator's last conv on reflect-padded rows: Conv1d(C -> 1, k7) of xpad [n, L + 6, C] with w [1, C, 7]
    (+ tanh) -> [n, L]; with the pre-activation y and M = the same conv on |x|, |w|, |b|."""
    x = torch.as_tensor(np.asarray(xpad, np.float64)).permute(0, 2, 1)
    w = torch.as_tensor(np.asarray(w, np.float64))
    y = F.conv1d(x, w, torch.tensor([float(b)], dtype=D))[:, 0]
    m = F.conv1d(x.abs(), w.abs(), torch.tensor([abs(float(b))], dtype=D))[:, 0]
    return (torch.tanh(y) if tanh else y).numpy(), y.numpy(), m.numpy()


def finalize(wav, peak, skip, n):
    """Peak normalise + trim_center of one clip in float32 (eval_gsr_voicefixer.py:68-72): the kernel divides by the peak
    when it exceeds 1, as numpy float32 does."""
    seg = np.asarray(wav, np.float32)[skip:skip + n]
    peak = np.float32(peak)
    return seg / peak if peak > np.float32(1.0) else seg.copy()


N_FFT, HOP = 2048, 441


def hann():
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(N_FFT) / N_FFT)


def stft64(wav, T):
    """The first T frames of the centred, reflect-padded float64 STFT of one clip: [T, 1025] complex, with Σ|x w| per frame."""
    x = np.pad(np.asarray(wav, np.float64), N_FFT // 2, mode="reflect")
    fr = np.stack([x[t * HOP:t * HOP + N_FFT] for t in range(T)]) * hann()
    return np.fft.rfft(fr, axis=-1), np.abs(fr).sum(axis=-1)


def phase(X, eps=1e-8):
    """fDomainHelper.py:60-65: cos, sin = re / m, im / m with m = sqrt(max(|X|^2, eps))."""
    m = np.sqrt(np.maximum(X.real ** 2 + X.imag ** 2, eps))
    return X.real / m, X.imag / m


def frontend64(wav, T, fb):
    """The front end of one clip (frontend.cu) in float64: the first T frames of the STFT X [T, 1025] and S_t = Σ|x w| per
    frame, the clamped magnitude and its cos / sin (fDomainHelper.py:62-64, power clamp 1e-8), mel = mag @ fb with the
    caller's fp32 filterbank [1025, 128] widened, and log-mel = log10(max(mel, 1e-8)) (pytorch_util.py:157-159)."""
    X, S = stft64(wav, T)
    mag = np.sqrt(np.maximum(X.real ** 2 + X.imag ** 2, 1e-8))
    cs, sn = phase(X)
    mel = mag @ np.asarray(fb, np.float32).astype(np.float64)
    return dict(X=X, S=S, mag=mag, cos=cs, sin=sn, mel=mel, logmel=np.log10(np.maximum(mel, 1e-8)))


def inverse_frames(Y, keep_dc_imag=False):
    """Windowed inverse DFT of every frame, Y [T, 1025] -> [T, 2048].  The imaginary parts of the DC and Nyquist bins do
    not reach a real signal; keep_dc_imag models a packed 1024-point inverse that forgets to drop them (they then leak into
    the even and odd samples as constants)."""
    fr = np.fft.irfft(Y, n=N_FFT, axis=-1)
    if keep_dc_imag:
        b, d = Y[:, 0].imag, Y[:, -1].imag
        fr[:, 0::2] += (-(b + d) / 2048.0)[:, None]
        fr[:, 1::2] += ((b - d) / 2048.0)[:, None]
    return fr * hann()


def overlap_add(frames, length):
    """y[i] = sum_t frames[t][p - 441 t] / max(sum_t win^2[p - 441 t], 1e-11), p = i + 1024, i < length; returns (y, the
    window sum at each p, sum_t |frames[t][p - 441 t]|)."""
    T = frames.shape[0]
    w2 = hann() ** 2
    L = (T - 1) * HOP + N_FFT
    acc, ws, ab = np.zeros(L), np.zeros(L), np.zeros(L)
    for t in range(T):
        acc[t * HOP:t * HOP + N_FFT] += frames[t]
        ab[t * HOP:t * HOP + N_FFT] += np.abs(frames[t])
        ws[t * HOP:t * HOP + N_FFT] += w2
    sl = slice(N_FFT // 2, N_FFT // 2 + length)
    wsc = np.maximum(ws[sl], 1e-11)
    return acc[sl] / wsc, wsc, ab[sl]


def istft_fused(mag, wav, T, keep_dc_imag=False):
    """unet_v2.py:96,136-139 then FDomainHelper.istft: the magnitude mag [T, 1025] with the phase of the float64 STFT of
    wav (1e-8 power clamp), inverse DFT, window, overlap-add, clamped window-sum divide, len(wav) samples."""
    X, _ = stft64(wav, T)
    cs, sn = phase(X)
    Y = np.asarray(mag, np.float64) * (cs + 1j * sn)
    return overlap_add(inverse_frames(Y, keep_dc_imag), len(wav))[0]
