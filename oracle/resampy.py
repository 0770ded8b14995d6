"""CPU restatement of librosa 0.8's `resample(y, orig_sr, target_sr, res_type="kaiser_best" / "kaiser_fast")`, the rate
conversion of `librosa.load(path, sr=...)` that the reference applies to every file (tools/utils.py:46-48,
evaluation_proc/metrics.py:33-34).  TEST INFRASTRUCTURE.

librosa 0.8 hands these res_types to the third-party resampy package.  Neither librosa nor resampy is in this image or in
the reference tree, so the arithmetic is restated here with numpy / scipy.  Parity status: restated, unpinned.  Every choice
below follows the published packages as recalled; NONE of it has been checked against resampy's or librosa's source.

Filter (resampy.filters.sinc_window, n = 2**precision * num_zeros), float64:
    interp_win = taper * (rolloff * sinc(rolloff * linspace(0, num_zeros, n + 1))),  taper = kaiser(2 n + 1, beta)[n:]
* kaiser_best: num_zeros 64, precision 9, rolloff 0.9475937167399596, beta 14.769656459379492;
  kaiser_fast: num_zeros 16, precision 7, rolloff 0.85, beta 8.555504641634386.
* The window is scipy's symmetric kaiser(M, beta).  The grouping of the three factors is the one recalled from
  sinc_window; it decides the table's last bits.
* resampy loads these tables from .npz files it ships.  Regenerating them from the parameters is an assumption: a table
  made with another scipy, or another grouping, differs in its last bits.
Resample (resampy >= 0.3, resample / _resample_loop):
* sample_ratio = sr_new / sr_orig, scale = min(1, sample_ratio).  When downsampling, interp_win *= sample_ratio; interp_delta
  = diff(interp_win) of the scaled table, with a final entry 0.  num_table = 2**precision, index_step = int(scale *
  num_table).
* n_out = int(n * sample_ratio) (a float product; ValueError when < 1), t_out = arange(n_out) / sample_ratio.
* For each t: n = int(t_out[t]), frac = scale * (t_out[t] - n), index_frac = frac * num_table, offset = int(index_frac),
  eta = index_frac - offset; left wing i < min(n + 1, (nwin - offset) // index_step) adds
  (win[offset + i step] + eta * delta[offset + i step]) * x[n - i]; then frac = scale - frac, offset and eta again, and the
  right wing k < min(n_orig - n - 1, (nwin - offset) // index_step) on x[n + k + 1].
* The output has x's dtype (float32): each y[t] += weight * x is a float64 product and sum, rounded back to float32 after
  every tap.  Nothing is contracted into an FMA.
librosa 0.8 resample(fix=True): y unchanged when the rates are equal; otherwise resampy's output zero-padded to
int(ceil(n * (float(target_sr) / orig_sr))), a float computation (`out_len`).

`VARIANTS` holds deliberately broken restatements (tests/test_resampy_cpu.py shows each one changes output bits).
"""
import numpy as np
import scipy.signal

FILTERS = {   # res_type: (num_zeros, precision, rolloff, Kaiser beta)
    "kaiser_best": (64, 9, 0.9475937167399596, 14.769656459379492),
    "kaiser_fast": (16, 7, 0.85, 8.555504641634386),
}
VARIANTS = ("time_register_sum", "periodic_window", "fma_weight", "f64_accumulate", "unscaled_window")


def sinc_window(res_type: str, periodic: bool = False):
    """(interp_win float64 [n + 1], num_table) of resampy's filter `res_type`; periodic=True uses a periodic Kaiser window
    (a broken variant)."""
    num_zeros, precision, rolloff, beta = FILTERS[res_type]
    num_table = 2 ** precision
    n = num_table * num_zeros
    sinc_win = rolloff * np.sinc(rolloff * np.linspace(0, num_zeros, num=n + 1, endpoint=True))
    taper = scipy.signal.windows.kaiser(2 * n + 1, beta, sym=not periodic)[n:]
    return taper * sinc_win, num_table


def out_len(n: int, orig_sr: int, target_sr: int) -> int:
    """librosa 0.8 resample's fix_length target: int(np.ceil(n * (float(target_sr) / orig_sr)))."""
    return int(np.ceil(n * (float(target_sr) / orig_sr)))


def tables(res_type: str, sample_ratio: float, variant: str = None):
    """(interp_win, interp_delta, num_table, scale) as resampy.resample hands them to its loop."""
    win, num_table = sinc_window(res_type, periodic=variant == "periodic_window")
    if sample_ratio < 1 and variant != "unscaled_window":
        win = win * sample_ratio
    delta = np.zeros_like(win)
    delta[:-1] = np.diff(win)
    return win, delta, num_table, min(1.0, sample_ratio)


def _fma(a, b, c):
    """a * b + c with one rounding of the exact product (extended-precision product, then float64): an FMA-contracted
    weight."""
    return (np.asarray(a, np.longdouble) * np.asarray(b, np.longdouble) + np.asarray(c, np.longdouble)).astype(np.float64)


def resampy_resample(x: np.ndarray, orig_sr: int, target_sr: int, res_type: str = "kaiser_best",
                     variant: str = None) -> np.ndarray:
    """resampy.resample(x, orig_sr, target_sr, filter=res_type) of a 1-D float32 signal, vectorised over the output samples
    with a masked tap loop.  variant: one of VARIANTS (tests only)."""
    assert variant is None or variant in VARIANTS, variant
    x = np.asarray(x, dtype=np.float32)
    sample_ratio = float(target_sr) / orig_sr
    n_orig = x.shape[0]
    n_out = int(n_orig * sample_ratio)
    if n_out < 1:
        raise ValueError(f"Input signal length={n_orig} is too small to resample from {orig_sr}->{target_sr}")
    win, delta, num_table, scale = tables(res_type, sample_ratio, variant)
    nwin = win.shape[0]
    index_step = int(scale * num_table)
    if variant == "time_register_sum":              # resampy 0.2.x: time_register += 1 / sample_ratio per output
        t_out = np.concatenate([[0.0], np.cumsum(np.full(n_out - 1, 1.0 / sample_ratio))])
    else:
        t_out = np.arange(n_out) / sample_ratio
    n = t_out.astype(np.int64)
    xd = x.astype(np.float64)
    y = np.zeros(n_out, np.float64 if variant == "f64_accumulate" else np.float32)

    def wing(frac, count, src):
        nonlocal y
        index_frac = frac * num_table
        offset = index_frac.astype(np.int64)
        eta = index_frac - offset
        k_max = np.minimum(count, (nwin - offset) // index_step)
        for i in range(int(k_max.max(initial=0))):
            live = i < k_max
            idx = np.where(live, offset + i * index_step, 0)
            if variant == "fma_weight":
                weight = _fma(eta, delta[idx], win[idx])
            else:
                weight = win[idx] + eta * delta[idx]
            acc = y.astype(np.float64) + weight * xd[np.where(live, src(i), 0)]
            y = np.where(live, acc.astype(y.dtype), y)
        return frac

    frac = wing(scale * (t_out - n), n + 1, lambda i: n - i)
    wing(scale - frac, n_orig - n - 1, lambda k: n + k + 1)
    return y.astype(np.float32)


def resample(y: np.ndarray, orig_sr: int, target_sr: int, res_type: str = "kaiser_best", variant: str = None) -> np.ndarray:
    """librosa 0.8 resample(y, orig_sr, target_sr, res_type, fix=True) of a 1-D float32 signal."""
    y = np.asarray(y, dtype=np.float32)
    if orig_sr == target_sr:
        return y
    out = resampy_resample(y, orig_sr, target_sr, res_type, variant)
    n = out_len(y.shape[0], orig_sr, target_sr)
    return np.pad(out, (0, n - out.shape[0])) if n > out.shape[0] else out[:n]
