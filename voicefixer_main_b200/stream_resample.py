"""The host bookkeeping of resampling a live stream: which outputs are final, which inputs must still be held, and how long
the output is once the stream ends.

A stream is resampled by vf_resample_rings (edges.cu / sinc.cu arithmetic, resample.cuh) from a device ring of its inputs.
An output can be computed as soon as it is *final*: every input the whole-signal kernel reads for it has arrived, and the
kernel's clamp to the signal's end cannot apply however long the stream turns out to be.  Then it has the bits it has in
the whole-signal resample, so a stream's outputs, emitted in order as they become final and the rest at close, are
`edges.resample_to` (res_type None: scipy's resample_poly) or `edges.resample` (kaiser_best / kaiser_fast: librosa 0.8's
resampy) of the whole stream, bit for bit and at the same length.

* poly (up, down reduced by their gcd, half = 10 max(up, down)): output m reads inputs ceil((m down - half) / up) ..
  floor((m down + half) / up), clamped to [0, n - 1].  With p inputs pushed, m is final iff floor((m down + half) / up) <=
  p - 1.  A closed stream has ceil(n up / down) outputs.
* sinc (ratio = rate_out / rate_in as a float64, scale = min(1, ratio), step = int(scale num_table)): output t has tr =
  t / ratio, n_t = int(tr), frac = scale (tr - n_t); its left wing reads x[n_t - i] for i < min(n_t + 1, K(frac)), its right
  wing x[n_t + 1 + k] for k < min(n - n_t - 1, K(scale - frac)), K(f) = (nwin - int(f num_table)) // step (resampy's loop
  bounds, oracle/resampy.py).  With p pushed, t is final iff n_t + K(scale - frac) <= p - 1 and t < int(p ratio).  A closed
  stream has int(ceil(n ratio)) outputs, zeros from int(n ratio) on; int(n ratio) == 0 raises ValueError.

Emission is a prefix: `final_count(p)` is the number of leading outputs that are all final.  The inputs still needed once
the first m outputs are out start at `keep_from(m)`: ceil((m down - half) / up) for poly, n_m - (K_max - 1) for sinc (K_max
= nwin // step, the wings' largest length).  After the final outputs of p inputs are out, at most `history` inputs are held;
`tail` bounds how many outputs close() adds to the final ones.
"""
import math
from fractions import Fraction

from .edges import RES_TYPES, check_res_type, sinc_lengths


class StreamResampling:
    """The finality rule of one stream converted from `rate` to `rate_out` with `res_type` (None: resample_poly)."""

    def __init__(self, rate: int, rate_out: int, res_type=None):
        check_res_type(res_type)
        rate, rate_out = int(rate), int(rate_out)
        if rate < 1 or rate_out < 1:
            raise ValueError(f"sample rates must be at least 1 Hz (got {rate} -> {rate_out})")
        self.rate, self.rate_out, self.res_type = rate, rate_out, res_type
        self.passthrough = rate == rate_out
        self.poly = res_type is None
        if self.passthrough:
            self.history = self.tail = 0
        elif self.poly:
            fr = Fraction(rate_out, rate)
            self.up, self.down = fr.numerator, fr.denominator
            self.half = 10 * max(self.up, self.down)
            self.history = 2 * self.half // self.up
            self.tail = -(-(self.half + 2 * self.down) // self.down)
        else:
            num_zeros, precision = RES_TYPES[res_type][:2]
            self.ratio = float(rate_out) / rate
            self.scale = min(1.0, self.ratio)
            self.num_table = 2 ** precision
            self.nwin = self.num_table * num_zeros + 1
            self.step = int(self.scale * self.num_table)
            self.k_max = self.nwin // self.step
            self.history = 2 * self.k_max + 1
            self.tail = int(math.ceil((self.k_max + 2) * self.ratio)) + 2

    # ---- the kernel's float64 time register
    def _sinc_t(self, t: int):
        """(n_t, frac) of output t, in the kernel's float64 arithmetic."""
        tr = t / self.ratio
        n_t = int(tr)
        return n_t, self.scale * (tr - n_t)

    def _wing(self, frac: float) -> int:
        return (self.nwin - int(frac * self.num_table)) // self.step

    # ---- finality
    def is_final(self, m: int, p: int) -> bool:
        """Output m of an open stream with p inputs pushed has the bits it has in the whole-signal output, whatever n >= p."""
        if self.passthrough:
            return m < p
        if self.poly:
            return (m * self.down + self.half) // self.up <= p - 1
        n_t, frac = self._sinc_t(m)
        return m < int(p * self.ratio) and n_t + self._wing(self.scale - frac) <= p - 1

    def final_count(self, p: int) -> int:
        """The number of leading outputs that are final with p inputs pushed (non-decreasing in p)."""
        if self.passthrough:
            return p
        if self.poly:
            x = p * self.up - 1 - self.half
            return x // self.down + 1 if x >= 0 else 0
        # every t whose n_t <= p - 1 - K_max is final; scan the few after that up to the first that is not
        t = max(0, int((p - self.k_max) * self.ratio) - 2)
        while self.is_final(t, p):
            t += 1
        return t

    def keep_from(self, m: int) -> int:
        """The first input that any output from m on reads (a lower bound for sinc, the one vf_resample_rings uses)."""
        if self.passthrough:
            return m
        if self.poly:
            return max(0, -(-(m * self.down - self.half) // self.up))
        return max(0, int(m / self.ratio) - (self.k_max - 1))

    def out_len(self, n: int) -> int:
        """The output length of a closed stream of n inputs (0 for none); sinc: ValueError when int(n ratio) == 0."""
        if n == 0 or self.passthrough:
            return n
        if self.poly:
            return -(-(n * self.up) // self.down)
        return sinc_lengths(n, self.rate, self.rate_out)[1]

    def due(self, n: int) -> int:
        """out_len(n) without the ValueError: the outputs a close after n inputs would make final."""
        if self.poly or self.passthrough:
            return self.out_len(n)
        return int(math.ceil(n * self.ratio))
