"""Restore many live audio streams at once: chunked boxcar-margin streaming over the engine's vf_restore_chunks.

`StreamingRestorer` runs `BoxcarOverlapAdd(RestoreNet(model, unify_energy), 1, W, M)` (longform.py, the reference's
tools/dsp/overlapadd_boxcar.py LambdaOverlapAdd) incrementally over streams whose samples arrive while they are restored:

    sr = StreamingRestorer(model, window_size=44100, in_margin=11025)
    a = sr.open()
    sr.push(a, samples)             # any number of samples, any split, host or device
    out = sr.step()                 # {id: the samples restored since the last step}
    sr.close(a)                     # the rest comes out of the following step()

The chunks and crops are exactly `BoxcarOverlapAdd.plan(n)`'s for a stream of n samples.  Chunk i is restored as soon as
it is known to be a middle chunk of that plan, i.e. once (i + 1) W + M samples have been pushed (W + M for the first), and
whatever is left after `close`.  So a stream's concatenated outputs are BoxcarOverlapAdd's result bit for bit, n samples in
all, however its pushes were split and whichever streams shared its steps: vf_restore_chunks gives each chunk the bits of a
one-clip restore().

Each stream owns one row of a device ring of 2 (W + 2M) samples.  After a step the ring holds less than W + 2M samples
still needed by the stream's next chunk, so a push of up to W + 2M samples always fits; a push that would overwrite needed
samples raises, and the caller must step() first.  Each step is one vf_restore_chunks call: one gather launch builds the
packed chunks from the rings and one crop launch packs the kept samples, whatever the number of streams.

The SSR_UNet / GSR_UNet models (denoising, declipping, dereverberation, super-resolution) stream the same way: with one of
them each step is one vf_ssr_restore_chunks call, the same gather and crop around the unet_v2 + ISTFT chain, and a stream's
outputs are `BoxcarOverlapAdd(RestoreNet(ssr_model), 1, W, M)`'s.  That path has no unify_energy, and none of the SSR
handler's peak normalisation either: the handler divides a whole segment by its peak, which a live stream only knows once it
has ended.

Both restorers take streams at their own sample rate (open(rate), res_type, max_input_rate): each step first resamples the
samples of every such stream that have become final into its 44.1 kHz ring row with one vf_resample_rings launch
(stream_resample.py has the finality rule), so the stream's outputs are the restorer's on edges.resample_to of the whole
stream, bit for bit.  `StreamingResampler` is that conversion on its own, to any rate: chain one on a restorer's output to
send it at 48 or 16 kHz.

`StreamingVocoder` vocodes live mel streams the same way, chunk by chunk from device frame rings: each step is one
vf_vocoder_chunks call (the geometry is vocoder.chunk_plan's, the composition its outputs equal vocoder.vocode_chunked).

`WindowedStreamingRestorer` runs the reference's other long-form scheme, `WindowedOverlapAdd(RestoreNet(model, unify_energy),
1, W, hop, window)` (longform.py, tools/dsp/overlapadd.py's LambdaOverlapAdd), incrementally the same way: windows of W
samples every hop, each restored, multiplied by the synthesis window and overlap-added, so adjacent windows cross-fade.
Each step is one vf_restore_windows call (vf_ssr_restore_windows): the gather, the restore chain, one overlap-add launch
per sub-batch into per-stream device accumulators, and one launch that emits the finished samples.
"""
import itertools
from typing import Dict, List, Optional, Tuple

import torch

from .arch import frames_for, vocoder_out_len
from .edges import check_res_type, stream_filter
from .longform import BoxcarOverlapAdd, WindowedOverlapAdd
from .model import SSR_UNet
from .stream_resample import StreamResampling
from .vocoder import check_chunking, chunk_plan

OPEN = (1 << 63) - 1              # `valid` of a chunk whose stream is still open: no position reads as zero padding
MAX_CHUNK = 1 << 30               # samples of one clip of vf_restore_varlen (engine.cu check_varlen_call)
MODEL_RATE = 44100                # the restorers' sample rate


def restore_rejects(engine, n: int, ssr: bool = False) -> Optional[str]:
    """Why restore() refuses a clip of n samples (the checks of vf_restore_ex / vf_restore_chunks), or None.  ssr: the
    SSR_UNet / GSR_UNet restore() (vf_ssr_restore_chunks), which has no vocoder and so no trim_center constraint."""
    if n <= 1024:
        return f"{n} samples (reflect padding needs more than 1024)"
    if n > MAX_CHUNK:
        return f"{n} samples (one restore takes at most 2^30)"
    if ssr:
        return None
    d = vocoder_out_len(frames_for(n), engine.voc_cfg) - n
    if d < 0 or d == 1:
        return f"{n} samples (a vocoder output of {n + d} samples, which trim_center cannot cut to {n})"
    return None


class _Stream:
    __slots__ = ("slot", "pushed", "next", "n", "emitted", "rs", "src_pushed", "src_n")

    def __init__(self, slot: int, first: int = 0):
        self.slot = slot
        self.pushed = 0           # samples pushed so far (absolute position of the next one)
        self.next = first         # index of the next chunk / window to restore
        self.n: Optional[int] = None    # total length once closed
        self.emitted = 0          # windowed: samples emitted so far; StreamingResampler: outputs emitted so far
        # a restorer's stream at another rate: its resampling, and its own samples pushed (and their count once closed);
        # `pushed` and `n` then count the 44.1 kHz samples resampled into the ring row
        self.rs: Optional[StreamResampling] = None
        self.src_pushed = 0
        self.src_n: Optional[int] = None


class _RingStreams:
    """The stream lifecycle and device ring shared by the streaming restorers and the streaming vocoder: open / push / close
    bookkeeping, one ring row of ring_len positions per stream, each position a sample (row shape ()) or a mel frame ((128,)).
    A subclass says from which position a stream's input is still needed (_keep_from)."""
    _first = 0                    # _Stream.next of a new stream
    _row = ()                     # the shape of one position
    _push_what = "samples must be a 1-D float32 tensor"
    _unit = "samples"

    def _init_model(self, model, unify_energy: bool, max_streams: int):
        if max_streams < 1:
            raise ValueError("max_streams must be at least 1")
        self.ssr = isinstance(model, SSR_UNet)          # GSR_UNet too
        if self.ssr and unify_energy:
            raise ValueError("unify_energy is a VoiceFixer option; SSR_UNet / GSR_UNet restore without it")
        self.engine = model._engine()
        self.unify_energy = unify_energy

    def _init_ring(self, ring_len: int, max_streams: int):
        self.ring_len = ring_len
        self.ring = torch.zeros(max_streams, ring_len, *self._row, device=self.engine.device)
        self._free = list(range(max_streams - 1, -1, -1))
        self._streams: Dict[int, _Stream] = {}
        self._ids = itertools.count()

    def open(self) -> int:
        """A new stream; its id is never reused."""
        if not self._free:
            raise RuntimeError(f"all {self.ring.shape[0]} streams are open (max_streams)")
        sid = next(self._ids)
        self._streams[sid] = _Stream(self._free.pop(), self._first)
        return sid

    def _get(self, sid: int, what: str) -> _Stream:
        st = self._streams.get(sid)
        if st is None:
            raise KeyError(f"{what}: no open stream {sid}")
        if st.n is not None:
            raise ValueError(f"{what}: stream {sid} is closed")
        return st

    def _keep_from(self, st: _Stream) -> int:
        raise NotImplementedError

    def _check_push(self, sid: int, samples) -> _Stream:
        st = self._get(sid, "push")
        if (not isinstance(samples, torch.Tensor) or samples.dtype != torch.float32 or samples.dim() != 1 + len(self._row)
                or tuple(samples.shape[1:]) != self._row):
            raise TypeError(f"push: stream {sid}: {self._push_what}")
        return st

    def push(self, sid: int, samples: torch.Tensor):
        """Appends 1-D float32 samples (host or device) to stream `sid`'s ring (StreamingVocoder: [k, 128] mel frames)."""
        st = self._check_push(sid, samples)
        k, L = samples.shape[0], self.ring_len
        held = st.pushed - self._keep_from(st)
        if held + k > L:
            raise OverflowError(f"push: stream {sid}: {k} {self._unit} do not fit its ring ({L - held} of {L} free); call step() first")
        _write(self.ring[st.slot], st.pushed, samples)
        st.pushed += k

    def _release(self, sid: int):
        self._free.append(self._streams.pop(sid).slot)


def _write(row: torch.Tensor, at: int, samples: torch.Tensor):
    """Copies samples into a ring row from absolute position `at` on, wrapping round its end."""
    L = row.shape[0]
    k, p = samples.shape[0], at % L
    first = min(k, L - p)
    row[p:p + first].copy_(samples[:first])
    if k > first:
        row[:k - first].copy_(samples[first:])


def _check_rate(rate, max_input_rate: int, what: str) -> int:
    if int(rate) != rate or not 1 <= rate <= max_input_rate:
        raise ValueError(f"{what}: rate {rate} Hz is not in 1 .. max_input_rate = {max_input_rate}")
    return int(rate)


def _history_bound(rate_out: int, res_type, max_input_rate: int) -> int:
    """The most inputs a stream at any rate up to max_input_rate holds after a step: StreamResampling.history grows with
    the input rate, and is the same for every upsampling rate."""
    rates = [max_input_rate] + ([rate_out - 1] if 1 < rate_out <= max_input_rate else [])
    return max(StreamResampling(r, rate_out, res_type).history for r in rates)


class _InputRates:
    """Streams at their own sample rate in front of a restorer's 44.1 kHz ring (mixed into StreamingRestorer and
    WindowedStreamingRestorer).  open(rate) with rate != 44100 gives the stream a row of a second ring, `in_ring`, of its
    own samples; each step first resamples the samples that have become final (stream_resample.py) into the stream's
    44.1 kHz ring row with one vf_resample_rings launch, then restores as for a 44.1 kHz stream.  `cap` is the 44.1 kHz push
    the restorer guarantees after a step (its ring holds 2 cap and fewer than cap samples are still needed after a step)."""

    def _init_rates(self, res_type, max_input_rate: int, max_streams: int, cap: int):
        check_res_type(res_type)
        if int(max_input_rate) != max_input_rate or max_input_rate < 1:
            raise ValueError(f"max_input_rate must be a positive integer (got {max_input_rate})")
        self.res_type, self.max_input_rate = res_type, int(max_input_rate)
        self._cap = cap
        self.in_len = cap * self.max_input_rate // MODEL_RATE + _history_bound(MODEL_RATE, res_type, self.max_input_rate) + 1
        self.in_ring = torch.zeros(max_streams, self.in_len, device=self.engine.device)

    def open(self, rate: int = MODEL_RATE) -> int:
        """A new stream of samples at `rate` Hz (1 .. max_input_rate, or 44100); its id is never reused."""
        rs = None
        if rate != MODEL_RATE:
            rs = StreamResampling(_check_rate(rate, self.max_input_rate, "open"), MODEL_RATE, self.res_type)
        sid = _RingStreams.open(self)
        self._streams[sid].rs = rs
        return sid

    def max_push(self, rate: int = MODEL_RATE) -> int:
        """The samples at `rate` that a push to a stream at that rate always fits after a step: cap at 44.1 kHz; at another
        rate floor((cap - tail - 2) rate / 44100), where tail (StreamResampling.tail, at most 60 samples for resample_poly
        and about 66 x 44100 / rate for kaiser_best) bounds the 44.1 kHz samples that close() adds."""
        if rate == MODEL_RATE:
            return self._cap
        rs = StreamResampling(_check_rate(rate, self.max_input_rate, "max_push"), MODEL_RATE, self.res_type)
        return max(0, min(self.in_len - rs.history, (self._cap - rs.tail - 2) * rs.rate // MODEL_RATE))

    def push(self, sid: int, samples: torch.Tensor):
        """Appends 1-D float32 samples (host or device) at the stream's own rate.  Raises OverflowError naming the stream,
        before anything is copied, when they would overrun its input ring or make more 44.1 kHz samples due than its
        restore ring holds; call step() first."""
        st = self._check_push(sid, samples)
        if st.rs is None:
            return _RingStreams.push(self, sid, samples)
        k = samples.shape[0]
        held = st.src_pushed - st.rs.keep_from(st.pushed)
        if held + k > self.in_len:
            raise OverflowError(f"push: stream {sid}: {k} samples at {st.rs.rate} Hz do not fit its input ring "
                                f"({self.in_len - held} of {self.in_len} free); call step() first")
        due = st.rs.due(st.src_pushed + k) - self._keep_from(st)      # held at 44.1 kHz if the stream closed next
        if due > self.ring_len:
            raise OverflowError(f"push: stream {sid}: {k} samples at {st.rs.rate} Hz would make {due} samples at 44.1 kHz "
                                f"due, more than its ring of {self.ring_len}; call step() first")
        _write(self.in_ring[st.slot], st.src_pushed, samples)
        st.src_pushed += k

    def _close_length(self, sid: int, st: _Stream) -> int:
        """The stream's 44.1 kHz length at close, its own count recorded (ValueError when a sinc resample has no output)."""
        if st.rs is None:
            return st.pushed
        try:
            n = st.rs.out_len(st.src_pushed)
        except ValueError as e:
            raise ValueError(f"close: stream {sid}: {e}") from None
        st.src_n = st.src_pushed
        return n

    def _resample(self):
        """Writes every other-rate stream's newly final 44.1 kHz samples (all that are left, once it is closed) into its ring
        row: one vf_resample_rings call, one launch per filter family present."""
        rows, ends = [], []
        for st in self._streams.values():
            if st.rs is None:
                continue
            m1 = st.rs.final_count(st.src_pushed) if st.n is None else st.n
            if m1 > st.pushed:
                rows.append((st.slot, stream_filter(self.engine, st.rs.rate, MODEL_RATE, self.res_type), st.pushed, m1,
                             OPEN if st.n is None else st.src_n, st.src_pushed, st.slot, 0))
                ends.append((st, m1))
        if rows:
            self.engine.resample_rings(self.in_ring, rows, self.ring)
        for st, m1 in ends:
            st.pushed = m1


class StreamingRestorer(_InputRates, _RingStreams):
    """Live streams restored chunk by chunk with `in_margin` samples of context on each side of every `window_size` window.

    model: a VoiceFixer, SSR_UNet or GSR_UNet on a CUDA device with weights loaded.  max_streams: the streams that may be open
    at once (one ring row each).  unify_energy: as VoiceFixer.restore(unify_energy=...); an SSR / GSR-UNet model has no such
    flag, and asking for it raises ValueError."""

    def __init__(self, model, window_size: int, in_margin: int, max_streams: int = 64, unify_energy: bool = False,
                 res_type: Optional[str] = None, max_input_rate: int = 48000):
        W, M = int(window_size), int(in_margin)
        if W % 2:
            raise ValueError("window_size must be even")
        if not 0 < M < W:
            raise ValueError("in_margin must be in (0, window_size)")
        self._init_model(model, unify_energy, max_streams)
        for n in (W + M, W + 2 * M):            # the first and middle chunks
            why = restore_rejects(self.engine, n, self.ssr)
            if why:
                raise ValueError(f"window_size {W} and in_margin {M} give chunks of {why}")
        self.window_size, self.in_margin = W, M
        self._ola = BoxcarOverlapAdd(None, 1, W, M)      # plan() is the chunk geometry of a closed stream
        self._init_ring(2 * (W + 2 * M), max_streams)
        self._init_rates(res_type, max_input_rate, max_streams, W + 2 * M)

    def _keep_from(self, st: _Stream) -> int:
        """First absolute position the stream's next chunk reads."""
        return 0 if st.next == 0 else st.next * self.window_size - self.in_margin

    def _final_chunks(self, st: _Stream) -> List[Tuple[int, int, int, int]]:
        """(start, length, crop_left, crop_right) of the chunks of a closed stream not restored yet: BoxcarOverlapAdd.plan(n)
        from st.next on, the only chunk of a stream of at most W samples cropped to n as ola_forward's final cut does."""
        plan, _ = self._ola.plan(st.n)
        out = []
        for i in range(st.next, len(plan)):
            start, stop, cl, cr = plan[i]
            if len(plan) == 1:
                cr = stop - st.n
            out.append((start, stop - start, cl, cr))
        return out

    def _ready_chunks(self, st: _Stream) -> List[Tuple[int, int, int, int]]:
        """The chunks of an open stream that are middle chunks of its final plan whatever its length: chunk i once (i + 1) W + M
        samples are in, as the plan's (i W - M, (i + 1) W + M, M, M), or (0, W + M, 0, M) for the first."""
        W, M = self.window_size, self.in_margin
        out = []
        i = st.next
        while st.pushed >= (i + 1) * W + M:
            out.append((0, W + M, 0, M) if i == 0 else (i * W - M, W + 2 * M, M, M))
            i += 1
        return out

    def close(self, sid: int):
        """Ends stream `sid`; its remaining samples come out of the next step().  Raises ValueError, and leaves the stream
        open, when its last chunk is one restore() would refuse (push more samples, then close again)."""
        st = self._get(sid, "close")
        st.n = self._close_length(sid, st)
        for start, length, _, _ in self._final_chunks(st):
            why = restore_rejects(self.engine, length, self.ssr)
            if why:
                st.n = st.src_n = None
                raise ValueError(f"close: stream {sid}: its last chunk (samples {start} .. {start + length - 1}) has {why}")
        if st.n == 0:                           # nothing was pushed: nothing to restore
            self._release(sid)

    def step(self) -> Dict[int, torch.Tensor]:
        """Restores every ready chunk of every stream in one vf_restore_chunks call (vf_ssr_restore_chunks for an SSR / GSR-UNet
        model) -> {id: 1-D device tensor of the samples restored since the last step} for the streams that have any.  A
        closed stream is gone once its last samples are out."""
        self._resample()
        table, owners = [], []
        for sid, st in self._streams.items():
            chunks = self._final_chunks(st) if st.n is not None else self._ready_chunks(st)
            valid = OPEN if st.n is None else st.n
            for start, length, cl, cr in chunks:
                table.append((st.slot, length, cl, cr, start, valid))
            if chunks:
                owners.append((sid, len(chunks), sum(length - cl - cr for _, length, cl, cr in chunks)))
        if not table:
            return {}
        if self.ssr:
            kept = self.engine.ssr_restore_chunks(self.ring, table)
        else:
            kept = self.engine.restore_chunks(self.ring, table, unify_energy=self.unify_energy)
        out, off = {}, 0
        for sid, n_chunks, n_kept in owners:
            out[sid] = kept[off:off + n_kept]
            off += n_kept
            st = self._streams[sid]
            st.next += n_chunks
            if st.n is not None:
                self._release(sid)              # a closed stream's step emits all its remaining chunks
        return out


class WindowedStreamingRestorer(_InputRates, _RingStreams):
    """Live streams restored as `WindowedOverlapAdd(RestoreNet(model, unify_energy), 1, window_size, hop_size, window=window,
    reorder_chunks=False)` restores a whole signal: window k reads positions [k hop - W, k hop) (zero before 0 and past the
    stream's end), is restored, weighted by the synthesis window (or by 1 / (W / hop) when window is None) and overlap-added.

    Window k is ready once k hop samples are in; it is then a window of the final plan whatever the stream's length.  Window
    0 reads only padding and the last one, when hop divides n + W, only samples past n: neither contributes to any output,
    so neither is restored.  Output sample t is final once the windows up to floor((t + W) / hop) (or the last) are added,
    so a sample leaves at most W samples after it arrives.  Each sample goes through the network W / hop times.

    Each stream owns one row of a device ring of 2W samples and one row of an accumulator of 2W partial sums.  After a step a
    stream holds fewer than W samples still needed by its next window, so a push of up to W samples always fits; a push
    that would overwrite needed samples raises OverflowError, and the caller must step() first.  model, max_streams and
    unify_energy as for StreamingRestorer."""
    _first = 1                    # window 0 contributes nothing

    def __init__(self, model, window_size: int, hop_size: Optional[int] = None, window="hanning", max_streams: int = 64,
                 unify_energy: bool = False, res_type: Optional[str] = None, max_input_rate: int = 48000):
        W = int(window_size)
        hop = W // 2 if hop_size is None else int(hop_size)
        if W % 2:
            raise ValueError("window_size must be even")
        if not 0 < hop <= W:
            raise ValueError("hop_size must be in (0, window_size]")
        self._init_model(model, unify_energy, max_streams)
        why = restore_rejects(self.engine, W, self.ssr)
        if why:
            raise ValueError(f"window_size {W} gives windows of {why}")
        self.window_size, self.hop_size = W, hop
        ola = WindowedOverlapAdd(None, 1, W, hop, window=window, reorder_chunks=False)
        if ola.use_window:
            synth = ola.window
        else:                     # frames / (W / hop) on the device: a product with the fp32 reciprocal of the fp32 divisor
            synth = torch.full((W,), float(torch.tensor(1.0) / torch.tensor(W / hop, dtype=torch.float32)))
        self.synthesis = synth.to(self.engine.device)
        self._init_ring(2 * W, max_streams)
        self.acc = torch.zeros(max_streams, 2 * W, device=self.engine.device)
        self._init_rates(res_type, max_input_rate, max_streams, W)

    def _keep_from(self, st: _Stream) -> int:
        """First absolute position the stream's next window reads; also the stream's first sample not emitted yet."""
        return max(0, st.next * self.hop_size - self.window_size)

    def _windows(self, st: _Stream) -> List[int]:
        """Indices of the windows to add now: on an open stream the ready ones (k hop <= pushed), on a closed one all that
        are left and contribute (k hop - W < n)."""
        W, hop = self.window_size, self.hop_size
        k, out = st.next, []
        while (k * hop <= st.pushed) if st.n is None else (k * hop - W < st.n):
            out.append(k)
            k += 1
        return out

    def close(self, sid: int):
        """Ends stream `sid`; its remaining samples come out of the next step()."""
        st = self._get(sid, "close")
        st.n = self._close_length(sid, st)
        if not self._windows(st):                # nothing left to add: everything is out already
            self._release(sid)

    def step(self) -> Dict[int, torch.Tensor]:
        """Restores every window ready to be added of every stream, adds it into the stream's accumulator and emits the
        samples that are final, in one vf_restore_windows call (vf_ssr_restore_windows for an SSR / GSR-UNet model) ->
        {id: 1-D device tensor of the samples finished since the last step} for the streams that have any.  A closed stream
        is gone once its last samples are out."""
        self._resample()
        W, hop = self.window_size, self.hop_size
        windows, emits, owners = [], [], []
        for sid, st in self._streams.items():
            ks = self._windows(st)
            if not ks:
                continue
            valid = OPEN if st.n is None else st.n
            windows += [(st.slot, k * hop - W, valid) for k in ks]
            end = st.n if st.n is not None else max(0, (ks[-1] + 1) * hop - W)
            emits.append((st.slot, st.emitted, end - st.emitted))
            owners.append((sid, ks[-1] + 1, end))
        if not windows:
            return {}
        if self.ssr:
            done = self.engine.ssr_restore_windows(self.ring, windows, W, self.synthesis, self.acc, emits)
        else:
            done = self.engine.restore_windows(self.ring, windows, W, self.synthesis, self.acc, emits,
                                               unify_energy=self.unify_energy)
        out, off = {}, 0
        for sid, nxt, end in owners:
            st = self._streams[sid]
            if end > st.emitted:
                out[sid] = done[off:off + end - st.emitted]
                off += end - st.emitted
            st.next, st.emitted = nxt, end
            if st.n is not None:
                self._release(sid)              # a closed stream's step adds its last windows and emits the rest
        return out


class StreamingVocoder(_RingStreams):
    """Live mel streams - a TTS or voice-conversion model's output, a few frames at a time - vocoded chunk by chunk with
    `margin_frames` frames of context on each side of every `window_frames` frames:

        sv = StreamingVocoder(vocoder, window_frames=64, margin_frames=16)
        a = sv.open()
        sv.push(a, mel)                 # [k, 128] float32 linear mel frames, any k, any split, host or device
        out = sv.step()                 # {id: the samples vocoded since the last step}
        sv.close(a)                     # the rest comes out of the following step()

    vocoder: a vocoder.Vocoder or a VoiceFixer (whose engine holds the vocoder) on a CUDA device with weights loaded.  W =
    window_frames and M = margin_frames must be even, W >= 2, M >= 0.  The chunks and crops of a stream of T frames are
    vocoder.chunk_plan(T, W, M)'s, so its concatenated outputs are vocoder.vocode_chunked(vocoder, mel, W, M) bit for bit,
    vocoder_out_len(T) samples in all, however its pushes were split and whichever streams shared its steps:
    vf_vocoder_chunks gives each chunk the bits of a one-mel forward on its frames.  A stream of at most W frames is one chunk,
    forward(mel) itself; with M >= arch.vocoder_receptive_field(cfg) (576 frames for the default config) every kept frame has
    the whole mel's context and the stream is forward(mel) on the whole mel.  A smaller M is an approximation whose error
    falls as M grows (DESIGN.md 5).

    Chunk i is vocoded once (i + 1) W + M frames have been pushed (with M = 0 one frame more: until then the stream could end
    at (i + 1) W, and then chunk i is the last one and keeps the tail padding's samples); its range is then final whatever
    the stream's length.  So the samples of frame t leave once M to W + M - 1 more frames have arrived after it (1 to W when
    M = 0), and the remaining chunks of a closed stream in the next step().

    Each stream owns one row of a device ring of 2 (W + 2M) frames.  After a step the ring holds fewer than W + 2M frames
    still needed by the stream's next chunk (at most W when M = 0), so a push of up to W + 2M frames always fits; a push
    that would overwrite needed frames raises OverflowError, and the caller must step() first.  Each step is one
    vf_vocoder_chunks call: per sub-batch one gather launch writes the chunks' frames from the rings straight into the
    vocoder plan and one crop launch reads the kept samples straight out of it, whatever the number of streams."""
    _row = (128,)
    _push_what = "mel must be a [k, 128] float32 tensor"
    _unit = "frames"

    def __init__(self, vocoder, window_frames: int, margin_frames: int, max_streams: int = 64):
        W, M = check_chunking(window_frames, margin_frames)
        if max_streams < 1:
            raise ValueError("max_streams must be at least 1")
        self.engine = vocoder._engine()
        self.voc_cfg = self.engine.voc_cfg
        self.window_frames, self.margin_frames = W, M
        self._init_ring(2 * (W + 2 * M), max_streams)

    def _keep_from(self, st: _Stream) -> int:
        """First absolute frame the stream's next chunk reads."""
        return max(0, st.next * self.window_frames - self.margin_frames)

    def _ready_chunks(self, st: _Stream) -> List[Tuple[int, int, int, int]]:
        """The chunks of an open stream whose range and crops are final whatever its length: chunk i once (i + 1) W + M
        frames are in (and more than (i + 1) W, so that it cannot be the last one), as chunk_plan gives it then."""
        W, M, hop = self.window_frames, self.margin_frames, self.voc_cfg.hop
        out = []
        i = st.next
        while st.pushed >= (i + 1) * W + max(M, 1):
            s = max(0, i * W - M)
            length = (i + 1) * W + M - s
            out.append((s, length, (i * W - s) * hop, vocoder_out_len(length, self.voc_cfg) - ((i + 1) * W - s) * hop))
            i += 1
        return out

    def close(self, sid: int):
        """Ends stream `sid`; its remaining samples come out of the next step()."""
        st = self._get(sid, "close")
        st.n = st.pushed
        if st.n == 0:                           # nothing was pushed: nothing to vocode
            self._release(sid)

    def step(self) -> Dict[int, torch.Tensor]:
        """Vocodes every ready chunk of every stream in one vf_vocoder_chunks call -> {id: 1-D device tensor of the samples
        vocoded since the last step} for the streams that have any.  A closed stream is gone once its last samples are out."""
        table, owners = [], []
        for sid, st in self._streams.items():
            if st.n is None:
                chunks = self._ready_chunks(st)
            else:
                chunks = chunk_plan(st.n, self.window_frames, self.margin_frames, self.voc_cfg)[st.next:]
            valid = OPEN if st.n is None else st.n
            for start, length, cl, cr in chunks:
                table.append((st.slot, length, cl, cr, start, valid))
            if chunks:
                n_kept = sum(vocoder_out_len(length, self.voc_cfg) - cl - cr for _, length, cl, cr in chunks)
                owners.append((sid, len(chunks), n_kept))
        if not table:
            return {}
        kept = self.engine.vocoder_chunks(self.ring, table)
        out, off = {}, 0
        for sid, n_chunks, n_kept in owners:
            out[sid] = kept[off:off + n_kept]
            off += n_kept
            st = self._streams[sid]
            st.next += n_chunks
            if st.n is not None:
                self._release(sid)              # a closed stream's step emits all its remaining chunks
        return out


class StreamingResampler(_RingStreams):
    """Live streams converted from their own sample rate to `rate_out` as they arrive:

        rs = StreamingResampler(model, rate_out=44100)      # or an Engine; res_type None, "kaiser_best" or "kaiser_fast"
        a = rs.open(16000)
        rs.push(a, samples)             # any number of samples at the stream's rate, any split, host or device
        out = rs.step()                 # {id: the samples at rate_out that became final since the last step}
        rs.close(a)                     # the rest comes out of the following step()

    A stream's concatenated outputs are `edges.resample_to(eng, whole[None], rate, rate_out)[0]` (res_type None: scipy's
    resample_poly) or `edges.resample(eng, [whole], rate, rate_out, res_type)[0]` (librosa 0.8's resampy) of the whole
    stream, bit for bit and at the same length, however its pushes were split and whichever streams shared its steps: each
    step computes the outputs that have become final (stream_resample.py) with the whole-signal kernels' arithmetic.  A
    stream at rate_out passes its samples through unchanged.  A stream's output lags its input by the filter's half-length:
    10 input samples for 16 kHz -> 44.1 kHz with resample_poly, about 64 with kaiser_best.

    Each stream owns one row of a device ring of max_input_rate + history samples at its own rate (history: the inputs a
    stream still holds after a step, StreamResampling.history at max_input_rate).  So a push of up to max_input_rate
    samples - one second at the highest rate - always fits after a step; a push that would overwrite needed samples raises
    OverflowError naming the stream, before anything is copied, and the caller must step() first.  Each step is one
    vf_resample_rings call: one launch for the streams of the family of res_type, whatever their number (up to 256)."""

    def __init__(self, owner, rate_out: int = MODEL_RATE, res_type: Optional[str] = None, max_streams: int = 64,
                 max_input_rate: int = 48000):
        check_res_type(res_type)
        if max_streams < 1:
            raise ValueError("max_streams must be at least 1")
        if int(rate_out) != rate_out or rate_out < 1 or int(max_input_rate) != max_input_rate or max_input_rate < 1:
            raise ValueError(f"rate_out and max_input_rate must be positive integers (got {rate_out}, {max_input_rate})")
        self.engine = owner._engine() if hasattr(owner, "_engine") else owner
        self.rate_out, self.res_type, self.max_input_rate = int(rate_out), res_type, int(max_input_rate)
        self._init_ring(self.max_input_rate + _history_bound(self.rate_out, res_type, self.max_input_rate), max_streams)
        self._through: Dict[int, List[torch.Tensor]] = {}    # pass-through streams' pushes since the last step

    def open(self, rate: int) -> int:
        """A new stream of samples at `rate` Hz (1 .. max_input_rate); its id is never reused."""
        rs = StreamResampling(_check_rate(rate, self.max_input_rate, "open"), self.rate_out, self.res_type)
        sid = _RingStreams.open(self)
        self._streams[sid].rs = rs
        if rs.passthrough:
            self._through[sid] = []
        return sid

    def _keep_from(self, st: _Stream) -> int:
        """First input the stream's next output reads."""
        return st.rs.keep_from(st.emitted)

    def push(self, sid: int, samples: torch.Tensor):
        """Appends 1-D float32 samples (host or device) at the stream's rate to stream `sid`."""
        st = self._check_push(sid, samples)
        if st.rs.passthrough:
            self._through[sid].append(samples.to(self.engine.device, copy=True))
            st.pushed += samples.shape[0]
            return
        _RingStreams.push(self, sid, samples)

    def close(self, sid: int):
        """Ends stream `sid`; its remaining samples come out of the next step().  A kaiser_best / kaiser_fast stream too short
        to resample (int(n * ratio) == 0, as librosa raises it) raises ValueError and stays open."""
        st = self._get(sid, "close")
        try:
            st.rs.out_len(st.pushed)
        except ValueError as e:
            raise ValueError(f"close: stream {sid}: {e}") from None
        st.n = st.pushed
        if st.rs.out_len(st.n) == st.emitted and not self._through.get(sid):
            self._release(sid)

    def _release(self, sid: int):
        self._through.pop(sid, None)
        _RingStreams._release(self, sid)

    def step(self) -> Dict[int, torch.Tensor]:
        """Resamples every stream's samples that have become final (all that are left of a closed one) in one
        vf_resample_rings call -> {id: 1-D device tensor of the samples at rate_out since the last step} for the streams that
        have any.  A closed stream is gone once its last samples are out."""
        rows, owners, off = [], [], 0
        out: Dict[int, torch.Tensor] = {}
        for sid, st in self._streams.items():
            rs = st.rs
            if rs.passthrough:
                if self._through[sid]:
                    out[sid] = torch.cat(self._through[sid])
                    self._through[sid] = []
                owners.append((sid, None, st.pushed))
                continue
            m1 = rs.final_count(st.pushed) if st.n is None else rs.out_len(st.n)
            if m1 > st.emitted:
                rows.append((st.slot, stream_filter(self.engine, rs.rate, self.rate_out, self.res_type), st.emitted, m1,
                             OPEN if st.n is None else st.n, st.pushed, -1, off))
                owners.append((sid, off, m1))
                off += m1 - st.emitted
        if rows:
            packed = self.engine.resample_rings(self.ring, rows, torch.empty(off, device=self.engine.device))
        for sid, at, m1 in owners:
            st = self._streams[sid]
            if at is not None:
                out[sid] = packed[at:at + m1 - st.emitted]
            st.emitted = m1
            if st.n is not None:
                self._release(sid)              # a closed stream's step emits all its remaining samples
        return out
