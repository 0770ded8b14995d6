"""Long-form restoration with context margins (SURVEY.md 8(f) row 2).

Mirror of `LambdaOverlapAdd` in the reference's tools/dsp/overlapadd_boxcar.py:338-534 ("boxcar" overlap-add:
hop = window, every chunk is processed with `in_margin` samples of real context on both sides and only its
centre is kept), with the same constructor arguments, the same `ola_forward` / `forward` results and the same
special cases (first chunk has no left margin, last chunk may be short, the signal is zero-padded to a multiple of
the window).  What differs is the schedule: the reference runs the chunks one by one through `nnet`; here all
middle chunks of all batch items have the same length and go through `nnet` as ONE batch when the network says it
is batch-invariant (`nnet.batch_invariant`, true for the CUDA engine, whose per-row peak normalisation and
vocoder are independent across rows), `max_batch` rows at a time: the engine's workspace grows linearly with
batch x length (~0.14 GB per clip-second), so an unbounded stack of a 20-minute file would not fit one GPU, and a
fixed group size also lets the per-shape plans be reused.  A 10-minute file is three launches of batch 8.

`RestoreNet` adapts `VoiceFixer.restore`, or `SSR_UNet.restore` / `GSR_UNet.restore`, to the
`nnet(x[B, C, L]) -> {key: [B, n_src, L]}` protocol the class expects.
"""
from typing import Optional

import torch
import torch.nn.functional as F

from .model import SSR_UNet


class RestoreNet:
    """`nnet` protocol of LambdaOverlapAdd over VoiceFixer.restore, or SSR_UNet / GSR_UNet.restore: [B, 1, L] ->
    {"wav": [B, 1, L]}.  unify_energy is VoiceFixer's restore flag; the SSR / GSR-UNet restore has none (ValueError)."""
    batch_invariant = True          # rows are independent: chunks may be stacked along the batch dimension
    in_channels = 1

    def __init__(self, model, unify_energy: bool = False):
        self.ssr = isinstance(model, SSR_UNet)          # GSR_UNet too
        if self.ssr and unify_energy:
            raise ValueError("unify_energy is a VoiceFixer option; SSR_UNet / GSR_UNet restore without it")
        self.model = model
        self.unify_energy = unify_energy

    def __call__(self, x: torch.Tensor):
        if x.ndim != 3 or x.shape[1] != 1:
            raise ValueError("RestoreNet expects [batch, 1, samples]")
        x = x[:, 0, :].contiguous()
        out = self.model.restore(x) if self.ssr else self.model.restore(x, unify_energy=self.unify_energy)
        return {"wav": out[:, None, :]}


class BoxcarOverlapAdd:
    """tools/dsp/overlapadd_boxcar.py:338-534.  nnet: callable [B, C, L] -> {key: [B, n_src, L]} (same length).

    window: None / False = plain boxcar (the frames are concatenated), or a scipy window name, multiplied onto every
    frame exactly as the reference does (`:497-498`).  reorder_chunks is only meaningful for n_src > 1 (source
    permutation, `:493-495`), which this path does not have: it must be False unless n_src == 1."""

    def __init__(self, nnet, n_src: Optional[int], window_size: int, in_margin: int, window=None,
                 reorder_chunks: bool = False, enable_grad: bool = False, device=None, max_batch: Optional[int] = 8):
        assert window_size % 2 == 0, "Window size must be even"          # :396
        self.max_batch = max_batch                                        # rows per nnet call when chunks are stacked
        self.reorder_chunks = reorder_chunks
        if in_margin <= 0 or in_margin >= window_size:
            raise ValueError("in_margin must be in (0, window_size)")     # :437-441: the unfold yields n/W chunks only then
        if reorder_chunks and n_src not in (None, 1):
            raise NotImplementedError("source reordering (n_src > 1) is outside this path")
        self.nnet = nnet
        self.window_size = window_size
        self.hop_size = window_size                                       # :399
        self.n_src = n_src
        self.in_margin = in_margin
        self.in_channels = getattr(nnet, "in_channels", None)
        self.enable_grad = enable_grad
        if window:
            from scipy.signal import get_window
            self.window = torch.from_numpy(get_window(window, window_size).astype("float32"))
            self.use_window = True
        else:
            self.window = None
            self.use_window = False

    # ------------------------------------------------------------------ chunk plan
    def plan(self, n_frames: int):
        """[(start, stop, crop_left, crop_right)] in samples of the zero-padded signal: chunk i feeds
        x_pad[start:stop] to the network and keeps out[crop_left : len - crop_right] (:452-470)."""
        W, M = self.window_size, self.in_margin
        last = n_frames - (n_frames // W) * W                                # :431
        n_chunks = (n_frames + W - 1) // W if n_frames > 0 else 0
        chunks = []
        for i in range(n_chunks):
            if i == 0:                                                      # :453-456 (also the single-chunk case)
                chunks.append((0, W + M, 0, M))
            elif i == n_chunks - 1 and last != 0:                           # :457-461
                chunks.append((i * W - M, i * W + last, M, 0))
            elif i == n_chunks - 1:                                         # :462-465
                chunks.append((i * W - M, (i + 1) * W, M, 0))
            else:                                                           # :466-473
                chunks.append((i * W - M, (i + 1) * W + M, M, M))
        return chunks, last

    # ------------------------------------------------------------------ forward
    def ola_forward(self, x: torch.Tensor, key: str = "wav") -> torch.Tensor:
        assert x.ndim == 3                                                  # :421
        batch, channels, n_frames = x.shape
        W, M = self.window_size, self.in_margin
        chunks, last = self.plan(n_frames)
        n_chunks = len(chunks)
        # zero padding: up to a multiple of the window (:432-433) plus the zero right margin of the final chunk (:445)
        xp = F.pad(x, (0, n_chunks * W + M - n_frames))
        frames = [None] * n_chunks

        def run(idx_list):
            """Run chunks of equal length; stacked along the batch dimension when the network allows it."""
            if not idx_list:
                return
            if getattr(self.nnet, "batch_invariant", False) and len(idx_list) > 1:
                per_call = len(idx_list) if not self.max_batch else max(1, self.max_batch // batch)
                for g0 in range(0, len(idx_list), per_call):
                    group = idx_list[g0:g0 + per_call]
                    stack = torch.cat([xp[..., chunks[i][0]:chunks[i][1]] for i in group], dim=0)
                    out = self.nnet(stack)[key]
                    for j, i in enumerate(group):
                        frames[i] = out[j * batch:(j + 1) * batch]
            else:
                for i in idx_list:
                    frames[i] = self.nnet(xp[..., chunks[i][0]:chunks[i][1]])[key]

        middle = [i for i in range(1, n_chunks - 1)]
        ends = [0] if n_chunks == 1 else [0, n_chunks - 1]
        run(middle)
        for i in ends:
            run([i])

        outs = []
        for i, (start, stop, cl, cr) in enumerate(chunks):
            f = frames[i]
            assert f.ndim == 3, "nnet should return (batch, n_src, time)"  # :477
            if self.n_src is not None:
                assert f.shape[1] == self.n_src, "nnet should return (batch, n_src, time)"
            if self.reorder_chunks and f.shape[1] > 1:                      # :493-495 would permute the sources here
                raise NotImplementedError("reorder_chunks with n_src > 1 (source permutation) is outside this path")
            f = f[..., cl:f.shape[-1] - cr]
            if f.shape[-1] < W:                                             # short last chunk (:461)
                f = F.pad(f, (0, W - f.shape[-1]))
            if self.use_window:
                f = f * self.window.to(f)                                   # :497-498
            else:
                f = f / (self.window_size / self.hop_size)                  # :499-500 (== 1 for the boxcar)
            outs.append(f)
        out = torch.cat(outs, dim=-1)                                       # fold with hop == window (:506-516)
        return out[..., :n_frames]                                          # :518

    def forward(self, x: torch.Tensor, key: str = "wav") -> torch.Tensor:
        with torch.autograd.set_grad_enabled(self.enable_grad):             # :522
            return self.ola_forward(x, key=key)

    __call__ = forward


class WindowedOverlapAdd:
    """tools/dsp/overlapadd.py:338-484 (`LambdaOverlapAdd`, windowed): the signal is zero-padded by one window on both
    sides, cut into windows of `window_size` every `hop_size` (default half a window), every window goes through
    `nnet`, is multiplied by the synthesis window and overlap-added back (`:419-466`).  All windows have the same
    length, so a batch-invariant network (the engine) processes them `max_batch` rows per call.

    window: scipy window name ("hanning", the reference's default spelling, is accepted for "hann"), or None/False for
    the unweighted average `frame / (window_size / hop_size)` (`:455-458`)."""

    def __init__(self, nnet, n_src: Optional[int], window_size: int, hop_size: Optional[int] = None, window="hanning",
                 reorder_chunks: bool = True, enable_grad: bool = False, device=None, max_batch: Optional[int] = 8):
        assert window_size % 2 == 0, "Window size must be even"          # :392
        self.max_batch = max_batch                                        # rows per nnet call when windows are stacked
        self.reorder_chunks = reorder_chunks
        if reorder_chunks and n_src not in (None, 1):
            raise NotImplementedError("source reordering (n_src > 1) is outside this path")
        self.nnet = nnet
        self.window_size = window_size
        self.hop_size = hop_size if hop_size is not None else window_size // 2   # :396
        self.n_src = n_src
        self.in_channels = getattr(nnet, "in_channels", None)
        self.enable_grad = enable_grad
        if window:
            from scipy.signal import get_window
            name = "hann" if window == "hanning" else window          # scipy dropped the old alias
            self.window = torch.from_numpy(get_window(name, window_size).astype("float32"))
            self.use_window = True
        else:
            self.window = None
            self.use_window = False

    def ola_forward(self, x: torch.Tensor, key: str = "wav") -> torch.Tensor:
        assert x.ndim == 3                                                  # :417
        batch, channels, n_frames = x.shape
        W, hop = self.window_size, self.hop_size
        unfolded = F.unfold(x.unsqueeze(-1), kernel_size=(W, 1), padding=(W, 0), stride=(hop, 1))   # :421-426
        n_chunks = unfolded.shape[-1]
        unfolded = unfolded.view(batch, channels, W, n_chunks)              # :431
        if getattr(self.nnet, "batch_invariant", False) and n_chunks > 1:
            stack = unfolded.permute(3, 0, 1, 2).reshape(n_chunks * batch, channels, W).contiguous()
            rows = stack.shape[0] if not self.max_batch else max(batch, self.max_batch // batch * batch)
            frames = torch.cat([self.nnet(stack[r0:r0 + rows])[key] for r0 in range(0, stack.shape[0], rows)], dim=0)
            assert frames.ndim == 3, "nnet should return (batch, n_src, time)"
            n_src = frames.shape[1]
            frames = frames.reshape(n_chunks, batch * n_src, W)
        else:
            outs = []
            n_src = None
            for i in range(n_chunks):                                       # :434-459
                f = self.nnet(unfolded[..., i])[key]
                assert f.ndim == 3, "nnet should return (batch, n_src, time)"
                n_src = f.shape[1]
                outs.append(f.reshape(batch * n_src, -1))
            frames = torch.stack(outs)
        if self.n_src is not None:
            assert n_src == self.n_src, "nnet should return (batch, n_src, time)"
        if self.reorder_chunks and n_src > 1:                               # :446-452 would run _reorder_sources here
            raise NotImplementedError("reorder_chunks with n_src > 1 (source permutation) is outside this path")
        if self.use_window:
            frames = frames * self.window.to(frames)                        # :455-456
        else:
            frames = frames / (W / hop)                                     # :457-458
        out = frames.reshape(n_chunks, batch * n_src, W).permute(1, 2, 0)   # :461-462
        out = F.fold(out, (n_frames, 1), kernel_size=(W, 1), padding=(W, 0), stride=(hop, 1))   # :464-470
        return out.squeeze(-1).reshape(batch, n_src, -1)

    def forward(self, x: torch.Tensor, key: str = "wav") -> torch.Tensor:
        with torch.autograd.set_grad_enabled(self.enable_grad):
            return self.ola_forward(x, key=key)

    __call__ = forward


def restore_longform(model, wav: torch.Tensor, window_size: int = 44100 * 30, in_margin: int = 44100 * 2,
                     unify_energy: bool = False, max_batch: Optional[int] = 8) -> torch.Tensor:
    """wav [B, N] on the model's device -> [B, N]: VoiceFixer.restore over 30 s windows with 2 s of context on
    both sides, middle windows batched `max_batch` rows per launch chain (8 x 34 s = ~38 GB of workspace).

    model may also be an SSR_UNet / GSR_UNet (restore() without unify_energy; unify_energy=True raises ValueError).  Its
    plans take about 1.4 times the bytes per frame, so 8 x 34 s would be a plan of about 60 GB, over the default plan budget
    (half the free memory) of an 80 GB card; the engine then runs the stack in sub-batches through smaller plans, with the
    same bits.  Measured on an NVIDIA H100 80GB HBM3 (700 W limit), B = 1, 300 s (eight middle chunks in one call): 0.6 s,
    3 plans of 15.2 GB cached at the end under a 41.9 GB budget, one plan evicted, and the bits of restoring every chunk
    alone."""
    ola = BoxcarOverlapAdd(RestoreNet(model, unify_energy=unify_energy), n_src=1, window_size=window_size, in_margin=in_margin,
                           max_batch=max_batch)
    return ola(wav[:, None, :])[:, 0, :]
