"""Static description of the two networks on the hot path.

The analysis ResUNet shape is fixed by the reference
(models/components/unet.py:13-55, models/components/modules.py:167-271): six
encoder stages of four pre-activation residual blocks, a bottleneck block, six
decoder stages (ConvTranspose2d k3 s2 + four residual blocks), one post block
and a 1x1 head.  State-dict key names follow the reference checkpoint layout
(SURVEY.md appendix B) so a reference checkpoint loads unchanged.

The vocoder is a third-party dependency of the reference (`voicefixer` PyPI
package, unpinned at requirements.txt:6; call sites models/gsr_voicefixer.py:113,
eval_gsr_voicefixer.py:66).  Its source is absent, so `VocoderConfig` restates
the published generator design (cond-net, k7 stem, four transposed-conv
upsamplers x441 with dilated residual stacks, k7 + tanh tail) with every
hyper-parameter exposed.  Parity for that stage is pinned only against
oracle/vf_oracle.py ("parity unpinned" by the reference itself).
"""
from dataclasses import dataclass, field
from typing import List, Tuple

UNET_PREFIX = "generator.analysis_module."      # VoiceFixer's mel UNet (models/gsr_voicefixer.py:50,139)
SSR_PREFIX = "generator.unet."                  # unet_v2 inside SSR_UNet / GSR_UNet (models/ssr_unet.py:49, gsr_unet.py:49)

ENC_CHANNELS = [(1, 32), (32, 64), (64, 128), (128, 256), (256, 384), (384, 384)]
DEC_CHANNELS = [(384, 384), (384, 384), (384, 256), (256, 128), (128, 64), (64, 32)]
BN_EPS = 1e-5            # nn.BatchNorm2d default, modules.py:232-233
LRELU_SLOPE = 0.01       # modules.py:265-266
DOWNSAMPLE = 64          # unet.py:20


def conv_block_res_keys(prefix: str, cin: int, cout: int) -> List[Tuple[str, Tuple[int, ...]]]:
    """Keys of one ConvBlockRes (modules.py:223-271) in state-dict order."""
    keys = []
    for bn, c in (("bn1", cin), ("bn2", cout)):
        keys += [(f"{prefix}.{bn}.weight", (c,)), (f"{prefix}.{bn}.bias", (c,)),
                 (f"{prefix}.{bn}.running_mean", (c,)), (f"{prefix}.{bn}.running_var", (c,)),
                 (f"{prefix}.{bn}.num_batches_tracked", ())]
    keys += [(f"{prefix}.conv1.weight", (cout, cin, 3, 3)),
             (f"{prefix}.conv2.weight", (cout, cout, 3, 3))]
    if cin != cout:
        keys += [(f"{prefix}.shortcut.weight", (cout, cin, 1, 1)),
                 (f"{prefix}.shortcut.bias", (cout,))]
    return keys


def unet_keys() -> List[Tuple[str, Tuple[int, ...]]]:
    """All UNet state-dict keys with shapes, relative to UNET_PREFIX, in
    the registration order of unet.py:22-53."""
    keys = []
    for i, (cin, cout) in enumerate(ENC_CHANNELS, 1):
        for j in range(1, 5):
            keys += conv_block_res_keys(f"encoder_block{i}.conv_block{j}", cin if j == 1 else cout, cout)
    keys += conv_block_res_keys("conv_block7", 384, 384)
    for i, (cin, cout) in enumerate(DEC_CHANNELS, 1):
        p = f"decoder_block{i}"
        keys += [(f"{p}.conv1.weight", (cin, cout, 3, 3))]          # ConvTranspose2d: [Cin,Cout,3,3]
        keys += [(f"{p}.bn1.weight", (cin,)), (f"{p}.bn1.bias", (cin,)),
                 (f"{p}.bn1.running_mean", (cin,)), (f"{p}.bn1.running_var", (cin,)),
                 (f"{p}.bn1.num_batches_tracked", ())]
        for j in range(2, 6):
            keys += conv_block_res_keys(f"{p}.conv_block{j}", 2 * cout if j == 2 else cout, cout)
    keys += conv_block_res_keys("after_conv_block1", 32, 32)
    keys += [("after_conv2.weight", (1, 32, 1, 1)), ("after_conv2.bias", (1,))]
    return keys


def _bn1_keys(prefix: str) -> List[Tuple[str, Tuple[int, ...]]]:
    """nn.BatchNorm2d(1) keys: the analysis modules normalise the [B, 1, T, F] tensor as one channel."""
    return [(f"{prefix}.weight", (1,)), (f"{prefix}.bias", (1,)), (f"{prefix}.running_mean", (1,)),
            (f"{prefix}.running_var", (1,)), (f"{prefix}.num_batches_tracked", ())]


def _linear_keys(prefix: str, cin: int, cout: int) -> List[Tuple[str, Tuple[int, ...]]]:
    return [(f"{prefix}.weight", (cout, cin)), (f"{prefix}.bias", (cout,))]


N_MEL = 128
GRU_HIDDEN = 2 * N_MEL      # BN_GRU(input_dim=n_mel*2, hidden_dim=n_mel*2, bidirectional=True, layer=2)


def bigru_keys() -> List[Tuple[str, Tuple[int, ...]]]:
    """State-dict keys of the `bi_gru` analysis module (models/gsr_voicefixer.py:54-64, BN_GRU :14-42) with shapes, relative
    to UNET_PREFIX, in registration order: 0 BatchNorm2d(1), 1 Linear, 2 BN_GRU (bn, then the nn.GRU), 4 and 6 Linear."""
    h = GRU_HIDDEN
    keys = _bn1_keys("0") + _linear_keys("1", N_MEL, h) + _bn1_keys("2.bn")
    for layer in range(2):
        cin = h if layer == 0 else 2 * h
        for sfx in ("", "_reverse"):
            keys += [(f"2.gru.weight_ih_l{layer}{sfx}", (3 * h, cin)), (f"2.gru.weight_hh_l{layer}{sfx}", (3 * h, h)),
                     (f"2.gru.bias_ih_l{layer}{sfx}", (3 * h,)), (f"2.gru.bias_hh_l{layer}{sfx}", (3 * h,))]
    return keys + _linear_keys("4", 2 * h, h) + _linear_keys("6", h, N_MEL)


DNN_WIDTHS = [N_MEL, 2 * N_MEL, 4 * N_MEL, 8 * N_MEL, 4 * N_MEL, 2 * N_MEL, N_MEL]
DNN_LINEARS = [0, 3, 6, 9, 12, 14]          # Sequential indices of the Linear layers; a BatchNorm2d(1) precedes 3, 6, 9, 12


def dnn_keys() -> List[Tuple[str, Tuple[int, ...]]]:
    """State-dict keys of the `dnn` analysis module (models/gsr_voicefixer.py:65-83) with shapes, relative to UNET_PREFIX, in
    registration order."""
    keys = []
    for i, idx in enumerate(DNN_LINEARS):
        if 1 <= i <= 4:
            keys += _bn1_keys(str(idx - 1))
        keys += _linear_keys(str(idx), DNN_WIDTHS[i], DNN_WIDTHS[i + 1])
    return keys


@dataclass
class VocoderConfig:
    """Frozen hyper-parameters of the stage-C generator restatement."""
    num_mels: int = 128
    cond_channels: int = 512
    cond_layers: int = 5
    channels: int = 1024
    upsample_scales: List[int] = field(default_factory=lambda: [7, 7, 3, 3])
    resstack_depth: List[int] = field(default_factory=lambda: [8, 8, 8, 8])
    resstack_kernel: int = 3
    stem_kernel: int = 7
    stage_slope: float = 0.2      # LeakyReLU between stages
    res_slope: float = 0.01       # nn.LeakyReLU() default inside the residual stacks
    min_db: float = -115.0
    ref_db: float = 20.0
    amp_floor: float = 1e-5
    tail_pad_value: float = -4.0
    tail_pad_base: int = 4        # pad frames = T % 2 + tail_pad_base
    mel_weight_a: float = 18.8927416350036
    mel_weight_b: float = 0.0269863588184314
    hop: int = 441
    tail_tanh: bool = True        # False: linear tail (test configurations whose output exceeds |1|)

    def stage_channels(self) -> List[Tuple[int, int]]:
        c = self.channels
        return [(c >> i, c >> (i + 1)) for i in range(len(self.upsample_scales))]

    def dilation(self, i: int) -> int:
        return 3 ** (i % 10)


def vocoder_keys(cfg: VocoderConfig) -> List[Tuple[str, Tuple[int, ...]]]:
    """State-dict keys of the vocoder restatement (weight-norm already folded),
    prefixed `vocoder.` inside a full VoiceFixer state dict."""
    keys = []
    cin = cfg.num_mels
    for i in range(cfg.cond_layers):
        keys += [(f"condnet.{i}.weight", (cfg.cond_channels, cin, 3)), (f"condnet.{i}.bias", (cfg.cond_channels,))]
        cin = cfg.cond_channels
    keys += [("stem.weight", (cfg.channels, cin, cfg.stem_kernel)), ("stem.bias", (cfg.channels,))]
    for s, ((ci, co), scale, depth) in enumerate(zip(cfg.stage_channels(), cfg.upsample_scales, cfg.resstack_depth)):
        keys += [(f"up.{s}.weight", (ci, co, 2 * scale)), (f"up.{s}.bias", (co,))]   # ConvTranspose1d: [Cin,Cout,k]
        for i in range(depth):
            for ab in ("a", "b"):
                keys += [(f"res.{s}.{i}.{ab}.weight", (co, co, cfg.resstack_kernel)),
                         (f"res.{s}.{i}.{ab}.bias", (co,))]
    c_last = cfg.stage_channels()[-1][1]
    keys += [("tail.weight", (1, c_last, cfg.stem_kernel)), ("tail.bias", (1,))]
    return keys


def frames_for(n_samples: int, hop: int = 441) -> int:
    """center=True STFT frame count (fDomainHelper.py:26-28 / torchlibrosa)."""
    return 1 + n_samples // hop


def metric_frames(n_samples: int, rate: int = 44100) -> int:
    """Frames of AudioMetrics.wav_to_spectrogram at `rate` (librosa's center=True count 1 + (n + 2 (n_fft // 2) - n_fft) //
    hop): frames_for(n) at 44.1 kHz (n_fft 2048, hop 441); 1 + (n - 1) // 160 at 16 kHz, where n_fft 743 is odd."""
    if rate == 16000:
        return 1 + (n_samples - 1) // 160
    if rate == 44100:
        return frames_for(n_samples)
    raise ValueError(f"Bad Samplerate: {rate} Hz")


def padded_frames(t: int) -> int:
    """unet.py:75-77: time axis zero-padded up to a multiple of 64."""
    return ((t + DOWNSAMPLE - 1) // DOWNSAMPLE) * DOWNSAMPLE


def vocoder_out_len(t: int, cfg: VocoderConfig) -> int:
    return (t + t % 2 + cfg.tail_pad_base) * cfg.hop


def vocoder_receptive_field(cfg: VocoderConfig = None) -> int:
    """R, in frames: the smallest margin such that mel frames outside [a - R, b + R) cannot change the vocoder's output
    samples of frames [a, b) (frame t's samples are [t hop, (t + 1) hop)).  A chunk with R frames of context on each side of
    its kept frames therefore gives those frames the samples of the whole mel; 576 frames (5.76 s) for the default config.

    Derived layer by layer: the interval a perturbation of one frame p reaches, in the units of each layer's output -
      - each of the cond_layers k3 convs (padding 1): +-1 frame;
      - the k7 reflect-padded stem: +-(stem_kernel // 2) frames;
      - each stage's ConvTranspose1d (stride s, kernel 2s, padding s // 2 + s % 2 = P): input [lo, hi] reaches output
        samples [lo s - P, hi s - P + 2s - 1] at the stage's rate;
      - each of the stage's resstack_depth residual pairs: the dilated k3 conv (dilation 3^i) +-3^i, the k3 conv after it
        +-1, in that stage's samples;
      - the k7 reflect-padded tail: +-(stem_kernel // 2) output samples.
    The frames of the samples reached, [floor(lo / hop), floor(hi / hop)], are then p - left .. p + right, and R =
    max(left, right).  Reflect and zero padding at a clip's edges and the constant tail frames only fold or drop what this
    interval holds, so no edge reaches farther; with every tap of the seeded weights non-zero the bound is tight."""
    cfg = cfg or VocoderConfig()
    h = cfg.resstack_kernel // 2
    hi = cfg.cond_layers + cfg.stem_kernel // 2          # frame p = 0 through the cond-net and the stem
    lo = -hi
    for scale, depth in zip(cfg.upsample_scales, cfg.resstack_depth):
        pad = scale // 2 + scale % 2
        lo, hi = lo * scale - pad, hi * scale - pad + 2 * scale - 1
        reach = sum(cfg.dilation(i) * h + h for i in range(depth))
        lo, hi = lo - reach, hi + reach
    lo, hi = lo - cfg.stem_kernel // 2, hi + cfg.stem_kernel // 2
    return max(-(lo // cfg.hop), hi // cfg.hop)
