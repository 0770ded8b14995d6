"""H100-native (sm_90a) VoiceFixer inference hot path (stages A/B/C of eval_gsr_voicefixer.py:handler) and the SSR/GSR-UNet path."""
from .arch import VocoderConfig  # noqa: F401
from .model import (Engine, FDomainHelper, GSR_UNet, HParams, MelScale, SSR_UNet, VoiceFixer, Vocoder,  # noqa: F401
                    default_hparams, get_hparams_from_file)
