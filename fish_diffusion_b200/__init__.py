"""fish_diffusion_b200 -- H100-native (sm_90a) implementation of fish-diffusion's data-parallel hot path:
the WaveNet and ConvNext diffusion denoisers + DDPM/PLMS/UniPC samplers and the NSF-HiFiGAN vocoder with its mel front end,
behind the reference's DENOISERS / DIFFUSIONS / VOCODERS registries.  See DESIGN.md and INTEGRATION.md.

Importing this package registers the native classes under the reference's registry names
("WaveNetDenoiser", "ConvNextDenoiser", "GaussianDiffusion", "NsfHifiGAN").  The compute path is libfishdiff_b200.so
(hand-written CUDA for sm_90a, C ABI in include/fishdiff_b200.h); there is no CPU or PyTorch fallback.
"""
from .registry import DENOISERS, DIFFUSIONS, VOCODERS, Registry  # noqa: F401
from .wavenet import WaveNet  # noqa: F401
from .convnext import ConvNext  # noqa: F401
from .diffusion import GaussianDiffusion, NaiveNoisePredictor, PLMSNoisePredictor, UNIPCNoisePredictor  # noqa: F401
from .nsf_hifigan import Generator, NsfHifiGAN  # noqa: F401
from .mel import (MelSpectrogram, PitchAdjustableMelSpectrogram, dynamic_range_compression, get_mel_from_audio,  # noqa: F401
                  get_mel_transform)
from .resample import resample, resample_length  # noqa: F401
from .diffsinger import ENCODERS, DiffSinger, NaiveProjectionEncoder, load_checkpoint, pitch_to_scale  # noqa: F401
from .fastspeech import FastSpeech2Encoder  # noqa: F401
from .pipeline import BatchedSynthesizer, plan_batches  # noqa: F401
from . import formats  # noqa: F401
from .vocoder_gan import (HifiGanTrainer, MultiPeriodDiscriminator, MultiScaleDiscriminator,  # noqa: F401
                          average_gradients)
from .vocoder_train import generator_forward_train  # noqa: F401
from .trainers import DiffSingerTrainer, WarmupCosine, ema_update  # noqa: F401

__version__ = "0.1.0"
