"""audio_diffusion_pytorch on H100: the reference's public names (reference __init__.py:1-20)
for the UNetV0 + VDiffusion/VSampler hot path, executed by hand-written sm_90a kernels.

Every name of the reference's export list is implemented; what is not supported inside one
(`use_text_conditioning=True`: T5 weights) raises on use instead of silently running something else."""
from .components import AppendChannelsPlugin, LTPlugin, MelSpectrogram, UNetV0
from .diffusion import (ARVDiffusion, ARVSampler, Diffusion, Distribution, Inpainter, LinearSchedule,
                        Sampler, Schedule, UniformDistribution, VDiffusion, VInpainter, VSampler)
from .models import (AdapterBase, DiffusionAE, DiffusionAR, DiffusionModel, DiffusionUpsampler,
                     DiffusionVocoder, EncoderBase)
from .unet import B200UNet


XUNet = B200UNet

__all__ = ["UNetV0", "XUNet", "LTPlugin", "MelSpectrogram", "VDiffusion", "VSampler", "VInpainter",
           "LinearSchedule", "UniformDistribution", "Diffusion", "Distribution", "Sampler",
           "Schedule", "DiffusionModel", "DiffusionUpsampler", "DiffusionVocoder", "DiffusionAE",
           "DiffusionAR", "ARVDiffusion", "ARVSampler", "EncoderBase", "AdapterBase", "AppendChannelsPlugin", "B200UNet", "Inpainter"]
