"""audio_diffusion_pytorch on H100: the reference's public names (reference __init__.py:1-20)
for the UNetV0 + VDiffusion/VSampler hot path, executed by hand-written sm_90a kernels.

Every name of the reference's export list is implemented; what is not supported inside one
(`use_text_conditioning=True`: T5 weights) raises on use instead of silently running something else."""
from .components import AppendChannelsPlugin, LTPlugin, MelSpectrogram, UNetV0
from .diffusion import (ARVDiffusion, ARVSampler, Diffusion, Distribution, DPMSolverSampler, Inpainter,
                        LinearSchedule, Sampler, Schedule, UniformDistribution, VDiffusion, VInpainter, VSampler)
from .losses import MultiResolutionSTFTLoss, STFTLoss
from .models import (AdapterBase, DiffusionAE, DiffusionAR, DiffusionModel, DiffusionUpsampler,
                     DiffusionVocoder, EncoderBase)
from .apex import ClassifierFreeGuidancePlugin, TimeConditioningPlugin, XUNet
from .unet import B200UNet

__all__ = ["UNetV0", "XUNet", "LTPlugin", "MelSpectrogram", "VDiffusion", "VSampler", "DPMSolverSampler", "VInpainter",
           "LinearSchedule", "UniformDistribution", "Diffusion", "Distribution", "Sampler",
           "Schedule", "DiffusionModel", "DiffusionUpsampler", "DiffusionVocoder", "DiffusionAE",
           "DiffusionAR", "ARVDiffusion", "ARVSampler", "EncoderBase", "AdapterBase", "AppendChannelsPlugin", "B200UNet", "Inpainter",
           "MultiResolutionSTFTLoss", "STFTLoss", "TimeConditioningPlugin", "ClassifierFreeGuidancePlugin"]
