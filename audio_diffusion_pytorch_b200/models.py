"""The model classes users instantiate.  Same names, constructor keywords, attribute names
(`net`, `diffusion`, `sampler`, `to_spectrogram`, `to_flat`) and call signatures as reference
models.py:22-45 (DiffusionModel), :134-165 (DiffusionUpsampler), :168-224 (DiffusionVocoder);
the arithmetic behind `net`, `diffusion` and `sampler` is the CUDA path.  U-Net weights of a
reference model are taken over with `model.net.load_reference_parameters(ref_model.net)`
(same parameter order and shapes as a_unet's module tree)."""
from abc import ABC, abstractmethod
from typing import Any, Callable, Optional, Sequence, Tuple, Union

import torch
import torch.nn.functional as F
from torch import Generator, Tensor, nn

from .components import AppendChannelsPlugin, MelSpectrogram
from .diffusion import ARVDiffusion, ARVSampler, VDiffusion, VSampler
from .unet import UNetV0
from .utils import closest_power_2, default, downsample, groupby, randn_like, upsample


class DiffusionModel(nn.Module):
    """Three plugin slots around ONE shared net: `net_t(dim=..., **net kwargs)` builds it,
    `diffusion_t(net=, loss_fn=, **diffusion_* kwargs)` is the training objective (`forward`),
    `sampler_t(net=, **sampler_* kwargs)` the generation loop (`sample`, under no_grad)."""

    def __init__(self, net_t: Callable = UNetV0, diffusion_t: Callable = VDiffusion,
                 sampler_t: Callable = VSampler, loss_fn: Callable = F.mse_loss, dim: int = 1,
                 **kwargs):
        super().__init__()
        for_diffusion, kwargs = groupby("diffusion_", kwargs)
        for_sampler, net_kwargs = groupby("sampler_", kwargs)
        self.net = net_t(dim=dim, **net_kwargs)
        self.diffusion = diffusion_t(net=self.net, loss_fn=loss_fn, **for_diffusion)
        self.sampler = sampler_t(net=self.net, **for_sampler)

    def forward(self, *args, **kwargs) -> Tensor:
        return self.diffusion(*args, **kwargs)

    @torch.no_grad()
    def sample(self, *args, **kwargs) -> Tensor:
        return self.sampler(*args, **kwargs)

    def load_reference_state_dict(self, state_dict) -> None:
        """Takes over a checkpoint of the REFERENCE model class built with the same kwargs
        (`ref_model.state_dict()`): the U-Net tensors (`net.*`; the copies under `diffusion.net.*` /
        `sampler.net.*` are the same tensors) are matched by position (B200UNet.load_reference_state_dict),
        everything else (`to_flat`, `to_spectrogram`, a DiffusionAE `encoder`, ...) by name -- those
        attributes carry the reference's names."""
        shared = ("net.", "diffusion.net.", "sampler.net.")
        self.net.load_reference_state_dict(state_dict, prefix="net.")
        rest = {k: v for k, v in state_dict.items() if not k.startswith(shared)}
        result = self.load_state_dict(rest, strict=False)
        assert not result.unexpected_keys, f"unexpected keys {result.unexpected_keys}"
        missing = [k for k in result.missing_keys if not k.startswith(shared)]
        assert not missing, f"missing keys {missing}"


class EncoderBase(nn.Module, ABC):
    """What DiffusionAE needs from an encoder: `out_channels`, `downsample_factor` and
    `forward(x, with_info=True) -> (latent, info)` (reference models.py:48-55)."""

    @abstractmethod
    def __init__(self):
        super().__init__()
        self.out_channels = None
        self.downsample_factor = None


class AdapterBase(nn.Module, ABC):
    """Optional fixed transform around the diffusion domain (reference models.py:58-67)."""

    @abstractmethod
    def encode(self, x: Tensor) -> Tensor:
        pass

    @abstractmethod
    def decode(self, x: Tensor) -> Tensor:
        pass


class DiffusionAE(DiffusionModel):
    """Diffusion autoencoder (reference models.py:70-131): the encoder's latent is injected at
    `inject_depth` of the U-Net (`InjectChannelsItem`: conv1x1 over cat([x, latent]) + x); training
    back-propagates into the encoder through the context gradient of the CUDA backward program."""

    def __init__(self, in_channels: int, channels: Sequence[int], encoder: nn.Module, inject_depth: int,
                 latent_factor: Optional[int] = None, adapter: Optional[nn.Module] = None, **kwargs):
        context_channels = [0] * len(channels)
        context_channels[inject_depth] = encoder.out_channels
        super().__init__(in_channels=in_channels, channels=channels, context_channels=context_channels,
                         **kwargs)
        self.in_channels = in_channels
        self.encoder = encoder
        self.inject_depth = inject_depth
        self.latent_factor = default(latent_factor, self.encoder.downsample_factor)
        self.adapter = adapter.requires_grad_(False) if adapter is not None else None

    def forward(self, x: Tensor, with_info: bool = False, **kwargs) -> Union[Tensor, Tuple[Tensor, Any]]:
        latent, info = self.encode(x, with_info=True)
        context = [None] * self.inject_depth + [latent]
        x = self.adapter.encode(x) if self.adapter is not None else x
        loss = super().forward(x, channels=context, **kwargs)
        return (loss, info) if with_info else loss

    def encode(self, *args, **kwargs):
        return self.encoder(*args, **kwargs)

    @torch.no_grad()
    def decode(self, latent: Tensor, generator: Optional[Generator] = None, **kwargs) -> Tensor:
        length = closest_power_2(latent.shape[2] * self.latent_factor)
        noise = torch.randn((latent.shape[0], self.in_channels, length), device=latent.device,
                            dtype=latent.dtype, generator=generator)
        context = [None] * self.inject_depth + [latent]
        out = super().sample(noise, channels=context, **kwargs)
        return self.adapter.decode(out) if self.adapter is not None else out


class DiffusionAR(DiffusionModel):
    """Autoregressive diffusion over a sliding window (reference models.py:227-250): the net sees
    the waveform plus one channel carrying the per-position noise level, has no time conditioning
    and no ModulationItems (use_modulation=False: SkipCat merges)."""

    def __init__(self, in_channels: int, length: int, num_splits: int,
                 diffusion_t: Callable = ARVDiffusion, sampler_t: Callable = ARVSampler, **kwargs):
        super().__init__(in_channels=in_channels + 1, out_channels=in_channels,
                         diffusion_t=diffusion_t, diffusion_length=length, diffusion_num_splits=num_splits,
                         sampler_t=sampler_t, sampler_in_channels=in_channels, sampler_length=length,
                         sampler_num_splits=num_splits, use_time_conditioning=False, use_modulation=False,
                         **kwargs)


class DiffusionUpsampler(DiffusionModel):
    """Band-limited copy of the target (down- then up-sampled by `upsample_factor`) as extra
    input channels of the net; sampling starts from a low-rate waveform."""

    def __init__(self, in_channels: int, upsample_factor: int, net_t: Callable = UNetV0, **kwargs):
        self.upsample_factor = upsample_factor
        conditioned_net_t = AppendChannelsPlugin(net_t, channels=in_channels)
        super().__init__(net_t=conditioned_net_t, in_channels=in_channels, **kwargs)

    def reupsample(self, x: Tensor) -> Tensor:
        low = downsample(x.clone(), factor=self.upsample_factor)
        return upsample(low, factor=self.upsample_factor)

    def forward(self, x: Tensor, *args, **kwargs) -> Tensor:
        kwargs["append_channels"] = self.reupsample(x)
        return super().forward(x, *args, **kwargs)

    @torch.no_grad()
    def sample(self, downsampled: Tensor, generator: Optional[Generator] = None, **kwargs) -> Tensor:
        guide = upsample(downsampled, factor=self.upsample_factor)
        start = randn_like(guide, generator=generator)
        return super().sample(start, append_channels=guide, **kwargs)


class _ToFlat(torch.autograd.Function):
    """DiffusionVocoder.to_flat = ConvTranspose1d(mel -> 1, bias-free) as the adp_to_flat kernel;
    backward = adp_to_flat_bwd (weight gradient: the only trainable part of the front-end)."""

    @staticmethod
    def forward(ctx, spec: Tensor, weight: Tensor, hop: int, pad: int) -> Tensor:
        from . import ops
        spec, w = spec.contiguous(), weight.detach().float().reshape(weight.shape[0], -1).contiguous()
        ctx.save_for_backward(spec, w)
        ctx.geom = (hop, pad, weight.shape, weight.dtype)
        return ops.to_flat(spec, w, hop, pad)

    @staticmethod
    def backward(ctx, dout: Tensor):
        from . import ops
        spec, w = ctx.saved_tensors
        hop, pad, w_shape, w_dtype = ctx.geom
        dspec, dw = ops.to_flat_bwd(spec, w, dout.float().contiguous(), hop, pad,
                                    need_dspec=ctx.needs_input_grad[0], need_dw=ctx.needs_input_grad[1])
        return dspec, (None if dw is None else dw.reshape(w_shape).to(w_dtype)), None, None


class DiffusionVocoder(DiffusionModel):
    """Mel spectrogram -> waveform.  Every audio channel becomes its own batch row; a bias-free
    transposed convolution (`to_flat`) stretches the spectrogram to one waveform-rate channel
    that is appended to the net input."""

    def __init__(self, net_t: Callable = UNetV0, mel_channels: int = 80, mel_n_fft: int = 1024,
                 mel_hop_length: Optional[int] = None, mel_win_length: Optional[int] = None,
                 in_channels: int = 1, **kwargs):
        hop = default(mel_hop_length, int(mel_n_fft) // 4)
        win = default(mel_win_length, mel_n_fft)
        front_end_kwargs, kwargs = groupby("mel_", kwargs)
        super().__init__(net_t=AppendChannelsPlugin(net_t, channels=1), in_channels=1, **kwargs)
        self.to_spectrogram = MelSpectrogram(n_fft=mel_n_fft, hop_length=hop, win_length=win,
                                             n_mel_channels=mel_channels, **front_end_kwargs)
        self.to_flat = nn.ConvTranspose1d(mel_channels, 1, kernel_size=win, stride=hop,
                                          padding=(win - hop) // 2, bias=False)

    def _unroll(self, spectrogram: Tensor) -> Tuple[Tensor, torch.Size]:
        """[..., mel, frames] -> ([rows, 1, samples], leading shape)."""
        lead = spectrogram.shape[:-2]
        spec = spectrogram.reshape(-1, *spectrogram.shape[-2:])
        if spec.is_cuda:         # adp_to_flat (+ its weight / input gradients)
            flat = _ToFlat.apply(spec.float(), self.to_flat.weight, self.to_flat.stride[0],
                                 self.to_flat.padding[0])
            return flat[:, None, :].to(spectrogram.dtype), lead
        return self.to_flat(spec), lead

    def forward(self, x: Tensor, *args, **kwargs) -> Tensor:
        guide, _ = self._unroll(self.to_spectrogram(x))
        rows = x.reshape(-1, 1, x.shape[-1])
        return super().forward(rows, *args, append_channels=guide, **kwargs)

    @torch.no_grad()
    def sample(self, spectrogram: Tensor, generator: Optional[Generator] = None, **kwargs) -> Tensor:
        guide, lead = self._unroll(spectrogram)
        start = randn_like(guide, generator=generator)
        rows = super().sample(start, append_channels=guide, **kwargs)
        return rows.reshape(*lead, rows.shape[-1])
