"""Plugins around the net (reference components.py:162-236)."""
from typing import Callable, Optional

import torch
import torch.nn.functional as F
from torch import Tensor, nn

from .unet import B200UNet, UNetV0  # noqa: F401  (UNetV0 re-exported like the reference)
from .utils import default


class _Appended(nn.Module):
    """Generic AppendChannelsPlugin for a net that is not the CUDA U-Net: concatenate, call."""

    def __init__(self, net: nn.Module):
        super().__init__()
        self.net = net

    def forward(self, x: Tensor, *args, append_channels: Tensor, **kwargs):
        return self.net(torch.cat([x, append_channels], dim=1), *args, **kwargs)


def AppendChannelsPlugin(net_t: Callable, channels: int):
    """reference components.py:162-180.  With the CUDA U-Net the concatenation is never
    materialised: the stem kernels read `x` and `append_channels` through two base pointers."""

    def Net(in_channels: int, out_channels: Optional[int] = None, **kwargs) -> nn.Module:
        out_channels = default(out_channels, in_channels)
        if net_t is UNetV0 or net_t is B200UNet:
            return B200UNet(in_channels=in_channels + channels, out_channels=out_channels,
                            append_channels=channels, **kwargs)
        return _Appended(net_t(in_channels=in_channels + channels, out_channels=out_channels,
                               **kwargs))

    return Net


class _LearnedTransform(nn.Module):
    """encode -> net -> decode; parameters registered in the reference's order (encode, decode, net)."""

    def __init__(self, encode: nn.Module, decode: nn.Module, net: nn.Module):
        super().__init__()
        self.encode, self.decode, self.net = encode, decode, net

    def forward(self, x: Tensor, *args, **kwargs) -> Tensor:
        return self.decode(self.net(self.encode(x), *args, **kwargs))


def LTPlugin(net_t: Callable, num_filters: int, window_length: int, stride: int):
    """Learned Transform plugin (reference components.py:113-157): a strided learned filterbank
    (Conv1d, reflect padding, bias-free) in front of the net and its transposed counterpart behind
    it; the net runs on `in_channels * num_filters` channels at 1/stride of the rate.  The two
    filterbank convolutions are PyTorch modules around the net call; with the CUDA U-Net inside, its
    boundary limits apply to the TRANSFORMED widths (in_channels * num_filters <= 64 inputs and
    outputs, in_channels * num_filters * factors[0] <= 128, channels[0] <= 256; stereo x 32 filters
    fits) and are asserted by its constructor."""

    def Net(dim: int, in_channels: int, out_channels: Optional[int] = None, **kwargs) -> nn.Module:
        assert dim == 1, "the reference builds a ConvTranspose1d decoder: dim must be 1"
        out_channels = default(out_channels, in_channels)
        wide_in, wide_out = in_channels * num_filters, out_channels * num_filters
        padding = window_length // 2 - stride // 2
        encode = nn.Conv1d(in_channels, wide_in, kernel_size=window_length, stride=stride,
                           padding=padding, padding_mode="reflect", bias=False)
        decode = nn.ConvTranspose1d(wide_out, out_channels, kernel_size=window_length, stride=stride,
                                    padding=padding, bias=False)
        net = net_t(dim=dim, in_channels=wide_in, out_channels=wide_out, **kwargs)
        return _LearnedTransform(encode, decode, net)

    return Net


class MelSpectrogram(nn.Module):
    """reference components.py:188-236 (DiffusionVocoder training front-end; runs once per
    call outside the step loop, torchaudio STFT + mel filterbank)."""

    def __init__(self, n_fft: int, hop_length: int, win_length: int, sample_rate: int,
                 n_mel_channels: int, center: bool = False, normalize: bool = False,
                 normalize_log: bool = False):
        super().__init__()
        from torchaudio import transforms
        self.padding = (n_fft - hop_length) // 2
        self.normalize, self.normalize_log, self.hop_length = normalize, normalize_log, hop_length
        self.to_spectrogram = transforms.Spectrogram(
            n_fft=n_fft, hop_length=hop_length, win_length=win_length, center=center, power=None)
        self.to_mel_scale = transforms.MelScale(
            n_mels=n_mel_channels, n_stft=n_fft // 2 + 1, sample_rate=sample_rate)

    def _kernel_tables(self, device):
        """Window padded to n_fft (torch.stft centres a shorter window) and, per mel filter, the
        bin range [lo, hi) it is non-zero on (a triangle): inputs of adp_mel_spectrogram."""
        cached = getattr(self, "_tables", None)
        stamp = (device, self.to_spectrogram.window._version, self.to_mel_scale.fb._version)
        if cached is None or cached[3] != stamp:
            n_fft = self.to_spectrogram.n_fft
            win = self.to_spectrogram.window.to(device=device, dtype=torch.float32)
            left = (n_fft - win.numel()) // 2
            window = F.pad(win, (left, n_fft - win.numel() - left)).contiguous()
            fb = self.to_mel_scale.fb.to(device=device, dtype=torch.float32).contiguous()
            nz = fb != 0
            bins = torch.arange(fb.shape[0], device=device)[:, None]
            lo = torch.where(nz, bins, fb.shape[0]).amin(0)
            hi = torch.where(nz, bins + 1, 0).amax(0)
            band = torch.stack([torch.minimum(lo, hi), hi], dim=1).to(torch.int32).contiguous()
            cached = self._tables = (window, fb, band, stamp)
        return cached[:3]

    def forward(self, waveform: Tensor) -> Tensor:
        lead, t = waveform.shape[:-1], waveform.shape[-1]
        if waveform.is_cuda and not (torch.is_grad_enabled() and waveform.requires_grad):
            # one kernel: framing, window, FFT, magnitude, mel filters (+ log); autograd through
            # the STFT (a waveform that requires grad) keeps the tensor-op route below.  center=True
            # reflects the padded signal once more by n_fft // 2, as torch.stft does
            from . import ops
            window, fb, band = self._kernel_tables(waveform.device)
            n_fft = self.to_spectrogram.n_fft
            mel = ops.mel_spectrogram(waveform.reshape(-1, t).float().contiguous(), window, fb, band,
                                      n_fft, self.hop_length, self.padding,
                                      apply_log=self.normalize_log and not self.normalize,
                                      center_pad=n_fft // 2 if self.to_spectrogram.center else 0)
            if self.normalize:
                mel = 2 * torch.pow(mel / torch.max(mel), 0.25) - 1
                if self.normalize_log:
                    mel = torch.log(torch.clamp(mel, min=1e-5))
            return mel.reshape(*lead, *mel.shape[-2:]).to(waveform.dtype)
        flat = F.pad(waveform.reshape(-1, t), [self.padding] * 2, mode="reflect")
        mel = self.to_mel_scale(torch.abs(self.to_spectrogram(flat)))
        if self.normalize:
            mel = mel / torch.max(mel)
            mel = 2 * torch.pow(mel, 0.25) - 1
        if self.normalize_log:
            mel = torch.log(torch.clamp(mel, min=1e-5))
        return mel.reshape(*lead, *mel.shape[-2:])
