"""Multi-resolution STFT loss, a `loss_fn` for the diffusion models (the loss of the reference's
`DiffusionAE` example, auraloss.freq.MultiResolutionSTFTLoss, with its keyword names).

Definition.  For each resolution (N = fft_size, hop = hop_size, W = win_length):
  1. rows are `input.reshape(-1, T)`: batch and channel are flattened;
  2. X = torch.stft(row, N, hop, W, torch.hann_window(W), center=True, pad_mode="reflect",
     onesided=True, return_complex=True): the periodic Hann window, zero-padded to the centre of N;
  3. mag = sqrt(clamp(re^2 + im^2, min=eps)), for `input` (Xmag) and `target` (Ymag);
  4. sc = mean over rows of ||Ymag - Xmag||_F / ||Ymag||_F, each norm over the row's bins and frames;
  5. log_mag = mean |log Xmag - log Ymag| and lin_mag = mean |Xmag - Ymag|, over all elements;
  6. L_r = w_sc * sc + w_log_mag * log_mag + w_lin_mag * lin_mag.
The multi-resolution loss is the mean of L_r over the resolutions.  The spectral-convergence ratio is
taken per row and then averaged (older auraloss releases took one ratio over the whole batch).
Gradients go to `input` only: a `target` that requires grad is refused.

On CUDA tensors (fp32 or bf16, fp32 arithmetic) the loss runs on csrc/stft_loss.cu: per resolution
one forward launch (one FFT per frame and signal) and one fixed-order reduction, and
in the backward one launch that recomputes the spectra and applies the adjoint of the transform and
one that overlap-adds the frame gradients onto dx.  The result and dx are bitwise reproducible.
Envelope of the CUDA route: fft_size in [32, 8192] with prime factors 2, 3, 5, 7 only,
win_length <= fft_size, hop_size >= 1, T > fft_size // 2, at most 65535 rows.  Host tensors take
the same definition in torch ops, at any size torch.stft accepts.
"""
from typing import List, Sequence, Tuple

import torch
from torch import Tensor, nn

from . import ops

# auraloss options this module does not implement, with the value that means "off": passing that
# value is accepted, anything else is refused with the option named
_OFF = {"w_phs": 0.0, "sample_rate": None, "scale": None, "n_bins": None, "perceptual_weighting": False,
        "scale_invariance": False, "output": "loss", "reduction": "mean", "mag_distance": "L1",
        "device": None}


def _refuse_options(cls: str, window: str, options: dict) -> None:
    if window != "hann_window":
        raise ValueError(f"{cls}: window={window!r} is not supported (only 'hann_window')")
    for name, value in options.items():
        if name not in _OFF:
            raise TypeError(f"{cls}: unknown option {name!r}")
        if value != _OFF[name]:
            raise ValueError(f"{cls}: {name}={value!r} is not supported (only {name}={_OFF[name]!r})")


def _host_loss(x: Tensor, y: Tensor, resolutions: Sequence[Tuple[int, int, int]], weights, eps: float) -> Tensor:
    """The definition above in torch ops (host tensors), in float64 for float64 inputs and in float32
    otherwise."""
    w_sc, w_log, w_lin = weights
    t = x.shape[-1]
    dtype = torch.float64 if x.dtype == torch.float64 else torch.float32
    x = x.reshape(-1, t).to(dtype)
    y = y.reshape(-1, t).to(dtype)
    total = 0.0
    for n_fft, hop, win in resolutions:
        window = torch.hann_window(win, dtype=x.dtype, device=x.device)

        def mag(s):
            z = torch.stft(s, n_fft, hop, win, window, center=True, pad_mode="reflect", onesided=True,
                           return_complex=True)
            return torch.sqrt(torch.clamp(z.real ** 2 + z.imag ** 2, min=eps))
        xm, ym = mag(x), mag(y)
        sc = ((ym - xm).flatten(1).norm(dim=1) / ym.flatten(1).norm(dim=1)).mean()
        log_mag = (torch.log(xm) - torch.log(ym)).abs().mean()
        lin_mag = (xm - ym).abs().mean()
        total = total + w_sc * sc + w_log * log_mag + w_lin * lin_mag
    return total / len(resolutions)


_WINDOWS = {}


def _window(n_fft: int, win: int, device) -> Tensor:
    """torch.hann_window(win) zero-padded to the centre of n_fft, as torch.stft applies it."""
    key = (n_fft, win, str(device))
    w = _WINDOWS.get(key)
    if w is None:
        left = (n_fft - win) // 2
        w = torch.nn.functional.pad(torch.hann_window(win, dtype=torch.float32), (left, n_fft - win - left))
        w = _WINDOWS[key] = w.to(device).contiguous()
    return w


def _frames(t: int, n_fft: int, hop: int) -> int:
    return 1 + (t + 2 * (n_fft // 2) - n_fft) // hop


def _fwd(x: Tensor, y: Tensor, res, weights, eps: float, scale: float, acc: Tensor, loss: Tensor,
         accumulate: bool) -> Tensor:
    """One resolution's forward (adp_stft_loss_fwd): acc / loss (+)= scale * L_r; returns the
    per-row norms {||Y - X||, ||Y||} the backward reads."""
    rows, t = x.shape
    n_fft, hop, win = res
    frames = _frames(t, n_fft, hop)
    window = _window(n_fft, win, x.device)
    partials = torch.empty(rows, (frames + 7) // 8, 4, device=x.device, dtype=torch.float64)
    stats = torch.empty(rows, 2, device=x.device, dtype=torch.float64)
    ops._launch("adp_stft_loss_fwd", (
        x.data_ptr(), y.data_ptr(), window.data_ptr(), partials.data_ptr(), stats.data_ptr(), acc.data_ptr(),
        loss.data_ptr(), rows, t, n_fft, hop, win, frames, 1 if x.dtype == torch.bfloat16 else 0, eps,
        *weights, scale, 1 if accumulate else 0),
        lambda: (f"stft_loss_fwd[n_fft={n_fft}]", 0, ops._nb(x, y)))
    return stats


def _bwd(x: Tensor, y: Tensor, res, weights, eps: float, scale: float, stats: Tensor, grad_out: Tensor,
         dx: Tensor, dx_bf16, accumulate: bool) -> None:
    """One resolution's backward (adp_stft_loss_bwd): dx (+)= grad_out * d(scale * L_r)/dx."""
    rows, t = x.shape
    n_fft, hop, win = res
    frames = _frames(t, n_fft, hop)
    window = _window(n_fft, win, x.device)
    frame_grad = torch.empty(rows, frames, win, device=x.device, dtype=torch.float32)
    ops._launch("adp_stft_loss_bwd", (
        x.data_ptr(), y.data_ptr(), window.data_ptr(), stats.data_ptr(), grad_out.data_ptr(),
        frame_grad.data_ptr(), dx.data_ptr(), ops._p(dx_bf16), rows, t, n_fft, hop, win, frames,
        1 if x.dtype == torch.bfloat16 else 0, eps, *weights, scale, 1 if accumulate else 0),
        lambda: (f"stft_loss_bwd[n_fft={n_fft}]", 0, ops._nb(x, y, dx)))


class _STFTLossFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor, y: Tensor, resolutions, weights, eps: float) -> Tensor:
        scale = 1.0 / len(resolutions)
        acc = torch.empty(1, device=x.device, dtype=torch.float64)
        loss = torch.empty((), device=x.device, dtype=torch.float32)
        stats = [_fwd(x, y, res, weights, eps, scale, acc, loss, i > 0) for i, res in enumerate(resolutions)]
        ctx.save_for_backward(x, y, *stats)
        ctx.config = (resolutions, weights, eps)
        return loss

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        x, y, *stats = ctx.saved_tensors
        resolutions, weights, eps = ctx.config
        scale = 1.0 / len(resolutions)
        grad_out = grad_out.detach().float().reshape(1).contiguous()
        dx = torch.empty(x.shape, device=x.device, dtype=torch.float32)
        dx_bf16 = torch.empty_like(x) if x.dtype == torch.bfloat16 else None
        last = len(resolutions) - 1
        for i, (res, st) in enumerate(zip(resolutions, stats)):
            _bwd(x, y, res, weights, eps, scale, st, grad_out, dx, dx_bf16 if i == last else None, i > 0)
        return (dx if dx_bf16 is None else dx_bf16), None, None, None, None


def _stft_loss(cls: str, input: Tensor, target: Tensor, resolutions, weights, eps: float) -> Tensor:
    if input.shape != target.shape:
        raise ValueError(f"{cls}: input {tuple(input.shape)} and target {tuple(target.shape)} differ in shape")
    if torch.is_grad_enabled() and target.requires_grad:
        raise ValueError(f"{cls}: gradients go to input only; detach the target")
    if not input.is_cuda:
        return _host_loss(input, target, resolutions, weights, eps)
    if input.dtype not in (torch.float32, torch.bfloat16) or target.dtype != input.dtype:
        raise TypeError(f"{cls}: CUDA input and target must both be float32 or both bfloat16 "
                        f"(got {input.dtype} and {target.dtype})")
    if target.device != input.device:
        raise ValueError(f"{cls}: input on {input.device}, target on {target.device}")
    t = input.shape[-1]
    x = input.reshape(-1, t).contiguous()
    y = target.detach().reshape(-1, t).contiguous()
    return _STFTLossFunction.apply(x, y, tuple(resolutions), tuple(float(w) for w in weights), float(eps))


class STFTLoss(nn.Module):
    """One resolution of the loss defined in this module's docstring (auraloss.freq.STFTLoss's
    keywords); called as loss(input, target) on [B, C, T] tensors, returns a 0-d tensor."""

    def __init__(self, fft_size: int = 1024, hop_size: int = 256, win_length: int = 1024,
                 window: str = "hann_window", w_sc: float = 1.0, w_log_mag: float = 1.0,
                 w_lin_mag: float = 0.0, eps: float = 1e-8, **options):
        super().__init__()
        _refuse_options("STFTLoss", window, options)
        self.fft_size, self.hop_size, self.win_length = int(fft_size), int(hop_size), int(win_length)
        self.window = window
        self.w_sc, self.w_log_mag, self.w_lin_mag, self.eps = float(w_sc), float(w_log_mag), float(w_lin_mag), float(eps)

    def forward(self, input: Tensor, target: Tensor) -> Tensor:
        return _stft_loss("STFTLoss", input, target, [(self.fft_size, self.hop_size, self.win_length)],
                          (self.w_sc, self.w_log_mag, self.w_lin_mag), self.eps)


class MultiResolutionSTFTLoss(nn.Module):
    """Mean of STFTLoss over (fft_sizes, hop_sizes, win_lengths) (auraloss.freq.MultiResolutionSTFTLoss's
    keywords and defaults); on CUDA tensors all resolutions run in one autograd node."""

    def __init__(self, fft_sizes: List[int] = (1024, 2048, 512), hop_sizes: List[int] = (120, 240, 50),
                 win_lengths: List[int] = (600, 1200, 240), window: str = "hann_window", w_sc: float = 1.0,
                 w_log_mag: float = 1.0, w_lin_mag: float = 0.0, eps: float = 1e-8, **options):
        super().__init__()
        if not (len(fft_sizes) == len(hop_sizes) == len(win_lengths)) or not fft_sizes:
            raise ValueError("MultiResolutionSTFTLoss: fft_sizes, hop_sizes and win_lengths must be "
                             "non-empty and of one length")
        _refuse_options("MultiResolutionSTFTLoss", window, options)
        self.stft_losses = nn.ModuleList(
            STFTLoss(fs, ss, wl, window, w_sc, w_log_mag, w_lin_mag, eps)
            for fs, ss, wl in zip(fft_sizes, hop_sizes, win_lengths))

    def forward(self, input: Tensor, target: Tensor) -> Tensor:
        first = self.stft_losses[0]
        return _stft_loss("MultiResolutionSTFTLoss", input, target,
                          [(f.fft_size, f.hop_size, f.win_length) for f in self.stft_losses],
                          (first.w_sc, first.w_log_mag, first.w_lin_mag), first.eps)
