"""`diffusion_t` / `sampler_t` plugin slots (reference diffusion.py), CUDA-native.

VDiffusion and VSampler keep the reference constructors and call signatures
(reference diffusion.py:68-95, :158-190).  When the wrapped net is the CUDA U-Net the
per-step arithmetic is fused into the net's last kernel and the loop launches one CUDA
graph per step; with any other `net` the same algebra runs as the generic fused
`adp_sampler_step` kernel after the net call.  DPMSolverSampler (DPM-Solver++(2M)) takes the same
slot: its update is the `adp_dpm_step` kernel, inside the step graph with the CUDA U-Net.
"""
from math import inf, isfinite, log, pi, sin
from typing import Any, List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch import Tensor
from tqdm import tqdm

from . import ops
from .unet import B200UNet


class Distribution:
    """Interface used by different distributions (reference diffusion.py:16-20)."""

    def __call__(self, num_samples: int, device: torch.device):
        raise NotImplementedError()


class UniformDistribution(Distribution):
    """reference diffusion.py:23-30"""

    def __init__(self, vmin: float = 0.0, vmax: float = 1.0):
        super().__init__()
        self.vmin, self.vmax = vmin, vmax

    def __call__(self, num_samples: int, device: torch.device = torch.device("cpu")):
        return (self.vmax - self.vmin) * torch.rand(num_samples, device=device) + self.vmin


class Diffusion(nn.Module):
    """Interface used by different diffusion methods"""


class Schedule(nn.Module):
    """Interface used by different sampling schedules (reference diffusion.py:135-139)."""

    def forward(self, num_steps: int, device: torch.device) -> Tensor:
        raise NotImplementedError()


class LinearSchedule(Schedule):
    """reference diffusion.py:142-148"""

    def __init__(self, start: float = 1.0, end: float = 0.0):
        super().__init__()
        self.start, self.end = start, end

    def forward(self, num_steps: int, device: Any) -> Tensor:
        return torch.linspace(self.start, self.end, num_steps, device=device)


class Sampler(nn.Module):
    pass


def _alpha_beta(sigmas: Tensor) -> Tuple[Tensor, Tensor]:
    angle = sigmas * pi / 2          # reference diffusion.py:77-80
    return torch.cos(angle), torch.sin(angle)


def _progress(label: str, num_steps: int, host_sig: Optional[List[float]]):
    """range(num_steps) through a tqdm bar, shown when `host_sig` is given: a host copy of the
    schedule, made once per call, whose next value the bar's description shows after each step (the
    reference formats a device scalar every step = one sync per step, reference diffusion.py:188)."""
    bar = tqdm(range(num_steps), disable=host_sig is None)
    for i in bar:
        yield i
        if host_sig is not None:
            bar.set_description(f"{label} (noise={host_sig[i + 1]:.2f})")


def _inner_b200(net: nn.Module) -> Optional[B200UNet]:
    return net if isinstance(net, B200UNet) else None


class VDiffusion(Diffusion):
    """v-objective diffusion loss (reference diffusion.py:68-95).

    RNG contract kept: `sigma_distribution(B)` is drawn first, then `randn_like(x)`, both on
    x.device.  With the CUDA net the noising (`alpha*x + beta*noise`) is fused into the first
    kernel and the MSE against `alpha*noise - beta*x` into the last."""

    def __init__(self, net: nn.Module, sigma_distribution: Distribution = UniformDistribution(),
                 loss_fn: Any = F.mse_loss):
        super().__init__()
        self.net = net
        self.sigma_distribution = sigma_distribution
        self.loss_fn = loss_fn

    def get_alpha_beta(self, sigmas: Tensor) -> Tuple[Tensor, Tensor]:
        return _alpha_beta(sigmas)

    def forward(self, x: Tensor, **kwargs) -> Tensor:
        batch_size, device = x.shape[0], x.device
        sigmas = self.sigma_distribution(num_samples=batch_size, device=device)   # :85
        noise = torch.randn_like(x)                                               # :88
        net = _inner_b200(self.net)
        if net is not None and self.loss_fn is F.mse_loss:
            from .training import fused_v_loss
            return fused_v_loss(net, x, noise, sigmas, **kwargs)
        sig_b = sigmas.view(-1, *([1] * (x.ndim - 1)))
        alphas, betas = _alpha_beta(sig_b)
        x_noisy = alphas * x + betas * noise                                      # :91
        v_target = alphas * noise - betas * x                                     # :92
        v_pred = self.net(x_noisy, sigmas, **kwargs)                              # :94
        return self.loss_fn(v_pred, v_target)                                     # :95


class ARVDiffusion(Diffusion):
    """v-objective with one noise level per SPLIT of the clip (reference diffusion.py:98-130): the
    per-position sigma rides along as an extra input channel, the net has no time conditioning.

    RNG contract kept: `rand((B, 1, num_splits))` first, then `randn_like(x)`, both on x.device.
    The pointwise noising runs as tensor ops (autograd records them for dL/dx); the net is the
    CUDA differentiable program (`B200UNet.forward` under grad mode)."""

    def __init__(self, net: nn.Module, length: int, num_splits: int, loss_fn: Any = F.mse_loss):
        super().__init__()
        assert length % num_splits == 0, "length must be divisible by num_splits"
        self.net = net
        self.length, self.num_splits = length, num_splits
        self.split_length = length // num_splits
        self.loss_fn = loss_fn

    def get_alpha_beta(self, sigmas: Tensor) -> Tuple[Tensor, Tensor]:
        return _alpha_beta(sigmas)

    def forward(self, x: Tensor, **kwargs) -> Tensor:
        b, t = x.shape[0], x.shape[2]
        assert t == self.length, "input length must match length"
        per_split = torch.rand((b, 1, self.num_splits), device=x.device, dtype=x.dtype)      # :118
        sigmas = per_split.repeat_interleave(self.split_length, dim=2)                      # :119
        noise = torch.randn_like(x)                                                          # :121
        alphas, betas = _alpha_beta(sigmas)
        x_noisy = alphas * x + betas * noise                                                 # :124
        v_target = alphas * noise - betas * x                                                # :125
        v_pred = self.net(torch.cat([x_noisy, sigmas], dim=1), **kwargs)                     # :127-129
        return self.loss_fn(v_pred, v_target)


class ARVSampler(Sampler):
    """Autoregressive sampler over a ladder of per-split noise levels (reference
    diffusion.py:193-298).  `sample_loop` keeps cat([current, sigma_i]) resident in the net's input
    buffer: one graph launch + one `adp_arv_step` per step (B200UNet.arv_loop)."""

    def __init__(self, net: nn.Module, in_channels: int, length: int, num_splits: int):
        super().__init__()
        assert length % num_splits == 0, "length must be divisible by num_splits"
        self.length, self.in_channels, self.num_splits = length, in_channels, num_splits
        self.split_length = length // num_splits
        self.net = net

    @property
    def device(self):
        return next(self.net.parameters()).device

    def get_alpha_beta(self, sigmas: Tensor) -> Tuple[Tensor, Tensor]:
        return _alpha_beta(sigmas)

    def get_sigmas_ladder(self, num_items: int, num_steps_per_split: int) -> Tensor:
        """[steps+1, B, 1, 2*(n//2)*l]: the first half of the window stays clean (context), the
        second half is a staircase of n//2 noise levels, lowest first, that one `sample_loop`
        lowers by exactly one stair; row `steps` is row 0 shifted by one split (reference :213-221)."""
        n_half, l, k = self.num_splits // 2, self.split_length, num_steps_per_split
        levels = torch.linspace(1, 0, k * n_half, device=self.device).view(n_half, k).t()    # [k, n_half]
        stairs = levels.repeat_interleave(l, dim=1).flip(-1)                                 # [k, n_half*l]
        stairs = torch.cat([stairs, torch.zeros_like(stairs[:1])], dim=0)
        stairs[-1, l:] = stairs[0, :-l]
        ladder = torch.cat([torch.zeros_like(stairs), stairs], dim=-1)
        return ladder[:, None, None, :].repeat(1, num_items, 1, 1)

    def sample_loop(self, current: Tensor, sigmas: Tensor, show_progress: bool = False, **kwargs) -> Tensor:
        num_steps = sigmas.shape[0] - 1
        progress = _progress("Sampling", num_steps, sigmas[:, 0, 0, 0].tolist() if show_progress else None)
        net = _inner_b200(self.net)
        if net is not None:
            return net.arv_loop(current, sigmas, progress=progress if show_progress else None, **kwargs)
        chan = torch.cat([current, sigmas[0]], dim=1).float().contiguous()
        sig = sigmas.float().reshape(num_steps + 1, current.shape[0], -1).contiguous()
        for i in progress:
            v = self.net(chan, **kwargs).float().contiguous()                                 # :231-232
            ops.arv_step(chan, v, sig[i + 1])                                                 # :233-235
        return chan[:, : current.shape[1]].to(current.dtype)

    def sample_start(self, num_items: int, num_steps: int, **kwargs) -> Tensor:
        b, c, t = num_items, self.in_channels, self.length
        sigmas = torch.linspace(1, 0, num_steps + 1, device=self.device)                      # :243
        sigmas = sigmas[:, None, None, None].repeat(1, b, 1, t)
        noise = torch.randn((b, c, t), device=self.device) * sigmas[0]                        # :245
        return self.sample_loop(current=noise, sigmas=sigmas, **kwargs)

    @torch.no_grad()
    def forward(self, num_items: int, num_chunks: int, num_steps: int, start: Optional[Tensor] = None,
                show_progress: bool = False, **kwargs) -> Tensor:
        n = self.num_splits
        assert num_chunks >= n, f"required at least {n} chunks"
        start = self.sample_start(num_items=num_items, num_steps=num_steps, **kwargs)         # :263
        if num_chunks == n:
            return start
        assert num_steps >= n, "num_steps must be greater than num_splits"
        sigmas = self.get_sigmas_ladder(num_items=num_items, num_steps_per_split=num_steps // n)
        alphas, betas = _alpha_beta(sigmas)
        # noise the start window up to the ladder, then slide: every pass lowers the last n chunks
        # by one stair and a fresh pure-noise chunk enters at the end (:278-296)
        noised = alphas[0] * start + betas[0] * torch.randn_like(start)
        chunks = list(noised.chunk(chunks=n, dim=-1))
        for _ in tqdm(range(num_chunks), disable=not show_progress):
            window = self.sample_loop(current=torch.cat(chunks[-n:], dim=-1), sigmas=sigmas, **kwargs)
            chunks[-n:] = list(window.chunk(chunks=n, dim=-1))
            chunks.append(torch.randn((num_items, self.in_channels, self.split_length), device=self.device))
        return torch.cat(chunks[:num_chunks], dim=-1)


class Inpainter(nn.Module):
    pass


class VInpainter(Inpainter):
    """reference diffusion.py:306-354: sampling with a known region.  `mask` (bool, True = keep
    `source`) selects what is replaced, after every net evaluation, by the source noised to the
    current level; `num_resamples` evaluations per step (RePaint-style)."""

    diffusion_types = [VDiffusion]

    def __init__(self, net: nn.Module, schedule: "Schedule" = None):
        super().__init__()
        self.net = net
        self.schedule = LinearSchedule() if schedule is None else schedule

    def get_alpha_beta(self, sigmas: Tensor) -> Tuple[Tensor, Tensor]:
        return _alpha_beta(sigmas)

    @torch.no_grad()
    def forward(self, source: Tensor, mask: Tensor, num_steps: int, num_resamples: int,
                show_progress: bool = False, x_noisy: Optional[Tensor] = None, **kwargs) -> Tensor:
        x_noisy = torch.randn_like(source) if x_noisy is None else x_noisy            # :331
        b = x_noisy.shape[0]
        sigmas_1d = self.schedule(num_steps + 1, device=x_noisy.device)              # :333
        sigmas = sigmas_1d[:, None].expand(-1, b)
        alphas, betas = _alpha_beta(sigmas_1d)
        progress = _progress("Inpainting", num_steps, sigmas_1d.tolist() if show_progress else None)
        net = _inner_b200(self.net)
        if net is not None:
            return net.inpaint_loop(x_noisy, source, mask, sigmas, alphas, betas, num_resamples,
                                    progress=progress if show_progress else None, **kwargs)
        x = x_noisy.float().contiguous().clone()
        src = source.float().expand_as(x).contiguous()
        mask_u8 = mask.expand_as(x).to(torch.uint8).contiguous()
        a, bt = alphas.float(), betas.float()
        for i in progress:
            for r in range(num_resamples):
                j = int(r == num_resamples - 1)
                ab = torch.stack([a[i], bt[i], a[i + j], bt[i + j]]).contiguous()
                v = self.net(x, sigmas[i], **kwargs).float().contiguous()             # :340
                ops.sampler_step(x, v, ab, x)                                         # :341-345
                noise = torch.randn_like(source).float().expand_as(x).contiguous()    # :346
                ops.inpaint_blend(x, src, noise, mask_u8, ab)                         # :346-350
        return x.to(x_noisy.dtype)


class VSampler(Sampler):
    """reference diffusion.py:158-190"""

    diffusion_types = [VDiffusion]

    def __init__(self, net: nn.Module, schedule: Schedule = LinearSchedule()):
        super().__init__()
        self.net = net
        self.schedule = schedule

    def get_alpha_beta(self, sigmas: Tensor) -> Tuple[Tensor, Tensor]:
        return _alpha_beta(sigmas)

    @torch.no_grad()
    def forward(self, x_noisy: Tensor, num_steps: int, show_progress: bool = False,
                **kwargs) -> Tensor:
        b = x_noisy.shape[0]
        sigmas_1d = self.schedule(num_steps + 1, device=x_noisy.device)           # :177
        sigmas = sigmas_1d[:, None].expand(-1, b)                                 # :178
        alphas, betas = _alpha_beta(sigmas_1d)                                    # :180
        progress = _progress("Sampling", num_steps, sigmas_1d.tolist() if show_progress else None)
        net = _inner_b200(self.net)
        if net is not None:
            return net.sample_loop(x_noisy, sigmas, alphas, betas,
                                   progress=progress if show_progress else None, **kwargs)
        ab = torch.stack([alphas[:-1], betas[:-1], alphas[1:], betas[1:]], 1).float().contiguous()
        x = x_noisy.float().contiguous().clone()
        for i in progress:
            v = self.net(x, sigmas[i], **kwargs).float().contiguous()             # :184
            ops.sampler_step(x, v, ab[i], x)                                      # :185-187
        return x.to(x_noisy.dtype)


def _log_snr(a: float, b: float) -> float:
    """lambda = log(alpha / beta): -inf at alpha = 0 (sigma = 1), +inf at beta = 0 (sigma = 0)."""
    if a <= 0.0:
        return -inf
    return inf if b <= 0.0 else log(a) - log(b)


def dpm_coefficients(sigmas: Tensor) -> Tensor:
    """The per-step rows (alpha_i, beta_i, c1, c2, k) of DPM-Solver++(2M) (Lu et al. 2022, Algorithm
    2) for a schedule sigmas [N + 1] in [0, 1], computed in float64 on the host and returned as fp32
    [N, 5] on the host.  With alpha = cos(pi sigma / 2), beta = sin(pi sigma / 2) and lambda =
    log(alpha / beta), step i (sigma_i -> sigma_i+1, h_i = lambda_i+1 - lambda_i) is
        x0_i = alpha_i x_i - beta_i v_i
        x_i+1 = c1 x_i + c2 ((1 + k) x0_i - k x0_i-1),   c1 = beta_i+1 / beta_i,   c2 = alpha_i+1 - alpha_i c1
    with k = h_i / (2 h_i-1), except k = 0 on the first step, on a last step to sigma = 0 (as
    k-diffusion's sample_dpmpp_2m) and after a step with h = inf.  alpha is evaluated as
    sin(pi (1 - sigma) / 2), clamped to >= 0, so that it is exactly 0 at sigma = 1: lambda = -inf
    there and the step from sigma = 1 has h = inf (cos(pi / 2) rounds to 6e-17 instead).  With
    k = 0 the step is VSampler's."""
    s = [float(v) for v in sigmas.detach().double().cpu()]
    a = [max(sin(pi * (1.0 - v) / 2), 0.0) for v in s]
    b = [sin(pi * v / 2) for v in s]
    lam = [_log_snr(ai, bi) for ai, bi in zip(a, b)]
    n = len(s) - 1
    rows = []
    h_prev = None
    for i in range(n):
        h = lam[i + 1] - lam[i]
        c1 = b[i + 1] / b[i]
        k = 0.0
        if h_prev is not None and isfinite(h_prev) and not (i == n - 1 and s[n] == 0.0):
            k = h / (2 * h_prev)
        rows.append([a[i], b[i], c1, a[i + 1] - a[i] * c1, k])
        h_prev = h
    return torch.tensor(rows, dtype=torch.float64).float()


def _dpm_step(x: Tensor, v: Tensor, hist: Tensor, table: Tensor, step: Tensor, rows: int) -> None:
    """One DPM-Solver++(2M) update (adp_dpm_step), in place on x and hist: the coefficients are row
    min(step[0], rows - 1) of table [rows, 5] (dpm_coefficients), step a device int32 counter."""
    ops._launch("adp_dpm_step", (x.data_ptr(), v.data_ptr(), hist.data_ptr(), table.data_ptr(),
                                 step.data_ptr(), rows, x.numel()),
                lambda: ("dpm_step", 0, ops._nb(x, v, hist, x, hist)))


def _check_schedule(sigmas: Tensor) -> None:
    s = sigmas.detach().double().cpu()
    if s.numel() < 2 or not bool(torch.all(s[1:] < s[:-1])):
        raise ValueError(f"DPMSolverSampler: the schedule must be strictly decreasing (got {s.tolist()})")
    if not bool(torch.all((s >= 0) & (s <= 1))):
        raise ValueError(f"DPMSolverSampler: the schedule leaves [0, 1] (got {s.tolist()})")


class DPMSolverSampler(Sampler):
    """Second-order multistep sampling of v-diffusion: DPM-Solver++(2M) (Lu et al. 2022, Algorithm
    2; the edge steps of k-diffusion's sample_dpmpp_2m), one net evaluation per step like VSampler
    and the same call.  The update (dpm_coefficients) runs as adp_dpm_step after the net: with the
    CUDA U-Net inside its sampling step graph (B200UNet.dpm_loop), with any other net after
    `net(x, sigma_i)`.  For num_steps <= 2 on a schedule from 1 to 0 it is VSampler's update."""

    diffusion_types = [VDiffusion]

    def __init__(self, net: nn.Module, schedule: Schedule = LinearSchedule()):
        super().__init__()
        self.net = net
        self.schedule = schedule

    def get_alpha_beta(self, sigmas: Tensor) -> Tuple[Tensor, Tensor]:
        return _alpha_beta(sigmas)

    @torch.no_grad()
    def forward(self, x_noisy: Tensor, num_steps: int, show_progress: bool = False,
                **kwargs) -> Tensor:
        b, c = x_noisy.shape[0], x_noisy.shape[1]
        out_channels = getattr(self.net, "out_channels", c)
        if out_channels != c:
            raise ValueError(f"DPMSolverSampler: the net's out_channels={out_channels} differs from the {c} "
                             f"channels of x (the update needs v of x's shape)")
        sigmas_1d = self.schedule(num_steps + 1, device=x_noisy.device)
        _check_schedule(sigmas_1d)
        sigmas = sigmas_1d[:, None].expand(-1, b)
        coef = dpm_coefficients(sigmas_1d).to(x_noisy.device)
        progress = _progress("Sampling", num_steps, sigmas_1d.tolist() if show_progress else None)
        net = _inner_b200(self.net)
        if net is not None:
            return net.dpm_loop(x_noisy, sigmas, coef, progress=progress if show_progress else None, **kwargs)
        x = x_noisy.float().contiguous().clone()
        hist = torch.empty_like(x)
        step = torch.zeros(1, dtype=torch.int32, device=x.device)
        for i in progress:
            v = self.net(x, sigmas[i], **kwargs).float().contiguous()
            if v.shape != x.shape:
                raise ValueError(f"DPMSolverSampler: the net returned {tuple(v.shape)} for x of shape "
                                 f"{tuple(x.shape)} (the update needs v of x's shape)")
            _dpm_step(x, v, hist, coef[i:], step, num_steps - i)
        return x.to(x_noisy.dtype)
