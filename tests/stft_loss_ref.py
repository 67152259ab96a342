"""fp64 restatements of the multi-resolution STFT loss (audio_diffusion_pytorch_b200/losses.py's
docstring) for the tests: the loss in torch ops, the same loss through an explicit DFT matrix, and
its input gradient written out as the adjoint the CUDA backward computes (Hermitian extension, two
frames per complex inverse transform, window, overlap-add, reflect-pad fold)."""
import math

import torch
import torch.nn.functional as F

DEFAULT = [(1024, 120, 600), (2048, 240, 1200), (512, 50, 240)]


def _mag(s, n_fft, hop, win, eps):
    window = torch.hann_window(win, dtype=s.dtype, device=s.device)
    z = torch.stft(s, n_fft, hop, win, window, center=True, pad_mode="reflect", onesided=True,
                   return_complex=True)
    return torch.sqrt(torch.clamp(z.real ** 2 + z.imag ** 2, min=eps))


def resolution_terms(x, y, n_fft, hop, win, eps=1e-8):
    """(sc, log_mag, lin_mag) of one resolution, x and y [..., T] in their own dtype."""
    t = x.shape[-1]
    xm, ym = _mag(x.reshape(-1, t), n_fft, hop, win, eps), _mag(y.reshape(-1, t), n_fft, hop, win, eps)
    sc = ((ym - xm).flatten(1).norm(dim=1) / ym.flatten(1).norm(dim=1)).mean()
    return sc, (torch.log(xm) - torch.log(ym)).abs().mean(), (xm - ym).abs().mean()


def loss(x, y, resolutions=DEFAULT, w=(1.0, 1.0, 0.0), eps=1e-8):
    """The multi-resolution loss in the dtype of x and y (call with float64 tensors)."""
    total = 0.0
    for res in resolutions:
        sc, lg, ln = resolution_terms(x, y, *res, eps=eps)
        total = total + w[0] * sc + w[1] * lg + w[2] * ln
    return total / len(resolutions)


def frames_of(s, n_fft, hop, win):
    """Windowed frames [rows, frames, n_fft] of s [rows, T] reflect-padded by n_fft // 2."""
    pad = n_fft // 2
    sp = F.pad(s[:, None], (pad, pad), mode="reflect")[:, 0]
    fr = sp.unfold(-1, n_fft, hop)
    left = (n_fft - win) // 2
    window = F.pad(torch.hann_window(win, dtype=s.dtype, device=s.device), (left, n_fft - win - left))
    return fr * window


def loss_dft(x, y, resolutions, w=(1.0, 1.0, 0.0), eps=1e-8):
    """The same loss through an explicit one-sided DFT matrix (small n_fft only)."""
    t = x.shape[-1]
    x, y = x.reshape(-1, t), y.reshape(-1, t)
    total = 0.0
    for n_fft, hop, win in resolutions:
        k = torch.arange(n_fft // 2 + 1, dtype=torch.float64)[:, None]
        n = torch.arange(n_fft, dtype=torch.float64)[None]
        ang = 2 * math.pi * k * n / n_fft
        cos, sin = torch.cos(ang), -torch.sin(ang)

        def mag(s):
            fr = frames_of(s, n_fft, hop, win)                      # [rows, frames, N]
            re, im = fr @ cos.T, fr @ sin.T                          # [rows, frames, bins]
            return torch.sqrt(torch.clamp(re ** 2 + im ** 2, min=eps))
        xm, ym = mag(x), mag(y)
        sc = ((ym - xm).flatten(1).norm(dim=1) / ym.flatten(1).norm(dim=1)).mean()
        total = total + w[0] * sc + w[1] * (torch.log(xm) - torch.log(ym)).abs().mean() \
            + w[2] * (xm - ym).abs().mean()
    return total / len(resolutions)


def adjoint_dx(x, y, resolutions, w=(1.0, 1.0, 0.0), eps=1e-8, grad_out=1.0):
    """dL/dx [rows, T] by the steps of the CUDA backward, in the dtype of x (float64)."""
    rows, t = x.shape
    dx = torch.zeros_like(x)
    scale = 1.0 / len(resolutions)
    for n_fft, hop, win in resolutions:
        pad, bins = n_fft // 2, n_fft // 2 + 1
        fx, fy = frames_of(x, n_fft, hop, win), frames_of(y, n_fft, hop, win)
        X, Y = torch.fft.rfft(fx, dim=-1), torch.fft.rfft(fy, dim=-1)
        p2 = X.real ** 2 + X.imag ** 2
        xm = torch.sqrt(torch.clamp(p2, min=eps))
        ym = torch.sqrt(torch.clamp(Y.real ** 2 + Y.imag ** 2, min=eps))
        frames = X.shape[1]
        count = rows * frames * bins
        dn = (ym - xm).flatten(1).norm(dim=1)[:, None, None]
        yn = ym.flatten(1).norm(dim=1)[:, None, None]
        a_sc = torch.where(dn > 0, scale * w[0] / rows / (dn * yn), torch.zeros_like(dn))
        g = a_sc * (xm - ym) + scale * w[1] / count * torch.sign(torch.log(xm) - torch.log(ym)) / xm \
            + scale * w[2] / count * torch.sign(xm - ym)
        G = torch.where(p2 >= eps, grad_out * g * X / xm, torch.zeros_like(X))
        # Hermitian extension of G, two frames per complex inverse transform
        H = G / 2
        H[..., 0] = G[..., 0].real
        if n_fft % 2 == 0:
            H[..., -1] = G[..., -1].real
        full = torch.zeros(rows, frames, n_fft, dtype=X.dtype)
        full[..., :bins] = H
        ks = torch.arange(1, (n_fft + 1) // 2)
        full[..., n_fft - ks] = H[..., ks].conj()
        if frames % 2:
            full = torch.cat([full, torch.zeros_like(full[:, :1])], dim=1)
        Z = full[:, 0::2] + 1j * full[:, 1::2]
        h = torch.fft.ifft(Z, dim=-1) * n_fft                       # sum_k Z_k e^{+2 pi i k n / N}
        fgrad = torch.stack([h.real, h.imag], dim=2).reshape(rows, -1, n_fft)[:, :frames]
        left = (n_fft - win) // 2
        window = F.pad(torch.hann_window(win, dtype=x.dtype), (left, n_fft - win - left))
        fgrad = fgrad * window
        # overlap-add onto the padded signal, then fold the reflect pad back onto x
        dp = torch.zeros(rows, t + 2 * pad, dtype=x.dtype)
        for f in range(frames):
            dp[:, f * hop:f * hop + n_fft] += fgrad[:, f]
        d = dp[:, pad:pad + t].clone()
        d[:, 1:pad + 1] += dp[:, :pad].flip(-1)
        d[:, t - 1 - pad:t - 1] += dp[:, t + pad:].flip(-1)
        dx += d
    return dx
