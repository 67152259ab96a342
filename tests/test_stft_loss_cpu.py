"""MultiResolutionSTFTLoss / STFTLoss without a GPU: defaults and refused options, the host route
against the fp64 restatement (tests/stft_loss_ref.py), the restatement against an explicit DFT
matrix, gradcheck of the restatement, and the adjoint the CUDA backward implements against autograd
of the restatement, all in float64."""
import pytest
import torch

import stft_loss_ref as ref
import audio_diffusion_pytorch_b200 as adp


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def test_defaults_follow_auraloss():
    loss = adp.MultiResolutionSTFTLoss()
    assert [(f.fft_size, f.hop_size, f.win_length) for f in loss.stft_losses] == ref.DEFAULT
    f = loss.stft_losses[0]
    assert (f.window, f.w_sc, f.w_log_mag, f.w_lin_mag, f.eps) == ("hann_window", 1.0, 1.0, 0.0, 1e-8)
    one = adp.STFTLoss()
    assert (one.fft_size, one.hop_size, one.win_length) == (1024, 256, 1024)
    # auraloss's "off" values are accepted
    adp.MultiResolutionSTFTLoss(w_phs=0.0, sample_rate=None, scale=None, n_bins=None, perceptual_weighting=False,
                                scale_invariance=False, output="loss", reduction="mean", mag_distance="L1")


@pytest.mark.parametrize("option,value", [("w_phs", 1.0), ("perceptual_weighting", True), ("scale", "mel"),
                                          ("n_bins", 128), ("sample_rate", 44100), ("scale_invariance", True),
                                          ("mag_distance", "L2"), ("reduction", "none"), ("output", "full"),
                                          ("window", "hamming_window")])
def test_unsupported_options_are_refused_by_name(option, value):
    for cls in (adp.MultiResolutionSTFTLoss, adp.STFTLoss):
        with pytest.raises(ValueError, match=option):
            cls(**{option: value})
    with pytest.raises(TypeError, match="bogus"):
        adp.STFTLoss(bogus=1)
    with pytest.raises(ValueError):
        adp.MultiResolutionSTFTLoss(fft_sizes=[512], hop_sizes=[128, 64], win_lengths=[512])


def test_target_requiring_grad_is_refused():
    x = torch.randn(1, 1, 2048)
    with pytest.raises(ValueError, match="input only"):
        adp.MultiResolutionSTFTLoss()(x, torch.randn(1, 1, 2048, requires_grad=True))
    with torch.no_grad():
        adp.MultiResolutionSTFTLoss()(x, torch.randn(1, 1, 2048, requires_grad=True))


def _grads(mod, x, y):
    xg = x.clone().requires_grad_(True)
    loss = mod(xg, y)
    loss.backward()
    return loss.detach(), xg.grad


@pytest.mark.parametrize("w", [(1.0, 1.0, 0.0), (0.5, 2.0, 1.5)])
def test_host_route_matches_the_fp64_restatement(w):
    g = torch.Generator().manual_seed(0)
    x, y = torch.randn(2, 2, 6000, generator=g), torch.randn(2, 2, 6000, generator=g)
    x[0, 1, 1000:3000] = 0.0                       # a silent stretch: bins reach the clamp
    y[1, 0, 2000:5000] = 0.0
    mod = adp.MultiResolutionSTFTLoss(w_sc=w[0], w_log_mag=w[1], w_lin_mag=w[2])
    x64 = x.double().requires_grad_(True)
    want = ref.loss(x64, y.double(), w=w)
    want.backward()
    # float64 inputs: the host route is the restatement
    got, dx = _grads(mod, x.double(), y.double())
    assert got.dim() == 0 and got.dtype == torch.float64
    assert abs(float(got) - float(want)) <= 1e-12 * float(want) and rel(dx, x64.grad) < 1e-12
    # float32: the loss to 1e-5.  The L1 terms' gradients are ill-conditioned in fp32 (the log term's
    # 1 / Xmag at the smallest bins, sign flips of |Xmag - Ymag| where the magnitudes agree to
    # rounding), so the whole dx is held to 3e-3 and the spectral-convergence term's dx to 1e-5
    got, dx = _grads(mod, x, y)
    assert got.dtype == torch.float32 and abs(float(got) - float(want)) / float(want) < 1e-5
    assert rel(dx, x64.grad) < 3e-3
    x64.grad = None
    ref.loss(x64, y.double(), w=(w[0], 0.0, 0.0)).backward()
    _, dx = _grads(adp.MultiResolutionSTFTLoss(w_sc=w[0], w_log_mag=0.0), x, y)
    assert rel(dx, x64.grad) < 1e-5
    one = adp.STFTLoss(fft_size=400, hop_size=100, win_length=300, w_sc=w[0], w_log_mag=w[1], w_lin_mag=w[2])
    want1 = ref.loss(x.double(), y.double(), [(400, 100, 300)], w=w)
    assert abs(float(one(x, y)) - float(want1)) / float(want1) < 1e-5


@pytest.mark.parametrize("n_fft,hop,win", [(32, 8, 32), (32, 5, 20), (33, 7, 33), (45, 10, 30), (48, 16, 17)])
def test_restatement_matches_an_explicit_dft(n_fft, hop, win):
    g = torch.Generator().manual_seed(n_fft + win)
    x = torch.randn(3, 2, 200, generator=g, dtype=torch.float64)
    y = torch.randn(3, 2, 200, generator=g, dtype=torch.float64)
    w = (1.0, 1.0, 0.7)
    a = ref.loss(x, y, [(n_fft, hop, win)], w=w)
    b = ref.loss_dft(x, y, [(n_fft, hop, win)], w=w)
    assert abs(float(a) - float(b)) <= 1e-12 * abs(float(b))


def test_gradcheck_of_the_restatement():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 2, 40, generator=g, dtype=torch.float64, requires_grad=True)
    y = torch.randn(1, 2, 40, generator=g, dtype=torch.float64)
    res = [(16, 4, 16), (15, 3, 10)]
    assert torch.autograd.gradcheck(lambda v: ref.loss(v, y, res, w=(1.0, 1.0, 0.5)), (x,))


@pytest.mark.parametrize("res,t", [(((32, 8, 32),), 100), (((33, 7, 20),), 17), (((48, 5, 30), (35, 9, 35)), 61),
                                   (((64, 16, 40),), 33), (((50, 12, 50),), 26)])
def test_adjoint_matches_autograd_of_the_restatement(res, t):
    """Short signals (t just above n_fft // 2) reach both folds of the reflect pad."""
    g = torch.Generator().manual_seed(t)
    x = torch.randn(3, t, generator=g, dtype=torch.float64)
    y = torch.randn(3, t, generator=g, dtype=torch.float64)
    x[1, : t // 3] = 0.0                           # silent stretches reach the clamp's mask
    y[2, t // 2:] = 0.0
    w = (1.0, 1.0, 0.6)
    xr = x.clone().requires_grad_(True)
    (0.7 * ref.loss(xr, y, list(res), w=w)).backward()
    got = ref.adjoint_dx(x, y, list(res), w=w, grad_out=0.7)
    assert rel(got, xr.grad) < 1e-12
