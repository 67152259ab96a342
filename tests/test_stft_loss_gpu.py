"""MultiResolutionSTFTLoss / STFTLoss on CUDA tensors (csrc/stft_loss.cu) against the fp64
restatement (tests/stft_loss_ref.py, torch ops in float64 on the same card).

Bounds: loss relative error <= LOSS_TOL; dx rel-L2 <= DX_TOL where the gradient is well-conditioned
in fp32 (the spectral-convergence term: measured <= 5.1e-7).  The gradients of the two L1 terms are
not everywhere: the log term's 1 / Xmag grows at the smallest bins of a frame, |Xmag - Ymag| changes
sign at bins where the two magnitudes agree to rounding, and the clamp's mask switches a bin of weight
1 / sqrt(eps) on or off where |X|^2 is within rounding of eps.  Any fp32 evaluation (the same
definition on cuFFT included) sits further from the fp64 gradient there, so these cases are held to
max(DX_TOL, COND_FACTOR x the fp32 torch restatement's own error), against the nearest of three fp64 references
with eps moved by 0 and +-1e-3 relative (an fp32 |X|^2 does not resolve the mask more finely)."""
import math

import pytest
import torch

import stft_loss_ref as ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
LOSS_TOL = 1e-5
DX_TOL = 1e-4
BF16_DX_TOL = 4e-3           # dx rounded to bf16 (2^-9 relative per element)
VERIFY_GRAD_TOL = 3e-3       # verify_fp32 parameter gradients of the default loss (L1 terms): measured 1.4e-3
COND_FACTOR = 12             # L1-term dx against the fp32 torch restatement's error: worst measured 5.6


@pytest.fixture(scope="module")
def adp():
    import audio_diffusion_pytorch_b200 as adp_
    return adp_


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def run(mod, x, y):
    xg = x.detach().clone().requires_grad_(True)
    loss = mod(xg, y)
    loss.backward()
    return loss.detach(), xg.grad


def reference(x, y, res, w, eps=1e-8):
    """fp64 loss and dx, and the rel-L2 of the fp32 torch restatement's dx against them."""
    x64 = x.detach().double().requires_grad_(True)
    want = ref.loss(x64, y.double(), res, w, eps)
    want.backward()
    x32 = x.detach().clone().float().requires_grad_(True)
    ref.loss(x32, y.float(), res, w, eps).backward()
    return float(want), x64.grad, rel(x32.grad, x64.grad)


def dx_error(dx, x, y, res, w):
    """(rel-L2 of dx against the nearest fp64 reference over eps * {1, 1 - 1e-3, 1 + 1e-3}, and the
    fp32 torch restatement's error at eps)."""
    _, dx_ref, err32 = reference(x, y, res, w)
    errs = [rel(dx, dx_ref)]
    if w[1:] != (0.0, 0.0):
        errs += [rel(dx, reference(x, y, res, w, 1e-8 * (1 + s))[1]) for s in (-1e-3, 1e-3)]
    return min(errs), err32


def signals(rows, t, seed, dtype, silent):
    g = torch.Generator().manual_seed(seed)
    x, y = torch.randn(rows, 1, t, generator=g), torch.randn(rows, 1, t, generator=g)
    if silent:                                   # silent stretches: bins reach the clamp
        x[0, :, t // 4: t // 2] = 0.0
        y[-1, :, t // 3:] = 0.0
        x[-1, :, t // 3 + t // 8:] = 0.0
    return x.to(DEV, dtype), y.to(DEV, dtype)


def fp32_dx(x, y, res, w):
    """The fp32 dx the backward accumulates before the bf16 rounding (the launches directly)."""
    from audio_diffusion_pytorch_b200 import losses
    x2, y2 = x.reshape(-1, x.shape[-1]).contiguous(), y.reshape(-1, y.shape[-1]).contiguous()
    acc = torch.empty(1, device=DEV, dtype=torch.float64)
    loss = torch.empty((), device=DEV)
    scale = 1.0 / len(res)
    stats = [losses._fwd(x2, y2, r, w, 1e-8, scale, acc, loss, i > 0) for i, r in enumerate(res)]
    dx = torch.empty(x2.shape, device=DEV)
    one = torch.ones(1, device=DEV)
    for i, (r, st) in enumerate(zip(res, stats)):
        losses._bwd(x2, y2, r, w, 1e-8, scale, st, one, dx, None, i > 0)
    return dx.reshape(x.shape)


CASES = [  # (resolutions, rows, T, dtype, silent)
    (ref.DEFAULT, 4, 1 << 15, torch.float32, False),
    (ref.DEFAULT, 8, 1 << 18, torch.float32, True),
    (ref.DEFAULT, 2, 1 << 16, torch.bfloat16, True),
    ([(400, 100, 400)], 1, 201, torch.float32, False),
    ([(400, 128, 300)], 3, 5000, torch.bfloat16, True),
    ([(441, 147, 441)], 2, 221, torch.float32, False),
    ([(441, 100, 300)], 5, 20000, torch.float32, True),
    ([(512, 128, 512)], 16, 1 << 16, torch.float32, False),
    ([(512, 50, 240)], 4, 1 << 18, torch.bfloat16, False),
    ([(1200, 240, 1200)], 2, 601, torch.float32, True),
    ([(1200, 300, 1000)], 8, 30000, torch.float32, False),
    ([(2048, 512, 2048)], 1, 1 << 18, torch.float32, False),
    ([(2048, 240, 1200)], 6, 1 << 17, torch.bfloat16, True),
    ([(8192, 2048, 8192)], 2, 4097, torch.float32, False),
    ([(8192, 1024, 6000)], 16, 1 << 16, torch.float32, True),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_loss_and_dx_match_the_fp64_restatement(adp, case):
    res, rows, t, dtype, silent = CASES[case]
    x, y = signals(rows, t, case, dtype, silent)
    for w in [(1.0, 1.0, 0.0), (0.5, 2.0, 1.5), (1.0, 0.0, 0.0)]:
        mod = adp.MultiResolutionSTFTLoss([r[0] for r in res], [r[1] for r in res], [r[2] for r in res],
                                          w_sc=w[0], w_log_mag=w[1], w_lin_mag=w[2])
        loss, dx = run(mod, x, y)
        want = float(ref.loss(x.double(), y.double(), res, w))
        e_loss = abs(float(loss) - want) / want
        assert dx.dtype == dtype and dx.shape == x.shape and loss.dim() == 0
        e_dx, err32 = dx_error(fp32_dx(x, y, res, w) if dtype == torch.bfloat16 else dx, x, y, res, w)
        bound = DX_TOL if w[1:] == (0.0, 0.0) else max(DX_TOL, COND_FACTOR * err32)
        print(f"{res} rows {rows} T {t} {dtype} silent {silent} w {w}: loss rel {e_loss:.2e}, "
              f"dx rel-L2 {e_dx:.2e} (fp32 torch {err32:.2e}, bound {bound:.1e})")
        assert e_loss <= LOSS_TOL
        assert e_dx <= bound
        if dtype == torch.bfloat16:
            assert dx_error(dx, x, y, res, w)[0] <= max(BF16_DX_TOL, COND_FACTOR * err32)


def test_two_calls_are_bitwise_identical(adp):
    x, y = signals(4, 1 << 16, 99, torch.float32, True)
    mod = adp.MultiResolutionSTFTLoss(w_lin_mag=0.5)
    l1, d1 = run(mod, x, y)
    l2, d2 = run(mod, x, y)
    assert torch.equal(l1, l2) and torch.equal(d1, d2)


def test_out_of_envelope_cuda_inputs_are_refused(adp):
    x, y = signals(2, 4096, 5, torch.float32, False)
    with pytest.raises(RuntimeError, match="prime factors"):
        adp.STFTLoss(fft_size=1100, hop_size=100, win_length=1100)(x, y)           # 11 * 100
    with pytest.raises(RuntimeError, match="8192"):
        adp.STFTLoss(fft_size=16384, hop_size=1024, win_length=16384)(torch.randn(1, 1, 20000, device=DEV),
                                                                     torch.randn(1, 1, 20000, device=DEV))
    with pytest.raises(RuntimeError, match="win_length"):
        adp.STFTLoss(fft_size=512, hop_size=128, win_length=600)(x, y)
    with pytest.raises(RuntimeError, match="reflect pad"):
        adp.STFTLoss(fft_size=512, hop_size=128, win_length=512)(x[..., :256], y[..., :256])
    with pytest.raises(ValueError, match="input only"):
        adp.MultiResolutionSTFTLoss()(x.requires_grad_(True), y.clone().requires_grad_(True))
    with pytest.raises(TypeError, match="float32"):
        adp.MultiResolutionSTFTLoss()(x.half(), y.half())


# --------------------------------------------------------------- training through the loss
CFG = dict(in_channels=2, channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 2, 2])


def compare_grads(ref_params, got_params):
    """Worst per-parameter rel-L2 (floored as in test_train_gpu.compare_grads) and the cosine of
    the whole gradient."""
    norms = torch.stack([p.grad.double().norm() for _, p in ref_params])
    floor = max(0.1 * float(norms.median()), 1e-3 * float(norms.max()))
    worst, dots, n1, n2 = 0.0, 0.0, 0.0, 0.0
    for (name, p), q in zip(ref_params, got_params):
        assert q.grad is not None, f"no gradient for {name}"
        g_ref, g = p.grad.double(), q.grad.double().cpu()
        worst = max(worst, float((g - g_ref).norm() / g_ref.norm().clamp_min(floor)))
        dots += float((g * g_ref).sum()); n1 += float((g * g).sum()); n2 += float((g_ref * g_ref).sum())
    return worst, dots / math.sqrt(n1 * n2)


def draws(shape, seed):
    """The sigma / noise draws VDiffusion makes on the GPU after torch.manual_seed(seed)."""
    torch.manual_seed(seed)
    sigma = torch.rand(shape[0], device=DEV).cpu()
    noise = torch.randn(*shape, device=DEV).cpu()
    a = torch.cos(sigma * math.pi / 2)[:, None, None]
    b = torch.sin(sigma * math.pi / 2)[:, None, None]
    return sigma, noise, a, b


def test_diffusion_model_step_with_the_loss(adp, oracle_port):
    """DiffusionModel(loss_fn=MultiResolutionSTFTLoss()) against the oracle port with the restated
    loss.  verify_fp32 against float64: the default loss, its value and every parameter gradient.
    bf16: the loss value at the custom-loss test's bound (test_train_gpu), and the gradients at its
    bounds for the spectral-convergence term alone: the L1 terms' gradients are not continuous in v at
    the scale of the bf16 net's error (see the module docstring), so no bf16 net can match them."""
    x = torch.randn(2, 2, 4096, generator=torch.Generator().manual_seed(6))
    for w_log, bf16 in ((1.0, False), (1.0, True), (0.0, True)):
        torch.manual_seed(0)
        ref_model = oracle_port.DiffusionModelPort(**CFG)
        model = adp.DiffusionModel(net_t=adp.UNetV0, loss_fn=adp.MultiResolutionSTFTLoss(w_log_mag=w_log),
                                   **CFG).to(DEV)
        model.net.load_reference_parameters(ref_model.net)
        dt = torch.float32 if bf16 else torch.float64
        if not bf16:
            ref_model.double()
            model.net.verify_fp32 = True
        torch.manual_seed(77)
        loss = model(x.to(DEV))
        loss.backward()
        sigma, noise, a, b = (v.to(dt) for v in draws(x.shape, 77))
        xr = x.to(dt)
        loss_ref = ref.loss(ref_model.net(a * xr + b * noise, sigma), a * noise - b * xr, w=(1.0, w_log, 0.0))
        loss_ref.backward()
        e = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
        worst, cos = compare_grads(list(ref_model.net.named_parameters()), list(model.net.parameters()))
        print(f"{'bf16' if bf16 else 'verify_fp32'} w_log_mag {w_log}: loss rel {e:.2e}, worst parameter "
              f"rel-L2 {worst:.3e}, cosine {cos:.9f}")
        if not bf16:
            assert e <= LOSS_TOL and worst <= VERIFY_GRAD_TOL
        else:
            assert e < 2e-3
            if w_log == 0.0:
                assert worst < 0.15 and cos > 1 - 5e-3


def test_diffusion_autoencoder_step_with_the_loss(adp, oracle_port):
    """The reference's DiffusionAE + MultiResolutionSTFTLoss example at a small size: a PyTorch
    encoder (oracle ToyEncoder) in place of MelE1d, its latent injected at depth 2; the default
    loss's value, and the gradients of the net and the encoder for the spectral-convergence term
    (as in the bf16 DiffusionModel step above), against the oracle port with the restated loss."""
    cfg = dict(CFG, inject_depth=2)
    x = torch.randn(1, 2, 8192, generator=torch.Generator().manual_seed(4))
    for w_log in (1.0, 0.0):
        torch.manual_seed(0)
        ref_model = oracle_port.DiffusionAEPort(encoder=oracle_port.ToyEncoder(), **cfg)
        torch.manual_seed(0)
        model = adp.DiffusionAE(encoder=oracle_port.ToyEncoder(), net_t=adp.UNetV0,
                                loss_fn=adp.MultiResolutionSTFTLoss(w_log_mag=w_log), **cfg).to(DEV)
        model.net.load_reference_parameters(ref_model.net)
        model.encoder.load_state_dict(ref_model.encoder.state_dict())
        torch.manual_seed(5)
        loss = model(x.to(DEV))
        loss.backward()
        sigma, noise, a, b = draws(x.shape, 5)
        latent = ref_model.encoder(x)
        v = ref_model.net(a * x + b * noise, sigma, channels=[None, None, latent])
        loss_ref = ref.loss(v, a * noise - b * x, w=(1.0, w_log, 0.0))
        loss_ref.backward()
        e = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
        worst, cos = compare_grads(list(ref_model.net.named_parameters()), list(model.net.parameters()))
        enc = rel(model.encoder.conv.weight.grad.cpu(), ref_model.encoder.conv.weight.grad)
        print(f"DiffusionAE w_log_mag {w_log}: loss rel {e:.2e}, worst net parameter rel-L2 {worst:.3e}, "
              f"cosine {cos:.6f}, encoder weight gradient rel-L2 {enc:.3e}")
        assert e < 2e-3
        if w_log == 0.0:
            assert worst < 0.15 and cos > 1 - 5e-3 and enc < 0.15
