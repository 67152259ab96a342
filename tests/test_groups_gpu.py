"""Whole-net parity at GroupNorm group counts other than the default 8 (UNetV0(resnet_groups=G)):
inference through every kernel path that carries statistics (the fused thin levels, gn_silu +
conv GEMM, the GroupNorm-fused conv GEMM), the fp32 verification mode and the training step,
each against the CPU oracle built with the same resnet_groups and evaluated in fp32.

Bounds are those of test_net_gpu.py / test_train_gpu.py.  The branch bound (rel-L2 of v - x) is
2x the error of the oracle itself under CPU bf16 autocast, recomputed here for every net and
never below the 1.2e-2 of the 8-group golden files."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
BRANCH_TOL = 1.2e-2
V_TOL = 1e-4
GRAD_TOL = 6e-2

TINY = dict(in_channels=2, channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 2, 2],
            attentions=[0, 0, 1], attention_heads=2, attention_features=64)
README = dict(in_channels=2, channels=[8, 32, 64, 128, 256, 512, 512, 1024, 1024],
              factors=[1, 4, 4, 4, 2, 2, 2, 2, 2], items=[1, 2, 2, 2, 2, 2, 2, 4, 4],
              attentions=[0, 0, 0, 0, 0, 1, 1, 1, 1], attention_heads=8, attention_features=64)
CFG = dict(in_channels=2, channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 2, 2])
ATT = dict(CFG, attentions=[0, 0, 1], attention_heads=2, attention_features=64)


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def check(v, v_ref, skip, what, branch_tol=BRANCH_TOL, v_tol=V_TOL):
    e_v, e_b = rel_l2(v, v_ref), rel_l2(v.cpu() - skip.cpu(), v_ref.cpu() - skip.cpu())
    print(f"{what}: rel-L2(v) {e_v:.3e}  rel-L2(branch) {e_b:.3e}")
    assert e_v <= v_tol, f"{what}: v error {e_v:.3e} > {v_tol}"
    assert e_b <= branch_tol, f"{what}: branch error {e_b:.3e} > {branch_tol}"


def close(got, want, what, rtol=1e-3, atol=1e-4):
    """The fp32 criterion: |got - want| <= atol + rtol * |want| elementwise."""
    got, want = got.detach().float().cpu(), want.detach().float().cpu()
    err = (got - want).abs()
    worst = float((err - rtol * want.abs()).max())
    print(f"{what}: max abs err {float(err.max()):.3e}, rel-L2 {rel_l2(got, want):.3e}, "
          f"max(err - rtol*|ref|) {worst:.3e} (atol {atol})")
    torch.testing.assert_close(got, want, rtol=rtol, atol=atol)


def oracle_loss(ref_net, x, noise, sigma, **kw):
    a, b = torch.cos(sigma * math.pi / 2)[:, None, None], torch.sin(sigma * math.pi / 2)[:, None, None]
    return F.mse_loss(ref_net(a * x + b * noise, sigma, **kw), a * noise - b * x)


def compare_grads(ref_params, got_params):
    worst, dots, n1, n2 = 0.0, 0.0, 0.0, 0.0
    # gradients that are analytically zero (a conv bias feeding a GroupNorm with one channel per
    # group) are compared on the scale of a typical parameter gradient, not on their own
    norms = torch.stack([p.grad.double().norm() for _, p in ref_params])
    floor = max(0.1 * float(norms.median()), 1e-3 * float(norms.max()))
    for (name, p), q in zip(ref_params, got_params):
        assert q.grad is not None, f"no gradient for {name}"
        g_ref, g = p.grad.double(), q.grad.double().cpu()
        rel = float((g - g_ref).norm() / g_ref.norm().clamp_min(floor))
        worst = max(worst, rel)
        dots += float((g * g_ref).sum()); n1 += float((g * g).sum()); n2 += float((g_ref * g_ref).sum())
        if rel > GRAD_TOL:
            print(f"  {name:60s} shape {tuple(p.shape)} rel-L2 {rel:.3e}")
    cos = dots / math.sqrt(n1 * n2)
    print(f"worst per-parameter rel-L2 {worst:.3e}; global cosine {cos:.6f}")
    return worst, cos


@pytest.fixture(scope="module")
def adp():
    import audio_diffusion_pytorch_b200 as adp
    return adp


def _pair(oracle_port, adp, cfg, groups):
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(resnet_groups=groups, **cfg)
    model = adp.DiffusionModel(net_t=adp.UNetV0, resnet_groups=groups, **cfg).to(DEV)
    model.net.load_reference_parameters(ref.net)
    return ref, model


def _oracle_v_and_branch_tol(ref, x, sigma, what):
    """fp32 oracle output and the branch bound: 2x the oracle's own error under bf16 autocast."""
    v_ref = ref.net(x, sigma)
    with torch.autocast("cpu", dtype=torch.bfloat16):
        v_bf16 = ref.net(x, sigma).float()
    e = rel_l2(v_bf16 - x, v_ref - x)
    print(f"{what}: oracle-under-bf16 branch rel-L2 {e:.3e}")
    return v_ref, max(BRANCH_TOL, 2 * e)


@pytest.mark.parametrize("groups", [1, 2, 4])
def test_tiny_net_forward(adp, oracle_port, groups):
    """Eager, capture and replay on the default path (C = 8 and C = 32 / 64 as fused ConvBlock
    kernels), then the C = 32 / 64 levels through gn_silu + conv GEMM and through the
    GroupNorm-fused conv GEMM."""
    ref, model = _pair(oracle_port, adp, TINY, groups)
    g = torch.Generator().manual_seed(1)
    x, sigma = torch.randn(2, 2, 4096, generator=g), torch.rand(2, generator=g)
    with torch.no_grad():
        v_ref, tol = _oracle_v_and_branch_tol(ref, x, sigma, f"tiny net G{groups}")
        for call in range(3):
            check(model.net(x.to(DEV), sigma.to(DEV)), v_ref, x, f"G{groups} forward (call {call})", tol)
        model.net.fuse_thin_levels = False
        model.net._plans.clear()
        check(model.net(x.to(DEV), sigma.to(DEV)), v_ref, x, f"G{groups} gn_silu + conv GEMM", tol)
        model.net.fuse_groupnorm = True
        model.net._plans.clear()
        check(model.net(x.to(DEV), sigma.to(DEV)), v_ref, x, f"G{groups} GroupNorm-fused conv GEMM", tol)


def test_readme_net_four_groups(adp, oracle_port):
    """The 9-level README net at 4 groups on a 2^13 clip: at C = 1024 each 256-channel group spans
    two 128-wide N tiles of the conv GEMM."""
    ref, model = _pair(oracle_port, adp, README, 4)
    g = torch.Generator().manual_seed(11)
    x, sigma = torch.randn(2, 2, 2 ** 13, generator=g), torch.rand(2, generator=g)
    with torch.no_grad():
        v_ref, tol = _oracle_v_and_branch_tol(ref, x, sigma, "README net G4")
        check(model.net(x.to(DEV), sigma.to(DEV)), v_ref, x, "README net G4, T=2^13", tol)


@pytest.mark.parametrize("groups", [1, 4])
def test_fp32_verification_mode(adp, oracle_port, groups):
    """verify_fp32 (fp32 storage and arithmetic, csrc/verify_f32.cu) at rtol 1e-3 / atol 1e-4."""
    ref, model = _pair(oracle_port, adp, TINY, groups)
    model.net.verify_fp32 = True
    g = torch.Generator().manual_seed(1)
    x, sigma = torch.randn(2, 2, 4096, generator=g), torch.rand(2, generator=g)
    with torch.no_grad():
        v_ref = ref.net(x, sigma)
        for call in range(3):                   # eager, capture, replay
            v = model.net(x.to(DEV), sigma.to(DEV))
    close(v, v_ref, f"fp32 mode G{groups}: tiny net forward")
    close(v.cpu() - x, v_ref - x, f"fp32 mode G{groups}: branch (v - skip)")


@pytest.mark.parametrize("cfg_name", ["no_attention", "attention"])
@pytest.mark.parametrize("groups", [1, 4])
def test_training_step(oracle_port, adp, groups, cfg_name):
    """fused_v_loss forward + hand-written backward against autograd through the oracle."""
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    ref, model = _pair(oracle_port, adp, CFG if cfg_name == "no_attention" else ATT, groups)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 2, 4096, generator=g)
    noise = torch.randn(2, 2, 4096, generator=g)
    sigma = torch.rand(2, generator=g)
    loss_ref = oracle_loss(ref.net, x, noise, sigma)
    loss_ref.backward()
    loss = fused_v_loss(model.net, x.to(DEV), noise.to(DEV), sigma.to(DEV))
    loss.backward()
    rel = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
    print(f"G{groups} {cfg_name}: loss {float(loss.detach()):.6f} vs oracle {float(loss_ref.detach()):.6f} "
          f"(rel {rel:.2e})")
    assert rel < 2e-3
    worst, cos = compare_grads(list(ref.net.named_parameters()), list(model.net.parameters()))
    assert worst < GRAD_TOL and cos > 1 - 1e-3
