"""Level, attention and embedding widths up to UNetV0.MAX_WIDTH (2048) on the GPU.

Kernels against fp64 restatements with the bounds of test_ops_gpu.py / test_bwd_ops_gpu.py:
ln_film (single and dual pass, with and without statistics) and ln_film_bwd at widths whose rows
do not fill a power of two of lanes (48, 80, 96, 320, 384, 640) and beyond 1024, at group sizes 6,
12, 20 and 24; the GroupNorm backward pair, skip_gate and skip_gate_bwd at 1536 and 2048; colsum at
3072 and 6144 (the q|k|v bias gradient at heads * D = 1024 and 2048).  T = 333 is not a multiple
of any kernel's rows per block.

Whole nets against the CPU oracle, as test_head_dims_gpu.py: v rel-L2 1e-4, branch
max(1.2e-2, 2 x the oracle's own bf16-autocast error), worst parameter gradient 6e-2 rel-L2, the
fp32 verification mode at rtol 1e-3 / atol 1e-4.  One wide net runs under the launch checker,
and every width the constructor accepts runs one forward and one backward."""
import math

import pytest
import torch
import torch.nn.functional as F

import launch_check as lc

pytestmark = pytest.mark.gpu
DEV = "cuda"
BRANCH_TOL, V_TOL, GRAD_TOL = 1.2e-2, 1e-4, 6e-2
T_ODD = 333
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

WIDTHS = [16, 48, 80, 96, 192, 320, 384, 640, 1280, 1536, 2048]
GROUP_SIZES = [6, 12, 20, 24]


def _groups(C):
    """Group counts of C: the UNetV0 default (8) and those giving the group sizes above (at most
    64 groups, the kernels' limit)."""
    gs = {8} if C % 8 == 0 else set()
    gs |= {C // s for s in GROUP_SIZES if C % s == 0 and C // s <= 64}
    return sorted(gs)


LN_CASES = [(C, g) for C in WIDTHS for g in _groups(C)]


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def bf(t):
    return t.to(torch.bfloat16)


def assert_close(got, ref, rtol, atol, what):
    got, ref = got.double(), ref.double()
    err = (got - ref).abs()
    bad = err > atol + rtol * ref.abs()
    msg = (f"{what}: max abs err {err.max().item():.4e}, ref max {ref.abs().max().item():.3e}, "
           f"violations {int(bad.sum())}/{bad.numel()}")
    print(msg)
    assert not bad.any(), msg


def close(got, ref, rtol, atol_frac, what):
    got, ref = got.double(), ref.double()
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item()
    print(f"{what}: max abs err {err:.4e} (ref max {scale:.3e})")
    assert err <= rtol * scale + atol_frac * scale + 1e-12, f"{what}: {err} vs scale {scale}"


def stats_of(y, groups):
    B, T, Cc = y.shape
    yg = y.double().reshape(B, T, groups, Cc // groups)
    return torch.stack([yg.sum(dim=(1, 3)), (yg * yg).sum(dim=(1, 3))], dim=-1).contiguous()


def layer_norm64(x, eps):
    x = x.double()
    m = x.mean(-1, keepdim=True)
    v = ((x - m) ** 2).mean(-1, keepdim=True)
    return (x - m) / torch.sqrt(v + eps)


@pytest.fixture(scope="module")
def ops():
    from audio_diffusion_pytorch_b200 import ops
    ops.device_check()
    return ops


@pytest.fixture(scope="module")
def adp():
    import audio_diffusion_pytorch_b200 as adp
    return adp


# ------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("C,groups", LN_CASES)
def test_ln_film_widths(ops, C, groups):
    B = 2
    x = bf(rnd(B, T_ODD, C, seed=19) * 2.0 + 0.5)
    ss = rnd(B, 2 * C, seed=20) * 0.3
    ref = layer_norm64(x, 1e-6) * (1 + ss.double()[:, None, :C]) + ss.double()[:, None, C:]
    for film in (True, False):
        stats = torch.zeros(B, groups, 2, dtype=torch.float64, device=DEV)
        y = torch.full_like(x, float("nan"))
        ops.ln_film(x, y, ss if film else None, 2 * C if film else 0, stats, groups, 1e-6)
        assert_close(y, ref if film else layer_norm64(x, 1e-6), 2 ** -7, 1e-2, f"ln_film C{C} film={film}")
        assert_close(stats, stats_of(y, groups), 1e-4, 1e-2, f"ln_film stats C{C} G{groups}")
    # without statistics (the attention pre-norm, the embedding LayerNorm)
    y = torch.full_like(x, float("nan"))
    ops.ln_film(x, y, None, 0, None, groups, 1e-5)
    assert_close(y, layer_norm64(x, 1e-5), 2 ** -7, 1e-2, f"ln_film no stats C{C}")


@pytest.mark.parametrize("C,groups", LN_CASES)
def test_ln_film_dual_widths(ops, C, groups):
    B = 2
    x = bf(rnd(B, T_ODD, C, seed=26) * 2.0 + 0.5)
    ss = rnd(B, 2 * C, seed=27) * 0.3
    for with_stats in (True, False):
        stats = torch.zeros(B, groups, 2, dtype=torch.float64, device=DEV) if with_stats else None
        y, y2 = torch.full_like(x, float("nan")), torch.full_like(x, float("nan"))
        ops.ln_film(x, y, ss, 2 * C, stats, groups, 1e-6, y2=y2, eps2=1e-5)
        y_single = torch.empty_like(x)         # the same kernel without the second LayerNorm
        ops.ln_film(x, y_single, ss, 2 * C, None if stats is None else torch.zeros_like(stats), groups, 1e-6)
        assert torch.equal(y, y_single), "dual pass changed the first output"
        assert_close(y2, layer_norm64(y, 1e-5), 2 ** -7, 1e-2, f"ln_film_dual y2 C{C}")
        if with_stats:
            assert_close(stats, stats_of(y, groups), 1e-4, 1e-2, f"ln_film_dual stats C{C} G{groups}")


@pytest.mark.parametrize("C", WIDTHS)
def test_ln_film_backward_widths(ops, C):
    B = 2
    x = bf(rnd(B, T_ODD, C, seed=10) * 2.0 + 0.5)
    dy = bf(rnd(B, T_ODD, C, seed=11))
    dres = bf(rnd(B, T_ODD, C, seed=13))
    ss = (rnd(B, 2 * C, seed=12) * 0.3).double().requires_grad_()
    xr = x.double().requires_grad_()
    y = layer_norm64(xr, 1e-6) * (1 + ss[:, None, :C]) + ss[:, None, C:]
    y.backward(dy.double())
    dx = torch.full_like(x, float("nan"))
    dss = torch.zeros(B, 2 * C, device=DEV)
    cs = torch.zeros(C, device=DEV)
    ops.ln_film_bwd(dy, x, ss.detach().float(), 2 * C, dx, dss=dss, dss_stride=2 * C, colsum=cs, dres=dres)
    want = xr.grad + dres.double()
    close(dx, want, 2 ** -6, 2e-3, f"ln_film bwd dx C{C}")
    close(dss, ss.grad, 1e-2, 2e-3, f"ln_film bwd dss C{C}")
    close(cs, want.sum(dim=(0, 1)), 2e-3, 2e-3, f"ln_film bwd colsum C{C}")


def _gn_silu64(x, stats_groups, gamma, beta):
    B, T, C = x.shape
    xg = x.reshape(B, T, stats_groups, C // stats_groups)
    m = xg.mean(dim=(1, 3), keepdim=True)
    v = ((xg - m) ** 2).mean(dim=(1, 3), keepdim=True)
    z = ((xg - m) / torch.sqrt(v + 1e-5)).reshape(B, T, C) * gamma + beta
    return F.silu(z)


@pytest.mark.parametrize("C,groups", [(1536, 8), (1536, 64), (2048, 8), (2048, 1), (1280, 64)])
def test_gn_backward_wide(ops, C, groups):
    B = 2
    x = bf(rnd(B, T_ODD, C, seed=5) * 1.5 + 0.3)
    da = bf(rnd(B, T_ODD, C, seed=6))
    dres = bf(rnd(B, T_ODD, C, seed=7))
    gamma = (rnd(C, seed=8) * 0.2 + 1.0).double().requires_grad_()
    beta = (rnd(C, seed=9) * 0.2).double().requires_grad_()
    xr = x.double().requires_grad_()
    _gn_silu64(xr, groups, gamma, beta).backward(da.double())
    stats = stats_of(x, groups)
    dxh, dx = torch.empty_like(x), torch.full_like(x, float("nan"))
    dg, db = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    S = torch.zeros(B, groups, 2, dtype=torch.float64, device=DEV)
    cs = torch.zeros(C, device=DEV)
    ops.gn_silu_bwd(da, x, stats, gamma.detach().float(), beta.detach().float(), dxh, dg, db, S, groups)
    ops.gn_bwd_apply(dxh, x, stats, S, dx, groups, dres=dres, colsum=cs)
    want = xr.grad + dres.double()
    close(dx, want, 2 ** -6, 2e-3, f"gn bwd dx C{C} G{groups}")
    close(dg, gamma.grad, 1e-2, 2e-3, f"gn bwd dgamma C{C} G{groups}")
    close(db, beta.grad, 1e-2, 2e-3, f"gn bwd dbeta C{C} G{groups}")
    close(cs, want.sum(dim=(0, 1)), 2e-3, 2e-3, f"gn bwd colsum C{C}")


@pytest.mark.parametrize("C,groups", [(1536, 8), (2048, 8), (2048, 64)])
def test_skip_gate_wide(ops, C, groups):
    B = 2
    y, skip, dout = (bf(rnd(B, T_ODD, C, seed=s)) for s in (13, 14, 15))
    gate = rnd(B, C + 8, seed=16)[:, :C]
    out = torch.full_like(y, float("nan"))
    stats = torch.zeros(B, groups, 2, dtype=torch.float64, device=DEV)
    ops.skip_gate(y, skip, gate, out, stats, groups)
    close(out, skip.double() + gate.double()[:, None, :] * y.double(), 2 ** -7, 1e-3, f"skip_gate out C{C}")
    close(stats, stats_of(out, groups), 1e-4, 1e-6, f"skip_gate stats C{C} G{groups}")
    out2 = torch.full_like(y, float("nan"))
    ops.skip_gate(y, skip, gate, out2, None, groups)
    assert torch.equal(out, out2)
    dys = torch.full_like(y, float("nan"))
    dgate = torch.zeros(B, C + 8, device=DEV)
    ops.skip_gate_bwd(dout, y, gate, dys, dgate[:, :C])
    close(dys, gate.double()[:, None, :] * dout.double(), 2 ** -7, 1e-3, f"skip_gate_bwd dys C{C}")
    close(dgate[:, :C], (dout.double() * y.double()).sum(1), 1e-3, 1e-3, f"skip_gate_bwd dgate C{C}")
    assert not dgate[:, C:].any()


@pytest.mark.parametrize("C", [3072, 6144])
def test_colsum_wide(ops, C):
    B = 2
    x = bf(rnd(B, T_ODD, C, seed=17))
    cs = torch.zeros(C, device=DEV)
    ops.colsum(x, cs)
    close(cs, x.double().sum(dim=(0, 1)), 1e-3, 1e-3, f"colsum C{C}")
    gate = rnd(B, C + 8, seed=18)[:, :C]
    cs = torch.zeros(C, device=DEV)
    ops.colsum(x, cs, gate)
    close(cs, (x.double() * gate.double()[:, None, :]).sum(dim=(0, 1)), 1e-3, 1e-3, f"colsum gated C{C}")


# ------------------------------------------------------------------------------ whole nets
NET_A = dict(in_channels=2, channels=[16, 48, 96, 192], factors=[1, 2, 2, 2], items=[1, 1, 1, 1],
             attentions=[0, 0, 1, 1], attention_heads=2, attention_features=32, resnet_groups=8)
NET_B = dict(in_channels=2, channels=[8, 64, 384, 1536, 2048], factors=[1, 4, 4, 2, 2], items=[1, 1, 1, 1, 1],
             attentions=[0, 0, 0, 1, 1], cross_attentions=[0, 0, 0, 1, 1], attention_heads=16,
             attention_features=64, use_embedding_cfg=True, embedding_max_length=8, embedding_features=2048)
NET_C = dict(in_channels=2, channels=[8, 32, 64, 1024], factors=[1, 4, 4, 2], items=[1, 1, 1, 1],
             attentions=[0, 0, 0, 1], attention_heads=8, attention_features=128)
NETS = {"a_thin_odd": (NET_A, 2 ** 12), "b_wide_deep": (NET_B, 2 ** 12), "c_8x128": (NET_C, 2 ** 12)}


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _pair(oracle_port, adp, cfg):
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**cfg)
    model = adp.DiffusionModel(net_t=adp.UNetV0, **cfg).to(DEV)
    model.net.load_reference_parameters(ref.net)
    return ref, model


def _inputs(cfg, T, seed):
    g = torch.Generator().manual_seed(seed)
    x, noise, sigma = torch.randn(2, 2, T, generator=g), torch.randn(2, 2, T, generator=g), torch.rand(2, generator=g)
    kw = {}
    if cfg.get("embedding_features"):
        kw = dict(embedding=torch.randn(2, cfg["embedding_max_length"], cfg["embedding_features"], generator=g))
    return x, noise, sigma, kw


def _dev(kw):
    return {k: v.to(DEV) if torch.is_tensor(v) else v for k, v in kw.items()}


def _check(v, v_ref, x, tol, what, v_tol=V_TOL):
    e_v, e_b = rel_l2(v, v_ref), rel_l2(v.cpu() - x, v_ref - x)
    print(f"{what}: rel-L2(v) {e_v:.3e}  rel-L2(branch) {e_b:.3e} (bound {tol:.3e})")
    assert e_v <= v_tol and e_b <= tol


@pytest.mark.parametrize("name", sorted(NETS))
def test_net_forward(adp, oracle_port, name):
    cfg, T = NETS[name]
    ref, model = _pair(oracle_port, adp, cfg)
    x, _, sigma, kw = _inputs(cfg, T, 1)
    with torch.no_grad():
        v_ref = ref.net(x, sigma, **kw)
        with torch.autocast("cpu", dtype=torch.bfloat16):
            v_bf = ref.net(x, sigma, **kw).float()
        tol = max(BRANCH_TOL, 2 * rel_l2(v_bf - x, v_ref - x))
        for call in range(3):                 # eager, capture, replay
            _check(model.net(x.to(DEV), sigma.to(DEV), **_dev(kw)), v_ref, x, tol, f"{name} call {call}")
        if kw:                                 # classifier-free guidance: two passes, amplified error
            v5_ref = ref.net(x, sigma, embedding_scale=5.0, **kw)
            v5 = model.net(x.to(DEV), sigma.to(DEV), embedding_scale=5.0, **_dev(kw))
            _check(v5, v5_ref, x, 2.5 * tol, f"{name} guidance 5", 3e-4)


def _oracle_loss(ref_net, x, noise, sigma, **kw):
    a, b = torch.cos(sigma * math.pi / 2)[:, None, None], torch.sin(sigma * math.pi / 2)[:, None, None]
    return F.mse_loss(ref_net(a * x + b * noise, sigma, **kw), a * noise - b * x)


def _grads(ref, model):
    worst, dots, n1, n2 = 0.0, 0.0, 0.0, 0.0
    pairs = [(n, p, q) for (n, p), q in zip(ref.net.named_parameters(), model.net.parameters()) if p.grad is not None]
    norms = torch.stack([p.grad.double().norm() for _, p, _ in pairs])
    floor = max(0.1 * float(norms.median()), 1e-3 * float(norms.max()))
    for name, p, q in pairs:
        assert q.grad is not None, f"no gradient for {name}"
        g_ref, g = p.grad.double(), q.grad.double().cpu()
        rel = float((g - g_ref).norm() / g_ref.norm().clamp_min(floor))
        if rel > worst:
            worst_name = name
        worst = max(worst, rel)
        dots += float((g * g_ref).sum()); n1 += float((g * g).sum()); n2 += float((g_ref * g_ref).sum())
    cos = dots / math.sqrt(n1 * n2)
    print(f"worst per-parameter rel-L2 {worst:.3e} ({worst_name}); global cosine {cos:.6f}")
    return worst, cos


@pytest.mark.parametrize("name", sorted(NETS))
def test_net_training(adp, oracle_port, name):
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    cfg, T = NETS[name]
    ref, model = _pair(oracle_port, adp, cfg)
    x, noise, sigma, kw = _inputs(cfg, T, 5)
    kw_mask = dict(kw, embedding_mask_proba=0.0) if kw else {}
    loss_ref = _oracle_loss(ref.net, x, noise, sigma, **kw_mask)
    loss_ref.backward()
    loss = fused_v_loss(model.net, x.to(DEV), noise.to(DEV), sigma.to(DEV), **_dev(kw_mask))
    loss.backward()
    rel = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
    print(f"{name}: loss {float(loss.detach()):.6f} vs oracle {float(loss_ref.detach()):.6f} (rel {rel:.2e})")
    assert rel < 2e-3
    worst, cos = _grads(ref, model)
    assert worst < GRAD_TOL and cos > 1 - 1e-3


@pytest.mark.parametrize("name", ["a_thin_odd", "b_wide_deep"])
def test_fp32_verification_mode(adp, oracle_port, name):
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    cfg, T = NETS[name]
    ref, model = _pair(oracle_port, adp, cfg)
    model.net.verify_fp32 = True
    x, noise, sigma, kw = _inputs(cfg, T, 1)
    with torch.no_grad():
        v_ref = ref.net(x, sigma, **kw)
        v = model.net(x.to(DEV), sigma.to(DEV), **_dev(kw))
    torch.testing.assert_close(v.cpu(), v_ref, rtol=1e-3, atol=1e-4)
    torch.testing.assert_close(v.cpu() - x, v_ref - x, rtol=1e-3, atol=1e-4)
    kw_mask = dict(kw, embedding_mask_proba=0.0) if kw else {}
    loss_ref = _oracle_loss(ref.net, x, noise, sigma, **kw_mask)
    loss_ref.backward()
    fused_v_loss(model.net, x.to(DEV), noise.to(DEV), sigma.to(DEV), **_dev(kw_mask)).backward()
    worst, _ = _grads(ref, model)
    assert worst <= 1e-4


# net (b)'s levels and self-attention; its cross-attention over 8 random tokens meets attention's lse
# bound only to err/bound 1.04 (DESIGN.md), a property of the attention kernel, not of the widths
NET_B_SELF = dict(NET_B, cross_attentions=[0, 0, 0, 0, 0], use_embedding_cfg=False, embedding_features=None)


def test_wide_net_under_launch_checker(adp):
    """Net (b)'s inference and training programs, self-attention only: every launch against its own
    bound."""
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    torch.manual_seed(0)
    model = adp.DiffusionModel(net_t=adp.UNetV0, **NET_B_SELF).to(DEV)
    net = model.net
    net.use_cuda_graph = False
    x, noise, sigma, _ = _inputs(NET_B_SELF, 2 ** 12, 7)
    with lc.Shadow() as sh:
        with torch.no_grad():
            net(x.to(DEV), sigma.to(DEV))
        fused_v_loss(net, x.to(DEV), noise.to(DEV), sigma.to(DEV)).backward()
    torch.cuda.synchronize()
    print(sh.table())
    assert sh.n_checked == sh.n_launch > 0
    assert {"ln_film", "ln_film_bwd", "colsum", "gn_silu_bwd", "gn_bwd_apply", "skip_gate_bwd"} <= \
        {k.split(".")[0] for k in sh.records}


from test_widths_cpu import ACCEPTED  # noqa: E402


@pytest.mark.parametrize("name", sorted(ACCEPTED))
def test_accepted_width_runs(adp, name):
    """Every net the constructor accepts in tests/test_widths_cpu.py: one forward, one backward."""
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    cfg = ACCEPTED[name]
    torch.manual_seed(0)
    model = adp.DiffusionModel(net_t=adp.UNetV0, **cfg).to(DEV)
    x, noise, sigma, kw = _inputs(cfg, 2 ** 11, 3)
    x, noise, sigma = x[:1], noise[:1], sigma[:1]
    kw = {k: v[:1] for k, v in kw.items()}
    with torch.no_grad():
        v = model.net(x.to(DEV), sigma.to(DEV), **_dev(kw))
    assert torch.isfinite(v).all()
    loss = fused_v_loss(model.net, x.to(DEV), noise.to(DEV), sigma.to(DEV), **_dev(kw))
    loss.backward()
    assert math.isfinite(float(loss))
    assert all(torch.isfinite(p.grad).all() for p in model.net.parameters() if p.grad is not None)
