"""Attention at head dims 32 and 128 (UNetV0(attention_features=D)) on the GPU.

Kernel cases reuse the shapes and bounds of test_ops_gpu.py::test_attention and
test_bwd_ops_gpu.py::test_attention_bwd, with heads chosen so that heads * D spans 32 to 512.
Whole-net cases follow test_groups_gpu.py: the CPU oracle is built with the same kwargs, weights
are loaded by position, and the branch bound is max(1.2e-2, 2x the oracle's own error under CPU
bf16 autocast), computed here for every net."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
BRANCH_TOL = 1.2e-2
V_TOL = 1e-4
GRAD_TOL = 6e-2
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

TINY = dict(in_channels=2, channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 2, 2], attentions=[0, 0, 1])
README = dict(in_channels=2, channels=[8, 32, 64, 128, 256, 512, 512, 1024, 1024],
              factors=[1, 4, 4, 4, 2, 2, 2, 2, 2], items=[1, 2, 2, 2, 2, 2, 2, 4, 4],
              attentions=[0, 0, 0, 0, 0, 1, 1, 1, 1])
TEXT_KW = dict(cross_attentions=[0, 1, 1], use_embedding_cfg=True, embedding_max_length=8,
               embedding_features=32)


def _tiny(heads, features, text=False):
    return dict(TINY, attention_heads=heads, attention_features=features, **(TEXT_KW if text else {}))


# (B, Tq, Tk) of test_ops_gpu.py::test_attention; per head dim, the heads of each shape
SHAPES = [(2, 256, 256), (1, 128, 128), (2, 1024, 1024), (2, 200, 200), (2, 512, 64), (1, 300, 8),
          (1, 64, 384)]
HEADS = {32: [8, 1, 16, 3, 8, 1, 3], 128: [2, 1, 4, 2, 4, 1, 1]}
KERNEL_CASES = [(D, HEADS[D][i], *shape) for D in (32, 128) for i, shape in enumerate(SHAPES)]


def rnd(*shape, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn(*shape, generator=g).to(DEV)


def assert_close(got, ref, rtol, atol, what):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    bad = err > atol + rtol * ref.abs()
    msg = (f"{what}: max abs err {err.max().item():.4e}, ref max {ref.abs().max().item():.3e}, "
           f"violations {int(bad.sum())}/{bad.numel()}")
    print(msg)
    assert not bad.any(), msg


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def check(v, v_ref, skip, what, branch_tol=BRANCH_TOL, v_tol=V_TOL):
    e_v, e_b = rel_l2(v, v_ref), rel_l2(v.cpu() - skip.cpu(), v_ref.cpu() - skip.cpu())
    print(f"{what}: rel-L2(v) {e_v:.3e}  rel-L2(branch) {e_b:.3e}")
    assert e_v <= v_tol, f"{what}: v error {e_v:.3e} > {v_tol}"
    assert e_b <= branch_tol, f"{what}: branch error {e_b:.3e} > {branch_tol}"


def close(got, want, what, rtol=1e-3, atol=1e-4):
    got, want = got.detach().float().cpu(), want.detach().float().cpu()
    print(f"{what}: max abs err {float((got - want).abs().max()):.3e}, rel-L2 {rel_l2(got, want):.3e}")
    torch.testing.assert_close(got, want, rtol=rtol, atol=atol)


def compare_grads(ref_params, got_params):
    worst, dots, n1, n2 = 0.0, 0.0, 0.0, 0.0
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
def ops():
    from audio_diffusion_pytorch_b200 import ops
    ops.device_check()
    return ops


@pytest.fixture(scope="module")
def adp():
    import audio_diffusion_pytorch_b200 as adp
    return adp


def _qkv(B, H, D, Tq, Tk, seed):
    """q, k, v read out of packed projection rows: q|k|v per row for self-attention (Tq == Tk),
    separate q and k|v rows otherwise."""
    mid = H * D
    if Tq == Tk:
        qkv = rnd(B, Tq, 3 * mid, seed=seed).bfloat16()
        return qkv, (qkv[..., :mid], qkv[..., mid:2 * mid], qkv[..., 2 * mid:])
    q = rnd(B, Tq, mid, seed=seed + 1).bfloat16()
    kv = rnd(B, Tk, 2 * mid, seed=seed + 2).bfloat16()
    return (q, kv), (q, kv[..., :mid], kv[..., mid:])


@pytest.mark.parametrize("D,H,B,Tq,Tk", KERNEL_CASES)
def test_attention_forward(ops, D, H, B, Tq, Tk):
    mid = H * D
    _, (q, k, v) = _qkv(B, H, D, Tq, Tk, seed=50)
    o = torch.full((B, Tq, mid), float("nan"), dtype=torch.bfloat16, device=DEV)
    ops.attention(q, k, v, o, H, D ** -0.5, head_dim=D)

    def heads(t):
        return t.float().reshape(B, -1, H, D).transpose(1, 2)
    ref = F.scaled_dot_product_attention(heads(q), heads(k), heads(v)).transpose(1, 2).reshape(B, Tq, mid)
    assert_close(o, ref, 2 ** -6, 2e-2, f"attention D{D} B{B} H{H} Tq{Tq} Tk{Tk}")


@pytest.mark.parametrize("D,H,B,Tq,Tk", KERNEL_CASES)
def test_attention_backward(ops, D, H, B, Tq, Tk):
    mid = H * D
    packed, (q, k, v) = _qkv(B, H, D, Tq, Tk, seed=70)
    if Tq == Tk:
        dqkv = torch.full_like(packed, float("nan"))
        dq, dk, dv = dqkv[..., :mid], dqkv[..., mid:2 * mid], dqkv[..., 2 * mid:]
    else:
        dq = torch.full_like(packed[0], float("nan"))
        dkv = torch.full_like(packed[1], float("nan"))
        dk, dv = dkv[..., :mid], dkv[..., mid:]
    d_o = rnd(B, Tq, mid, seed=73).bfloat16()
    o = torch.empty(B, Tq, mid, dtype=torch.bfloat16, device=DEV)
    lse = torch.full((B, H, Tq), float("nan"), device=DEV)
    delta = torch.empty(B, H, Tq, device=DEV)
    scale = D ** -0.5
    ops.attention(q, k, v, o, H, scale, lse=lse, head_dim=D)
    ops.attention_bwd(q, k, v, o, d_o, lse, delta, dq, dk, dv, H, scale, head_dim=D)

    def heads(t):
        return t.float().reshape(B, -1, H, D).transpose(1, 2)
    qf, kf, vf = (heads(t).detach().requires_grad_(True) for t in (q, k, v))
    F.scaled_dot_product_attention(qf, kf, vf).backward(heads(d_o))
    lse_ref = torch.logsumexp(qf.detach() @ kf.detach().transpose(-1, -2) * scale, dim=-1)
    assert_close(lse, lse_ref, 1e-3, 1e-3, f"lse D{D}")

    def flat(t):
        return t.transpose(1, 2).reshape(B, -1, mid)
    what = f"D{D} B{B} H{H} Tq{Tq} Tk{Tk}"
    assert_close(dq, flat(qf.grad), 2 ** -6, 1.5e-2, f"dq {what}")
    assert_close(dk, flat(kf.grad), 2 ** -6, 1.5e-2, f"dk {what}")
    assert_close(dv, flat(vf.grad), 2 ** -6, 1.5e-2, f"dv {what}")


def _pair(oracle_port, adp, cfg, **model_kw):
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**cfg)
    model = adp.DiffusionModel(net_t=adp.UNetV0, **cfg, **model_kw).to(DEV)
    model.net.load_reference_parameters(ref.net)
    return ref, model


def _oracle_v_and_branch_tol(ref, x, sigma, what, **kw):
    """fp32 oracle output and the branch bound: 2x the oracle's own error under bf16 autocast."""
    v_ref = ref.net(x, sigma, **kw)
    with torch.autocast("cpu", dtype=torch.bfloat16):
        v_bf16 = ref.net(x, sigma, **kw).float()
    e = rel_l2(v_bf16 - x, v_ref - x)
    print(f"{what}: oracle-under-bf16 branch rel-L2 {e:.3e}")
    return v_ref, max(BRANCH_TOL, 2 * e)


@pytest.mark.parametrize("heads,D", [(4, 32), (1, 128), (1, 32), (3, 32)])
def test_tiny_net_forward(adp, oracle_port, heads, D):
    """Eager, graph capture and graph replay; heads * D = 128, 32 and 96 (the q|k|v pack, the
    LayerNorm fold and the output projection at those widths)."""
    ref, model = _pair(oracle_port, adp, _tiny(heads, D))
    g = torch.Generator().manual_seed(1)
    x, sigma = torch.randn(2, 2, 4096, generator=g), torch.rand(2, generator=g)
    with torch.no_grad():
        v_ref, tol = _oracle_v_and_branch_tol(ref, x, sigma, f"tiny net H{heads} D{D}")
        for call in range(3):
            check(model.net(x.to(DEV), sigma.to(DEV)), v_ref, x, f"H{heads} D{D} forward (call {call})", tol)


@pytest.mark.parametrize("D", [32, 128])
def test_text_net_with_guidance(adp, oracle_port, D):
    """Cross-attention net at guidance 1 and 5 (the CFG double evaluation).  Guidance 5 amplifies
    both passes' error: v bound 3e-4, branch bound 2.5x the single-pass bound."""
    heads = {32: 1, 128: 2}[D]        # heads * D = 32 and 256
    ref, model = _pair(oracle_port, adp, _tiny(heads, D, text=True))
    g = torch.Generator().manual_seed(2)
    x, sigma = torch.randn(2, 2, 4096, generator=g), torch.rand(2, generator=g)
    emb = torch.randn(2, 8, 32, generator=g)
    with torch.no_grad():
        v1_ref, tol = _oracle_v_and_branch_tol(ref, x, sigma, f"text net D{D}", embedding=emb)
        v5_ref = ref.net(x, sigma, embedding=emb, embedding_scale=5.0)
        for call in range(3):
            v1 = model.net(x.to(DEV), sigma.to(DEV), embedding=emb.to(DEV))
            v5 = model.net(x.to(DEV), sigma.to(DEV), embedding=emb.to(DEV), embedding_scale=5.0)
            check(v1, v1_ref, x, f"text D{D} guidance 1 (call {call})", tol)
            check(v5, v5_ref, x, f"text D{D} guidance 5 (call {call})", 2.5 * tol, 3e-4)


def test_readme_net_head_dim_128(adp, oracle_port):
    """The 9-level README net with 4 heads of 128 (the parameter count of 8 heads of 64)."""
    ref, model = _pair(oracle_port, adp, dict(README, attention_heads=4, attention_features=128))
    g = torch.Generator().manual_seed(11)
    x, sigma = torch.randn(2, 2, 2 ** 13, generator=g), torch.rand(2, generator=g)
    with torch.no_grad():
        v_ref, tol = _oracle_v_and_branch_tol(ref, x, sigma, "README net H4 D128")
        check(model.net(x.to(DEV), sigma.to(DEV)), v_ref, x, "README net H4 D128, T=2^13", tol)


def test_sampler_50_steps_head_dim_128(adp, oracle_port):
    ref, model = _pair(oracle_port, adp, _tiny(1, 128))
    noise = torch.randn(2, 2, 4096, generator=torch.Generator().manual_seed(4))
    with torch.no_grad():
        s_ref = ref.sample(noise, num_steps=50)
        s = model.sample(noise.to(DEV), num_steps=50)
    e = rel_l2(s, s_ref)
    print(f"VSampler 50 steps (tiny, D128): rel-L2 {e:.3e}")
    assert e <= 1e-2


@pytest.mark.parametrize("text", [False, True])
@pytest.mark.parametrize("D", [32, 128])
def test_fp32_verification_mode(adp, oracle_port, D, text):
    ref, model = _pair(oracle_port, adp, _tiny({32: 3, 128: 2}[D], D, text=text))
    model.net.verify_fp32 = True
    g = torch.Generator().manual_seed(1)
    x, sigma = torch.randn(2, 2, 4096, generator=g), torch.rand(2, generator=g)
    kw = dict(embedding=torch.randn(2, 8, 32, generator=g)) if text else {}
    with torch.no_grad():
        v_ref = ref.net(x, sigma, **kw)
        for call in range(3):                   # eager, capture, replay
            v = model.net(x.to(DEV), sigma.to(DEV), **{k: t.to(DEV) for k, t in kw.items()})
    what = f"fp32 mode D{D}{' text' if text else ''}"
    close(v, v_ref, f"{what}: forward")
    close(v.cpu() - x, v_ref - x, f"{what}: branch (v - skip)")


def oracle_loss(ref_net, x, noise, sigma, **kw):
    a, b = torch.cos(sigma * math.pi / 2)[:, None, None], torch.sin(sigma * math.pi / 2)[:, None, None]
    return F.mse_loss(ref_net(a * x + b * noise, sigma, **kw), a * noise - b * x)


@pytest.mark.parametrize("case", ["self_attention", "cross_attention"])
@pytest.mark.parametrize("D", [32, 128])
def test_training_step(adp, oracle_port, D, case):
    """fused_v_loss forward + hand-written backward against autograd through the oracle."""
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    # heads * D: self-attention 96 / 256, cross-attention 32 / 128
    heads = {(32, "self_attention"): 3, (128, "self_attention"): 2,
             (32, "cross_attention"): 1, (128, "cross_attention"): 1}[D, case]
    ref, model = _pair(oracle_port, adp, _tiny(heads, D, text=case == "cross_attention"))
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 2, 4096, generator=g)
    noise = torch.randn(2, 2, 4096, generator=g)
    sigma = torch.rand(2, generator=g)
    kw_ref, kw = {}, {}
    if case == "cross_attention":
        emb = torch.randn(2, 8, 32, generator=g)
        kw_ref = dict(embedding=emb, embedding_mask_proba=0.0)
        kw = dict(embedding=emb.to(DEV), embedding_mask_proba=0.0)
    loss_ref = oracle_loss(ref.net, x, noise, sigma, **kw_ref)
    loss_ref.backward()
    loss = fused_v_loss(model.net, x.to(DEV), noise.to(DEV), sigma.to(DEV), **kw)
    loss.backward()
    rel = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
    print(f"D{D} {case}: loss {float(loss.detach()):.6f} vs oracle {float(loss_ref.detach()):.6f} (rel {rel:.2e})")
    assert rel < 2e-3
    ref_named = [(n, p) for n, p in ref.net.named_parameters() if p.grad is not None]
    got = [q for (n, p), q in zip(ref.net.named_parameters(), model.net.parameters()) if p.grad is not None]
    worst, cos = compare_grads(ref_named, got)
    assert worst < GRAD_TOL and cos > 1 - 1e-3


def test_custom_loss_through_differentiable_forward(adp, oracle_port):
    """A user loss (not F.mse_loss itself) runs the net through differentiable_forward."""
    def loss_fn(pred, target):
        return 0.5 * F.mse_loss(pred, target)

    ref, model = _pair(oracle_port, adp, _tiny(1, 128), loss_fn=loss_fn)
    x = torch.randn(2, 2, 4096, generator=torch.Generator().manual_seed(6))
    # identical sigma / noise on both sides: drive the oracle by hand with the GPU's draws
    torch.manual_seed(77)
    loss = model(x.to(DEV))
    loss.backward()
    torch.manual_seed(77)
    sigma = torch.rand(2, device=DEV).cpu()
    noise = torch.randn(2, 2, 4096, device=DEV).cpu()
    a, b = torch.cos(sigma * math.pi / 2)[:, None, None], torch.sin(sigma * math.pi / 2)[:, None, None]
    loss_ref = loss_fn(ref.net(a * x + b * noise, sigma), a * noise - b * x)
    loss_ref.backward()
    rel = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
    print(f"custom loss D128: {float(loss.detach()):.6f} vs oracle {float(loss_ref.detach()):.6f} (rel {rel:.2e})")
    assert rel < 2e-3
    worst, cos = compare_grads(list(ref.net.named_parameters()), list(model.net.parameters()))
    assert worst < GRAD_TOL and cos > 1 - 1e-3
