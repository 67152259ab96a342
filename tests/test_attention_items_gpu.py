"""Repeated attention items (UNetV0 attentions[i] / cross_attentions[i] above 1) on the GPU, for the
configs of tests/test_attention_items_cpu.py, against the CPU oracle built with the same kwargs:

  * the net (eager, captured, replayed): rel-L2 of v <= 1e-4 and of the branch (v - skip) <= 1.2e-2;
    a SkipCat net has no identity skip and is held to DiffusionAR's v bound of test_net_gpu.py, 5e-3;
    guidance 5 at 3e-4 / 3e-2; a 3-step sample at 5e-3;
  * the training step, fused_v_loss and differentiable_forward: the loss, every parameter gradient
    and d(embedding) against autograd through the oracle, worst parameter rel-L2 6e-2 and global
    cosine >= 0.999;
  * the fp32 verification mode: forward at rtol 1e-3 / atol 1e-4 and every gradient within rel-L2
    1e-4 of the float64 oracle's (the bounds of test_train_fp32_gpu.py);
  * a reference-style checkpoint of the oracle loaded with load_reference_state_dict;
  * one repeated-items net under the per-launch checker (tests/launch_check.py): one evaluation under
    guidance and one training step."""
import math

import pytest
import torch
import torch.nn.functional as F

import launch_check as lc
from test_attention_items_cpu import CONFIGS, inputs, n_items, oracle_kw

pytestmark = pytest.mark.gpu
DEV = "cuda"
V_TOL, BRANCH_TOL = 1e-4, 1.2e-2
CFG_V_TOL, CFG_BRANCH_TOL = 3e-4, 3e-2
SKIPCAT_V_TOL = 5e-3
SAMPLE_TOL = 5e-3
GRAD_TOL, GRAD_COS = 6e-2, 0.999
FP32_LOSS_TOL, FP32_GRAD_TOL = 1e-5, 1e-4
T = 4096
TIMED = sorted(n for n in CONFIGS if CONFIGS[n].get("use_time_conditioning", True))


@pytest.fixture(scope="module")
def adp():
    import audio_diffusion_pytorch_b200 as adp_
    from audio_diffusion_pytorch_b200 import ops
    ops.device_check()
    return adp_


def rel_l2(a, b, floor=1e-30):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(floor))


def pair(oracle_port, adp, cfg):
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**cfg)
    model = adp.DiffusionModel(net_t=adp.UNetV0, **cfg).to(DEV)
    model.net.load_reference_parameters(ref.net)
    return ref, model


def dev_kw(kw):
    out = {}
    for k, v in kw.items():
        if isinstance(v, torch.Tensor):
            out[k] = v.to(DEV)
        elif isinstance(v, list):
            out[k] = [None if t is None else t.to(DEV) for t in v]
        else:
            out[k] = v
    return out


def net_call(net, x, sigma, kw):
    return net(x, sigma, **kw) if sigma is not None else net(x, **kw)


def check(v, want, x, what, v_tol, b_tol):
    e_v, e_b = rel_l2(v, want), rel_l2(v.cpu() - x, want - x)
    print(f"{what}: rel-L2(v) {e_v:.3e}  rel-L2(branch) {e_b:.3e}")
    assert e_v <= v_tol and e_b <= b_tol, what


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_net_vs_oracle(adp, oracle_port, name):
    cfg = CONFIGS[name]
    ref, model = pair(oracle_port, adp, cfg)
    x, sigma, emb, channels = inputs(cfg, T=T)
    skipcat = not cfg.get("use_modulation", True)
    cases = [(1.0, SKIPCAT_V_TOL if skipcat else V_TOL, BRANCH_TOL)]
    if emb is not None:
        cases.append((5.0, CFG_V_TOL, CFG_BRANCH_TOL))
    with torch.no_grad():
        for scale, v_tol, b_tol in cases:
            kw = oracle_kw(emb, channels, scale)
            want = net_call(ref.net, x, sigma, kw)
            for call in range(3):               # eager, capture + replay, replay
                v = net_call(model.net, x.to(DEV), None if sigma is None else sigma.to(DEV), dev_kw(kw))
                check(v, want, x, f"{name} scale {scale} call {call}", v_tol, b_tol)


@pytest.mark.parametrize("name", TIMED)
def test_sample_vs_oracle(adp, oracle_port, name):
    cfg = CONFIGS[name]
    ref, model = pair(oracle_port, adp, cfg)
    noise, _, emb, channels = inputs(cfg, T=T, seed=4)
    kw = oracle_kw(emb, channels)
    with torch.no_grad():
        want = ref.sample(noise, num_steps=3, **kw)
        for call in range(2):
            s = model.sample(noise.to(DEV), num_steps=3, **dev_kw(kw))
            e = rel_l2(s, want)
            print(f"{name} 3-step sample call {call}: rel-L2 {e:.3e}")
            assert e <= SAMPLE_TOL


def compare_grads(ref_named, got_params):
    """(worst per-parameter rel-L2, global cosine), floored as in test_train_gpu.compare_grads."""
    worst, at, dots, n1, n2 = 0.0, None, 0.0, 0.0, 0.0
    norms = torch.stack([p.grad.double().norm() for _, p in ref_named])
    floor = max(0.1 * float(norms.median()), 1e-3 * float(norms.max()))
    for (name, p), q in zip(ref_named, got_params):
        assert q.grad is not None, f"no gradient for {name}"
        g_ref, g = p.grad.double(), q.grad.double().cpu()
        rel = float((g - g_ref).norm() / g_ref.norm().clamp_min(floor))
        if rel > worst:
            worst, at = rel, name
        dots += float((g * g_ref).sum()); n1 += float((g * g).sum()); n2 += float((g_ref * g_ref).sum())
    cos = dots / math.sqrt(n1 * n2)
    print(f"worst per-parameter rel-L2 {worst:.3e} ({at}); global cosine {cos:.6f}")
    return worst, cos


def named_grads(ref, model):
    ref_named = [(n, p) for n, p in ref.net.named_parameters() if p.grad is not None]
    got = [q for (_, p), q in zip(ref.net.named_parameters(), model.net.parameters()) if p.grad is not None]
    return ref_named, got


def oracle_loss(ref_net, x, noise, sigma, timed, **kw):
    a, b = torch.cos(sigma * math.pi / 2)[:, None, None], torch.sin(sigma * math.pi / 2)[:, None, None]
    xn = a * x + b * noise
    return F.mse_loss(ref_net(xn, sigma, **kw) if timed else ref_net(xn, **kw), a * noise - b * x)


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_training_step(adp, oracle_port, name):
    """fused_v_loss forward + hand-written backward against autograd through the oracle; d(embedding)
    sums the cross-attention items of every level."""
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    cfg = CONFIGS[name]
    timed = cfg.get("use_time_conditioning", True)
    ref, model = pair(oracle_port, adp, cfg)
    x, _, emb, channels = inputs(cfg, T=T, seed=5)
    g = torch.Generator().manual_seed(6)
    noise, sigma = torch.randn(x.shape, generator=g), torch.rand(x.shape[0], generator=g)
    kw = oracle_kw(None, channels)
    e_ref = e = None
    if emb is not None:
        e_ref = emb.clone().requires_grad_(True)
        kw.update(embedding=e_ref, embedding_mask_proba=0.0)
    loss_ref = oracle_loss(ref.net, x, noise, sigma, timed, **kw)
    loss_ref.backward()
    for call in range(2):
        model.zero_grad(set_to_none=True)
        kw_d = dev_kw({k: v for k, v in kw.items() if k != "embedding"})
        if emb is not None:
            e = emb.to(DEV).requires_grad_(True)
            kw_d["embedding"] = e
        loss = fused_v_loss(model.net, x.to(DEV), noise.to(DEV), sigma.to(DEV), **kw_d)
        loss.backward()
        rel = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
        print(f"{name} call {call}: loss {float(loss.detach()):.6f} vs oracle {float(loss_ref.detach()):.6f} "
              f"(rel {rel:.2e})")
        assert rel < 2e-3
        worst, cos = compare_grads(*named_grads(ref, model))
        assert worst < GRAD_TOL and cos >= GRAD_COS
        if emb is not None:
            e_rel = rel_l2(e.grad, e_ref.grad)
            print(f"{name} call {call}: d(embedding) rel-L2 {e_rel:.3e}")
            assert e_rel < GRAD_TOL


@pytest.mark.parametrize("name", ["mixed", "skipcat_2"])
def test_differentiable_forward(adp, oracle_port, name):
    """v = net(x, ...) under autograd with a weighted-sum loss: input, embedding and parameter gradients."""
    cfg = CONFIGS[name]
    ref, model = pair(oracle_port, adp, cfg)
    x, sigma, emb, channels = inputs(cfg, T=T, seed=7)
    wgt = torch.randn(x.shape[0], 2, T, generator=torch.Generator().manual_seed(8))
    x_ref = x.clone().requires_grad_(True)
    kw = oracle_kw(None, channels)
    if emb is not None:
        e_ref = emb.clone().requires_grad_(True)
        kw["embedding"] = e_ref
    v_ref = net_call(ref.net, x_ref, sigma, kw)
    (v_ref * wgt).sum().backward()
    xd = x.to(DEV).requires_grad_(True)
    kw_d = dev_kw({k: v for k, v in kw.items() if k != "embedding"})
    if emb is not None:
        ed = emb.to(DEV).requires_grad_(True)
        kw_d["embedding"] = ed
    v = net_call(model.net, xd, None if sigma is None else sigma.to(DEV), kw_d)
    (v * wgt.to(DEV)).sum().backward()
    worst, cos = compare_grads(*named_grads(ref, model))
    assert worst < GRAD_TOL and cos >= GRAD_COS
    e_x = rel_l2(xd.grad, x_ref.grad)
    print(f"{name}: dx rel-L2 {e_x:.3e}")
    assert e_x < GRAD_TOL
    if emb is not None:
        e_e = rel_l2(ed.grad, e_ref.grad)
        print(f"{name}: d(embedding) rel-L2 {e_e:.3e}")
        assert e_e < GRAD_TOL


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_fp32_verification_mode(adp, oracle_port, name):
    """Forward at rtol 1e-3 / atol 1e-4 and the training step's loss and gradients against the float64
    oracle (test_train_fp32_gpu.py's bounds)."""
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    cfg = CONFIGS[name]
    timed = cfg.get("use_time_conditioning", True)
    ref, model = pair(oracle_port, adp, cfg)
    ref.double()
    model.net.verify_fp32 = True
    x, sigma, emb, channels = inputs(cfg, T=T, seed=9)
    kw = {k: (v.double() if isinstance(v, torch.Tensor) else
              [None if t is None else t.double() for t in v] if isinstance(v, list) else v)
          for k, v in oracle_kw(emb, channels).items()}
    with torch.no_grad():
        want = net_call(ref.net, x.double(), None if sigma is None else sigma.double(), kw)
        for call in range(3):
            v = net_call(model.net, x.to(DEV), None if sigma is None else sigma.to(DEV), dev_kw(kw))
        print(f"{name} fp32 forward: max abs err {float((v.double().cpu() - want).abs().max()):.3e}")
        torch.testing.assert_close(v.double().cpu(), want, rtol=1e-3, atol=1e-4)
        torch.testing.assert_close(v.double().cpu() - x.double(), want - x.double(), rtol=1e-3, atol=1e-4)

    g = torch.Generator().manual_seed(10)
    noise, sig = torch.randn(x.shape, generator=g), torch.rand(x.shape[0], generator=g)
    tkw = {k: v for k, v in kw.items() if k != "embedding_scale"}
    if emb is not None:
        tkw["embedding_mask_proba"] = 0.0
    loss_ref = oracle_loss(ref.net, x.double(), noise.double(), sig.double(), timed, **tkw)
    loss_ref.backward()
    ref_named = [(n, p) for n, p in ref.net.named_parameters() if p.grad is not None]
    got = dict((n, q) for (n, _), q in zip(ref.net.named_parameters(), model.net.parameters()))
    norms = torch.stack([p.grad.norm() for _, p in ref_named])
    floor = max(0.1 * float(norms.median()), 1e-3 * float(norms.max()))
    for call in range(2):
        model.zero_grad(set_to_none=True)
        loss = fused_v_loss(model.net, x.to(DEV), noise.to(DEV), sig.to(DEV), **dev_kw(tkw))
        loss.backward()
        rel = abs(float(loss.detach()) - float(loss_ref.detach())) / abs(float(loss_ref.detach()))
        worst, at = 0.0, None
        for n, p in ref_named:
            assert got[n].grad is not None, f"no gradient for {n}"
            e = rel_l2(got[n].grad, p.grad, floor)
            if e > worst:
                worst, at = e, n
        print(f"{name} fp32 training call {call}: loss rel {rel:.2e}, worst gradient rel-L2 {worst:.2e} ({at})")
        assert rel <= FP32_LOSS_TOL and worst <= FP32_GRAD_TOL


@pytest.mark.parametrize("name", ["mixed", "inject_2"])
def test_reference_checkpoint_gives_the_oracle_outputs(adp, oracle_port, tmp_path, name):
    cfg = CONFIGS[name]
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**cfg)
    torch.save(ref.state_dict(), tmp_path / "ref.pt")
    torch.manual_seed(1)                          # other initial weights than the checkpoint's
    model = adp.DiffusionModel(net_t=adp.UNetV0, **cfg).to(DEV)
    model.load_reference_state_dict(torch.load(tmp_path / "ref.pt"))
    x, sigma, emb, channels = inputs(cfg, T=T, seed=11)
    kw = oracle_kw(emb, channels)
    with torch.no_grad():
        want = net_call(ref.net, x, sigma, kw)
        v = net_call(model.net, x.to(DEV), sigma.to(DEV), dev_kw(kw))
    check(v, want, x, f"{name} from a reference checkpoint", V_TOL, BRANCH_TOL)


def test_launch_checker_eval_and_training_step(adp):
    """The mixed config at B = 2, T = 2^14: one guidance-5 evaluation and one training step with input
    and embedding gradients, every launch against its fp64 restatement."""
    cfg = CONFIGS["mixed"]
    torch.manual_seed(1234)
    model = adp.DiffusionModel(net_t=adp.UNetV0, **cfg).to(DEV)
    net = model.net
    net.use_cuda_graph = False
    g = torch.Generator().manual_seed(12)
    Tl = 2 ** 14
    x, sigma = torch.randn(2, 2, Tl, generator=g).to(DEV), torch.rand(2, generator=g).to(DEV)
    emb = torch.randn(2, 8, 32, generator=g).to(DEV)
    wgt = (torch.randn(2, 2, Tl, generator=g) / Tl).to(DEV)
    n_att = n_items(cfg, "attentions") + n_items(cfg, "cross_attentions")
    with torch.no_grad(), lc.Shadow() as sh:
        net(x, sigma, embedding=emb, embedding_scale=5.0)
    print(f"\nmixed v, guidance 5, B=2 T=2^14\n{sh.table()}")
    assert sh.n_checked == sh.n_launch > 0
    assert sh.records["attention.o"].count == n_att
    xg, eg = x.clone().requires_grad_(), emb.clone().requires_grad_()
    with lc.Shadow() as sh:
        v = net(xg, sigma, embedding=eg)
        (v * wgt).sum().backward()
    print(f"\nmixed training step, B=2 T=2^14\n{sh.table()}")
    assert sh.n_checked == sh.n_launch > 0
    assert sh.records["attention_bwd.dq"].count == n_att
    assert xg.grad is not None and eg.grad is not None and float(eg.grad.abs().sum()) > 0
