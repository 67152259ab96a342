"""XUNet nets on the GPU, for the item lists of tests/test_xunet_cpu.py, against the oracle's XUNet
built from the same blocks (the bounds of tests/test_attention_items_gpu.py):

  * the net (eager, captured, replayed): rel-L2 of v <= 1e-4 and of the branch (v - x) <= 1.2e-2, a
    SkipCat net (no identity skip) 5e-3 on v; guidance 5 with cross-attention at 3e-4 / 3e-2.  A SkipAdd
    net adds its level-0 branch with no gate, so v carries the branch's bf16 error (3.1e-3 and 3.2e-3 on
    an H100 80GB HBM3, 700 W) and is held to SkipCat's 5e-3;
  * DiffusionModel(net_t=TimeConditioningPlugin(XUNet)).sample, 10 steps, against the oracle's
    sampler at 5e-3 (guidance 5 for the cross-attention net); a SkipAdd net at 1e-2 (6.0e-3 measured
    on that card);
  * the fused-loss training step: the loss, every parameter gradient and d(embedding) against autograd
    through the oracle, worst parameter rel-L2 6e-2 and global cosine >= 0.999;
  * the fp32 verification mode: forward at rtol 1e-3 / atol 1e-4 and every gradient within rel-L2 1e-4
    of the float64 oracle's;
  * a SkipAdd net at T = 2^18 under the per-launch checker, with and without guard bands: v, and one
    training step; the graph runs of v against the checked run and against each other within
    SKIPADD_RUN_SPREAD."""
import pytest
import torch

import launch_check as lc
from test_attention_items_gpu import (BRANCH_TOL, CFG_BRANCH_TOL, CFG_V_TOL, FP32_GRAD_TOL, FP32_LOSS_TOL,
                                      GRAD_COS, GRAD_TOL, SAMPLE_TOL, SKIPCAT_V_TOL, V_TOL, check, compare_grads,
                                      dev_kw, named_grads, net_call, oracle_loss, rel_l2)
from test_xunet_cpu import CASES, EMBEDDING_MAX_LENGTH, oracle_modules, xunet_t

pytestmark = pytest.mark.gpu
DEV = "cuda"
T = 4096
GPU_CASES = sorted(c for c in CASES if c != "cfg_outer")
TIMED = [c for c in GPU_CASES if "time" in CASES[c][1]]
SKIPADD_SAMPLE_TOL = 1e-2
# run-to-run spread of v of the full-size SkipAdd net: on an H100 80GB HBM3 (700 W) its output took one
# of two values, 1.243e-3 apart, between plain eager runs (no graph) as often as between graph
# replays; the bound is twice that
SKIPADD_RUN_SPREAD = 2.5e-3


@pytest.fixture(scope="module")
def adp():
    import audio_diffusion_pytorch_b200 as adp_
    from audio_diffusion_pytorch_b200 import ops
    ops.device_check()
    return adp_


def pair(oracle_port, adp, case):
    from audio_diffusion_pytorch_b200 import apex
    top, oapex = oracle_modules(oracle_port)
    torch.manual_seed(0)
    ref_t, ref_kw = xunet_t(top, oapex, case)
    ref = oracle_port.DiffusionModelPort(net_t=ref_t, **ref_kw)
    net_t, kw = xunet_t(adp, apex, case)
    model = adp.DiffusionModel(net_t=net_t, **kw).to(DEV)
    model.net.load_reference_parameters(ref.net)
    return ref, model


def inputs(case, B=2, T=T, seed=3):
    """(x, sigma or None, embedding or None, context channels or None) for a case."""
    _, plugins, blocks = CASES[case]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 2, T, generator=g)
    sigma = torch.rand(B, generator=g) if "time" in plugins else None
    cross = "cfg" in plugins or any("C" in b[2] + (b[3] or "") for b in blocks)
    emb = torch.randn(B, EMBEDDING_MAX_LENGTH, 32, generator=g) if cross else None
    channels, t = None, T
    if any(b[4] for b in blocks):
        channels = []
        for b in blocks:
            t //= b[1]
            channels.append(torch.randn(B, b[4], t, generator=g) if b[4] else None)
    return x, sigma, emb, channels


def oracle_kw(emb, channels, scale=1.0):
    kw = {}
    if emb is not None:
        kw.update(embedding=emb, embedding_scale=scale)
    if channels is not None:
        kw["channels"] = channels
    return kw


@pytest.mark.parametrize("case", GPU_CASES)
def test_net_vs_oracle(adp, oracle_port, case):
    ref, model = pair(oracle_port, adp, case)
    x, sigma, emb, channels = inputs(case)
    cases = [(1.0, SKIPCAT_V_TOL if CASES[case][0] in ("cat", "add") else V_TOL, BRANCH_TOL)]
    if "cfg" in CASES[case][1]:
        cases.append((5.0, CFG_V_TOL, CFG_BRANCH_TOL))
    with torch.no_grad():
        for scale, v_tol, b_tol in cases:
            kw = oracle_kw(emb, channels, scale)
            want = net_call(ref.net, x, sigma, kw)
            for call in range(3):               # eager, capture + replay, replay
                v = net_call(model.net, x.to(DEV), None if sigma is None else sigma.to(DEV), dev_kw(kw))
                check(v, want, x, f"{case} scale {scale} call {call}", v_tol, b_tol)


@pytest.mark.parametrize("case", TIMED)
def test_sample_vs_oracle(adp, oracle_port, case):
    ref, model = pair(oracle_port, adp, case)
    noise, _, emb, channels = inputs(case, seed=4)
    kw = oracle_kw(emb, channels, 5.0 if "cfg" in CASES[case][1] else 1.0)
    with torch.no_grad():
        want = ref.sample(noise, num_steps=10, **kw)
        for call in range(2):
            s = model.sample(noise.to(DEV), num_steps=10, **dev_kw(kw))
            e = rel_l2(s, want)
            print(f"{case} 10-step sample call {call}: rel-L2 {e:.3e}")
            assert e <= (SKIPADD_SAMPLE_TOL if CASES[case][0] == "add" else SAMPLE_TOL)


def training_inputs(case, seed):
    x, _, emb, channels = inputs(case, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    noise, sigma = torch.randn(x.shape, generator=g), torch.rand(x.shape[0], generator=g)
    return x, noise, sigma, emb, channels


@pytest.mark.parametrize("case", GPU_CASES)
def test_training_step(adp, oracle_port, case):
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    timed = "time" in CASES[case][1]
    ref, model = pair(oracle_port, adp, case)
    x, noise, sigma, emb, channels = training_inputs(case, 5)
    kw = oracle_kw(None, channels)
    e_ref = None
    if emb is not None:
        e_ref = emb.clone().requires_grad_(True)
        kw["embedding"] = e_ref
        if "cfg" in CASES[case][1]:
            kw["embedding_mask_proba"] = 0.0
    loss_ref = oracle_loss(ref.net, x, noise, sigma, timed, **kw)
    loss_ref.backward()
    for call in range(2):
        model.zero_grad(set_to_none=True)
        kw_d = dev_kw({k: v for k, v in kw.items() if k != "embedding"})
        e = None
        if emb is not None:
            e = emb.to(DEV).requires_grad_(True)
            kw_d["embedding"] = e
        loss = fused_v_loss(model.net, x.to(DEV), noise.to(DEV), sigma.to(DEV), **kw_d)
        loss.backward()
        rel = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
        print(f"{case} call {call}: loss {float(loss.detach()):.6f} vs oracle {float(loss_ref.detach()):.6f}")
        assert rel < 2e-3
        worst, cos = compare_grads(*named_grads(ref, model))
        assert worst < GRAD_TOL and cos >= GRAD_COS
        if e is not None:
            assert rel_l2(e.grad, e_ref.grad) < GRAD_TOL
        if not model.net.use_modulation and model.net.time is not None:
            # nothing reads the time features: the time MLP gets no gradient, as under autograd
            assert all(p.grad is None for p in model.net.time.parameters())


@pytest.mark.parametrize("case", GPU_CASES)
def test_fp32_verification_mode(adp, oracle_port, case):
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    timed = "time" in CASES[case][1]
    ref, model = pair(oracle_port, adp, case)
    ref.double()
    model.net.verify_fp32 = True
    x, sigma, emb, channels = inputs(case, seed=9)

    def dbl(kw):
        return {k: (v.double() if isinstance(v, torch.Tensor) else
                    [None if t is None else t.double() for t in v] if isinstance(v, list) else v)
                for k, v in kw.items()}
    kw = dbl(oracle_kw(emb, channels))
    with torch.no_grad():
        want = net_call(ref.net, x.double(), None if sigma is None else sigma.double(), kw)
        for call in range(3):
            v = net_call(model.net, x.to(DEV), None if sigma is None else sigma.to(DEV), dev_kw(kw))
        print(f"{case} fp32 forward: max abs err {float((v.double().cpu() - want).abs().max()):.3e}")
        torch.testing.assert_close(v.double().cpu(), want, rtol=1e-3, atol=1e-4)

    x, noise, sig, emb, channels = training_inputs(case, 10)
    tkw = dbl(oracle_kw(emb, channels))
    tkw.pop("embedding_scale", None)
    if emb is not None and "cfg" in CASES[case][1]:
        tkw["embedding_mask_proba"] = 0.0
    loss_ref = oracle_loss(ref.net, x.double(), noise.double(), sig.double(), timed, **tkw)
    loss_ref.backward()
    ref_named = [(n, p) for n, p in ref.net.named_parameters() if p.grad is not None]
    got = dict((n, q) for (n, _), q in zip(ref.net.named_parameters(), model.net.parameters()))
    norms = torch.stack([p.grad.norm() for _, p in ref_named])
    floor = max(0.1 * float(norms.median()), 1e-3 * float(norms.max()))
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
    print(f"{case} fp32 training: loss rel {rel:.2e}, worst gradient rel-L2 {worst:.2e} ({at})")
    assert rel <= FP32_LOSS_TOL and worst <= FP32_GRAD_TOL


# a SkipAdd net whose attention runs on levels of at most 4096 positions at T = 2^18 (the checker's
# fp64 attention holds the whole score matrix)
FULL_BLOCKS = [(8, 1, "RM", None), (32, 4, "MR", "RR"), (64, 4, "RM", None), (128, 4, "ARM", "RMA"),
               (256, 4, "RMA", "MRA")]


@pytest.mark.parametrize("guard", [False, True])
def test_full_size_skipadd_under_launch_checker(adp, guard):
    from audio_diffusion_pytorch_b200 import apex
    kinds = {"R": apex.ResnetItem, "M": apex.ModulationItem, "A": apex.AttentionItem}
    blocks = [apex.XBlock(channels=c, factor=f, items=[kinds[k] for k in it],
                          items_up=None if up is None else [kinds[k] for k in up]) for c, f, it, up in FULL_BLOCKS]
    torch.manual_seed(1234)
    model = adp.DiffusionModel(net_t=adp.TimeConditioningPlugin(adp.XUNet), in_channels=2, blocks=blocks,
                               skip_t=apex.SkipAdd, resnet_groups=8, attention_features=64, attention_heads=4,
                               modulation_features=1024).to(DEV)
    net = model.net
    net.use_cuda_graph = False
    g = torch.Generator().manual_seed(0)
    x, sigma = torch.randn(2, 2, 2 ** 18, generator=g).to(DEV), torch.rand(2, generator=g).to(DEV)
    try:
        with torch.no_grad(), lc.Shadow(guard=guard) as sh:
            v = net(x, sigma).clone()
        torch.cuda.synchronize()
        print(f"SkipAdd v T=2^18 guard={guard}\n{sh.table()}")
        assert sh.n_checked == sh.n_launch > 0 and (sh.n_guarded == sh.n_launch if guard else True)
        net.use_cuda_graph = True
        net._plans.clear()
        with torch.no_grad():
            runs = [net(x, sigma).clone() for _ in range(3)]
        # every run (eager, capture + replay, replay) against the checked one and against each other
        errs = [rel_l2(r, v) for r in runs] + [rel_l2(runs[2], runs[1]), rel_l2(runs[1], runs[0])]
        print("runs vs checked run, replay vs replay, first replay vs eager: " + " ".join(f"{e:.3e}" for e in errs))
        assert max(errs) <= SKIPADD_RUN_SPREAD
        net.use_cuda_graph = False
        with lc.Shadow(guard=guard) as sh:
            model.zero_grad(set_to_none=True)
            torch.manual_seed(77)
            model(x).backward()
        torch.cuda.synchronize()
        print(f"SkipAdd training step T=2^18 guard={guard}\n{sh.table()}")
        assert sh.n_checked == sh.n_launch > 0 and (sh.n_guarded == sh.n_launch if guard else True)
        assert all(p.grad is not None for p in model.parameters())
    finally:
        del model, net
        torch.cuda.empty_cache()
