"""Wide network boundary on the GPU: the stem kernels at up to 64 input / output channels,
(cx+ca)*f up to 128 and c0 up to 256, and UNetV0 nets that use them.

  - each kernel against a float64 restatement (forward) or float64 autograd (backward), every
    epilogue: append, adapter, noising + loss_sum + dv, x_next, CFG, GroupNorm statistics at 1 / 4 / 8
    groups; the backward also at c0 = 128 / 256 with narrow in / out widths;
  - whole nets against the CPU oracle with the same kwargs, eager / captured / replayed, and a
    sample; the branch bound (rel-L2 of v - x) is max(1.2e-2, 2x the oracle's own bf16-autocast
    error), computed here;
  - every launch of the LTPlugin and 5.1 inference / sampling programs held to its fp64
    restatement (launch_check.Shadow);
  - training: fused_v_loss loss and every parameter gradient against autograd through the oracle
    (bounds of test_train_gpu.py), and the fp32 verification mode against the float64 oracle
    (bounds of test_train_fp32_gpu.py)."""
import gc
import math

import pytest
import torch
import torch.nn.functional as F

import launch_check as lc

pytestmark = pytest.mark.gpu
DEV = "cuda"
BRANCH_TOL = 1.2e-2
V_TOL = 1e-4
GRAD_TOL = 6e-2              # test_train_gpu.GRAD_TOL
F32_GRAD_TOL = 1e-4          # test_train_fp32_gpu.GRAD_TOL
F32_LOSS_TOL = 1e-5


@pytest.fixture(scope="module")
def adp():
    import audio_diffusion_pytorch_b200 as adp_
    from audio_diffusion_pytorch_b200 import ops
    ops.device_check()
    return adp_


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def rel_l2(a, b, floor=0.0):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(max(floor, 1e-30)))


def close(got, ref, rtol, what):
    """max |got - ref| <= rtol * max |ref|"""
    got, ref = got.detach().double(), ref.detach().double()
    err, scale = float((got - ref).abs().max()), float(ref.abs().max())
    print(f"{what}: max abs err {err:.3e} = {err / max(scale, 1e-30):.2e} of max |ref| (bound {rtol:.1e})")
    assert err <= rtol * scale + 1e-12, f"{what}: {err:.3e} > {rtol} * {scale:.3e}"


# ------------------------------------------------------------------------------ per kernel
def _xin(x, app, noise, alpha, beta):
    xi = x.double()
    if noise is not None:
        xi = alpha.double()[:, None, None] * xi + beta.double()[:, None, None] * noise.double()
    return torch.cat([xi, app.double()], 1) if app is not None else xi


@pytest.mark.parametrize("cx,ca,c0,f,groups", [(9, 0, 8, 4, 1), (6, 6, 128, 4, 4), (64, 0, 256, 2, 8),
                                               (32, 0, 128, 4, 8), (12, 0, 256, 4, 4), (40, 24, 128, 2, 1),
                                               (9, 0, 256, 1, 8)])
@pytest.mark.parametrize("noised", [False, True])
def test_stem_in_wide(adp, cx, ca, c0, f, groups, noised):
    from audio_diffusion_pytorch_b200 import ops
    B, T = 2, 1024 * f
    cin = cx + ca
    x, app = rnd(B, cx, T, seed=1), (rnd(B, ca, T, seed=2) if ca else None)
    noise = rnd(B, cx, T, seed=3) if noised else None
    alpha, beta = (torch.rand(B, device=DEV), torch.rand(B, device=DEV)) if noised else (None, None)
    w, bias = rnd(c0, cin, f, scale=(cin * f) ** -0.5, seed=4), rnd(c0, seed=5)
    out = torch.full((B, T // f, c0), float("nan"), dtype=torch.bfloat16, device=DEV)
    stats = torch.zeros(B, groups, 2, dtype=torch.float64, device=DEV)
    ops.stem_in(x, w, bias, out, f, append=app, noise=noise, alpha=alpha, beta=beta, stats=stats, groups=groups)
    ref = F.conv1d(_xin(x, app, noise, alpha, beta), w.double(), bias.double(), stride=f).transpose(1, 2)
    close(out, ref, 2 ** -7, f"stem_in cin={cin} c0={c0} f={f}")
    o = out.double().view(B, T // f, groups, c0 // groups)
    st_ref = torch.stack([o.sum((1, 3)), (o * o).sum((1, 3))], -1)
    close(stats, st_ref, 1e-5, f"stem_in statistics G{groups}")


@pytest.mark.parametrize("cx,ca,co,c0,f,adapter", [(9, 0, 5, 8, 1, True), (6, 6, 6, 128, 2, True),
                                                   (64, 0, 64, 256, 2, False), (8, 0, 8, 128, 4, False),
                                                   (12, 0, 6, 8, 4, True), (64, 0, 64, 128, 1, True)])
@pytest.mark.parametrize("epilogue", ["v", "loss", "x_next", "cfg"])
def test_stem_out_wide(adp, cx, ca, co, c0, f, adapter, epilogue):
    from audio_diffusion_pytorch_b200 import ops
    B, T = 2, 1024
    cin = cx + ca
    if not adapter and cin != co:
        pytest.skip("identity skip needs cx+ca == co")
    cfg = epilogue == "cfg"
    Bh = 2 * B if cfg else B
    h = rnd(Bh, T // f, c0, seed=10).to(torch.bfloat16)
    x, app = rnd(B, cx, T, seed=11), (rnd(B, ca, T, seed=12) if ca else None)
    w, bias = rnd(co, c0, 3, scale=(3 * c0) ** -0.5, seed=13), rnd(co, seed=14)
    wa, ba = (rnd(co, cin, scale=cin ** -0.5, seed=15), rnd(co, seed=16)) if adapter else (None, None)
    gate = rnd(Bh, co + 3, seed=17)                 # a pitch other than co
    noise = rnd(B, cx, T, seed=18) if epilogue == "loss" else None
    alpha, beta = (torch.rand(B, device=DEV), torch.rand(B, device=DEV)) if noise is not None else (None, None)
    ab = torch.rand(4, device=DEV)

    xin = _xin(x, app, noise, alpha, beta)
    skip = F.conv1d(xin, wa.double()[:, :, None], ba.double()) if adapter else xin

    def branch(hh):
        up = F.interpolate(hh.double().transpose(1, 2), scale_factor=f, mode="nearest")
        return F.conv1d(up, w.double(), bias.double(), padding=1)
    v_ref = skip + gate.double()[:B, :co, None] * branch(h[:B])
    if cfg:
        vm = skip + gate.double()[B:, :co, None] * branch(h[B:])
        v_ref = vm + (v_ref - vm) * 3.0
    v = torch.full((B, co, T), float("nan"), device=DEV)
    kw = dict(append=app, w_adapt=wa, b_adapt=ba)
    if epilogue == "x_next":
        # in place when x and the output have the same channels, as the sampler runs it
        x_in = x.clone()
        x_next = x_in if co == cx else torch.full((B, co, T), float("nan"), device=DEV)
        ops.stem_out(h, x_in, w, bias, gate, f, x_next=x_next, ab=ab, **kw)
        a0, b0, a1, b1 = ab.double().tolist()
        xo = xin[:, :co]
        ref = a1 * (a0 * xo - b0 * v_ref) + b1 * (b0 * xo + a0 * v_ref)
        close(x_next, ref, 2e-5, f"stem_out x_next co={co} c0={c0}")
        return
    if epilogue == "loss":
        loss_sum = torch.zeros(1, dtype=torch.float64, device=DEV)
        dv = torch.full_like(v, float("nan"))
        ops.stem_out(h, x, w, bias, gate, f, v_out=v, noise=noise, alpha=alpha, beta=beta, loss_sum=loss_sum,
                     dv=dv, **kw)
        vt = alpha.double()[:, None, None] * noise.double()[:, :co] - beta.double()[:, None, None] * x.double()[:, :co]
        d = v_ref - vt
        close(loss_sum, (d * d).sum().reshape(1), 1e-5, "stem_out loss_sum")
        close(dv, 2 * d / d.numel(), 1e-5, "stem_out dv")
    else:
        ops.stem_out(h, x, w, bias, gate, f, v_out=v, cfg_scale=3.0 if cfg else None, **kw)
    close(v, v_ref, 2e-5, f"stem_out {epilogue} cin={cin} co={co} c0={c0} f={f} adapter={adapter}")


@pytest.mark.parametrize("cx,ca,co,c0,f,adapter", [(9, 0, 5, 8, 1, True), (6, 6, 6, 128, 2, True),
                                                   (64, 0, 64, 256, 2, False), (2, 0, 2, 128, 1, False),
                                                   (2, 0, 2, 256, 2, False), (1, 1, 1, 256, 4, True),
                                                   (64, 0, 64, 128, 1, True), (32, 0, 32, 128, 4, False)])
def test_stem_backward_wide(adp, cx, ca, co, c0, f, adapter):
    """adp_stem_out_bwd / adp_stem_in_bwd against float64 autograd, input gradient included."""
    from audio_diffusion_pytorch_b200 import ops
    B, T = 2, 1024
    cin = cx + ca
    h = rnd(B, T // f, c0, seed=26).to(torch.bfloat16)
    x, app = rnd(B, cx, T, seed=27), (rnd(B, ca, T, seed=28) if ca else None)
    noise = rnd(B, cx, T, seed=29)
    alpha, beta = torch.rand(B, device=DEV), torch.rand(B, device=DEV)
    w = rnd(co, c0, 3, scale=(3 * c0) ** -0.5, seed=30)
    bias, gate = rnd(co, seed=31), rnd(B, co + 2, seed=32)
    wa, ba = (rnd(co, cin, scale=cin ** -0.5, seed=33), rnd(co, seed=34)) if adapter else (None, None)
    dv = rnd(B, co, T, seed=35)
    gscale = torch.full((1,), 0.75, device=DEV)
    leaf = lambda t: t.detach().double().requires_grad_()  # noqa: E731
    hr, wr, br, gr = leaf(h), leaf(w), leaf(bias), leaf(gate)
    xin = leaf(_xin(x, app, noise, alpha, beta))
    war, bar = (leaf(wa), leaf(ba)) if adapter else (None, None)
    up = F.interpolate(hr.transpose(1, 2), scale_factor=f, mode="nearest")
    y = F.conv1d(up, wr, br, padding=1)
    skip = F.conv1d(xin, war[:, :, None], bar) if adapter else xin
    (skip + gr[:, :co, None] * y).backward(dv.double() * 0.75)
    dh = torch.full_like(h, float("nan"))
    dw, db = torch.zeros(co, c0, 3, device=DEV), torch.zeros(co, device=DEV)
    dgate = torch.zeros(B, co + 2, device=DEV)
    dwa, dba = (torch.zeros(co, cin, device=DEV), torch.zeros(co, device=DEV)) if adapter else (None, None)
    dxin = torch.full((B, cin, T), float("nan"), device=DEV)
    ops.stem_out_bwd(dv, h, x, w, bias, gate, f, dh, dw, db, dgate, gscale=gscale, append=app, noise=noise,
                     alpha=alpha, beta=beta, w_adapt=wa, dw_adapt=dwa, db_adapt=dba, dxin=dxin)
    what = f"stem_out_bwd cin={cin} co={co} c0={c0} f={f}"
    close(dh, hr.grad, 2 ** -7, what + " dh")
    close(dw, wr.grad, 1e-4, what + " dw")
    close(db, br.grad, 1e-4, what + " dbias")
    close(dgate[:, :co], gr.grad[:, :co], 1e-4, what + " dgate")
    assert float(dgate[:, co:].abs().max()) == 0.0
    if adapter:
        close(dwa, war.grad, 1e-4, what + " dw_adapt")
        close(dba, bar.grad, 1e-4, what + " db_adapt")
    # stem_in backward on top of the skip path's input gradient
    w_in, b_in = rnd(c0, cin, f, scale=(cin * f) ** -0.5, seed=36), rnd(c0, seed=37)
    dout = rnd(B, T // f, c0, seed=38).to(torch.bfloat16)
    wir, bir = leaf(w_in), leaf(b_in)
    xin2 = leaf(xin)
    F.conv1d(xin2, wir, bir, stride=f).transpose(1, 2).backward(dout.double())
    dwi, dbi = torch.zeros(c0, cin, f, device=DEV), torch.zeros(c0, device=DEV)
    ops.stem_in_bwd(dout, x, dwi, dbi, f, append=app, noise=noise, alpha=alpha, beta=beta, w=w_in, dxin=dxin)
    what = f"stem_in_bwd cin={cin} c0={c0} f={f}"
    close(dwi, wir.grad, 1e-4, what + " dw")
    close(dbi, bir.grad, 1e-4, what + " dbias")
    close(dxin, xin.grad + xin2.grad, 1e-4, what + " dxin (skip + downsample paths)")


# ------------------------------------------------------------------------------ whole nets
TINY = dict(channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 2, 2], attentions=[0, 0, 1],
            attention_heads=2, attention_features=64)
LT = dict(num_filters=32, window_length=64, stride=32)
LT_NET = dict(channels=[128, 256, 256], factors=[1, 2, 2], items=[1, 1, 1], attentions=[0, 0, 1],
              attention_heads=2, attention_features=64)


def _make(oracle_port, adp, kind):
    """(oracle model, GPU model, x, what) for one of the wide configurations."""
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(7)
    if kind == "surround_51":
        ref = oracle_port.DiffusionModelPort(in_channels=6, **TINY)
        model = adp.DiffusionModel(net_t=adp.UNetV0, in_channels=6, **TINY)
        x = torch.randn(2, 6, 4096, generator=g)
    elif kind == "upsampler_51":
        ref = oracle_port.DiffusionUpsamplerPort(upsample_factor=4, in_channels=6, **TINY)
        model = adp.DiffusionUpsampler(net_t=adp.UNetV0, upsample_factor=4, in_channels=6, **TINY)
        x = torch.randn(2, 6, 4096, generator=g)
    elif kind == "ltplugin":
        ref = oracle_port.DiffusionModelPort(net_t=oracle_port.lt_plugin(oracle_port.build_unet_v0, **LT),
                                             in_channels=2, **LT_NET)
        model = adp.DiffusionModel(net_t=adp.LTPlugin(adp.UNetV0, **LT), in_channels=2, **LT_NET)
        x = torch.randn(2, 2, 2 ** 15, generator=g)
    elif kind == "ar_8ch":
        cfg = dict(TINY, in_channels=8, length=4096, num_splits=4)
        ref = oracle_port.DiffusionARPort(**cfg)
        model = adp.DiffusionAR(net_t=adp.UNetV0, **cfg)
        x = torch.randn(2, 9, 4096, generator=g)
    elif kind in ("c0_128", "c0_256"):
        c0 = int(kind[3:])
        cfg = dict(in_channels=2, channels=[c0, 256, 256], factors=[2, 2, 2], items=[1, 1, 1])
        ref = oracle_port.DiffusionModelPort(**cfg)
        model = adp.DiffusionModel(net_t=adp.UNetV0, **cfg)
        x = torch.randn(2, 2, 4096, generator=g)
    else:
        raise KeyError(kind)
    model = model.to(DEV)
    if kind == "ltplugin":                          # filterbanks + net, registered in the same order
        with torch.no_grad():
            for p, q in zip(model.parameters(), ref.parameters()):
                p.copy_(q)
    else:
        model.net.load_reference_parameters(ref.net)
    return ref, model, x


def _net(model, adp):
    return [m for m in model.modules() if isinstance(m, adp.B200UNet)][0]


@pytest.mark.parametrize("kind", ["surround_51", "upsampler_51", "ltplugin", "ar_8ch"])
def test_net_forward_and_sample(adp, oracle_port, kind):
    ref, model, x = _make(oracle_port, adp, kind)
    if kind == "upsampler_51":                      # x and the appended low-rate signal
        x = torch.cat([x, torch.randn(x.shape, generator=torch.Generator().manual_seed(10))], 1)
    sigma = torch.rand(2, generator=torch.Generator().manual_seed(8))
    with torch.no_grad():
        if kind == "ar_8ch":
            v_ref = ref.net(x)
            with torch.autocast("cpu", dtype=torch.bfloat16):
                v_bf = ref.net(x).float()
            run = lambda: model.net(x.to(DEV))  # noqa: E731
            skip = x[:, :8]
        elif kind == "upsampler_51":
            v_ref = ref.net(x[:, :6], sigma, append_channels=x[:, 6:])
            with torch.autocast("cpu", dtype=torch.bfloat16):
                v_bf = ref.net(x[:, :6], sigma, append_channels=x[:, 6:]).float()
            run = lambda: model.net(x[:, :6].to(DEV), sigma.to(DEV), append_channels=x[:, 6:].to(DEV))  # noqa: E731
            skip = x[:, :6]
        else:
            v_ref = ref.net(x, sigma)
            with torch.autocast("cpu", dtype=torch.bfloat16):
                v_bf = ref.net(x, sigma).float()
            run = lambda: model.net(x.to(DEV), sigma.to(DEV))  # noqa: E731
            skip = x
        tol = max(BRANCH_TOL, 2 * rel_l2(v_bf - skip, v_ref - skip))
        for call in range(3):                       # eager, capture, replay
            v = run().cpu()
            e_v, e_b = rel_l2(v, v_ref), rel_l2(v - skip, v_ref - skip)
            print(f"{kind} call {call}: rel-L2 v {e_v:.3e}  v - x {e_b:.3e} (bound {tol:.3e})")
            assert e_b <= tol
        if kind in ("surround_51", "ltplugin"):
            s_ref = ref.sample(x, num_steps=3)
            s = model.sample(x.to(DEV), num_steps=3).cpu()
            e = rel_l2(s, s_ref)
            print(f"{kind}: 3-step sample rel-L2 {e:.3e} (bound {tol:.3e})")
            assert e <= tol


def test_cfg_net_with_embedding(adp, oracle_port):
    """Guidance at a 64-channel boundary: v under embedding_scale 3 (2B trunk rows, the combine in
    the wide stem_out) and a 2-step guided sample against the oracle."""
    cfg = dict(in_channels=64, channels=[128, 256, 256], factors=[1, 2, 2], items=[1, 1, 1],
               attentions=[0, 0, 1], cross_attentions=[0, 1, 1], attention_heads=2, attention_features=64,
               use_embedding_cfg=True, embedding_max_length=8, embedding_features=32)
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**cfg)
    model = adp.DiffusionModel(net_t=adp.UNetV0, **cfg).to(DEV)
    model.net.load_reference_parameters(ref.net)
    g = torch.Generator().manual_seed(9)
    x, sigma, emb = torch.randn(2, 64, 2048, generator=g), torch.rand(2, generator=g), torch.randn(2, 8, 32, generator=g)
    with torch.no_grad():
        kw = dict(embedding=emb, embedding_scale=3.0)
        v_ref = ref.net(x, sigma, **kw)
        with torch.autocast("cpu", dtype=torch.bfloat16):
            v_bf = ref.net(x, sigma, **kw).float()
        tol = max(BRANCH_TOL, 2 * rel_l2(v_bf - x, v_ref - x))
        for call in range(3):
            v = model.net(x.to(DEV), sigma.to(DEV), embedding=emb.to(DEV), embedding_scale=3.0).cpu()
            e = rel_l2(v - x, v_ref - x)
            print(f"CFG 64/64 call {call}: branch rel-L2 {e:.3e} (bound {tol:.3e})")
            assert e <= tol and rel_l2(v, v_ref) <= 1e-2
        s_ref = ref.sample(x, num_steps=2, **kw)
        s = model.sample(x.to(DEV), num_steps=2, embedding=emb.to(DEV), embedding_scale=3.0).cpu()
        e = rel_l2(s, s_ref)
        print(f"CFG 64/64: 2-step guided sample rel-L2 {e:.3e} (bound {tol:.3e})")
        assert e <= tol


@pytest.mark.parametrize("kind", ["surround_51", "ltplugin"])
def test_launch_check(adp, oracle_port, kind):
    """Every launch of the inference and sampling programs against its fp64 restatement."""
    _, model, x = _make(oracle_port, adp, kind)
    net = _net(model, adp)
    net.use_cuda_graph = False
    sigma = torch.rand(2, generator=torch.Generator().manual_seed(8)).to(DEV)
    try:
        with torch.no_grad():
            for what, call in (("v", lambda: model.net(x.to(DEV), sigma)),
                               ("sample", lambda: model.sample(x.to(DEV), num_steps=2))):
                with lc.Shadow() as sh:
                    call()
                print(f"\n{kind} {what}\n{sh.table()}")
                assert sh.n_checked == sh.n_launch > 0
    finally:
        del model, net
        gc.collect()
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------ training
def _train_inputs(model, x, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(x.shape, generator=g), torch.rand(x.shape[0], generator=g)


def _compare_grads(ref_named, got_params, tol, what):
    """Worst per-parameter rel-L2 with test_train_gpu.compare_grads' floor.  A gradient that is zero
    in float64 (a conv bias feeding a GroupNorm with one channel per group) has no relative error:
    what the GPU program returns there is the round-off of a cancelling sum, bounded at 1e-3 of the
    floor (10x the fp32-mode bound of the others), and reported separately."""
    pairs = [(n, p, q) for (n, p), q in zip(ref_named, got_params) if p.grad is not None]
    norms = torch.stack([p.grad.double().norm() for _, p, _ in pairs])
    floor = max(0.1 * float(norms.median()), 1e-3 * float(norms.max()))
    worst, at, worst0, at0 = 0.0, None, 0.0, None
    for n, p, q in pairs:
        assert q.grad is not None, f"{what}: no gradient for {n}"
        e = rel_l2(q.grad, p.grad, floor)
        if float(p.grad.double().norm()) <= 1e-9 * floor:
            if e > worst0:
                worst0, at0 = e, n
        elif e > worst:
            worst, at = e, n
    print(f"{what}: worst parameter-gradient rel-L2 {worst:.3e} ({at}) (bound {tol:.1e}); "
          f"analytically-zero gradients: worst {worst0:.3e} of the floor ({at0})")
    assert worst <= tol and worst0 <= 1e-3


@pytest.mark.parametrize("kind", ["surround_51", "ltplugin", "ar_8ch", "c0_128", "c0_256"])
@pytest.mark.parametrize("fp32", [False, True])
def test_training(adp, oracle_port, kind, fp32):
    """fused_v_loss (DiffusionModel nets) or the model's own loss (DiffusionAR, LTPlugin: the
    differentiable forward) and every parameter gradient, the filterbanks included, against autograd
    through the oracle: bf16 bounds of test_train_gpu.py, or fp32 mode against float64."""
    ref, model, x = _make(oracle_port, adp, kind)
    net = _net(model, adp)
    if fp32:
        ref.double()
        net.verify_fp32 = True
    dt = torch.float64 if fp32 else torch.float32
    seed = 40
    if kind == "ar_8ch":
        audio = x[:, :8]
        for _ in range(3 if fp32 else 1):
            model.zero_grad(set_to_none=True)
            torch.manual_seed(seed)
            loss = model(audio.to(DEV))
            loss.backward()
        torch.manual_seed(seed)
        per_split = torch.rand((2, 1, 4), device=DEV).cpu().to(dt)
        noise = torch.randn(2, 8, 4096, device=DEV).cpu().to(dt)
        sig = per_split.repeat_interleave(1024, dim=2)
        a, b = torch.cos(sig * math.pi / 2), torch.sin(sig * math.pi / 2)
        a64 = audio.to(dt)
        loss_ref = F.mse_loss(ref.net(torch.cat([a * a64 + b * noise, sig], dim=1)), a * noise - b * a64)
        ref_named, got = list(ref.net.named_parameters()), list(model.net.parameters())
    elif kind == "ltplugin":
        for _ in range(3 if fp32 else 1):
            model.zero_grad(set_to_none=True)
            torch.manual_seed(seed)
            loss = model(x.to(DEV))
            loss.backward()
        torch.manual_seed(seed)
        sigma = torch.rand(2, device=DEV).cpu().to(dt)
        eps = torch.randn(x.shape, device=DEV).cpu().to(dt)
        a, b = torch.cos(sigma * math.pi / 2)[:, None, None], torch.sin(sigma * math.pi / 2)[:, None, None]
        xd = x.to(dt)
        loss_ref = F.mse_loss(ref.net(a * xd + b * eps, sigma), a * eps - b * xd)
        ref_named, got = list(ref.named_parameters()), list(model.parameters())
    else:
        from audio_diffusion_pytorch_b200.training import fused_v_loss
        noise, sigma = _train_inputs(model, x, seed)
        for _ in range(3 if fp32 else 1):
            model.zero_grad(set_to_none=True)
            loss = fused_v_loss(model.net, x.to(DEV), noise.to(DEV), sigma.to(DEV))
            loss.backward()
        a, b = torch.cos(sigma * math.pi / 2)[:, None, None], torch.sin(sigma * math.pi / 2)[:, None, None]
        xd, nd, a, b = x.to(dt), noise.to(dt), a.to(dt), b.to(dt)
        loss_ref = F.mse_loss(ref.net(a * xd + b * nd, sigma.to(dt)), a * nd - b * xd)
        ref_named, got = list(ref.net.named_parameters()), list(model.net.parameters())
    loss_ref.backward()
    rel = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
    what = f"{kind} {'fp32 mode' if fp32 else 'bf16'}"
    print(f"{what}: loss {float(loss.detach()):.6f} vs oracle {float(loss_ref.detach()):.6f} (rel {rel:.2e})")
    assert rel <= (F32_LOSS_TOL if fp32 else 2e-3)
    _compare_grads(ref_named, got, F32_GRAD_TOL if fp32 else GRAD_TOL, what)


@pytest.mark.parametrize("kind", ["surround_51", "ltplugin", "upsampler_51"])
def test_fp32_forward(adp, oracle_port, kind):
    """verify_fp32 inference at rtol 1e-3 / atol 1e-4 against the float64 oracle."""
    ref, model, x = _make(oracle_port, adp, kind)
    ref.double()
    _net(model, adp).verify_fp32 = True
    sigma = torch.rand(2, generator=torch.Generator().manual_seed(8))
    with torch.no_grad():
        if kind == "upsampler_51":
            app = torch.randn(2, 6, 4096, generator=torch.Generator().manual_seed(10))
            v_ref = ref.net(x.double(), sigma.double(), append_channels=app.double())
            run = lambda: model.net(x.to(DEV), sigma.to(DEV), append_channels=app.to(DEV))  # noqa: E731
        else:
            v_ref = ref.net(x.double(), sigma.double())
            run = lambda: model.net(x.to(DEV), sigma.to(DEV))  # noqa: E731
        for call in range(3):
            v = run().cpu()
        err = float((v.double() - v_ref).abs().max())
        print(f"{kind} fp32 mode: max abs err {err:.3e}")
        torch.testing.assert_close(v.double(), v_ref, rtol=1e-3, atol=1e-4)
