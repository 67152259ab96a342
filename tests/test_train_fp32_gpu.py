"""The training program in the fp32 verification mode (B200UNet.verify_fp32 under autograd) against
torch.autograd through the CPU oracle in float64, on the same x / noise / sigma / embedding, so that
the comparison measures only the GPU program's fp32 round-off.  Every case runs eager, captured and
replayed (three calls).  Bounds, fixed before measuring:
  - loss relative error <= 1e-5;
  - v, dx, d append: torch.testing.assert_close(rtol=1e-3, atol=1e-4);
  - every parameter gradient (and embedding / encoder / filterbank / to_flat gradient) within a
    rel-L2 of 1e-4 of the float64 gradient, floored as in test_train_gpu.compare_grads for
    analytically-zero gradients (600x tighter than the bf16 bound there).
The unmodified reference's gradients in tests/golden are checked at rtol 1e-3 / atol 1e-4 where the
draws that produced them can be replayed."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
CFG = dict(in_channels=2, channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 2, 2])
ATT = dict(CFG, attentions=[0, 0, 1], attention_heads=2, attention_features=64)
TEXT = dict(ATT, cross_attentions=[0, 1, 1], use_embedding_cfg=True, embedding_max_length=8,
            embedding_features=32)
README = dict(in_channels=2, channels=[8, 32, 64, 128, 256, 512, 512, 1024, 1024],
              factors=[1, 4, 4, 4, 2, 2, 2, 2, 2], items=[1, 2, 2, 2, 2, 2, 2, 4, 4],
              attentions=[0, 0, 0, 0, 0, 1, 1, 1, 1], attention_heads=8, attention_features=64)
LOSS_TOL = 1e-5
GRAD_TOL = 1e-4
BF16_GRAD_TOL = 6e-2         # test_train_gpu.GRAD_TOL


def ab(sigma):
    return torch.cos(sigma * math.pi / 2)[:, None, None], torch.sin(sigma * math.pi / 2)[:, None, None]


def oracle_loss(ref_net, x, noise, sigma, **kw):
    a, b = ab(sigma)
    return F.mse_loss(ref_net(a * x + b * noise, sigma, **kw), a * noise - b * x)


def d64(*ts):
    return [t.detach().double() for t in ts]


def rel_l2(got, want, floor=0.0):
    want = want.double()
    return float((got.detach().double().cpu() - want).norm() / want.norm().clamp_min(floor))


def check_loss(what, loss, loss_ref):
    rel = abs(float(loss.detach()) - float(loss_ref.detach())) / abs(float(loss_ref.detach()))
    print(f"{what}: loss {float(loss.detach()):.8f} vs float64 {float(loss_ref.detach()):.8f} (rel {rel:.2e})")
    assert rel <= LOSS_TOL


def check_grads(what, ref_named, got_params, tol=GRAD_TOL):
    """Worst per-parameter rel-L2 against the float64 gradients (compare_grads' floor)."""
    ref_named = [(n, p) for n, p in ref_named if p.grad is not None]
    got = dict(got_params)
    norms = torch.stack([p.grad.norm() for _, p in ref_named])
    floor = max(0.1 * float(norms.median()), 1e-3 * float(norms.max()))
    worst, at = 0.0, None
    for n, p in ref_named:
        q = got[n]
        assert q.grad is not None, f"{what}: no gradient for {n}"
        e = rel_l2(q.grad, p.grad, floor)
        if e > worst:
            worst, at = e, n
    print(f"{what}: worst parameter-gradient rel-L2 {worst:.2e} ({at})")
    assert worst <= tol
    return worst


def close(what, got, want):
    err = float((got.detach().double().cpu() - want.detach().double()).abs().max())
    print(f"{what}: max abs err {err:.2e}")
    torch.testing.assert_close(got.detach().double().cpu(), want.detach().double(), rtol=1e-3, atol=1e-4)


def named(ref_net, net):
    """(reference name, GPU parameter) pairs: both trees register parameters in a_unet order."""
    return [(n, q) for (n, _), q in zip(ref_net.named_parameters(), net.parameters())]


def pair(oracle_port, adp, cfg, kind="model", **kw):
    torch.manual_seed(0)
    if kind == "upsampler":
        cfg = {k: v for k, v in cfg.items() if k != "in_channels"}
        ref = oracle_port.DiffusionUpsamplerPort(upsample_factor=16, in_channels=2, **cfg)
        model = adp.DiffusionUpsampler(net_t=adp.UNetV0, upsample_factor=16, in_channels=2, **cfg).to(DEV)
    else:
        ref = oracle_port.DiffusionModelPort(**cfg, **kw)
        model = adp.DiffusionModel(net_t=adp.UNetV0, **cfg, **kw).to(DEV)
    model.net.load_reference_parameters(ref.net)
    ref.double()
    model.net.verify_fp32 = True
    return ref, model


def fused_case(what, ref, model, x, noise, sigma, ref_kw=None, kw=None):
    """loss = mse(...) through fused_v_loss, eager / captured / replayed, against the float64 oracle."""
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    ref_kw, kw = ref_kw or {}, kw or {}
    loss_ref = oracle_loss(ref.net, *d64(x, noise, sigma), **ref_kw)
    loss_ref.backward()
    for call in range(3):
        model.zero_grad(set_to_none=True)
        loss = fused_v_loss(model.net, x.to(DEV), noise.to(DEV), sigma.to(DEV), **kw)
        loss.backward()
        check_loss(f"{what} call {call}", loss, loss_ref)
        check_grads(f"{what} call {call}", list(ref.net.named_parameters()), named(ref.net, model.net))
    return loss_ref


def inputs(seed, shape=(2, 2, 4096)):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g), torch.randn(*shape, generator=g), torch.rand(shape[0], generator=g)


@pytest.fixture(scope="module")
def adp():
    import audio_diffusion_pytorch_b200 as adp_
    return adp_


def test_attention_free_net_and_golden_gradients(adp, oracle_port, golden_dir):
    """The attention-free net; then the attention net of tests/golden/tiny_unconditional.npz on its
    own x and replayed draws: loss and the stored reference gradients at rtol 1e-3 / atol 1e-4."""
    ref, model = pair(oracle_port, adp, CFG)
    fused_case("attention-free", ref, model, *inputs(3))
    g = np.load(f"{golden_dir}/tiny_unconditional.npz")
    ref, model = pair(oracle_port, adp, ATT)
    x = torch.from_numpy(g["x"])
    torch.manual_seed(2)                 # the reference's draws: sigma, then noise
    sigma = torch.rand(2)
    noise = torch.randn(x.shape)
    fused_case("golden tiny_unconditional", ref, model, x, noise, sigma)
    got = dict(named(ref.net, model.net))
    for k in g.files:
        if k.startswith("grad:net."):
            close(k, got[k[len("grad:net."):]].grad, torch.from_numpy(g[k]))


def test_upsampler(adp, oracle_port):
    ref, model = pair(oracle_port, adp, CFG, kind="upsampler")
    x, noise, sigma = inputs(4)
    app = ref.reupsample(x.double())
    fused_case("DiffusionUpsampler", ref, model, x, noise, sigma, dict(append_channels=app),
               dict(append_channels=app.float().to(DEV)))


@pytest.mark.parametrize("head_dim", [32, 64, 128])
def test_self_attention_head_dims(adp, oracle_port, head_dim):
    cfg = dict(ATT, attention_features=head_dim, attention_heads=1 if head_dim == 128 else 2)
    ref, model = pair(oracle_port, adp, cfg)
    fused_case(f"self-attention D={head_dim}", ref, model, *inputs(5))


@pytest.mark.parametrize("groups", [1, 4])
def test_resnet_groups(adp, oracle_port, groups):
    ref, model = pair(oracle_port, adp, dict(ATT, resnet_groups=groups))
    fused_case(f"resnet_groups={groups}", ref, model, *inputs(6))


def test_cross_attention_embedding_gradient_and_guidance(adp, oracle_port):
    """Text net: the embedding's gradient through the fused loss; then guidance 5.0 under autograd
    (two differentiable passes, the mask embedding's gradient included)."""
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    ref, model = pair(oracle_port, adp, TEXT)
    x, noise, sigma = inputs(7)
    emb = torch.randn(2, 8, 32, generator=torch.Generator().manual_seed(8))
    e_ref = emb.double().requires_grad_(True)
    loss_ref = oracle_loss(ref.net, *d64(x, noise, sigma), embedding=e_ref)
    loss_ref.backward()
    for call in range(3):
        model.zero_grad(set_to_none=True)
        e = emb.to(DEV).requires_grad_(True)
        loss = fused_v_loss(model.net, x.to(DEV), noise.to(DEV), sigma.to(DEV), embedding=e)
        loss.backward()
        check_loss(f"text call {call}", loss, loss_ref)
        check_grads(f"text call {call}", list(ref.net.named_parameters()), named(ref.net, model.net))
        e_rel = rel_l2(e.grad, e_ref.grad)
        print(f"text call {call}: embedding gradient rel-L2 {e_rel:.2e}")
        assert e_rel <= GRAD_TOL

    ref.zero_grad(set_to_none=True)
    wgt = torch.randn(2, 2, 4096, generator=torch.Generator().manual_seed(9))
    v_ref = ref.net(*d64(x, sigma), embedding=emb.double(), embedding_scale=5.0)
    (v_ref * wgt.double()).sum().backward()
    for call in range(3):
        model.zero_grad(set_to_none=True)
        v = model.net(x.to(DEV), sigma.to(DEV), embedding=emb.to(DEV), embedding_scale=5.0)
        (v * wgt.to(DEV)).sum().backward()
        close(f"guidance 5.0 call {call}: v", v, v_ref)
        # out_masked + (out - out_masked) * 5: the gradient is 5 g_cond - 4 g_masked, so each pass's fp32
        # round-off enters with weight 5 and 4 while the combination is smaller than either pass's
        # gradient (they nearly cancel on the conv biases in front of a GroupNorm): the bound scales
        # with the 5 + 4 weights
        check_grads(f"guidance 5.0 call {call}", list(ref.net.named_parameters()), named(ref.net, model.net),
                    tol=(5 + 4) * GRAD_TOL)


def test_custom_loss_with_input_gradients(adp, oracle_port):
    """differentiable_forward (custom loss_fn / diffusion_t): v, dL/dx and dL/d append_channels."""
    ref, model = pair(oracle_port, adp, CFG, kind="upsampler")
    x, app, sigma = inputs(10)
    wgt = torch.randn(2, 2, 4096, generator=torch.Generator().manual_seed(11))
    target = torch.randn(2, 2, 4096, generator=torch.Generator().manual_seed(12))

    def loss_fn(v, w, t):               # a smooth user loss: weighted sum + squared error
        return (v * w).mean() + ((v - t) ** 2).mean()
    xr, ar = [t.requires_grad_(True) for t in d64(x, app)]
    v_ref = ref.net(xr, sigma.double(), append_channels=ar)
    loss_fn(v_ref, wgt.double(), target.double()).backward()
    for call in range(3):
        model.zero_grad(set_to_none=True)
        xg, ag = x.to(DEV).requires_grad_(True), app.to(DEV).requires_grad_(True)
        v = model.net(xg, sigma.to(DEV), append_channels=ag)
        loss_fn(v, wgt.to(DEV), target.to(DEV)).backward()
        close(f"custom loss call {call}: v", v, v_ref)
        close(f"custom loss call {call}: dx", xg.grad, xr.grad)
        close(f"custom loss call {call}: d append", ag.grad, ar.grad)
        check_grads(f"custom loss call {call}", list(ref.net.named_parameters()), named(ref.net, model.net))


def test_vocoder_to_flat_gradient(adp, oracle_port):
    kw = dict(mel_n_fft=64, mel_channels=8, mel_sample_rate=48000, mel_normalize_log=True, **CFG)
    kw.pop("in_channels")
    torch.manual_seed(0)
    ref = oracle_port.DiffusionVocoderPort(**kw)
    model = adp.DiffusionVocoder(net_t=adp.UNetV0, **kw).to(DEV)
    model.net.load_reference_parameters(ref.net)
    model.to_flat.load_state_dict(ref.to_flat.state_dict())
    ref.double()
    model.net.verify_fp32 = True
    audio = torch.randn(2, 2, 4096, generator=torch.Generator().manual_seed(13))
    for call in range(3):
        model.zero_grad(set_to_none=True)
        torch.manual_seed(31)
        loss = model(audio.to(DEV))
        loss.backward()
    torch.manual_seed(31)                 # the draws of the CUDA run, replayed for the oracle
    sigma = torch.rand(4, device=DEV).cpu()
    noise = torch.randn(4, 1, 4096, device=DEV).cpu()
    a64 = audio.double()
    mel = ref.to_spectrogram(a64)
    guide = ref.to_flat(mel.reshape(-1, *mel.shape[-2:]))
    loss_ref = oracle_loss(ref.net, a64.reshape(-1, 1, 4096), *d64(noise, sigma), append_channels=guide)
    loss_ref.backward()
    check_loss("vocoder", loss, loss_ref)
    e = rel_l2(model.to_flat.weight.grad, ref.to_flat.weight.grad)
    print(f"vocoder: to_flat.weight.grad rel-L2 {e:.2e}")
    assert e <= GRAD_TOL
    check_grads("vocoder", list(ref.net.named_parameters()), named(ref.net, model.net))


def test_autoencoder_encoder_gradient(adp, oracle_port):
    cfg = dict(ATT, inject_depth=2)
    torch.manual_seed(0)
    ref = oracle_port.DiffusionAEPort(encoder=oracle_port.ToyEncoder(), **cfg)
    torch.manual_seed(0)
    model = adp.DiffusionAE(encoder=oracle_port.ToyEncoder(), net_t=adp.UNetV0, **cfg).to(DEV)
    model.net.load_reference_parameters(ref.net)
    model.encoder.load_state_dict(ref.encoder.state_dict())
    ref.double()
    model.net.verify_fp32 = True
    audio = torch.randn(2, 2, 4096, generator=torch.Generator().manual_seed(24))
    for call in range(3):
        model.zero_grad(set_to_none=True)
        torch.manual_seed(91)
        loss = model(audio.to(DEV))
        loss.backward()
    torch.manual_seed(91)
    sigma = torch.rand(2, device=DEV).cpu()
    noise = torch.randn(2, 2, 4096, device=DEV).cpu()
    a64 = audio.double()
    loss_ref = oracle_loss(ref.net, a64, *d64(noise, sigma), channels=[None, None, ref.encoder(a64)])
    loss_ref.backward()
    check_loss("autoencoder", loss, loss_ref)
    check_grads("autoencoder", list(ref.net.named_parameters()), named(ref.net, model.net))
    e = rel_l2(model.encoder.conv.weight.grad, ref.encoder.conv.weight.grad)
    print(f"autoencoder: encoder conv.weight.grad rel-L2 {e:.2e}")
    assert e <= GRAD_TOL


def test_autoregressive_skipcat(adp, oracle_port):
    """use_modulation=False: SkipCat merges, the level-0 merge folded into the stems and unfolded."""
    cfg = dict(ATT, in_channels=2, length=4096, num_splits=4)
    torch.manual_seed(0)
    ref = oracle_port.DiffusionARPort(**cfg)
    model = adp.DiffusionAR(net_t=adp.UNetV0, **cfg).to(DEV)
    model.net.load_reference_parameters(ref.net)
    ref.double()
    model.net.verify_fp32 = True
    audio = torch.randn(2, 2, 4096, generator=torch.Generator().manual_seed(25))
    for call in range(3):
        model.zero_grad(set_to_none=True)
        torch.manual_seed(92)
        loss = model(audio.to(DEV))
        loss.backward()
    torch.manual_seed(92)
    per_split = torch.rand((2, 1, 4), device=DEV).cpu().double()
    noise = torch.randn(2, 2, 4096, device=DEV).cpu().double()
    sig = per_split.repeat_interleave(1024, dim=2)
    a, b = torch.cos(sig * math.pi / 2), torch.sin(sig * math.pi / 2)
    a64 = audio.double()
    loss_ref = F.mse_loss(ref.net(torch.cat([a * a64 + b * noise, sig], dim=1)), a * noise - b * a64)
    loss_ref.backward()
    check_loss("DiffusionAR", loss, loss_ref)
    check_grads("DiffusionAR", list(ref.net.named_parameters()), named(ref.net, model.net))


def test_learned_transform_filterbanks(adp, oracle_port):
    lt = dict(num_filters=4, window_length=8, stride=4)
    cfg = dict(ATT, in_channels=1)
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(net_t=oracle_port.lt_plugin(oracle_port.build_unet_v0, **lt), **cfg)
    model = adp.DiffusionModel(net_t=adp.LTPlugin(adp.UNetV0, **lt), **cfg).to(DEV)
    with torch.no_grad():
        for p, q in zip(model.parameters(), ref.parameters()):
            p.copy_(q)
    ref.double()
    nets = [m for m in model.modules() if isinstance(m, adp.B200UNet)]
    nets[0].verify_fp32 = True
    x = torch.randn(2, 1, 16384, generator=torch.Generator().manual_seed(26))
    for call in range(3):
        model.zero_grad(set_to_none=True)
        torch.manual_seed(93)
        loss = model(x.to(DEV))
        loss.backward()
    torch.manual_seed(93)
    sigma = torch.rand(2, device=DEV).cpu()
    eps = torch.randn(2, 1, 16384, device=DEV).cpu()
    loss_ref = oracle_loss(ref.net, *d64(x, eps, sigma))
    loss_ref.backward()
    check_loss("LTPlugin", loss, loss_ref)
    # every parameter, the two filterbanks included
    check_grads("LTPlugin", list(ref.named_parameters()), list(zip([n for n, _ in ref.named_parameters()],
                                                                   model.parameters())))


def test_readme_net(adp, oracle_port):
    """The README 9-level net on a 2^13 clip (B = 1): loss and every parameter gradient."""
    ref, model = pair(oracle_port, adp, README)
    fused_case("README net 2^13", ref, model, *inputs(14, (1, 2, 2 ** 13)))


def test_adamw_step_refreshes_the_fp32_packs(adp, oracle_port):
    """One AdamW step on the GPU model, the same weights written into the oracle, then a second loss
    and backward: the fp32 forward and dgrad packs must have been refreshed in place."""
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    ref, model = pair(oracle_port, adp, ATT)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-2)
    x, noise, sigma = inputs(15)
    for step in range(2):
        ref.zero_grad(set_to_none=True)
        loss_ref = oracle_loss(ref.net, *d64(x, noise, sigma))
        loss_ref.backward()
        opt.zero_grad(set_to_none=True)
        loss = fused_v_loss(model.net, x.to(DEV), noise.to(DEV), sigma.to(DEV))
        loss.backward()
        check_loss(f"AdamW step {step}", loss, loss_ref)
        check_grads(f"AdamW step {step}", list(ref.named_parameters()),
                    list(zip([n for n, _ in ref.named_parameters()], model.parameters())))
        opt.step()
        with torch.no_grad():
            for p, q in zip(ref.parameters(), model.parameters()):
                p.copy_(q.double().cpu())
        x, noise, sigma = inputs(16)


def test_switching_back_to_bf16(adp, oracle_port):
    """verify_fp32 = False afterwards: the bf16 training step is rebuilt and meets the bf16 bounds."""
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    ref, model = pair(oracle_port, adp, ATT)
    x, noise, sigma = inputs(17)
    fused_case("fp32 before switching", ref, model, x, noise, sigma)
    model.net.verify_fp32 = False
    loss_ref = oracle_loss(ref.net, *d64(x, noise, sigma))
    for call in range(3):
        model.zero_grad(set_to_none=True)
        loss = fused_v_loss(model.net, x.to(DEV), noise.to(DEV), sigma.to(DEV))
        loss.backward()
        rel = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
        assert rel < 2e-3
        check_grads(f"bf16 again call {call}", list(ref.net.named_parameters()), named(ref.net, model.net),
                    tol=BF16_GRAD_TOL)
