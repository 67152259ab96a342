"""Training step parity: fused VDiffusion loss + hand-written backward of the CUDA U-Net against
torch.autograd through the CPU oracle (same weights, same x / noise / sigma): attention-free
nets (BASELINE cfg4/cfg5 shape), nets with AttentionItem / CrossAttentionItem (README config,
cfg3), the 9-level shape, custom loss functions through the differentiable net forward, the
DiffusionVocoder front-end gradient, and the autograd contracts (accumulation, stale plans).
bf16 storage: loss within 2e-3 relative; every parameter gradient within GRAD_TOL rel-L2 of the
fp32 oracle gradient (floored at 10 % of the median gradient norm for analytically-zero
gradients) and the global gradient direction within 1e-3 cosine distance."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
CFG = dict(in_channels=2, channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 2, 2])
ATT = dict(CFG, attentions=[0, 0, 1], attention_heads=2, attention_features=64)
TEXT = dict(ATT, cross_attentions=[0, 1, 1], use_embedding_cfg=True, embedding_max_length=8,
            embedding_features=32)
GRAD_TOL = 6e-2


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


@pytest.mark.parametrize("upsampler", [False, True])
def test_loss_and_gradients_match_oracle(oracle_port, upsampler):
    import audio_diffusion_pytorch_b200 as adp
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    torch.manual_seed(0)
    if upsampler:
        kw = {k: v for k, v in CFG.items() if k != "in_channels"}
        ref = oracle_port.DiffusionUpsamplerPort(upsample_factor=16, in_channels=2, **kw)
        model = adp.DiffusionUpsampler(net_t=adp.UNetV0, upsample_factor=16, in_channels=2, **kw).to(DEV)
    else:
        ref = oracle_port.DiffusionModelPort(**CFG)
        model = adp.DiffusionModel(net_t=adp.UNetV0, **CFG).to(DEV)
    model.net.load_reference_parameters(ref.net)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 2, 4096, generator=g)
    noise = torch.randn(2, 2, 4096, generator=g)
    sigma = torch.rand(2, generator=g)
    extra_ref, extra = {}, {}
    if upsampler:
        app = ref.reupsample(x)
        extra_ref, extra = dict(append_channels=app), dict(append_channels=app.to(DEV))
    loss_ref = oracle_loss(ref.net, x, noise, sigma, **extra_ref)
    loss_ref.backward()
    for call in range(3):                       # eager, graph capture, graph replay
        model.zero_grad(set_to_none=True)
        loss = fused_v_loss(model.net, x.to(DEV), noise.to(DEV), sigma.to(DEV), **extra)
        loss.backward()
        rel = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
        print(f"call {call}: loss {float(loss.detach()):.6f} vs oracle {float(loss_ref.detach()):.6f} (rel {rel:.2e})")
        assert rel < 2e-3
        worst, cos = compare_grads(list(ref.net.named_parameters()), list(model.net.parameters()))
        assert worst < GRAD_TOL and cos > 1 - 1e-3


def test_optimizer_step_refreshes_packed_weights(oracle_port):
    """After optimizer.step() the next loss must see the new weights (in-place re-pack)."""
    import audio_diffusion_pytorch_b200 as adp
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**CFG)
    model = adp.DiffusionModel(net_t=adp.UNetV0, **CFG).to(DEV)
    model.net.load_reference_parameters(ref.net)
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    opt_ref = torch.optim.SGD(ref.parameters(), lr=0.05)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 2, 4096, generator=g)
    losses, losses_ref = [], []
    for step in range(4):
        torch.manual_seed(100 + step)
        sigma = torch.rand(2)
        noise = torch.randn(2, 2, 4096)
        from audio_diffusion_pytorch_b200.training import fused_v_loss
        opt.zero_grad(); opt_ref.zero_grad()
        loss = fused_v_loss(model.net, x.to(DEV), noise.to(DEV), sigma.to(DEV))
        loss.backward(); opt.step()
        lr_ = oracle_loss(ref.net, x, noise, sigma)
        lr_.backward(); opt_ref.step()
        losses.append(float(loss.detach())); losses_ref.append(float(lr_.detach()))
    print("losses", losses, "oracle", losses_ref)
    for a, b in zip(losses, losses_ref):
        assert abs(a - b) / b < 5e-3


def test_model_forward_is_the_reference_call(oracle_port):
    """`loss = model(x); loss.backward()` -- the reference's own training call (README.md:37-38)."""
    import audio_diffusion_pytorch_b200 as adp
    torch.manual_seed(0)
    model = adp.DiffusionModel(net_t=adp.UNetV0, **CFG).to(DEV)
    x = torch.randn(2, 2, 4096, device=DEV)
    loss = model(x)
    loss.backward()
    assert loss.ndim == 0 and torch.isfinite(loss)
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in model.parameters())


def _pair(oracle_port, adp, cfg):
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**cfg)
    model = adp.DiffusionModel(net_t=adp.UNetV0, **cfg).to(DEV)
    model.net.load_reference_parameters(ref.net)
    return ref, model


@pytest.mark.parametrize("case", ["self_attention", "cross_attention", "cross_attention_all_masked"])
def test_attention_gradients_match_oracle(oracle_port, case):
    """AttentionItem / CrossAttentionItem backward (adp_attention_bwd + LayerNorm-folded projection
    backward): `loss = model(x); loss.backward()` on nets WITH attention (README.md:37-38)."""
    import audio_diffusion_pytorch_b200 as adp
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    cfg = ATT if case == "self_attention" else TEXT
    ref, model = _pair(oracle_port, adp, cfg)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 2, 4096, generator=g)
    noise = torch.randn(2, 2, 4096, generator=g)
    sigma = torch.rand(2, generator=g)
    kw_ref, kw = {}, {}
    if case != "self_attention":
        emb = torch.randn(2, 8, 32, generator=g)
        # proba 1.0: every sample uses the learned mask embedding (deterministic), so the
        # gradient reaches `fixed_embedding` through torch.where
        proba = 1.0 if case.endswith("all_masked") else 0.0
        kw_ref = dict(embedding=emb, embedding_mask_proba=proba)
        kw = dict(embedding=emb.to(DEV), embedding_mask_proba=proba)
    loss_ref = oracle_loss(ref.net, x, noise, sigma, **kw_ref)
    loss_ref.backward()
    for call in range(3):
        model.zero_grad(set_to_none=True)
        loss = fused_v_loss(model.net, x.to(DEV), noise.to(DEV), sigma.to(DEV), **kw)
        loss.backward()
        rel = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
        print(f"{case} call {call}: loss {float(loss.detach()):.6f} vs oracle {float(loss_ref.detach()):.6f} (rel {rel:.2e})")
        assert rel < 2e-3
        ref_named = [(n, p) for n, p in ref.net.named_parameters() if p.grad is not None]
        got = [q for (n, p), q in zip(ref.net.named_parameters(), model.net.parameters()) if p.grad is not None]
        worst, cos = compare_grads(ref_named, got)
        assert worst < GRAD_TOL and cos > 1 - 1e-3
    if case.endswith("all_masked"):
        assert model.net.fixed_embedding.weight.grad is not None


@pytest.mark.parametrize("cfg_name", ["noatt", "att"])
def test_custom_loss_through_differentiable_forward(oracle_port, cfg_name):
    """DiffusionModel(loss_fn=F.l1_loss): VDiffusion calls net(x_noisy, sigma) and a user loss
    (reference models.py:28,37; tests/testcustomloss.py:28) -- the net forward carries autograd."""
    import audio_diffusion_pytorch_b200 as adp
    cfg = CFG if cfg_name == "noatt" else ATT
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**cfg)
    model = adp.DiffusionModel(net_t=adp.UNetV0, loss_fn=F.l1_loss, **cfg).to(DEV)
    model.net.load_reference_parameters(ref.net)
    g = torch.Generator().manual_seed(6)
    x = torch.randn(2, 2, 4096, generator=g)
    # identical sigma / noise on both sides: drive the oracle by hand with the GPU's draws
    torch.manual_seed(77)
    loss = model(x.to(DEV))
    loss.backward()
    torch.manual_seed(77)
    sigma = torch.rand(2, device=DEV).cpu()
    noise = torch.randn(2, 2, 4096, device=DEV).cpu()
    a = torch.cos(sigma * math.pi / 2)[:, None, None]
    b = torch.sin(sigma * math.pi / 2)[:, None, None]
    loss_ref = F.l1_loss(ref.net(a * x + b * noise, sigma), a * noise - b * x)
    loss_ref.backward()
    rel = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
    print(f"l1 loss {float(loss.detach()):.6f} vs oracle {float(loss_ref.detach()):.6f} (rel {rel:.2e})")
    assert rel < 2e-3
    worst, cos = compare_grads(list(ref.net.named_parameters()), list(model.net.parameters()))
    # d|e|/de = sign(e): elements whose bf16 error flips the sign contribute O(1) changes
    assert worst < 0.15 and cos > 1 - 5e-3


def test_input_gradients_of_the_differentiable_forward(oracle_port):
    """d v / d x and d v / d append_channels (the DiffusionVocoder trains `to_flat` through it)."""
    import audio_diffusion_pytorch_b200 as adp
    kw = {k: v for k, v in CFG.items() if k != "in_channels"}
    torch.manual_seed(0)
    ref = oracle_port.DiffusionUpsamplerPort(upsample_factor=16, in_channels=2, **kw)
    model = adp.DiffusionUpsampler(net_t=adp.UNetV0, upsample_factor=16, in_channels=2, **kw).to(DEV)
    model.net.load_reference_parameters(ref.net)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(2, 2, 4096, generator=g, requires_grad=True)
    app = torch.randn(2, 2, 4096, generator=g, requires_grad=True)
    sigma = torch.rand(2, generator=g)
    wgt = torch.randn(2, 2, 4096, generator=g)
    (ref.net(x, sigma, append_channels=app) * wgt).sum().backward()
    xg = x.detach().to(DEV).requires_grad_(True)
    ag = app.detach().to(DEV).requires_grad_(True)
    v = model.net(xg, sigma.to(DEV), append_channels=ag)
    (v * wgt.to(DEV)).sum().backward()
    for name, got, want in (("dx", xg.grad, x.grad), ("d append", ag.grad, app.grad)):
        e = float((got.cpu() - want).norm() / want.norm())
        print(f"{name}: rel-L2 {e:.3e}")
        assert e < 2e-2


def test_vocoder_forward_trains_to_flat(oracle_port):
    """DiffusionVocoder.forward (reference models.py:203-209): mel -> to_flat -> append_channels.
    Loss parity and the gradient of `to_flat.weight` (it only receives one through d append)."""
    import audio_diffusion_pytorch_b200 as adp
    kw = dict(mel_n_fft=64, mel_channels=8, mel_sample_rate=48000, mel_normalize_log=True,
              channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 2, 2])
    torch.manual_seed(0)
    ref = oracle_port.DiffusionVocoderPort(**kw)
    model = adp.DiffusionVocoder(net_t=adp.UNetV0, **kw).to(DEV)
    model.net.load_reference_parameters(ref.net)
    model.to_flat.load_state_dict(ref.to_flat.state_dict())
    g = torch.Generator().manual_seed(9)
    audio = torch.randn(2, 2, 4096, generator=g)
    torch.manual_seed(31)
    loss = model(audio.to(DEV))
    loss.backward()
    # the same sigma / noise draws for the oracle (drawn on the GPU generator, rows = b*c)
    torch.manual_seed(31)
    sigma = torch.rand(4, device=DEV).cpu()
    noise = torch.randn(4, 1, 4096, device=DEV).cpu()
    mel = ref.to_spectrogram(audio)
    guide = ref.to_flat(mel.reshape(-1, *mel.shape[-2:]))
    rows = audio.reshape(-1, 1, audio.shape[-1])
    loss_ref = oracle_loss(ref.net, rows, noise, sigma, append_channels=guide)
    loss_ref.backward()
    rel = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
    print(f"vocoder loss {float(loss.detach()):.6f} vs oracle {float(loss_ref.detach()):.6f} (rel {rel:.2e})")
    assert rel < 2e-3
    got, want = model.to_flat.weight.grad, ref.to_flat.weight.grad
    assert got is not None, "to_flat.weight received no gradient"
    e = float((got.cpu() - want).norm() / want.norm())
    print(f"to_flat.weight.grad rel-L2 {e:.3e}")
    assert e < GRAD_TOL
    worst, cos = compare_grads(list(ref.net.named_parameters()), list(model.net.parameters()))
    assert worst < GRAD_TOL and cos > 1 - 1e-3


def test_gradient_accumulation_and_zero_grad_in_place(oracle_port):
    """.grad must not alias the plan's arenas: two backward passes accumulate g1 + g2, and
    zero_grad(set_to_none=False) followed by a backward gives exactly that backward's gradient."""
    import audio_diffusion_pytorch_b200 as adp
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    _, model = _pair(oracle_port, adp, CFG)
    g = torch.Generator().manual_seed(12)
    xs = [torch.randn(2, 2, 4096, generator=g).to(DEV) for _ in range(2)]
    ns = [torch.randn(2, 2, 4096, generator=g).to(DEV) for _ in range(2)]
    sg = [torch.rand(2, generator=g).to(DEV) for _ in range(2)]
    singles = []
    for i in range(2):
        model.zero_grad(set_to_none=True)
        fused_v_loss(model.net, xs[i], ns[i], sg[i]).backward()
        singles.append([p.grad.clone() for p in model.net.parameters()])
    model.zero_grad(set_to_none=True)
    for i in range(2):
        fused_v_loss(model.net, xs[i], ns[i], sg[i]).backward()
    # run-to-run reproducibility is ~1e-4 (GroupNorm statistics accumulate with atomics); gradients
    # that are analytically zero are compared on the scale of a typical gradient
    floor = 0.1 * float(torch.stack([g_.norm() for g_ in singles[0]]).median())
    for p, g1, g2 in zip(model.net.parameters(), *singles):
        want = g1 + g2
        assert float((p.grad - want).norm()) <= 2e-3 * float(want.norm()) + 2e-2 * floor
    model.zero_grad(set_to_none=False)
    fused_v_loss(model.net, xs[0], ns[0], sg[0]).backward()
    for p, g1 in zip(model.net.parameters(), singles[0]):
        assert float((p.grad - g1).norm()) <= 2e-3 * float(g1.norm()) + 2e-2 * floor


def test_stale_plan_raises(oracle_port):
    """Two forwards on one shape before a backward: the first graph's activations are gone."""
    import audio_diffusion_pytorch_b200 as adp
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    _, model = _pair(oracle_port, adp, CFG)
    x = torch.randn(2, 2, 4096, device=DEV)
    l1 = fused_v_loss(model.net, x, torch.randn_like(x), torch.rand(2, device=DEV))
    l2 = fused_v_loss(model.net, x, torch.randn_like(x), torch.rand(2, device=DEV))
    l2.backward()
    with pytest.raises(RuntimeError, match="another forward"):
        l1.backward()


def test_untracked_weight_update_is_seen_by_inference(oracle_port):
    """EMA-style `p.data.copy_()` updates bump no version counter (ADVICE r1): the inference
    entry points fingerprint the parameters and re-pack."""
    import audio_diffusion_pytorch_b200 as adp
    ref, model = _pair(oracle_port, adp, CFG)
    torch.manual_seed(1)
    other = oracle_port.DiffusionModelPort(**CFG)          # a second set of weights
    x = torch.randn(2, 2, 4096, device=DEV)
    sig = torch.rand(2, device=DEV)
    with torch.no_grad():
        v0 = model.net(x, sig).clone()
        for p, q in zip(model.net.parameters(), other.net.parameters()):
            p.data.lerp_(q.to(DEV), 0.5)                   # EMA-style update through .data
        for p, q in zip(ref.net.parameters(), other.net.parameters()):
            p.lerp_(q, 0.5)
        v1 = model.net(x, sig)
        v_ref = ref.net(x.cpu(), sig.cpu())
    assert float((v1 - v0).norm()) > 0, "stale packed weights"
    e = float(((v1.cpu() - x.cpu()) - (v_ref - x.cpu())).norm() / (v_ref - x.cpu()).norm())
    print(f"after .data update: branch rel-L2 {e:.3e}")
    assert e < 1.2e-2


def test_nine_level_gradients(oracle_port):
    """The 9-level attention-free shape of BASELINE configs[3] (DiffusionUpsampler channels up to
    1024: split-K wgrad, C = 1024 dgrad) at a short length the CPU oracle back-propagates in seconds."""
    import audio_diffusion_pytorch_b200 as adp
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    kw = dict(channels=[8, 32, 64, 128, 256, 512, 512, 1024, 1024], factors=[1, 4, 4, 4, 2, 2, 2, 2, 2],
              items=[1, 2, 2, 2, 2, 2, 2, 4, 4])
    torch.manual_seed(0)
    ref = oracle_port.DiffusionUpsamplerPort(upsample_factor=16, in_channels=2, **kw)
    model = adp.DiffusionUpsampler(net_t=adp.UNetV0, upsample_factor=16, in_channels=2, **kw).to(DEV)
    model.net.load_reference_parameters(ref.net)
    g = torch.Generator().manual_seed(13)
    T = 2 ** 14
    x = torch.randn(2, 2, T, generator=g)
    noise = torch.randn(2, 2, T, generator=g)
    sigma = torch.rand(2, generator=g)
    app = ref.reupsample(x)
    loss_ref = oracle_loss(ref.net, x, noise, sigma, append_channels=app)
    loss_ref.backward()
    loss = fused_v_loss(model.net, x.to(DEV), noise.to(DEV), sigma.to(DEV), append_channels=app.to(DEV))
    loss.backward()
    rel = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
    print(f"9-level loss {float(loss.detach()):.6f} vs oracle {float(loss_ref.detach()):.6f} (rel {rel:.2e})")
    assert rel < 2e-3
    worst, cos = compare_grads(list(ref.net.named_parameters()), list(model.net.parameters()))
    assert worst < 0.1 and cos > 1 - 2e-3


def test_guidance_under_autograd(oracle_port):
    """embedding_scale != 1 with gradients enabled: two differentiable evaluations combined as
    out_masked + (out - out_masked) * scale (a_unet ClassifierFreeGuidancePlugin)."""
    import audio_diffusion_pytorch_b200 as adp
    ref, model = _pair(oracle_port, adp, TEXT)
    g = torch.Generator().manual_seed(15)
    x = torch.randn(2, 2, 4096, generator=g)
    sigma = torch.rand(2, generator=g)
    emb = torch.randn(2, 8, 32, generator=g)
    wgt = torch.randn(2, 2, 4096, generator=g)
    (ref.net(x, sigma, embedding=emb, embedding_scale=3.0) * wgt).sum().backward()
    v = model.net(x.to(DEV), sigma.to(DEV), embedding=emb.to(DEV), embedding_scale=3.0)
    (v * wgt.to(DEV)).sum().backward()
    ref_named = [(n, p) for n, p in ref.net.named_parameters() if p.grad is not None]
    got = [q for (n, p), q in zip(ref.net.named_parameters(), model.net.parameters()) if p.grad is not None]
    worst, cos = compare_grads(ref_named, got)
    assert worst < 0.1 and cos > 1 - 2e-3


def test_autoencoder_trains_encoder_through_injected_context(oracle_port):
    """DiffusionAE.forward (reference models.py:99-110): loss parity, U-Net gradients incl. the
    InjectChannelsItem convs, and the ENCODER's gradient, which only arrives through d(context)."""
    import audio_diffusion_pytorch_b200 as adp
    cfg = dict(ATT, inject_depth=2)
    torch.manual_seed(0)
    ref = oracle_port.DiffusionAEPort(encoder=oracle_port.ToyEncoder(), **cfg)
    torch.manual_seed(0)
    model = adp.DiffusionAE(encoder=oracle_port.ToyEncoder(), net_t=adp.UNetV0, **cfg).to(DEV)
    model.net.load_reference_parameters(ref.net)
    model.encoder.load_state_dict(ref.encoder.state_dict())
    g = torch.Generator().manual_seed(24)
    audio = torch.randn(2, 2, 4096, generator=g)
    for call in range(3):
        model.zero_grad(set_to_none=True)
        torch.manual_seed(91)
        loss = model(audio.to(DEV))
        loss.backward()
    torch.manual_seed(91)
    sigma = torch.rand(2, device=DEV).cpu()
    noise = torch.randn(2, 2, 4096, device=DEV).cpu()
    latent = ref.encoder(audio)
    loss_ref = oracle_loss(ref.net, audio, noise, sigma, channels=[None, None, latent])
    loss_ref.backward()
    rel = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
    print(f"autoencoder loss {float(loss.detach()):.6f} vs oracle {float(loss_ref.detach()):.6f} (rel {rel:.2e})")
    assert rel < 2e-3
    worst, cos = compare_grads(list(ref.net.named_parameters()), list(model.net.parameters()))
    assert worst < GRAD_TOL and cos > 1 - 1e-3
    got, want = model.encoder.conv.weight.grad, ref.encoder.conv.weight.grad
    assert got is not None, "the encoder received no gradient"
    e = float((got.cpu() - want).norm() / want.norm())
    print(f"encoder conv.weight.grad rel-L2 {e:.3e}")
    assert e < GRAD_TOL


def test_autoregressive_loss_and_gradients(oracle_port):
    """DiffusionAR.forward (reference models.py:227-250, diffusion.py:98-130): a
    use_modulation=False net -- no ModulationItems, SkipCat merges (conv1x1 over
    cat([skip * 2^-0.5, y])), the level-0 merge folded into the stem kernels -- under the
    per-split-sigma loss; every parameter gradient against autograd through the CPU oracle.
    Level 1 (8-channel output) exercises the paired-position merge GEMMs, level 2 the plain ones."""
    import audio_diffusion_pytorch_b200 as adp
    cfg = dict(ATT, in_channels=2, length=4096, num_splits=4)
    torch.manual_seed(0)
    ref = oracle_port.DiffusionARPort(**cfg)
    model = adp.DiffusionAR(net_t=adp.UNetV0, **cfg).to(DEV)
    model.net.load_reference_parameters(ref.net)
    audio = torch.randn(2, 2, 4096, generator=torch.Generator().manual_seed(25))
    for call in range(3):                    # eager, capture, replay
        model.zero_grad(set_to_none=True)
        torch.manual_seed(92)
        loss = model(audio.to(DEV))
        loss.backward()
    torch.manual_seed(92)                    # the draws the CUDA run consumed, replayed for the oracle
    per_split = torch.rand((2, 1, 4), device=DEV).cpu()
    noise = torch.randn(2, 2, 4096, device=DEV).cpu()
    sig = per_split.repeat_interleave(1024, dim=2)
    a, b = torch.cos(sig * math.pi / 2), torch.sin(sig * math.pi / 2)
    loss_ref = F.mse_loss(ref.net(torch.cat([a * audio + b * noise, sig], dim=1)), a * noise - b * audio)
    loss_ref.backward()
    rel = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
    print(f"DiffusionAR loss {float(loss.detach()):.6f} vs oracle {float(loss_ref.detach()):.6f} (rel {rel:.2e})")
    assert rel < 2e-3
    worst, cos = compare_grads(list(ref.net.named_parameters()), list(model.net.parameters()))
    assert worst < GRAD_TOL and cos > 1 - 1e-3


def test_learned_transform_plugin(oracle_port):
    """LTPlugin (reference components.py:113-157) around the CUDA net: forward / 3-step sample
    against the oracle and, through the differentiable net (the filterbanks are PyTorch modules on
    both sides of it: d(input) of the hand-written backward feeds the encoder), the loss and every
    gradient incl. the two filterbanks."""
    import audio_diffusion_pytorch_b200 as adp
    lt = dict(num_filters=4, window_length=8, stride=4)
    cfg = dict(ATT, in_channels=1)
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(net_t=oracle_port.lt_plugin(oracle_port.build_unet_v0, **lt), **cfg)
    model = adp.DiffusionModel(net_t=adp.LTPlugin(adp.UNetV0, **lt), **cfg).to(DEV)
    with torch.no_grad():
        for p, q in zip(model.parameters(), ref.parameters()):
            assert p.shape == q.shape
            p.copy_(q)
    g = torch.Generator().manual_seed(26)
    x = torch.randn(2, 1, 16384, generator=g)
    sig = torch.rand(2, generator=g)
    noise = torch.randn(2, 1, 16384, generator=g)
    with torch.no_grad():
        v, v_ref = model.net(x.to(DEV), sig.to(DEV)), ref.net(x, sig)
        e = float((v.cpu() - v_ref).norm() / v_ref.norm())
        s, s_ref = model.sample(noise.to(DEV), num_steps=3), ref.sample(noise, num_steps=3)
        e_s = float((s.cpu() - s_ref).norm() / s_ref.norm())
    print(f"LTPlugin forward rel-L2 {e:.3e}, 3-step sample rel-L2 {e_s:.3e}")
    assert e <= 5e-3 and e_s <= 5e-3
    for call in range(3):
        model.zero_grad(set_to_none=True)
        torch.manual_seed(93)
        loss = model(x.to(DEV))
        loss.backward()
    torch.manual_seed(93)
    sigma = torch.rand(2, device=DEV).cpu()
    eps = torch.randn(2, 1, 16384, device=DEV).cpu()
    loss_ref = oracle_loss(ref.net, x, eps, sigma)
    loss_ref.backward()
    rel = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
    print(f"LTPlugin loss {float(loss.detach()):.6f} vs oracle {float(loss_ref.detach()):.6f} (rel {rel:.2e})")
    assert rel < 2e-3
    worst, cos = compare_grads(list(ref.net.named_parameters()), list(model.net.parameters()))
    assert worst < GRAD_TOL and cos > 1 - 1e-3
