"""Host-side logic that needs no GPU: weight packers (the algebra the kernels rely on), the
liveness pool, the product path's refusal to run without a CUDA device."""
import pytest
import torch
import torch.nn.functional as F


@pytest.fixture(scope="module")
def ops():
    from audio_diffusion_pytorch_b200 import ops
    return ops


def test_pack_conv_is_tap_major(ops):
    w = torch.randn(24, 16, 3)
    p = ops.pack_conv(w).float()
    assert p.shape == (32, 48)                         # rows padded to 16
    for tap in range(3):
        assert torch.equal(p[:24, tap * 16:(tap + 1) * 16], w[:, :, tap].to(torch.bfloat16).float())
    assert torch.count_nonzero(p[24:]) == 0


def test_pack_mid_conv_layout(ops):
    w = torch.randn(32, 32, 3)
    p = ops.pack_mid_conv(w).float()
    assert p.shape == (32, 96)
    for tap in range(3):
        assert torch.equal(p[:, tap * 32:(tap + 1) * 32], w[:, :, tap].to(torch.bfloat16).float())


@pytest.mark.parametrize("f", [2, 4])
def test_upsample_fold_equals_upsample_then_conv(ops, f):
    """nearest-upsample(f) + conv3 == f phases x <= 2 taps on the low-res signal with pre-summed
    weights (the a_unet Upsample block, evaluated the way adp_conv_gemm(up_factor=f) does)."""
    torch.manual_seed(0)
    co, ci, T = 8, 16, 12
    w = torch.randn(co, ci, 3).to(torch.bfloat16).float()      # bf16-exact values: sums exact enough
    x = torch.randn(1, ci, T)
    ref = F.conv1d(F.interpolate(x, scale_factor=f, mode="nearest"), w, padding=1)   # [1, co, T*f]
    packed = ops.pack_upsample_conv(w, f).float()
    n_pad = packed.shape[0] // f
    xp = F.pad(x, (1, 1))                                       # zero rows outside [0, T)
    out = torch.zeros(1, co, T * f)
    for p in range(f):
        wp = packed[p * n_pad:p * n_pad + co]                   # [co, 2*ci]: tap slot 0, 1
        if p == 0:
            offs = (-1, 0)
        elif p == f - 1:
            offs = (0, 1)
        else:
            offs = (0,)
        acc = torch.zeros(1, co, T)
        for slot, off in enumerate(offs):
            xs = xp[:, :, 1 + off:1 + off + T]
            acc += torch.einsum("oc,bct->bot", wp[:, slot * ci:(slot + 1) * ci], xs)
        out[:, :, p::f] = acc
    err = float((out - ref).norm() / ref.norm())                # pre-summed weights are rounded to bf16
    assert err <= 5e-3, err


def test_pack_conv_dgrad_is_the_transposed_conv(ops):
    """Data gradient of conv3 = conv3 of the output gradient with flipped, transposed weights."""
    torch.manual_seed(1)
    co, ci, T = 16, 16, 20
    w = torch.randn(co, ci, 3).to(torch.bfloat16).float()
    x = torch.randn(1, ci, T, requires_grad=True)
    g = torch.randn(1, co, T)
    F.conv1d(x, w, padding=1).backward(g)
    p = ops.pack_conv_dgrad(w).float()[:ci]                     # [ci, 3*co] tap-major
    wt = torch.stack([p[:, k * co:(k + 1) * co] for k in range(3)], dim=2)   # [ci, co, 3]
    dx = F.conv1d(g, wt, padding=1)
    assert torch.allclose(dx, x.grad, rtol=1e-4, atol=1e-4)


def test_product_path_refuses_to_run_on_cpu():
    """No CPU / PyTorch fallback: a CPU tensor must raise, never silently compute."""
    import audio_diffusion_pytorch_b200 as adp
    model = adp.DiffusionModel(net_t=adp.UNetV0, in_channels=2, channels=[8, 32], factors=[1, 4],
                               items=[1, 1], attentions=[0, 0])
    with pytest.raises((AssertionError, RuntimeError)):
        model.sample(torch.randn(1, 2, 64), num_steps=2)


_GROUPS = [([16, 32, 64], 16, False), ([32, 64, 128], 32, False),
           ([8, 32, 64], 1, True), ([8, 32, 64], 2, True), ([8, 32, 64], 4, True), ([8, 32, 64], 8, True)]


@pytest.mark.parametrize("channels,groups,ok", _GROUPS, ids=[f"c{c[0]}-g{g}" for c, g, _ in _GROUPS])
def test_resnet_groups_beyond_the_fused_statistics_are_refused(channels, groups, ok):
    """The conv GEMM sums GroupNorm statistics for at most 8 groups: the constructor refuses more
    instead of failing inside the first forward."""
    import audio_diffusion_pytorch_b200 as adp
    kw = dict(dim=1, in_channels=2, channels=channels, factors=[1, 4, 4], items=[1, 1, 1],
              resnet_groups=groups)
    if ok:
        assert adp.UNetV0(**kw).groups == groups
    else:
        with pytest.raises(AssertionError, match="at most 8 groups"):
            adp.UNetV0(**kw)


def test_resampler_matches_the_oracle(oracle_port):
    """utils.resample (cached polyphase bank) == the oracle's windowed-sinc resampler, which
    make_golden.py proved bit-identical to the reference's."""
    from audio_diffusion_pytorch_b200 import utils
    torch.manual_seed(3)
    x = torch.randn(2, 2, 512)
    for f in (2, 4, 16):
        assert torch.equal(utils.upsample(x, f), oracle_port.sinc_upsample(x, f))
        assert torch.equal(utils.downsample(x, f), oracle_port.sinc_downsample(x, f))
    assert torch.equal(utils.upsample(x, 4), utils.upsample(x, 4))       # cached bank, same result
    y = utils.resample(x, 3, 2)
    assert torch.equal(y, oracle_port.sinc_resample(x, 3, 2))


def test_kwarg_routing_helpers():
    from audio_diffusion_pytorch_b200.utils import default, groupby
    taken, rest = groupby("mel_", {"mel_n_fft": 64, "channels": [8], "mel_sample_rate": 48000})
    assert taken == {"n_fft": 64, "sample_rate": 48000} and rest == {"channels": [8]}
    kept, _ = groupby("mel_", {"mel_n_fft": 64}, keep_prefix=True)
    assert kept == {"mel_n_fft": 64}
    assert default(None, 3) == 3 and default(0, 3) == 0 and default(None, lambda: 7) == 7
    assert default(None, int) is int          # classes are values, not factories


def test_model_classes_take_over_reference_parameters(oracle_port):
    """The U-Net registers its parameters in a_unet's order with a_unet's shapes, so
    `load_reference_parameters` can adopt the weights of a reference model; the vocoder's own
    layers keep the reference's names."""
    import audio_diffusion_pytorch_b200 as adp
    tiny = dict(channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 2, 2])
    voc_kw = dict(mel_n_fft=64, mel_channels=8, mel_sample_rate=48000, mel_normalize_log=True, **tiny)
    pairs = [
        (adp.DiffusionModel(net_t=adp.UNetV0, in_channels=2, attentions=[0, 0, 1], attention_heads=2,
                            attention_features=64, **tiny),
         oracle_port.DiffusionModelPort(in_channels=2, attentions=[0, 0, 1], attention_heads=2,
                                        attention_features=64, **tiny)),
        (adp.DiffusionUpsampler(net_t=adp.UNetV0, upsample_factor=16, in_channels=2, **tiny),
         oracle_port.DiffusionUpsamplerPort(upsample_factor=16, in_channels=2, **tiny)),
        (adp.DiffusionVocoder(net_t=adp.UNetV0, **voc_kw), oracle_port.DiffusionVocoderPort(**voc_kw)),
    ]
    for ours, ref in pairs:
        want = [tuple(p.shape) for p in ref.net.parameters()]
        got = [tuple(p.shape) for p in ours.net.parameters()]
        assert got == want
        ours.net.load_reference_parameters(ref.net)
        for a, b in zip(ours.net.parameters(), ref.net.parameters()):
            assert torch.equal(a, b)
        assert ours.diffusion.net is ours.net and ours.sampler.net is ours.net
    voc, vref = pairs[2]
    for key in ("to_flat.weight",):
        assert voc.state_dict()[key].shape == vref.state_dict()[key].shape


def test_reference_checkpoints_load_by_position(oracle_port, tmp_path):
    """`model.load_reference_state_dict(torch.load(ckpt))`: a state_dict saved from the reference
    model classes (a_unet key names, the shared net listed under three prefixes, the time MLP's
    Linear listed twice) is taken over without knowing a_unet's module names -- text-conditional
    net, vocoder (own layers by name), autoregressive (SkipCat) and autoencoder (user encoder)."""
    import audio_diffusion_pytorch_b200 as adp
    tiny = dict(channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 2, 2])
    text = dict(tiny, in_channels=2, attentions=[0, 0, 1], cross_attentions=[0, 1, 1], attention_heads=2,
                attention_features=64, use_embedding_cfg=True, embedding_max_length=8, embedding_features=32)
    voc_kw = dict(mel_n_fft=64, mel_channels=8, mel_sample_rate=48000, **tiny)
    ar_kw = dict(tiny, in_channels=2, length=1024, num_splits=4)
    ae_kw = dict(tiny, in_channels=2, inject_depth=2)
    pairs = [
        (adp.DiffusionModel(net_t=adp.UNetV0, **text), oracle_port.DiffusionModelPort(**text)),
        (adp.DiffusionVocoder(net_t=adp.UNetV0, **voc_kw), oracle_port.DiffusionVocoderPort(**voc_kw)),
        (adp.DiffusionAR(net_t=adp.UNetV0, **ar_kw), oracle_port.DiffusionARPort(**ar_kw)),
        (adp.DiffusionAE(net_t=adp.UNetV0, encoder=oracle_port.ToyEncoder(), **ae_kw),
         oracle_port.DiffusionAEPort(encoder=oracle_port.ToyEncoder(), **ae_kw)),
    ]
    for i, (ours, ref) in enumerate(pairs):
        path = tmp_path / f"ref{i}.pt"
        torch.save(ref.state_dict(), path)
        ckpt = torch.load(path)
        assert not any(torch.equal(a, b) for a, b in zip(ours.net.parameters(), ref.net.parameters())
                       if a.numel() > 64 and a.std() > 0)
        ours.load_reference_state_dict(ckpt)
        for a, b in zip(ours.net.parameters(), ref.net.parameters()):
            assert torch.equal(a, b)
        for key, val in ref.state_dict().items():
            if not key.startswith(("net.", "diffusion.", "sampler.")):
                assert torch.equal(ours.state_dict()[key], val), key
    # a checkpoint of a different architecture is refused, not half-loaded
    with pytest.raises(AssertionError):
        pairs[0][0].load_reference_state_dict(pairs[2][1].state_dict())


def test_upsampler_and_vocoder_conditioning_paths(oracle_port):
    """Host-side halves of DiffusionUpsampler / DiffusionVocoder (everything before the net)."""
    import audio_diffusion_pytorch_b200 as adp
    tiny = dict(channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 2, 2])
    up = adp.DiffusionUpsampler(net_t=adp.UNetV0, upsample_factor=16, in_channels=2, **tiny)
    ref = oracle_port.DiffusionUpsamplerPort(upsample_factor=16, in_channels=2, **tiny)
    x = torch.randn(2, 2, 4096)
    assert torch.equal(up.reupsample(x), ref.reupsample(x))
    kw = dict(mel_n_fft=64, mel_channels=8, mel_sample_rate=48000, mel_normalize_log=True, **tiny)
    torch.manual_seed(0)
    voc = adp.DiffusionVocoder(net_t=adp.UNetV0, **kw)
    vref = oracle_port.DiffusionVocoderPort(**kw)
    voc.to_flat.load_state_dict(vref.to_flat.state_dict())
    mel = torch.randn(2, 2, 8, 256)
    guide, lead = voc._unroll(mel)
    assert lead == (2, 2) and guide.shape == (4, 1, 4096)
    assert torch.equal(guide, vref.to_flat(mel.reshape(-1, 8, 256)))
    audio = torch.randn(2, 2, 4096)
    assert torch.allclose(voc.to_spectrogram(audio), vref.to_spectrogram(audio), atol=1e-6)


def test_skipcat_packs_reproduce_the_merge():
    """Host side of the use_modulation=False (SkipCat) path: the 1x1 merge conv folded into the
    level-0 stem weights, and the block-diagonal (two positions per row) packs of an 8-channel
    level, both reproduce conv1x1(cat([skip * 2^-0.5, y])) in fp32."""
    import audio_diffusion_pytorch_b200 as adp
    torch.manual_seed(3)
    net = adp.UNetV0(dim=1, in_channels=3, out_channels=2, channels=[8, 32], factors=[1, 4], items=[1, 1],
                     use_modulation=False, use_time_conditioning=False)
    with ops_pack_fp32():
        P = net._compute_packed_impl()
    lv0, lv1 = net.levels()
    L0, L1 = P["levels"]
    x, h = torch.randn(2, 3, 64), torch.randn(2, 8, 64)
    with torch.no_grad():
        want = lv0.merge(torch.cat([lv0.adapter(x) * 2 ** -0.5, lv0.up(h)], dim=1))
    got = F.conv1d(x, L0["adapt_w"][:, :, None], L0["adapt_b"]) + F.conv1d(h, L0["up_w"], L0["up_b"], padding=1)
    assert float((got - want).abs().max()) <= 1e-5
    # level 1: out = Wc1 (skip * s) + Wc2 y + bc on [B, T/2, 16] views of 8-channel tensors
    skip, y = torch.randn(2, 64, 8), torch.randn(2, 64, 8)
    with torch.no_grad():
        want = lv1.merge(torch.cat([skip.transpose(1, 2) * 2 ** -0.5, y.transpose(1, 2)], dim=1)).transpose(1, 2)
    w1, w2 = L1["cat_w1"].float(), L1["cat_w2"].float()
    assert w1.shape == (16, 16)
    got = (skip.reshape(2, 32, 16) @ w1.t() + L1["cat_b"] + y.reshape(2, 32, 16) @ w2.t()).reshape(2, 64, 8)
    assert float((got - want).abs().max()) <= 1e-5


def ops_pack_fp32():
    from audio_diffusion_pytorch_b200 import ops
    return ops.pack_dtype(torch.float32)


def test_arv_diffusion_algebra_and_rng_order(oracle_port):
    """ARVDiffusion (reference diffusion.py:98-130) around an arbitrary net, on the host: the
    product class draws rand((B,1,n)) then randn_like(x) and forms the same noised input, sigma
    channel and target as the oracle port (bit-identical with a pointwise toy net)."""
    from audio_diffusion_pytorch_b200.diffusion import ARVDiffusion

    class Toy(torch.nn.Module):
        def forward(self, chan, **kw):
            return torch.tanh(chan[:, :2]) * (1.0 + chan[:, 2:3])

    x = torch.randn(3, 2, 64, generator=torch.Generator().manual_seed(4))
    ours, theirs = ARVDiffusion(net=Toy(), length=64, num_splits=4), oracle_port.ARVDiffusionPort(Toy(), 64, 4)
    torch.manual_seed(11)
    a = ours(x)
    torch.manual_seed(11)
    b = theirs(x)
    assert torch.equal(a, b)
    with pytest.raises(AssertionError):
        ours(x[..., :32])                       # input length must match `length`
    with pytest.raises(AssertionError):
        ARVDiffusion(net=Toy(), length=64, num_splits=5)


@pytest.mark.parametrize("n_fft,n_mels,sr", [(1024, 80, 48000), (256, 16, 16000), (2048, 128, 44100), (64, 8, 48000)])
def test_mel_filter_bands_cover_every_nonzero(n_fft, n_mels, sr):
    """Host tables of adp_mel_spectrogram: every mel filter's non-zero bins lie inside the
    [lo, hi) range handed to the kernel (so the banded product equals the full matmul), the window
    is padded to n_fft the way torch.stft centres it, and empty filters get an empty range."""
    from audio_diffusion_pytorch_b200.components import MelSpectrogram
    front = MelSpectrogram(n_fft=n_fft, hop_length=n_fft // 4, win_length=n_fft // 2, sample_rate=sr,
                           n_mel_channels=n_mels)
    window, fb, band = front._kernel_tables(torch.device("cpu"))
    assert window.shape == (n_fft,) and fb.shape == (n_fft // 2 + 1, n_mels) and band.shape == (n_mels, 2)
    quarter = n_fft // 4
    assert torch.equal(window[quarter:quarter + n_fft // 2], front.to_spectrogram.window)
    assert float(window[:quarter].abs().sum() + window[quarter + n_fft // 2:].abs().sum()) == 0.0
    mag = torch.rand(n_fft // 2 + 1)
    full = mag @ fb
    banded = torch.stack([(mag[lo:hi] * fb[lo:hi, m]).sum() for m, (lo, hi) in enumerate(band.tolist())])
    assert torch.allclose(banded, full, rtol=1e-6, atol=1e-7)
    for m, (lo, hi) in enumerate(band.tolist()):
        assert 0 <= lo <= hi <= n_fft // 2 + 1
        if not bool((fb[:, m] != 0).any()):
            assert lo == hi


@pytest.mark.parametrize("fi,fo", [(1, 16), (16, 1), (3, 2), (4, 1)])
def test_polyphase_bank_geometry(fi, fo):
    """adp_resample's contract with the host filter bank: [factor_out, taps] with
    taps = 2*half + factor_in."""
    from audio_diffusion_pytorch_b200.utils import _polyphase_bank
    bank, half = _polyphase_bank(fi, fo, 0.99, 6, torch.float32, "cpu")
    assert bank.shape == (fo, 1, 2 * half + fi)


def test_a_fused_optimizer_step_moves_the_pack_version():
    """`fused=True` optimizers update the parameters without bumping their version counters: the
    packs must still be refreshed after the step."""
    from audio_diffusion_pytorch_b200.unet import UNetV0
    torch.manual_seed(0)
    net = UNetV0(dim=1, in_channels=2, channels=[8, 32], factors=[1, 4], items=[1, 1])
    for fused in (True, False):
        opt = torch.optim.AdamW(net.parameters(), lr=1e-2, fused=fused)
        for p in net.parameters():
            p.grad = torch.ones_like(p)
        before, w0 = net._version(), net.net.down.weight.detach().clone()
        opt.step()
        assert not torch.equal(w0, net.net.down.weight.detach())
        assert net._version() != before, f"fused={fused}: the optimizer step left the pack version unchanged"
