"""DPMSolverSampler (DPM-Solver++(2M)) on the GPU.

  * adp_dpm_step against its float64 restatement, between guard bands around every buffer: k = 0 with
    a NaN-filled history, k != 0, the step counter past the table (the last row), lengths that are
    not a multiple of the float4 width and buffers off 16-byte alignment (the scalar route);
  * the generic path (a module that is not the CUDA U-Net) on Gaussian data x0 ~ N(0, s^2), for
    which v = alpha beta (1 - s^2) x / (alpha^2 s^2 + beta^2) is exact and the exact sample is s x_1:
    the CUDA loop equals the fp64 loop to fp32 rounding, and its error is below half of VSampler's at
    N = 20 and 40;
  * tiny nets against the oracle net driven by the fp64 DPM loop (tests/test_dpm_sampler_cpu.py), at
    the 5e-3 of the VSampler sample tests: unconditional, guidance 5, DiffusionUpsampler,
    DiffusionAE.decode and an XUNet; 1 and 2 steps against VSampler;
  * eager runs, one graph per step, steps_per_graph = 10, the progress bar and a blocked
    conditioning table agree with each other and with the oracle;
  * the fp32 verification mode at rtol 1e-3 / atol 1e-4 against the fp64 loop."""
import math

import pytest
import torch

from test_dpm_sampler_cpu import FEW_STEPS, DpmRef, dpm_loop_f64

pytestmark = pytest.mark.gpu
DEV = "cuda"
SAMPLE_TOL = 5e-3
STEPS = 5                 # 2 first-order steps at the ends, 3 second-order ones
# DPM against VSampler at N <= 2 (every k = 0): on the GPU also GroupNorm's fp64 atomics, not only
# last-bit differences of x, flip bf16 roundings (tests/test_dpm_sampler_cpu.py, FEW_STEPS)
FEW_STEPS_TOL = 5e-4
POISON = 1.2345e30
GUARD = 36                # elements: 144 bytes

TINY = dict(in_channels=2, channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 2, 2],
            attentions=[0, 0, 1], attention_heads=2, attention_features=64)
TINY_TEXT = dict(TINY, cross_attentions=[0, 1, 1], use_embedding_cfg=True,
                 embedding_max_length=8, embedding_features=32)
TINY_NOATT = dict(channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 2, 2])


@pytest.fixture(scope="module")
def adp():
    import audio_diffusion_pytorch_b200 as adp_
    from audio_diffusion_pytorch_b200 import ops
    ops.device_check()
    return adp_


@pytest.fixture(autouse=True)
def no_grad():
    with torch.no_grad():
        yield


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ------------------------------------------------------------------------------ the kernel
def guarded(values, offset=0):
    """values (1-D, 4-byte elements) in a buffer between guard bands (POISON, or -7 for integers),
    `offset` elements past a 16-byte boundary (torch allocations are 16-byte aligned and GUARD
    elements are a multiple of 16 bytes); returns (buffer, view)."""
    n = values.numel()
    fill = POISON if values.dtype.is_floating_point else -7
    buf = torch.full((GUARD + offset + n + GUARD,), fill, dtype=values.dtype, device=DEV)
    view = buf[GUARD + offset:GUARD + offset + n]
    view.copy_(values.to(DEV))
    return buf, view


def outside(buf, view):
    """buf's elements outside `view`."""
    s = view.storage_offset() - buf.storage_offset()
    return torch.cat([buf[:s], buf[s + view.numel():]])


ROWS = torch.tensor([[0.0, 1.0, 0.70710678, 0.70710678, 0.0],        # sigma 1 -> 0.5: first order
                     [0.38268343, 0.92387953, 0.6532815, 0.41421356, 0.31546488],
                     [0.92387953, 0.38268343, 0.0, 1.0, 0.0]])        # last step to sigma = 0


@pytest.mark.parametrize("n", [1, 3, 4, 4099, 1 << 20])
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("step", [0, 1, 2, 9])
def test_dpm_step_kernel_vs_float64(adp, n, offset, step):
    from audio_diffusion_pytorch_b200 import diffusion
    g = torch.Generator().manual_seed(n + 7 * offset + step)
    x0, v0 = torch.randn(n, generator=g), torch.randn(n, generator=g)
    row = ROWS[min(step, 2)]
    k = float(row[4])
    h0 = torch.full((n,), float("nan")) if k == 0 else torch.randn(n, generator=g)
    bufs = {name: guarded(t, offset) for name, t in (("x", x0), ("v", v0), ("hist", h0))}
    tbuf, table = guarded(ROWS.reshape(-1))
    sbuf, step_t = guarded(torch.tensor([step], dtype=torch.int32))
    diffusion._dpm_step(bufs["x"][1], bufs["v"][1], bufs["hist"][1], table.view(3, 5), step_t, 3)
    torch.cuda.synchronize()
    a, b, c1, c2, kk = row.double().tolist()
    xd, vd = x0.double(), v0.double()
    x0d = a * xd - b * vd
    want = c1 * xd + c2 * (x0d if kk == 0 else (1 + kk) * x0d - kk * h0.double())
    absref = abs(c1) * xd.abs() + abs(c2) * ((1 + abs(kk)) * (abs(a) * xd.abs() + abs(b) * vd.abs()) +
                                             (0 if kk == 0 else abs(kk) * h0.double().abs()))
    got_x, got_h = bufs["x"][1].double().cpu(), bufs["hist"][1].double().cpu()
    assert torch.isfinite(got_x).all() and torch.isfinite(got_h).all()
    assert ((got_x - want).abs() <= 2 ** -20 * absref + 1e-30).all(), float((got_x - want).abs().max())
    assert ((got_h - x0d).abs() <= 2 ** -21 * (abs(a) * xd.abs() + abs(b) * vd.abs()) + 1e-30).all()
    assert torch.equal(bufs["v"][1].cpu(), v0), "v is read-only"
    assert torch.equal(table.cpu(), ROWS.reshape(-1)) and int(step_t) == step, "table and step are read-only"
    for name, (buf, view) in bufs.items():
        assert (outside(buf, view) == POISON).all(), f"{name}: a guard band changed"
    assert (outside(tbuf, table) == POISON).all() and (outside(sbuf, step_t) == -7).all()


# ------------------------------------------------------------------------------ Gaussian data
class GaussianV(torch.nn.Module):
    """The exact v of x0 ~ N(0, s^2) (not the CUDA U-Net: the sampler's generic path)."""

    def __init__(self, s: float):
        super().__init__()
        self.s = s

    def forward(self, x, sigma):
        sig = sigma.double().view(-1, 1, 1)
        a, b = torch.cos(sig * math.pi / 2), torch.sin(sig * math.pi / 2)
        s2 = self.s ** 2
        return (a * b * (1 - s2) * x.double() / (a * a * s2 + b * b)).to(x.dtype)


@pytest.mark.parametrize("steps", [10, 20, 40])
def test_gaussian_data_generic_path(adp, steps):
    s = 0.5
    noise = torch.randn(4, 2, 4096, generator=torch.Generator().manual_seed(1))
    exact = s * noise.double()
    net = GaussianV(s)
    got = adp.DPMSolverSampler(net)(noise.to(DEV), num_steps=steps).cpu()
    sig = torch.linspace(1, 0, steps + 1).tolist()
    want = dpm_loop_f64(lambda x, sg: net(x, torch.full((4,), sg, dtype=torch.float64)), noise, sig)
    e_impl = rel_l2(got, want)
    e_dpm, e_v = rel_l2(want, exact), rel_l2(adp.VSampler(net)(noise.to(DEV), num_steps=steps), exact)
    print(f"N={steps}: CUDA vs fp64 loop {e_impl:.2e}; error vs exact: DPM++(2M) {e_dpm:.3e}, VSampler {e_v:.3e}")
    assert e_impl <= 1e-5
    assert rel_l2(got, exact) <= e_dpm + 1e-5
    if steps >= 20:
        assert e_dpm < 0.5 * e_v


# ------------------------------------------------------------------------------ tiny nets
def model_pair(adp, oracle_port, port_cls, model_cls, **cfg):
    torch.manual_seed(0)
    ref = port_cls(sampler_t=DpmRef, **cfg)
    model = model_cls(net_t=adp.UNetV0, sampler_t=adp.DPMSolverSampler, **cfg).to(DEV)
    model.net.load_reference_parameters(ref.net)
    return ref, model


def noise_of(seed, shape=(2, 2, 4096)):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def test_unconditional_vs_oracle(adp, oracle_port):
    ref, model = model_pair(adp, oracle_port, oracle_port.DiffusionModelPort, adp.DiffusionModel, **TINY)
    noise = noise_of(4)
    e = rel_l2(model.sample(noise.to(DEV), num_steps=STEPS), ref.sample(noise, num_steps=STEPS))
    print(f"unconditional {STEPS} steps: rel-L2 {e:.3e}")
    assert e <= SAMPLE_TOL


def test_guidance_vs_oracle(adp, oracle_port):
    ref, model = model_pair(adp, oracle_port, oracle_port.DiffusionModelPort, adp.DiffusionModel, **TINY_TEXT)
    noise = noise_of(5)
    emb = torch.randn(2, 8, 32, generator=torch.Generator().manual_seed(6))
    s = model.sample(noise.to(DEV), num_steps=STEPS, embedding=emb.to(DEV), embedding_scale=5.0)
    e = rel_l2(s, ref.sample(noise, num_steps=STEPS, embedding=emb, embedding_scale=5.0))
    print(f"guidance 5, {STEPS} steps: rel-L2 {e:.3e}")
    assert e <= SAMPLE_TOL


def test_upsampler_vs_oracle(adp, oracle_port):
    ref, model = model_pair(adp, oracle_port, oracle_port.DiffusionUpsamplerPort, adp.DiffusionUpsampler,
                            upsample_factor=16, in_channels=2, **TINY_NOATT)
    low = noise_of(7, (2, 2, 256))
    s = model.sample(low.to(DEV), num_steps=STEPS, generator=torch.Generator().manual_seed(8))
    e = rel_l2(s, ref.sample(low, num_steps=STEPS, generator=torch.Generator().manual_seed(8)))
    print(f"DiffusionUpsampler {STEPS} steps: rel-L2 {e:.3e}")
    assert e <= SAMPLE_TOL


def test_autoencoder_decode_vs_oracle(adp, oracle_port):
    cfg = dict(TINY, inject_depth=2)
    torch.manual_seed(0)
    ref = oracle_port.DiffusionAEPort(encoder=oracle_port.ToyEncoder(), sampler_t=DpmRef, **cfg)
    torch.manual_seed(0)
    model = adp.DiffusionAE(encoder=oracle_port.ToyEncoder(), net_t=adp.UNetV0, sampler_t=adp.DPMSolverSampler,
                            **cfg).to(DEV)
    model.net.load_reference_parameters(ref.net)
    model.encoder.load_state_dict(ref.encoder.state_dict())
    latent = ref.encoder(noise_of(9))
    noise = noise_of(10)
    out = model.sampler(noise.to(DEV), num_steps=STEPS, channels=[None, None, latent.to(DEV)])
    e = rel_l2(out, ref.sampler(noise, num_steps=STEPS, channels=[None, None, latent]))
    print(f"DiffusionAE decode {STEPS} steps: rel-L2 {e:.3e}")
    assert e <= SAMPLE_TOL
    assert model.decode(latent.to(DEV), num_steps=STEPS).shape == (2, 2, 4096)


def test_xunet_vs_oracle(adp, oracle_port):
    from test_xunet_gpu import inputs, pair
    ref, model = pair(oracle_port, adp, "att_first")
    noise = inputs("att_first", seed=4)[0]
    s = adp.DPMSolverSampler(model.net)(noise.to(DEV), num_steps=10)
    e = rel_l2(s, DpmRef(ref.net)(noise, num_steps=10))
    print(f"XUNet att_first 10 steps: rel-L2 {e:.3e}")
    assert e <= SAMPLE_TOL


@pytest.mark.parametrize("steps,schedule", FEW_STEPS, ids=["1_step", "2_steps"])
def test_few_steps_agree_with_vsampler(adp, oracle_port, steps, schedule):
    _, model = model_pair(adp, oracle_port, oracle_port.DiffusionModelPort, adp.DiffusionModel, **TINY)
    noise = noise_of(11).to(DEV)
    s_dpm = adp.DPMSolverSampler(model.net, schedule=schedule)(noise, num_steps=steps)
    s_v = adp.VSampler(model.net, schedule=schedule)(noise, num_steps=steps)
    e = rel_l2(s_dpm, s_v)
    print(f"{steps} steps: DPM vs VSampler rel-L2 {e:.3e}")
    assert e <= FEW_STEPS_TOL


# ------------------------------------------------------------------------------ execution variants
def test_execution_variants_agree(adp, oracle_port):
    ref, model = model_pair(adp, oracle_port, oracle_port.DiffusionModelPort, adp.DiffusionModel, **TINY)
    net, steps = model.net, 20
    noise = noise_of(12)
    want = ref.sample(noise, num_steps=steps)
    runs = {}

    def run(name, **attrs):
        saved = {k: getattr(net, k) for k in attrs}
        for k, v in attrs.items():
            setattr(net, k, v)
        runs[name] = model.sample(noise.to(DEV), num_steps=steps, show_progress=name == "progress").cpu()
        for k, v in saved.items():
            setattr(net, k, v)
    run("eager", use_cuda_graph=False)
    run("graph_per_step", steps_per_graph=1)
    run("graph_per_step_replayed", steps_per_graph=1)
    run("steps_per_graph_10", steps_per_graph=10)
    run("steps_per_graph_10_replayed", steps_per_graph=10)
    run("progress")
    run("blocks", cond_table_rows=6)          # 3 steps per conditioning block at batch 2
    for name, s in runs.items():
        e, e_eager = rel_l2(s, want), rel_l2(s, runs["eager"])
        print(f"{name}: rel-L2 vs oracle {e:.3e}, vs eager {e_eager:.3e}")
        assert torch.isfinite(s).all() and e <= SAMPLE_TOL and e_eager <= SAMPLE_TOL


# ------------------------------------------------------------------------------ fp32 mode
def close(got, want, what, rtol=1e-3, atol=1e-4):
    got, want = got.detach().float().cpu(), want.detach().float().cpu()
    err = (got - want).abs()
    print(f"{what}: max abs err {float(err.max()):.3e}, rel-L2 {rel_l2(got, want):.3e}")
    torch.testing.assert_close(got, want, rtol=rtol, atol=atol)


def test_fp32_verification_mode(adp, oracle_port):
    ref, model = model_pair(adp, oracle_port, oracle_port.DiffusionModelPort, adp.DiffusionModel, **TINY)
    model.net.verify_fp32 = True
    noise = noise_of(13)
    want = ref.sample(noise, num_steps=STEPS)
    for call in range(2):
        close(model.sample(noise.to(DEV), num_steps=STEPS), want, f"fp32 mode: {STEPS} steps (call {call})")

    ref, model = model_pair(adp, oracle_port, oracle_port.DiffusionModelPort, adp.DiffusionModel, **TINY_TEXT)
    model.net.verify_fp32 = True
    emb = torch.randn(2, 8, 32, generator=torch.Generator().manual_seed(14))
    close(model.sample(noise.to(DEV), num_steps=STEPS, embedding=emb.to(DEV), embedding_scale=5.0),
          ref.sample(noise, num_steps=STEPS, embedding=emb, embedding_scale=5.0), "fp32 mode: guidance 5")

