"""DPMSolverSampler (DPM-Solver++(2M) for v-diffusion) on the CPU.

  * the host coefficient rows (alpha_i, beta_i, c1, c2, k) against an independent restatement in the
    log-SNR form of Lu et al. (2022), Algorithm 2: c2 = -alpha_i+1 expm1(-h_i), at the limits
    sigma_0 = 1 (lambda = -inf) and sigma_N = 0 (lambda = +inf), and at N = 1, 2;
  * the refusals (schedule not strictly decreasing, outside [0, 1], out_channels other than x's)
    name their condition;
  * the 'sample_dpm' plan launches the 'sample' plan's program with stem_out writing v and the
    update before step_advance;
  * a tiny net runs its 'sample_dpm' program here (fake kernels writing the launch checker's fp64
    restatements, tests/launch_check.py; the update as its fp64 restatement) against the oracle net
    driven by an fp64 DPM-Solver++(2M) loop: plain, in blocks of the conditioning table and with
    the progress bar.

DpmRef and reference_rows are also the references of tests/test_dpm_sampler_gpu.py."""
import math

import numpy as np
import pytest
import torch
from torch import nn

import launch_check as lc
from audio_diffusion_pytorch_b200 import _lib, diffusion, ops
from audio_diffusion_pytorch_b200.diffusion import (DPMSolverSampler, LinearSchedule, Schedule, VSampler,
                                                    dpm_coefficients)
from audio_diffusion_pytorch_b200.models import DiffusionModel
from audio_diffusion_pytorch_b200.unet import UNetV0


def reference_rows(sigmas) -> np.ndarray:
    """float64 [N, 5] rows (alpha_i, beta_i, c1, c2, k) in the log-SNR form: lambda = log(alpha / beta)
    with lambda(1) = -inf and lambda(0) = +inf, h_i = lambda_i+1 - lambda_i, c1 = beta_i+1 / beta_i,
    c2 = -alpha_i+1 expm1(-h_i); k = h_i / (2 h_i-1), 0 on the first step, after an infinite h and on
    a last step to sigma = 0."""
    s = np.asarray(sigmas, dtype=np.float64)
    a = np.where(s == 1.0, 0.0, np.cos(np.pi * s / 2))
    b = np.sin(np.pi * s / 2)
    with np.errstate(divide="ignore"):
        lam = np.where(s == 1.0, -np.inf, np.where(s == 0.0, np.inf, np.log(a / b)))
    h = lam[1:] - lam[:-1]
    n = len(h)
    k = np.zeros(n)
    for i in range(1, n):
        if np.isfinite(h[i - 1]) and not (i == n - 1 and s[-1] == 0.0):
            k[i] = h[i] / (2 * h[i - 1])
    return np.stack([a[:-1], b[:-1], b[1:] / b[:-1], -a[1:] * np.expm1(-h), k], axis=1)


def dpm_loop_f64(net_fn, x, sigmas):
    """The fp64 DPM-Solver++(2M) loop over sigmas (a list): net_fn(x float64, sigma_i) -> v; returns x_N
    in float64."""
    rows = reference_rows(sigmas)
    x, prev = x.double(), None
    for i, (a, b, c1, c2, k) in enumerate(rows):
        v = net_fn(x, float(sigmas[i])).double()
        x0 = a * x - b * v
        x = c1 * x + c2 * (x0 if k == 0 else (1 + k) * x0 - k * prev)
        prev = x0
    return x


class DpmRef(nn.Module):
    """A `sampler_t` for the oracle models: dpm_loop_f64 with the linear schedule from 1 to 0, as
    LinearSchedule makes it (fp32 linspace)."""

    def __init__(self, net: nn.Module):
        super().__init__()
        self.net = net

    @torch.no_grad()
    def forward(self, x_noisy, num_steps: int, show_progress: bool = False, **kwargs):
        sig = torch.linspace(1.0, 0.0, num_steps + 1).tolist()
        b = x_noisy.shape[0]

        def net_fn(x, s):
            return self.net(x.float().to(x_noisy.device), torch.full((b,), s, device=x_noisy.device), **kwargs).cpu()
        return dpm_loop_f64(net_fn, x_noisy.cpu(), sig).float()


def dpm_step_f64(x, v, hist, table, step, rows):
    """adp_dpm_step restated in float64 (reads hist only when k != 0)."""
    r = min(max(int(step[0]), 0), rows - 1)
    a, b, c1, c2, k = table[r].double().tolist()
    x0 = a * x.double() - b * v.double()
    d = x0 if k == 0 else (1 + k) * x0 - k * hist.double()
    x.copy_(c1 * x.double() + c2 * d)
    hist.copy_(x0)


# ------------------------------------------------------------------------------ coefficients
SCHEDULES = {
    "linear_1": torch.linspace(1, 0, 2),
    "linear_2": torch.linspace(1, 0, 3),
    "linear_3": torch.linspace(1, 0, 4),
    "linear_50": torch.linspace(1, 0, 51),
    "from_1_to_0.05": torch.linspace(1, 0.05, 8),
    "from_0.9_to_0": torch.linspace(0.9, 0, 8),
    "inside": torch.tensor([0.95, 0.7, 0.4, 0.2, 0.1, 0.02]),
    "inside_2": torch.tensor([0.8, 0.5, 0.3]),
}


@pytest.mark.parametrize("name", sorted(SCHEDULES))
def test_coefficients_match_log_snr_form(name):
    sig = SCHEDULES[name]
    got = dpm_coefficients(sig)
    want = reference_rows(sig.double().numpy())
    assert got.dtype == torch.float32 and got.shape == (len(sig) - 1, 5)
    assert torch.isfinite(got).all()
    np.testing.assert_allclose(got.double().numpy(), want, rtol=1e-6, atol=1e-7)
    assert got[0, 4] == 0.0                                   # first step: first order
    if float(sig[0]) == 1.0:
        assert got[0, 0] == 0.0 and (len(got) < 2 or got[1, 4] == 0.0)   # h_0 = inf
    if float(sig[-1]) == 0.0:
        assert got[-1, 2] == 0.0 and got[-1, 3] == 1.0 and got[-1, 4] == 0.0   # x_N = x0
    if name == "inside":
        assert (got[1:, 4] != 0).all()


@pytest.mark.parametrize("n", [1, 2])
def test_first_order_steps_are_vsampler_steps(n):
    """k = 0 on every step for N <= 2 from 1 to 0, and the step is then VSampler's update."""
    sig = torch.linspace(1, 0, n + 1).double()
    rows = dpm_coefficients(sig).double()
    assert (rows[:, 4] == 0).all()
    x, v = torch.randn(64, dtype=torch.float64), torch.randn(64, dtype=torch.float64)
    a, b = torch.cos(sig * math.pi / 2), torch.sin(sig * math.pi / 2)
    for i, (ai, bi, c1, c2, _) in enumerate(rows.tolist()):
        dpm = c1 * x + c2 * (ai * x - bi * v)
        vs = a[i + 1] * (a[i] * x - b[i] * v) + b[i + 1] * (b[i] * x + a[i] * v)
        torch.testing.assert_close(dpm, vs, rtol=1e-6, atol=1e-6)


# ------------------------------------------------------------------------------ refusals
class Fixed(Schedule):
    def __init__(self, values):
        super().__init__()
        self.values = values

    def forward(self, num_steps, device):
        return torch.tensor(self.values, device=device)


class Echo(nn.Module):
    def __init__(self, out_channels=None, drop=0):
        super().__init__()
        if out_channels is not None:
            self.out_channels = out_channels
        self.drop = drop

    def forward(self, x, sigma, **kw):
        return x[:, self.drop:]


REFUSALS = [
    ("not_decreasing", Echo(), Fixed([1.0, 0.5, 0.5, 0.0]), "strictly decreasing"),
    ("increasing", Echo(), Fixed([0.0, 0.5, 1.0, 1.0]), "strictly decreasing"),
    ("above_1", Echo(), LinearSchedule(1.2, 0.0), r"leaves \[0, 1\]"),
    ("below_0", Echo(), LinearSchedule(1.0, -0.5), r"leaves \[0, 1\]"),
    ("out_channels", Echo(out_channels=1), LinearSchedule(), "out_channels=1 differs from the 2 channels of x"),
    ("returned_shape", Echo(drop=1), LinearSchedule(), r"returned \(2, 1, 16\) for x of shape \(2, 2, 16\)"),
]


@pytest.mark.parametrize("name,net,schedule,msg", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_refusals_name_their_condition(name, net, schedule, msg):
    with pytest.raises(ValueError, match=msg):
        DPMSolverSampler(net, schedule=schedule)(torch.randn(2, 2, 16), num_steps=3)


def test_refuses_cuda_net_with_fewer_output_channels():
    net = UNetV0(dim=1, in_channels=2, out_channels=1, channels=[8, 32], factors=[1, 2], items=[1, 1])
    with pytest.raises(ValueError, match="out_channels=1 differs from the 2 channels of x"):
        DPMSolverSampler(net)(torch.randn(1, 2, 64), num_steps=2)


# ------------------------------------------------------------------------------ programs
TINY = dict(in_channels=2, channels=[16, 48, 96], factors=[1, 2, 2], items=[1, 1, 1],
            attentions=[0, 0, 1], attention_heads=2, attention_features=32)


@pytest.fixture
def cpu_launches(monkeypatch):
    monkeypatch.setattr(ops, "device_check", lambda: None)
    monkeypatch.setattr(ops, "require_cuda", lambda x: None)

    def no_library():
        raise AssertionError("a launch reached the CUDA library")
    monkeypatch.setattr(_lib, "lib", no_library)


def test_sample_dpm_program_is_the_sample_program_with_the_update(monkeypatch):
    from test_launch_programs_cpu import install
    rec = install(monkeypatch)
    monkeypatch.setattr(diffusion, "_dpm_step", rec.make("dpm_step", diffusion._dpm_step))
    torch.manual_seed(0)
    net = UNetV0(dim=1, **TINY)
    progs = {}
    for mode in ("sample", "sample_dpm"):
        plan = net._plan(2, 1024, 2, 0, mode, (None, False))
        plan.run_eager()
        progs[mode] = [(k[0], dict((a, v) for a, v in k[1:])) for k in rec.take()]
    sample, dpm = progs["sample"], progs["sample_dpm"]
    assert [n for n, _ in dpm] == [n for n, _ in sample[:-1]] + ["dpm_step", "step_advance"]
    so_s, so_d = sample[-2][1], dpm[-3][1]
    assert so_s["x_next"] is not None and so_s["ab"] is not None and so_s["v_out"] is None
    assert so_d["x_next"] is None and so_d["ab"] is None and so_d["v_out"] is not None
    upd = dpm[-2][1]
    assert upd["v"] == so_d["v_out"] and upd["step"] == dpm[-1][1]["step"] and upd["rows"] == net.max_table_steps


def _pair(oracle_port, cfg):
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**cfg)
    model = DiffusionModel(net_t=UNetV0, sampler_t=DPMSolverSampler, **cfg)
    model.net.load_reference_parameters(ref.net)
    model.net.use_cuda_graph = False
    return ref, model


@pytest.mark.parametrize("variant", ["plain", "blocks", "progress"])
def test_sample_dpm_program_vs_oracle(cpu_launches, oracle_port, monkeypatch, variant):
    ref, model = _pair(oracle_port, TINY)
    used = []

    def update(x, v, hist, table, step, rows):
        r = min(int(step[0]), rows - 1)
        if table[r, 4] == 0:
            hist.fill_(float("nan"))          # k = 0 must not read the history
        used.append(table[r].clone())
        dpm_step_f64(x, v, hist, table, step, rows)
    monkeypatch.setattr(diffusion, "_dpm_step", update)
    if variant == "blocks":
        model.net.cond_table_rows = 4         # 2 steps per block at batch 2
    noise = torch.randn(2, 2, 1024, generator=torch.Generator().manual_seed(4))
    steps = 5
    with torch.no_grad():
        want = DpmRef(ref.net)(noise, num_steps=steps)
        with lc.Shadow(fake=True) as sh:
            s = model.sample(noise, num_steps=steps, show_progress=variant == "progress")
    assert sh.n_checked == sh.n_launch > 0
    assert torch.equal(torch.stack(used), dpm_coefficients(torch.linspace(1, 0, steps + 1)))
    e = float((s.double() - want.double()).norm() / want.double().norm())
    print(f"{variant}: 5-step DPM-Solver++(2M) sample rel-L2 {e:.3e}")
    assert torch.isfinite(s).all() and e <= 5e-3


# For N <= 2 from sigma = 1 every k is 0 (the first step, then h_0 = inf).  The schedules end at
# 0.3, not 0: the last step to sigma = 0 returns x0 = alpha x - beta v, which for an untrained net
# (v ~ x) is a cancellation to ~1 % of |x| that turns a last-bit difference of x into a flipped bf16
# rounding and a ~2 % change of the sample (VSampler against itself on x (1 + 1e-7) moves as much).
# Ending at 0.3 keeps that amplification near 1e-4 (7e-5 on this program's fake kernels)
FEW_STEPS_TOL = 2e-4
FEW_STEPS = [(1, LinearSchedule()), (2, LinearSchedule(1.0, 0.3))]


@pytest.mark.parametrize("steps,schedule", FEW_STEPS, ids=["1_step", "2_steps"])
def test_few_steps_agree_with_vsampler_program(cpu_launches, oracle_port, monkeypatch, steps, schedule):
    monkeypatch.setattr(diffusion, "_dpm_step", dpm_step_f64)
    _, model = _pair(oracle_port, TINY)
    noise = torch.randn(2, 2, 1024, generator=torch.Generator().manual_seed(5))
    with torch.no_grad(), lc.Shadow(fake=True):
        s_dpm = DPMSolverSampler(model.net, schedule=schedule)(noise, num_steps=steps)
        s_v = VSampler(model.net, schedule=schedule)(noise, num_steps=steps)
    e = float((s_dpm - s_v).norm() / s_v.norm())
    print(f"{steps} steps: DPM vs VSampler rel-L2 {e:.3e}")
    assert e <= FEW_STEPS_TOL
