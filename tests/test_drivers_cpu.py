"""The drivers above the launch programs, run on the CPU: B200UNet.forward, sample_loop,
inpaint_loop and arv_loop, training.fused_v_loss and differentiable_forward with their backward.

The drivers stage the inputs, pick the plan, walk the sampling steps through the conditioning
table and decide when a program runs eagerly, is captured into a CUDA graph or is replayed.  Here
every launch function is replaced by the recorder of test_launch_programs_cpu.py, and the CUDA
graph capture by a fake that logs ("capture", early_weights) and, on replay(), logs ("replay",) and
runs the captured function.  Each step_select also records the conditioning block it points at
(the table by storage index, the iterations per table row, the rows) and the alpha/beta rows of the
block.  Progress iterators log each step they hand out and their end.  The log of every scenario
is compared with tests/golden/drivers.json.gz.

    python tests/test_drivers_cpu.py --write     # re-record the fixture
"""
import gzip
import inspect
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
TESTS = os.path.join(ROOT, "tests")
if TESTS not in sys.path:
    sys.path.insert(0, TESTS)

import launch_check as lc  # noqa: E402
from audio_diffusion_pytorch_b200 import ops, training, unet  # noqa: E402
from audio_diffusion_pytorch_b200.diffusion import ARVSampler, VInpainter, _alpha_beta  # noqa: E402
from audio_diffusion_pytorch_b200.models import DiffusionAR, DiffusionModel  # noqa: E402
from test_launch_check_cpu import _draws_from, _golden, cpu_launches, rel_l2  # noqa: E402,F401  (fixture)
from test_launch_programs_cpu import TINY, TINY_TEXT, build_net, first_difference, install  # noqa: E402

FIXTURE = os.path.join(ROOT, "tests", "golden", "drivers.json.gz")


class _FakeGraph:
    def __init__(self, log, run):
        self.log, self.run = log, run

    def replay(self):
        self.log.append(["replay"])
        self.run()


def install_drivers(mp):
    """The launch recorder (plus the sampler, inpainting and autoregressive steps), the table log of
    step_select and the fake capture."""
    sig = inspect.signature(ops.step_select)
    rec = install(mp)
    mp.setattr(ops, "require_cuda", lambda x: None)
    for name in ("sampler_step", "inpaint_blend", "arv_step"):
        mp.setattr(ops, name, rec.make(name, getattr(ops, name)))
    recorded = ops.step_select

    def step_select(*args, **kwargs):
        recorded(*args, **kwargs)
        a = sig.bind(*args, **kwargs).arguments
        addr, share, rows = a["ctrl"].tolist()
        table = [i for (ptr, _), i in rec.storages.items() if ptr == addr]
        rec.launches.append(["table", table, share, rows, a["ab_table"][:share * rows].tolist()])
    mp.setattr(ops, "step_select", step_select)

    def capture(run, early_weights=False):
        rec.launches.append(["capture", early_weights])
        return _FakeGraph(rec.launches, run)
    for mod in (unet, training):
        if hasattr(mod, "_capture"):
            mp.setattr(mod, "_capture", capture)
    return rec


def _progress(log, n):
    for i in range(n):
        log.append(["progress", i])
        yield i
    log.append(["progress", "end"])


def _inputs(B=2, C=2, T=4096, seed=1):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, C, T, generator=g), torch.rand(B, generator=g)


def _schedule(num_steps, B=2):
    sig = torch.linspace(1, 0, num_steps + 1)
    alphas, betas = _alpha_beta(sig)
    return sig[:, None].expand(-1, B), alphas, betas


def forward(rec):
    net = build_net(TINY, {})
    x, sigma = _inputs()
    with torch.no_grad():
        for _ in range(3):
            net(x, sigma)


def sample(rec):
    """5 steps in conditioning blocks of 2, 2 and 1 steps, two steps per multi-step graph."""
    net = build_net(TINY, {"cond_table_rows": 4, "steps_per_graph": 2})
    x, _ = _inputs()
    net.sample_loop(x, *_schedule(5))
    net.sample_loop(x, *_schedule(5), progress=_progress(rec.launches, 5))


def sample_cfg(rec):
    net = build_net(TINY_TEXT, {"cond_table_rows": 8, "steps_per_graph": 2})
    x, _ = _inputs()
    emb = torch.randn(2, 8, 32, generator=torch.Generator().manual_seed(2))
    net.sample_loop(x, *_schedule(5), embedding=emb, embedding_scale=5.0)


def inpaint(rec):
    """3 steps x 2 resamples in conditioning blocks of 2 and 1 steps."""
    net = build_net(TINY, {"cond_table_rows": 4, "steps_per_graph": 2})
    x, _ = _inputs()
    source, _ = _inputs(seed=3)
    mask = torch.zeros(2, 2, 4096, dtype=torch.bool)
    mask[:, :, :1000] = True
    net.inpaint_loop(x, source, mask, *_schedule(3), 2)
    net.inpaint_loop(x, source, mask, *_schedule(3), 2, progress=_progress(rec.launches, 3))


def autoregressive(rec):
    torch.manual_seed(0)
    kw = {k: v for k, v in TINY.items() if k != "in_channels"}
    net = DiffusionAR(net_t=unet.UNetV0, in_channels=2, length=4096, num_splits=4, **kw).net
    current, _ = _inputs()
    sigmas = torch.linspace(1, 0, 4)[:, None, None, None].repeat(1, 2, 1, 4096)
    net.arv_loop(current, sigmas)
    net.arv_loop(current, sigmas, progress=_progress(rec.launches, 3))


def train(rec):
    """Three loss + backward steps with an optimizer step between them: the forward and backward
    graphs and the re-packs after a weight update."""
    net = build_net(TINY, {})
    x, sigma = _inputs()
    noise, _ = _inputs(seed=4)
    opt = torch.optim.SGD(net.parameters(), lr=1e-3)
    for i in range(3):
        if i:
            opt.step()
            opt.zero_grad()
        training.fused_v_loss(net, x, noise, sigma).backward()


def train_cfg(rec):
    """Guidance under autograd: the 'v' and 'v1' plans of differentiable_forward."""
    net = build_net(TINY_TEXT, {})
    x, sigma = _inputs()
    emb = torch.randn(2, 8, 32, generator=torch.Generator().manual_seed(2))
    for _ in range(2):
        net(x, sigma, embedding=emb, embedding_scale=5.0).sum().backward()


SCENARIOS = {f.__name__: f for f in (forward, sample, sample_cfg, inpaint, autoregressive, train, train_cfg)}


def record(name, rec):
    rec.storages, rec.slots, rec.keep = {}, {}, []
    rec.take()
    SCENARIOS[name](rec)
    return rec.take()


@pytest.fixture
def recorder(monkeypatch):
    return install_drivers(monkeypatch)


@pytest.fixture(scope="module")
def fixture():
    with gzip.open(FIXTURE, "rt") as f:
        return json.load(f)


@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_driver_log(name, recorder, fixture):
    got = json.loads(json.dumps({"prog": record(name, recorder)}))
    d = first_difference(got, {"prog": fixture[name]}, name)
    assert d is None, "driver log differs from the fixture at " + d


def test_fixture_covers_every_scenario(fixture):
    assert sorted(fixture) == sorted(SCENARIOS)


# ------------------------------------------------------------------------------ fp32 fake kernels
def _fp32(model, ref):
    model.net.load_reference_parameters(ref.net)
    model.net.verify_fp32 = True
    model.net.use_cuda_graph = False           # every call runs the plan's launches eagerly
    return model.net


def test_inpaint_loop_fp32_vs_golden(cpu_launches, oracle_port, golden_dir, monkeypatch):
    """B200UNet.inpaint_loop (the sampling plan, step_select over the conditioning table,
    inpaint_blend), 4 steps x 2 resamples in two conditioning blocks on fp32 fake kernels, fed the
    golden run's draws.  Measured rel-L2 against the unmodified reference: 1.8e-8; bound 1e-7."""
    g = _golden(golden_dir, "tiny_inpaint.npz")
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**TINY)
    net = _fp32(DiffusionModel(net_t=unet.UNetV0, **TINY), ref)
    net.cond_table_rows = 4                    # 2 steps per conditioning block at batch 2
    source = torch.randn(2, 2, 4096, generator=torch.Generator().manual_seed(int(g["source_seed"])))
    mask = torch.zeros(2, 2, 4096, dtype=torch.bool)
    for b_, lo, hi in g["mask_spans"].tolist():
        mask[b_, :, lo:hi] = True
    steps, resamples = int(g["num_steps"]), int(g["num_resamples"])
    torch.manual_seed(int(g["rng_seed"]))
    left = _draws_from(monkeypatch, [torch.randn(2, 2, 4096) for _ in range(1 + steps * resamples)])
    with torch.no_grad(), lc.Shadow(fake=True, probe=True) as sh:
        out = VInpainter(net=net)(source, mask, num_steps=steps, num_resamples=resamples)
    monkeypatch.undo()
    e = rel_l2(out, g["out"])
    print(f"B200UNet.inpaint_loop {steps} steps x {resamples} resamples on fp32 fake kernels: rel-L2 {e:.3e}")
    assert e <= 1e-7
    assert next(left, None) is None
    assert sh.n_checked == sh.n_launch > 0
    assert sh.records["inpaint_blend.x"].count == steps * resamples
    assert {"step_select", "stem_out", "inpaint_blend"} <= {k for k, _ in sh.probed}
    assert torch.equal(out[mask], source[mask])


def test_arv_loop_fp32_vs_golden(cpu_launches, oracle_port, golden_dir, monkeypatch):
    """B200UNet.arv_loop (the 'v' plan over cat([current, sigma]), arv_step) under ARVSampler: start
    window (4 steps) and 6 ladder passes on fp32 fake kernels, fed the golden run's draws.
    Measured rel-L2 against the unmodified reference: 1.2e-7; bound 5e-7."""
    g = _golden(golden_dir, "tiny_autoregressive.npz")
    cfg = dict(TINY, in_channels=2, length=4096, num_splits=4)
    torch.manual_seed(0)
    ref = oracle_port.DiffusionARPort(**cfg)
    net = _fp32(DiffusionAR(net_t=unet.UNetV0, **cfg), ref)
    torch.manual_seed(int(g["sample_seed"]))
    draws = [torch.randn(2, 2, 4096), torch.randn(2, 2, 4096)] + [torch.randn(2, 2, 1024) for _ in range(6)]
    left = _draws_from(monkeypatch, draws)
    sampler = ARVSampler(net=net, in_channels=2, length=4096, num_splits=4)
    with torch.no_grad(), lc.Shadow(fake=True, probe=True) as sh:
        out = sampler(num_items=2, num_chunks=6, num_steps=4)
    monkeypatch.undo()
    e = rel_l2(out, g["sample"])
    print(f"B200UNet.arv_loop 6 chunks x 4 steps on fp32 fake kernels: rel-L2 {e:.3e}")
    assert out.shape == (2, 2, 6144) and e <= 5e-7
    assert next(left, None) is None
    assert sh.n_checked == sh.n_launch > 0
    assert sh.records["arv_step.chan"].count == 4 + 6
    assert {"arv_step", "stem_out"} <= {k for k, _ in sh.probed}


if __name__ == "__main__" and "--write" in sys.argv:
    mp = pytest.MonkeyPatch()
    rec = install_drivers(mp)
    data = {name: record(name, rec) for name in sorted(SCENARIOS)}
    mp.undo()
    with gzip.GzipFile(FIXTURE, "wb", mtime=0) as f:
        f.write(json.dumps(data, separators=(",", ":"), sort_keys=True).encode())
    for name, log in data.items():
        print(name, len(log), [e for e in log if e[0] in ("capture", "replay", "progress")][:40])
    print(f"wrote {FIXTURE} ({os.path.getsize(FIXTURE)} bytes)")
