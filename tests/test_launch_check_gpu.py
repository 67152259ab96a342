"""Every kernel launch of the benchmark's sampling programs, at the benchmark's shapes, checked
against an fp64 restatement (tests/launch_check.py): each launch on the activations the real
program gives it, with the real buffer aliasing, held to its own bf16 bound.

The wrapped runs are eager and synchronised; each test then runs the same model and inputs
unwrapped through the captured CUDA graph (programmatic-dependent launch, early weight fetch)
and requires the same result within rel-L2 1e-4 (GroupNorm statistics are accumulated with
atomics, so runs are not bit-identical).  For the sampling programs that comparison runs on a
one-step sample, also checked launch by launch: x_1 = -v(x, sigma = 1) is well conditioned,
while a two-step sample of an untrained net from sigma = 1 is the branch applied twice
(x_pred = -beta gate branch at each step; the skip cancels), a few 1e-4 of v, so the atomics'
last-bit jitter is already ~1e-2 of it from one eager run to the next.  The one-step program
goes through the same conditioning table, device step selector and in-place x_next update.
Run with -s for the per-kind table (count, worst err/bound, label of the worst launch)."""
import gc
import time

import pytest
import torch

import launch_check as lc

pytestmark = pytest.mark.gpu

DEV = "cuda"
T_FULL = 2 ** 18
# the benchmark's workloads (bench.py)
README = dict(in_channels=2, channels=[8, 32, 64, 128, 256, 512, 512, 1024, 1024],
              factors=[1, 4, 4, 4, 2, 2, 2, 2, 2], items=[1, 2, 2, 2, 2, 2, 2, 4, 4],
              attentions=[0, 0, 0, 0, 0, 1, 1, 1, 1], attention_heads=8, attention_features=64)
CFG3 = dict(README, cross_attentions=[0, 0, 0, 1, 1, 1, 1, 1, 1], use_embedding_cfg=True,
            embedding_max_length=64, embedding_features=768)


@pytest.fixture(scope="module")
def adp():
    import audio_diffusion_pytorch_b200 as adp
    from audio_diffusion_pytorch_b200 import ops
    ops.device_check()
    return adp


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


def _checked(call, model, what):
    t0 = time.perf_counter()
    with lc.Shadow() as sh:
        out = call(model).clone()
    print(f"\n{what}: {time.perf_counter() - t0:.1f} s\n{sh.table()}")
    assert sh.n_checked == sh.n_launch > 0
    return out


def _run(adp, cfg, what, call, attrs=None, compare=None):
    """call(model) under Shadow (eager); then compare(model) (default: call) under Shadow and three
    times unwrapped with the CUDA graph on (eager, capture + replay, replay)."""
    torch.manual_seed(1234)
    model = adp.DiffusionModel(net_t=adp.UNetV0, **cfg).to(DEV)
    net = model.net
    for k, v in (attrs or {}).items():
        setattr(net, k, v)
    net.use_cuda_graph = False
    try:
        with torch.no_grad():
            out = _checked(call, model, what)
            if compare is not None:
                what = what + ", one-step sample for the graph comparison"
                out = _checked(compare, model, what)
            net.use_cuda_graph = True
            net._plans.clear()
            runs = [(compare or call)(model).clone() for _ in range(3)]
            e = rel_l2(runs[2], out)
            print(f"{what}: graph replay vs checked eager run: rel-L2 {e:.3e} "
                  f"(replay vs replay {rel_l2(runs[2], runs[1]):.3e})")
            assert e <= 1e-4, f"{what}: the captured graph disagrees with the checked run ({e:.3e})"
    finally:
        del model, net
        gc.collect()
        torch.cuda.empty_cache()


def _inputs(B, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 2, T_FULL, generator=g).to(DEV), torch.rand(B, generator=g).to(DEV)


def test_cfg2_sample(adp):
    """README net, batch 8, 2^18 samples: the conditioning-table plan, the device step selector
    and two sampling steps."""
    x, _ = _inputs(8)
    _run(adp, README, "cfg2 sample(num_steps=2) B=8", lambda m: m.sample(x, num_steps=2),
         compare=lambda m: m.sample(x, num_steps=1))


def test_cfg2_v(adp):
    """README net, batch 8: one evaluation of v with its own conditioning GEMMs."""
    x, sigma = _inputs(8, 1)
    _run(adp, README, "cfg2 v B=8", lambda m: m.net(x, sigma))


def test_cfg3_sample(adp):
    """Text-conditional net, batch 16 under guidance 5 (32 trunk rows), 64 x 768 context."""
    x, _ = _inputs(16, 2)
    emb = torch.randn(16, 64, 768, generator=torch.Generator().manual_seed(3)).to(DEV)
    _run(adp, CFG3, "cfg3 sample(num_steps=2) B=16 CFG 5",
         lambda m: m.sample(x, num_steps=2, embedding=emb, embedding_scale=5.0),
         compare=lambda m: m.sample(x, num_steps=1, embedding=emb, embedding_scale=5.0))


@pytest.mark.parametrize("attrs", [{"fuse_groupnorm": True, "fuse_thin_levels": True},
                                   {"fuse_thin_levels": False}],
                         ids=["fuse_groupnorm", "unfused_thin_levels"])
def test_readme_alternative_paths(adp, attrs):
    """The optional GroupNorm-in-GEMM path and the unfused thin levels at full size."""
    x, sigma = _inputs(8, 4)
    _run(adp, README, f"README v B=8 {attrs}", lambda m: m.net(x, sigma), attrs)
