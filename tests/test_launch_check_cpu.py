"""The per-launch checker of tests/launch_check.py, without a GPU.

  * coverage: the checkers are exactly the launch kinds of the recorded inference, sampling,
    conditioning and training programs plus the generic sampler step, the resampler, the vocoder
    front-end and the VInpainter / ARVSampler steps -- every launching function of `ops` -- and
    every tensor argument of a checked kind in those programs has exactly one declared role;
  * the VInpainter and ARVSampler loops around the oracle's nets on fake kernels reproduce the
    reference's golden vectors;
  * probes: changing any input a launch reads must move its reference;
  * end to end: the tiny programs run on the CPU with fake kernels that write the checker's own
    fp64 restatement rounded to the output dtype; v must match the golden vectors made from the
    unmodified reference, which pins the restatements themselves;
  * mutations: the same programs with one launch's output damaged after the fake write must fail.
"""
import gzip
import inspect
import json
import os

import numpy as np
import pytest
import torch

import launch_check as lc
from audio_diffusion_pytorch_b200 import _lib, ops
from audio_diffusion_pytorch_b200.diffusion import VSampler
from audio_diffusion_pytorch_b200.models import DiffusionModel
from audio_diffusion_pytorch_b200.unet import UNetV0
from test_launch_programs_cpu import FIXTURE, LAUNCHES, TINY, TINY_TEXT

V_TOL, BRANCH_TOL = 1e-4, 1.2e-2


def _fixture_launches(inference_only=True):
    """Launches of the recorded programs: the inference / sampling plans ('infer_*') and the
    conditioning tables ('cond_*'), or also the training programs."""
    with gzip.open(FIXTURE, "rt") as f:
        data = json.load(f)
    for net in data.values():
        for key, case in net.items():
            if inference_only and not key.startswith(("infer_", "cond_")):
                continue
            for part in ("pre", "prog", "fwd", "bwd"):
                yield from case.get(part, [])


def test_checker_table_matches_ops():
    fns = set(lc.launching_functions())
    assert set(LAUNCHES) <= fns
    assert {"fir_resample", "mel_spectrogram", "to_flat", "to_flat_bwd", "sampler_step", "inpaint_blend",
            "arv_step"} <= fns
    recorded = {launch[0] for launch in _fixture_launches(inference_only=False)}
    assert {launch[0] for launch in _fixture_launches()} < recorded
    # outside the recorded programs: the generic VSampler step (a net that is not a B200UNet), the
    # upsampler's resampling of the clip and the vocoder front-end (host tensors, as recorded, take
    # the tensor-op route), and the VInpainter / ARVSampler steps
    assert set(lc.CHECKERS) == recorded | {"sampler_step", "fir_resample", "mel_spectrogram", "to_flat",
                                           "to_flat_bwd", "inpaint_blend", "arv_step"}
    assert set(lc.ARGS) == set(lc.CHECKERS)
    assert set(lc.UNCHECKED) == fns - set(lc.CHECKERS)
    assert not lc.UNCHECKED
    for name in lc.RESULT:          # the returned tensors' names are stored roles, not parameters
        params = set(inspect.signature(getattr(ops, name)).parameters)
        assert not lc.ARGS[name][1] & params, name


def _tensor_args(v):
    if isinstance(v, list) and v and v[0] == "T":
        return True
    return isinstance(v, list) and any(_tensor_args(x) for x in v)


def test_every_tensor_argument_is_classified():
    """Each tensor argument of a checked kind in the recorded inference and training programs is
    declared as read, stored or accumulated (statistics, fp32 / fp64 accumulators), in exactly one of the three (the declarations are enforced at run time:
    Shadow._check_roles and the probes of the program tests below)."""
    seen = {}
    for launch in _fixture_launches(inference_only=False):
        seen.setdefault(launch[0], set()).update(k for k, v in launch[1:] if _tensor_args(v))
    for name, names in seen.items():
        read, stored, acc = lc.ARGS[name]
        assert not (read & stored) and not (read & acc) and not (stored & acc), name
        params = set(inspect.signature(getattr(ops, name)).parameters)
        assert read | stored | acc <= params, f"{name}: declared roles name unknown arguments"
        unclassified = sorted(names - (read | stored | acc))
        assert not unclassified, f"{name}: arguments {unclassified} have no declared role"


# ------------------------------------------------------------------------------ programs
@pytest.fixture
def cpu_launches(monkeypatch):
    monkeypatch.setattr(ops, "device_check", lambda: None)
    monkeypatch.setattr(ops, "require_cuda", lambda x: None)

    def no_library():
        raise AssertionError("a launch reached the CUDA library")
    monkeypatch.setattr(_lib, "lib", no_library)


def _model(oracle_port, cfg):
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**cfg)
    model = DiffusionModel(net_t=UNetV0, **cfg)
    model.net.load_reference_parameters(ref.net)
    model.net.use_cuda_graph = False           # every call runs the plan's launches eagerly
    return model.net


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


def _golden(golden_dir, name):
    return {k: torch.from_numpy(np.asarray(v)) for k, v in np.load(os.path.join(golden_dir, name)).items()
            if np.asarray(v).dtype.kind != "U"}            # numbers only (some files carry a note)


def test_tiny_program_vs_golden(cpu_launches, oracle_port, golden_dir):
    g = _golden(golden_dir, "tiny_unconditional.npz")
    net = _model(oracle_port, TINY)
    with torch.no_grad(), lc.Shadow(fake=True, probe=True) as sh:
        v = net(g["x"], g["sigma"])
    print(sh.table())
    e_v, e_b = rel_l2(v, g["v"]), rel_l2(v - g["x"], g["v"] - g["x"])
    print(f"tiny: rel-L2(v) {e_v:.3e} rel-L2(branch) {e_b:.3e}")
    assert e_v <= V_TOL and e_b <= BRANCH_TOL
    assert sh.n_checked == sh.n_launch > 0


def test_tiny_sampling_program_vs_golden(cpu_launches, oracle_port, golden_dir):
    """5 VSampler steps: conditioning table, step_select, x_next in place, step_advance."""
    g = _golden(golden_dir, "tiny_unconditional.npz")
    net = _model(oracle_port, TINY)
    with torch.no_grad(), lc.Shadow(fake=True, probe=True) as sh:
        s = VSampler(net=net)(g["noise"], num_steps=5)
    print(sh.table())
    e = rel_l2(s, g["sample5"])
    print(f"tiny 5-step sample: rel-L2 {e:.3e}")
    assert e <= 5e-3                       # the GPU bound of test_net_gpu.py
    assert {"step_select", "step_advance", "stem_out"} <= {k for k, _ in sh.probed}


def test_text_cfg_program_vs_golden(cpu_launches, oracle_port, golden_dir):
    g = _golden(golden_dir, "tiny_text_cfg.npz")
    net = _model(oracle_port, TINY_TEXT)
    with torch.no_grad(), lc.Shadow(fake=True, probe=True) as sh:
        v1 = net(g["x"], g["sigma"], embedding=g["embedding"])
        v5 = net(g["x"], g["sigma"], embedding=g["embedding"], embedding_scale=5.0)
    print(sh.table())
    for v, want, v_tol, b_tol in ((v1, g["v_scale1"], V_TOL, BRANCH_TOL), (v5, g["v_scale5"], 3e-4, 3e-2)):
        e_v, e_b = rel_l2(v, want), rel_l2(v - g["x"], want - g["x"])
        print(f"text_cfg: rel-L2(v) {e_v:.3e} rel-L2(branch) {e_b:.3e}")
        assert e_v <= v_tol and e_b <= b_tol
    assert {"attention", "ln_film", "stem_out"} <= {k.split(".")[0] for k in sh.records}


def _draws_from(monkeypatch, draws):
    """torch.randn / randn_like hand out the golden run's CPU draws, in order."""
    it = iter(draws)
    monkeypatch.setattr(torch, "randn", lambda *a, **kw: next(it).to(kw.get("device", "cpu")))
    monkeypatch.setattr(torch, "randn_like", lambda t_, **kw: next(it).to(t_))
    return it


def test_inpainter_program_vs_golden(cpu_launches, oracle_port, golden_dir, monkeypatch):
    """VInpainter's generic loop (sampler_step, inpaint_blend) around the oracle's tiny net, 4 steps x
    2 resamples on fake kernels: only the fp32 rounding of the writes separates it from the golden
    run of the unmodified reference."""
    from audio_diffusion_pytorch_b200.diffusion import VInpainter
    g = _golden(golden_dir, "tiny_inpaint.npz")
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**TINY)
    source = torch.randn(2, 2, 4096, generator=torch.Generator().manual_seed(int(g["source_seed"])))
    mask = torch.zeros(2, 2, 4096, dtype=torch.bool)
    for b_, lo, hi in g["mask_spans"].tolist():
        mask[b_, :, lo:hi] = True
    steps, resamples = int(g["num_steps"]), int(g["num_resamples"])
    torch.manual_seed(int(g["rng_seed"]))
    draws = [torch.randn(2, 2, 4096) for _ in range(1 + steps * resamples)]
    left = _draws_from(monkeypatch, draws)
    with torch.no_grad(), lc.Shadow(fake=True, probe=True) as sh:
        out = VInpainter(net=ref.net)(source, mask, num_steps=steps, num_resamples=resamples)
    monkeypatch.undo()
    print(sh.table())
    e = rel_l2(out, g["out"])
    print(f"VInpainter {steps} steps x {resamples} resamples on fake kernels: rel-L2 {e:.3e}")
    assert e <= 1e-5
    assert next(left, None) is None
    assert sh.records["inpaint_blend.x"].count == sh.records["sampler_step.x_next"].count == steps * resamples
    assert {k for k, _ in sh.probed} == {"sampler_step", "inpaint_blend"}
    assert torch.equal(out[mask], source[mask])           # sigma = 0 at the end: the known region is the source


def test_autoregressive_program_vs_golden(cpu_launches, oracle_port, golden_dir, monkeypatch):
    """ARVSampler's generic loop (arv_step) around the oracle's DiffusionAR net: start window (4 steps)
    and 6 ladder passes on fake kernels, against the golden run of the unmodified reference."""
    from audio_diffusion_pytorch_b200.diffusion import ARVSampler
    g = _golden(golden_dir, "tiny_autoregressive.npz")
    cfg = dict(TINY, in_channels=2, length=4096, num_splits=4)
    torch.manual_seed(0)
    ref = oracle_port.DiffusionARPort(**cfg)
    torch.manual_seed(int(g["sample_seed"]))
    draws = [torch.randn(2, 2, 4096), torch.randn(2, 2, 4096)] + [torch.randn(2, 2, 1024) for _ in range(6)]
    left = _draws_from(monkeypatch, draws)
    sampler = ARVSampler(net=ref.net, in_channels=2, length=4096, num_splits=4)
    with torch.no_grad(), lc.Shadow(fake=True, probe=True) as sh:
        out = sampler(num_items=2, num_chunks=6, num_steps=4)
    monkeypatch.undo()
    print(sh.table())
    e = rel_l2(out, g["sample"])
    print(f"ARVSampler 6 chunks x 4 steps on fake kernels: rel-L2 {e:.3e}")
    assert out.shape == (2, 2, 6144) and e <= 1e-5
    assert next(left, None) is None
    assert sh.records["arv_step.chan"].count == sh.records["arv_step.chan.sigma"].count == 4 + 6
    assert {k for k, _ in sh.probed} == {"arv_step"}


def test_unfused_program_probes(cpu_launches, oracle_port):
    """gn_silu -> conv_gemm -> ln_film(+ statistics, + pre-norm) and the fused GroupNorm A tile."""
    torch.manual_seed(0)
    x, sigma = torch.randn(2, 2, 4096), torch.rand(2)
    for attrs, kinds in (({"fuse_thin_levels": False}, {"gn_silu", "ln_film"}),
                         ({"fuse_thin_levels": False, "fuse_groupnorm": True}, {"ln_film"})):
        net = _model(oracle_port, TINY)
        for k, v in attrs.items():
            setattr(net, k, v)
        with torch.no_grad(), lc.Shadow(fake=True, probe=True) as sh:
            net(x, sigma)
        assert kinds <= {k for k, _ in sh.probed}
        if attrs.get("fuse_groupnorm"):
            assert any(k == "conv_gemm" and "gn" in args for k, args in sh.probed)


def _direct(kind):
    """One small launch of a kind the tiny programs do not reach."""
    g = torch.Generator().manual_seed(5)
    if kind == "gn_stats":
        x = torch.randn(2, 300, 64, generator=g).to(torch.bfloat16)
        ops.gn_stats(x, torch.zeros(2, 4, 2, dtype=torch.float64), 4)
    else:
        x, v = torch.randn(2, 2, 500, generator=g), torch.randn(2, 2, 500, generator=g)
        ops.sampler_step(x, v, torch.tensor([0.8, 0.6, 0.9, 0.43589]), torch.empty_like(x))


@pytest.mark.parametrize("kind", ["gn_stats", "sampler_step"])
def test_direct_launch_probe(cpu_launches, kind):
    with lc.Shadow(fake=True, probe=True) as sh:
        _direct(kind)
    assert {k for k, _ in sh.probed} == {kind}


def test_probe_catches_an_ignored_input(cpu_launches, monkeypatch):
    """A restatement that reads a constant in place of one of its inputs must be refused."""
    real = lc.CHECKERS["sampler_step"]

    def ignores_ab(a, ctx):
        return real(dict(a, ab=torch.tensor([0.8, 0.6, 0.9, 0.43589])), ctx)
    monkeypatch.setitem(lc.CHECKERS, "sampler_step", ignores_ab)
    with lc.Shadow(fake=True, probe=True), pytest.raises(lc.CheckError, match="does not depend on `ab`"):
        _direct("sampler_step")


# ------------------------------------------------------------------------------ mutations
_V_KINDS = ("conv_gemm", "ln_film", "attention", "skinny_linear", "time_features", "silu_bf16", "stem_in",
            "stem_out", "narrow_conv", "gn_silu")
_SAMPLE_KINDS = ("step_select", "step_advance")          # reached by the sampling program
_DIRECT_KINDS = ("gn_stats", "sampler_step")             # one direct launch each
_ALL = _V_KINDS + _SAMPLE_KINDS + _DIRECT_KINDS
MUTANTS = ([("scale_largest", k) for k in _ALL if k != "gn_stats"] +
           [("stale_tile", k) for k in ("conv_gemm", "ln_film", "attention", "stem_in", "stem_out",
                                        "narrow_conv", "gn_silu", "sampler_step")] +
           [("stats_slot", k) for k in ("conv_gemm", "ln_film", "stem_in", "narrow_conv", "gn_stats")] +
           [("outside_view", k) for k in ("conv_gemm", "ln_film", "stem_in", "narrow_conv")] +
           [("readonly", k) for k in _ALL if k != "step_advance"])


@pytest.fixture(scope="module")
def tiny_nets():
    from conftest import ORACLE
    import sys
    if ORACLE not in sys.path:
        sys.path.insert(0, ORACLE)
    import reference_port
    nets = {"fused": _model(reference_port, TINY)}
    nets["unfused"] = _model(reference_port, TINY)
    nets["unfused"].fuse_thin_levels = False           # gn_silu -> conv_gemm -> ln_film at C = 32, 64
    return nets


@pytest.mark.parametrize("mutation,kind", MUTANTS, ids=[f"{m}-{k}" for m, k in MUTANTS])
def test_mutation_is_caught(cpu_launches, tiny_nets, mutation, kind):
    net = tiny_nets["unfused" if kind in ("gn_silu", "ln_film") else "fused"]
    # a fresh input per case: the plans' buffers still hold the previous case's values, and a tile
    # left stale must differ from the value it should have been given
    g = torch.Generator().manual_seed(1 + MUTANTS.index((mutation, kind)))
    x, sigma = torch.randn(2, 2, 4096, generator=g), torch.rand(2, generator=g)
    with torch.no_grad(), lc.Shadow(fake=True, mutate=(kind, lc.MUTATIONS[mutation])) as sh:
        with pytest.raises(lc.CheckError) as err:
            if kind in _DIRECT_KINDS:
                _direct(kind)
            elif kind in _SAMPLE_KINDS:
                VSampler(net=net)(x, num_steps=2)
            else:
                net(x, sigma)
    assert sh.mutate is None, f"{mutation} never applied to a {kind} launch"
    assert f"): {kind}:" in str(err.value), str(err.value)
    print(f"caught {mutation} in {kind}: {err.value}")
