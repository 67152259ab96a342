"""The per-launch checker of tests/launch_check.py in the fp32 verification mode, without a GPU.

  * coverage: every launch kind of the recorded fp32 inference, sampling and training programs has
    a checker, and every tensor argument of those launches has exactly one declared role;
  * end to end: the tiny fp32 programs (v, the text net at CFG 5, a 5-step sample, a training step)
    run on fake kernels that write the checker's fp64 restatement rounded to fp32; they must meet
    the float64 oracle at fp32 round-off, which pins the fp32 restatements themselves;
  * probes on every fp32 kind those programs reach, and f32_conv_gemm's residual is read;
  * mutations: the classes of test_launch_check_cpu.py caught in the fp32 mode -- acc_stored on
    direct launches into accumulators that hold values before the launch (a training step's gradient
    arena starts at zero), as is silu's 2^-12 case (the tiny programs do not reach silu) -- and a 2^-12 relative
    change of the largest element caught on every fp32 kind whose chain is at most 256 long.  The
    long-chain reductions (wgrad, colsum, stem_in_bwd: chains of B T terms) catch, at the largest
    element of the 2 x 1024 tiny training step, a relative change of 2^-5 (what the checker's
    acc_lost_split mutation applies); `test_long_chain_resolution` prints the smallest relative
    change their bound catches there and requires it to be at most 2^-9.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import launch_check as lc
from audio_diffusion_pytorch_b200 import _lib, ops, training
from audio_diffusion_pytorch_b200.diffusion import VSampler
from audio_diffusion_pytorch_b200.models import DiffusionModel
from audio_diffusion_pytorch_b200.unet import UNetV0
from test_launch_programs_cpu import NETS, TINY, TINY_TEXT, build_net, install
from test_train_fp32_cpu import record_train

F64 = torch.float64
BRANCH_TOL = 1e-5              # fake fp32 writes: the rounding of each stored value only
SAMPLE_TOL = 1e-5
LOSS_TOL, GRAD_TOL = 1e-5, 1e-4


@pytest.fixture
def cpu_launches(monkeypatch):
    monkeypatch.setattr(ops, "device_check", lambda: None)
    monkeypatch.setattr(ops, "require_cuda", lambda x: None)

    def no_library():
        raise AssertionError("a launch reached the CUDA library")
    monkeypatch.setattr(_lib, "lib", no_library)


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ------------------------------------------------------------------------------ coverage
def _recorded_fp32():
    """(kind, recorded launch) of the fp32 programs of the tiny configs: inference, sampling with its
    conditioning table, and training in every mode the configs train in."""
    mp = pytest.MonkeyPatch()
    rec = install(mp)
    out = []
    try:
        for name in ("tiny", "text_cfg", "skipcat_adapter", "append", "head32_g4", "head128_g4"):
            kw, attrs, B, T, M, modes, trains = NETS[name]
            net = build_net(kw, attrs)
            net.verify_fp32 = True
            for m in modes:
                cfg = m.endswith("_cfg")
                plan = net._plan(B, T, 2 * B if cfg else B, M, m[:-4] if cfg else m, (5.0 if cfg else None, False))
                plan.cfg_scale = 5.0 if cfg else None
                for fn in getattr(plan, "pre", []):
                    fn()
                plan.run_eager()
                out += rec.take()
            if net.use_modulation:
                net._cond_table(torch.zeros(6), None)
                out += rec.take()
            for mode, want_dxin in trains:
                _, fwd, bwd, _ = record_train(net, rec, B, T, M, mode, want_dxin)
                out += fwd + bwd
    finally:
        mp.undo()
    return out


def _tensor_args(v):
    if isinstance(v, list) and v and v[0] == "T":
        return True
    return isinstance(v, list) and any(_tensor_args(x) for x in v)


def test_fp32_programs_are_covered_and_classified():
    launches = _recorded_fp32()
    kinds = {launch[0] for launch in launches}
    assert kinds <= set(lc.CHECKERS), sorted(kinds - set(lc.CHECKERS))
    # the fp32 routes these programs take (narrow_conv / narrow_conv_bwd run unfused in the fp32 mode)
    assert {"conv_gemm", "gn_silu", "ln_film", "attention", "skinny_linear", "stem_in", "stem_out", "wgrad",
            "gn_silu_bwd", "gn_bwd_apply", "ln_film_bwd", "colsum", "skip_gate_bwd", "cond_bwd", "stem_out_bwd",
            "stem_in_bwd", "attention_bwd"} <= kinds
    assert not {"narrow_conv", "narrow_conv_bwd"} & kinds
    seen = {}
    for launch in launches:
        for k, v in launch[1:]:
            if isinstance(v, list) and v and v[0] == "T":
                assert v[5] != "bfloat16", f"{launch[0]}: `{k}` is bf16 in the fp32 mode"
        seen.setdefault(launch[0], set()).update(k for k, v in launch[1:] if _tensor_args(v))
    for name, names in seen.items():
        read, stored, acc = lc.ARGS[name]
        assert not (read & stored) and not (read & acc) and not (stored & acc), name
        unclassified = sorted(names - (read | stored | acc))
        assert not unclassified, f"{name}: arguments {unclassified} have no declared role"


# ------------------------------------------------------------------------------ programs
def _pair(oracle_port, cfg):
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**cfg)
    model = DiffusionModel(net_t=UNetV0, **cfg)
    model.net.load_reference_parameters(ref.net)
    model.net.verify_fp32 = True
    model.net.use_cuda_graph = False           # every call runs the plan's launches eagerly
    ref.double()
    return ref, model.net


def _inputs(seed, B=2, T=4096, C=2):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, C, T, generator=g), torch.randn(B, C, T, generator=g), torch.rand(B, generator=g)


def _f32_kinds(sh):
    return {k for k, _ in sh.probed}


def test_tiny_v_fp32(cpu_launches, oracle_port):
    ref, net = _pair(oracle_port, TINY)
    x, _, sigma = _inputs(1)
    with torch.no_grad(), lc.Shadow(fake=True, probe=True) as sh:
        v = net(x, sigma)
    want = ref.net(x.double(), sigma.double())
    print(sh.table())
    e = rel_l2(v - x, want - x.double())
    print(f"tiny fp32 v on fake kernels: branch rel-L2 {e:.3e}")
    assert e <= BRANCH_TOL
    assert sh.n_checked == sh.n_launch > 0
    assert {"conv_gemm", "gn_silu", "ln_film", "attention", "skinny_linear", "stem_in", "stem_out"} <= _f32_kinds(sh)


def test_text_cfg5_fp32(cpu_launches, oracle_port):
    ref, net = _pair(oracle_port, TINY_TEXT)
    x, _, sigma = _inputs(2)
    emb = torch.randn(2, 8, 32, generator=torch.Generator().manual_seed(3))
    with torch.no_grad(), lc.Shadow(fake=True, probe=True) as sh:
        v = net(x, sigma, embedding=emb, embedding_scale=5.0)
    want = ref.net(x.double(), sigma.double(), embedding=emb.double(), embedding_scale=5.0)
    e = rel_l2(v - x, want - x.double())
    print(f"text net fp32 CFG 5 on fake kernels: branch rel-L2 {e:.3e}")
    assert e <= BRANCH_TOL * (5 + 4)             # guidance s: (|s| + |1 - s|) times the bound
    assert sh.n_checked == sh.n_launch > 0


def test_tiny_sample_fp32(cpu_launches, oracle_port):
    ref, net = _pair(oracle_port, TINY)
    noise, _, _ = _inputs(4)
    with torch.no_grad(), lc.Shadow(fake=True, probe=True) as sh:
        s = VSampler(net=net)(noise, num_steps=5)
    want = ref.sample(noise.double(), num_steps=5)
    e = rel_l2(s, want)
    print(f"tiny fp32 5-step sample on fake kernels: rel-L2 {e:.3e}")
    assert e <= SAMPLE_TOL
    assert {"step_select", "step_advance", "stem_out"} <= _f32_kinds(sh)


def test_tiny_training_step_fp32(cpu_launches, oracle_port):
    ref, net = _pair(oracle_port, TINY)
    x, noise, sigma = _inputs(5, T=1024)
    a, b = torch.cos(sigma * math.pi / 2)[:, None, None], torch.sin(sigma * math.pi / 2)[:, None, None]
    x64, n64, a64, b64 = x.double(), noise.double(), a.double(), b.double()
    loss_ref = F.mse_loss(ref.net(a64 * x64 + b64 * n64, sigma.double()), a64 * n64 - b64 * x64)
    loss_ref.backward()
    with lc.Shadow(fake=True, probe=True) as sh:
        loss = training.fused_v_loss(net, x, noise, sigma)
        loss.backward()
    assert sh.n_checked == sh.n_launch > 0
    rel = abs(float(loss) - float(loss_ref)) / float(loss_ref)
    worst = max((rel_l2(p.grad, q.grad), n) for (n, q), p in zip(ref.net.named_parameters(), net.parameters())
                if q.grad is not None and float(q.grad.norm()) > 1e-6 * float(loss_ref))
    print(f"tiny fp32 training step on fake kernels: loss rel {rel:.2e}, worst gradient rel-L2 {worst[0]:.2e} "
          f"({worst[1]})")
    assert rel <= LOSS_TOL and worst[0] <= GRAD_TOL
    assert {"wgrad", "gn_silu_bwd", "gn_bwd_apply", "ln_film_bwd", "colsum", "cond_bwd", "stem_out_bwd",
            "stem_in_bwd", "attention_bwd"} <= _f32_kinds(sh)


# ------------------------------------------------------------------------------ probes
def test_f32_conv_gemm_reads_its_residual(cpu_launches):
    """f32_conv_gemm adds the residual (verify_f32.cu): the probe must demand it, while the
    tensor-core kernel's fp32 epilogue (bf16 operands, no residual) stays exempt."""
    g = torch.Generator().manual_seed(9)
    a = torch.randn(2, 40, 16, generator=g)
    w = torch.randn(16, 48, generator=g)
    out = torch.randn(2, 40, 16, generator=g)
    with lc.Shadow(fake=True, probe=True) as sh:
        ops.conv_gemm(a, w, out, c_in=16, n_valid=16, taps=(-1, 0, 1), residual=out)
    assert ("conv_gemm", frozenset({"a", "w", "out", "residual"})) in sh.probed
    assert "residual" not in lc.NOT_READ["conv_gemm"]({"a": a, "out": out})
    assert "residual" in lc.NOT_READ["conv_gemm"]({"a": a.bfloat16(), "out": out})

    def ignores_residual(args, ctx):
        return real(dict(args, residual=None), ctx)
    real = lc.CHECKERS["conv_gemm"]
    mp = pytest.MonkeyPatch()
    mp.setitem(lc.CHECKERS, "conv_gemm", ignores_residual)
    try:
        with lc.Shadow(fake=True, probe=True), pytest.raises(lc.CheckError, match="does not depend on `residual`"):
            ops.conv_gemm(a, w, out, c_in=16, n_valid=16, taps=(-1, 0, 1), residual=out)
    finally:
        mp.undo()


def test_nested_statistics_launch_is_part_of_its_caller(cpu_launches, monkeypatch):
    """In the fp32 mode conv_gemm(stats=) launches gn_stats from inside ops: one checked launch,
    labelled by the caller, its statistics checked as the caller's `stats` output."""
    calls = []

    class Lib:
        def __getattr__(self, sym):
            def fn(*a):
                calls.append(sym)
                return 0
            return fn
    monkeypatch.setattr(_lib, "lib", lambda: Lib())
    monkeypatch.setattr(_lib, "check", lambda rc, what: None)
    monkeypatch.setattr(ops, "_stream", lambda: None)
    g = torch.Generator().manual_seed(3)
    a, w = torch.randn(1, 8, 16, generator=g), torch.randn(16, 16, generator=g)
    out = torch.zeros(1, 8, 16)
    stats = torch.zeros(1, 8, 2, dtype=F64)
    sh = lc.Shadow()
    sh._check = lambda *args: None           # no kernel ran: nothing to compare, only the bookkeeping
    with sh:
        ops.conv_gemm(a, w, out, c_in=16, n_valid=16, stats=stats)
    assert calls == ["adp_f32_conv_gemm", "adp_f32_gn_stats"]
    assert sh.n_launch == sh.n_checked == 1
    assert sh.symbols == {"adp_f32_conv_gemm", "adp_f32_gn_stats"}
    assert all(lab.startswith("conv_gemm[") for lab in sh.labels), sh.labels      # not f32_gn_stats[


# ------------------------------------------------------------------------------ mutations
_INFER = ("conv_gemm", "gn_silu", "ln_film", "attention", "skinny_linear", "stem_in", "stem_out")
_TRAIN = ("skip_gate", "gn_silu_bwd", "gn_bwd_apply", "ln_film_bwd", "skip_gate_bwd", "cond_bwd", "stem_out_bwd",
          "attention_bwd")             # skip_gate: the training forward keeps y_up, so the merge is its own pass
_LONG = ("wgrad", "colsum", "stem_in_bwd")          # accumulators over B T terms only
MUTANTS = ([("scale_largest", k) for k in _INFER + _TRAIN] +
           [("scale_largest_f32", k) for k in _INFER + _TRAIN] +
           [("stale_tile", k) for k in ("conv_gemm", "ln_film", "attention", "stem_in", "gn_silu", "gn_silu_bwd")] +
           [("stats_slot", k) for k in ("conv_gemm", "stem_in")] +
           [("outside_view", k) for k in ("conv_gemm", "ln_film", "stem_in", "wgrad")] +
           [("readonly", k) for k in _INFER + _TRAIN + _LONG] +
           [("acc_lost_split", k) for k in _LONG + ("gn_silu_bwd", "ln_film_bwd", "stem_out_bwd")])


@pytest.fixture(scope="module")
def tiny_fp32():
    from conftest import ORACLE
    import sys
    if ORACLE not in sys.path:
        sys.path.insert(0, ORACLE)
    import reference_port
    return _pair(reference_port, TINY)[1]


@pytest.mark.parametrize("mutation,kind", MUTANTS, ids=[f"{m}-{k}" for m, k in MUTANTS])
def test_fp32_mutation_is_caught(cpu_launches, tiny_fp32, mutation, kind):
    net = tiny_fp32
    x, noise, sigma = _inputs(20 + MUTANTS.index((mutation, kind)), T=1024)
    with lc.Shadow(fake=True, mutate=(kind, lc.MUTATIONS[mutation])) as sh:
        with pytest.raises(lc.CheckError) as err:
            if kind in _TRAIN + _LONG:
                training.fused_v_loss(net, x, noise, sigma).backward()
            else:
                with torch.no_grad():
                    net(x, sigma)
    assert sh.mutate is None, f"{mutation} never applied to a {kind} launch"
    assert f"): {kind}:" in str(err.value), str(err.value)
    print(f"caught {mutation} in {kind}: {err.value}")


def test_long_chain_resolution(cpu_launches, tiny_fp32):
    """The smallest relative change of the largest element that the bound of each long-chain
    reduction catches in the tiny training step (2 x 1024): bound / |ref| there."""
    net = tiny_fp32
    x, noise, sigma = _inputs(7, T=1024)
    seen = {}
    real = {k: lc.CHECKERS[k] for k in _LONG}

    def spy(kind):
        def checker(a, ctx):
            outs = real[kind](a, ctx)
            o = outs[0]
            ref, absr = (o.ref, o.absref) if not callable(o.ref) else o.ref(a)
            i = int(ref.abs().reshape(-1).argmax())
            r, ab = float(ref.reshape(-1)[i]), float(absr.reshape(-1)[i])
            bound = lc.F32_REL * abs(r) + lc.F32_LAMBDA * math.sqrt(o.chain) * lc.F32_U * ab
            seen[kind] = max(seen.get(kind, 0.0), bound / abs(r))
            return outs
        return checker
    mp = pytest.MonkeyPatch()
    for k in _LONG:
        mp.setitem(lc.CHECKERS, k, spy(k))
    try:
        with lc.Shadow(fake=True):
            training.fused_v_loss(net, x, noise, sigma).backward()
    finally:
        mp.undo()
    for k, r in sorted(seen.items()):
        print(f"{k}: smallest caught relative change of the largest element 2^{math.log2(r):.1f}")
    assert set(seen) == set(_LONG)
    assert max(seen.values()) <= 2.0 ** -9


# -------------------------------------------------- direct launches into non-zero accumulators
def _direct(kind, seed=13):
    """One small fp32 launch of `kind`, every accumulator holding values before it."""
    g = torch.Generator().manual_seed(seed)

    def n(*shape):
        return torch.randn(*shape, generator=g)
    B, T, C = 2, 24, 16
    if kind == "wgrad":
        ops.wgrad(n(B, T, C), n(B, T, C), n(3, C, C), n=C, k=C, off=-1, ntaps=3)
    elif kind == "colsum":
        ops.colsum(n(B, T, C), n(C), gate=n(B, 2 * C)[:, :C])
    elif kind == "gn_silu_bwd":
        x = n(B, T, C)
        ops.gn_silu_bwd(n(B, T, C), x, lc.stats_of(x, 4), n(C), n(C), torch.empty_like(x), n(C), n(C),
                        n(B, 4, 2).double(), 4)
    elif kind == "ln_film_bwd":
        x = n(B, T, C)
        ops.ln_film_bwd(n(B, T, C), x, n(B, 2 * C), 2 * C, torch.empty_like(x), dss=n(B, 2 * C), dss_stride=2 * C,
                        colsum=n(C))
    elif kind == "skip_gate_bwd":
        y = n(B, T, C)
        ops.skip_gate_bwd(n(B, T, C), y, n(B, C), torch.empty_like(y), n(B, C))
    elif kind == "cond_bwd":
        ops.cond_bwd(n(B, 32), n(B, 8), n(32, 8), torch.empty(32, 8), torch.empty(32), n(B, 8), 32)
    elif kind == "stem_in_bwd":
        ops.stem_in_bwd(n(B, T // 4, 8), n(B, 2, T), n(8, 2, 4), n(8), 4, w=n(8, 2, 4), dxin=n(B, 2, T))
    elif kind == "stem_out_bwd":
        ops.stem_out_bwd(n(B, 2, T), n(B, T // 2, 8), n(B, 2, T), n(2, 8, 3), n(2), n(B, 2), 2,
                         torch.empty(B, T // 2, 8), n(2, 8, 3), n(2), n(B, 2))
    elif kind == "silu_bf16":
        ops.silu_bf16(n(3, 40), torch.empty(3, 40))


DIRECT_MUTANTS = ([("acc_stored", k) for k in ("wgrad", "colsum", "gn_silu_bwd", "ln_film_bwd", "skip_gate_bwd",
                                                "cond_bwd", "stem_in_bwd", "stem_out_bwd")] +
                  [("scale_largest_f32", "silu_bf16"), ("scale_largest", "silu_bf16"), ("readonly", "silu_bf16")])


@pytest.mark.parametrize("mutation,kind", DIRECT_MUTANTS, ids=[f"{m}-{k}" for m, k in DIRECT_MUTANTS])
def test_fp32_direct_mutation_is_caught(cpu_launches, mutation, kind):
    with lc.Shadow(fake=True, probe=True) as sh:
        _direct(kind)                          # the unmutated launch passes, probes included
    assert sh.n_checked == sh.n_launch == 1
    with lc.Shadow(fake=True, mutate=(kind, lc.MUTATIONS[mutation])) as sh:
        with pytest.raises(lc.CheckError) as err:
            _direct(kind)
    assert sh.mutate is None, f"{mutation} never applied to a {kind} launch"
    assert f"): {kind}:" in str(err.value), str(err.value)


def test_only_the_statistics_pass_may_nest(cpu_launches, monkeypatch):
    """A launch of any other kind inside a checked ops call fails the caller."""
    class Lib:
        def __getattr__(self, sym):
            return lambda *a: 0
    monkeypatch.setattr(_lib, "lib", lambda: Lib())
    monkeypatch.setattr(_lib, "check", lambda rc, what: None)
    monkeypatch.setattr(ops, "_stream", lambda: None)
    monkeypatch.setattr(ops, "gn_stats", lambda x, stats, groups: ops.silu_bf16(x, x))
    g = torch.Generator().manual_seed(3)
    a, w = torch.randn(1, 8, 16, generator=g), torch.randn(16, 16, generator=g)
    sh = lc.Shadow()
    sh._check = lambda *args: None
    with sh, pytest.raises(lc.CheckError, match="adp_f32_silu"):
        ops.conv_gemm(a, w, torch.zeros(1, 8, 16), c_in=16, n_valid=16, stats=torch.zeros(1, 8, 2, dtype=F64))
