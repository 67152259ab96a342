"""Every kernel launch between poisoned guard bands (`Shadow(guard=True)`, tests/launch_check.py).

Each launch runs on copies of its storages placed between 2 MiB guards, at the original address
modulo 4096, with the guards and every unviewed byte poisoned (floating storages 0x7F bytes, a
finite 3.39e38 in bf16 / fp32; integer storages zero).  A launch fails if a poisoned byte changed
(a store before the start, past the end or into a gap of an allocation), and a kernel that reads
poison shows it in the fp64 value check that follows.

  a. per-kernel: the parametrised bodies of the kernel test modules, and shapes aimed at the last
     bytes of an allocation (ragged tiles of the conv GEMM and attention, vector tails of the
     row-wise kernels, stems, thin levels, wgrad, the front-end kernels);
  b. the STFT loss, whose launches do not go through `ops`: its arguments and its scratch buffers
     between guards, the results bitwise equal to an unguarded run;
  c. whole programs: the small cases of test_lengths_gpu.py, the README net and the CFG3 sampler
     at full size, a full-size README training step, and the front-end programs of
     test_launch_check_frontends_gpu.py, through those files' own drivers.
"""
import importlib
import inspect
import itertools
import time

import pytest
import torch

import launch_check as lc

pytestmark = pytest.mark.gpu

DEV = "cuda"
KERNEL_MODULES = ["test_ops_gpu", "test_bwd_ops_gpu", "test_frontend_gpu", "test_conv_tiles_gpu", "test_head_dims_gpu"]


@pytest.fixture(scope="module")
def ops():
    from audio_diffusion_pytorch_b200 import ops
    ops.device_check()
    return ops


@pytest.fixture(scope="module")
def adp():
    import audio_diffusion_pytorch_b200 as adp
    from audio_diffusion_pytorch_b200 import ops
    ops.device_check()
    print("\n" + torch.cuda.get_device_name(0))
    return adp


def _parametrized(module):
    """(module, test name, keyword arguments) of every parameter set of module's tests that take
    no fixture but `ops`."""
    mod = importlib.import_module(module)
    out = []
    for name, fn in sorted(vars(mod).items()):
        if not name.startswith("test_") or not inspect.isfunction(fn):
            continue
        grids = []
        for mark in getattr(fn, "pytestmark", []):
            if mark.name != "parametrize":
                continue
            names = [s.strip() for s in mark.args[0].split(",")]
            grids.append([dict(zip(names, v if len(names) > 1 else (v,))) for v in mark.args[1]])
        given = {n for g in grids for n in g[0]}
        if set(inspect.signature(fn).parameters) - given - {"ops"}:
            continue                                   # needs the oracle or a whole net
        for combo in itertools.product(*grids):
            out.append((module, name, {k: v for d in combo for k, v in d.items()}))
    return out


def _run_guarded(ops, module, name, kw):
    fn = getattr(importlib.import_module(module), name)
    if "ops" in inspect.signature(fn).parameters:
        kw = dict(kw, ops=ops)
    with lc.Shadow(guard=True) as sh:
        fn(**kw)
    torch.cuda.synchronize()
    # a launch the body expects to be refused (the 256-row plan below T = 256) is neither checked nor guarded
    assert sh.n_guarded == sh.n_checked > 0, sh.table()
    return sh


def _id(case):
    module, name, kw = case
    return f"{module[5:-8]}.{name[5:]}[" + "-".join(
        str(v[0]) if isinstance(v, tuple) else str(v) for v in kw.values()) + "]"


# ------------------------------------------------------------------ a. per-kernel
KERNEL_CASES = [c for m in KERNEL_MODULES for c in _parametrized(m)]


@pytest.mark.parametrize("case", KERNEL_CASES, ids=[_id(c) for c in KERNEL_CASES])
def test_kernel_bodies_guarded(ops, case):
    _run_guarded(ops, *case)


# Shapes aimed at the last bytes of an allocation, through the kernel modules' own bodies: tails of
# 1 and 127 rows past a 128-row tile and of 129 past a 256-row tile at odd B, n_valid 8 / 24 / 40
# (padded to 16 / 32 / 48), upsample phases at ragged T, fp32 output; attention at Tq = 65 over one
# key or 65 at head dims 32, 64 and 128 (forward without lse, backward with it); row-wise kernels
# at B T C / 8 just past a multiple of a vector tile; wgrad at off = +-1; odd lengths and frame
# counts of the front-end kernels.
TAIL_CASES = (
    [("test_ops_gpu", "test_conv_gemm_linear", dict(B=B, T=T, cin=ci, n=n, res=r))
     for B, T, ci, n, r in [(3, 129, 64, 8, None), (3, 127, 64, 24, None), (3, 385, 64, 40, "residual"),
                            (5, 385, 128, 40, "inplace"), (1, 1, 64, 8, None)]] +
    [("test_ops_gpu", "test_conv_gemm_conv3", dict(B=B, T=T, C=C, co=co))
     for B, T, C, co in [(3, 383, 64, 64), (3, 385, 128, 128), (5, 129, 256, 256), (3, 127, 32, 24)]] +
    [("test_ops_gpu", "test_conv_gemm_upsample", dict(B=B, T=T, ci=ci, co=co, f=f))
     for B, T, ci, co, f in [(3, 117, 64, 32, 2), (3, 129, 32, 8, 4), (1, 65, 128, 40, 2)]] +
    [("test_conv_tiles_gpu", "test_tile_plans_agree", dict(case=c)) for c in [
        ("tail-fp32-385", "k3", 3, 385, 128, 128, 0, False, False, True),
        ("tail-k3-641", "k3", 5, 641, 256, 256, 8, True, False, False),
        ("tail-up2-129", "up2", 3, 129, 256, 128, 8, True, False, False),
        ("tail-k1-257-gate", "k1", 3, 257, 256, 512, 8, False, True, False)]] +
    [("test_head_dims_gpu", fn, dict(D=D, H=2, B=3, Tq=65, Tk=tk))
     for fn in ("test_attention_forward", "test_attention_backward") for D in (32, 64, 128) for tk in (1, 65)] +
    [("test_ops_gpu", "test_gn_silu_and_stats", dict(B=B, T=T, C=C, groups=8))
     for B, T, C in [(3, 129, 8), (3, 1025, 64), (1, 3001, 32)]] +
    [("test_ops_gpu", "test_ln_film", dict(B=B, T=T, C=C, film=film, groups=8))
     for B, T, C, film in [(3, 129, 64, True), (3, 257, 8, False)]] +
    [("test_bwd_ops_gpu", "test_wgrad", dict(B=B, T=T, n=n, k=k, off=off))
     for B, T, n, k, off in [(3, 129, 64, 64, 1), (3, 129, 64, 64, -1), (1, 65, 8, 32, 1), (3, 385, 128, 128, -1)]] +
    [("test_bwd_ops_gpu", "test_gn_silu_backward", dict(B=3, T=129, C=64, groups=8)),
     ("test_bwd_ops_gpu", "test_ln_film_backward", dict(B=3, T=129, C=64))] +
    [("test_frontend_gpu", "test_resample_kernel_and_its_adjoint", dict(factor_in=fi, factor_out=fo, t=t))
     for fi, fo, t in [(3, 2, 3001), (1, 16, 1001), (4, 1, 1001)]] +
    [("test_frontend_gpu", "test_to_flat_kernel_forward_and_gradients", dict(mel=m, win=w, hop=h, frames=fr))
     for m, w, h, fr in [(8, 64, 16, 7), (16, 256, 64, 31)]]
)


@pytest.mark.parametrize("case", TAIL_CASES, ids=[_id(c) for c in TAIL_CASES])
def test_tails_guarded(ops, case):
    _run_guarded(ops, *case)


def _rnd(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


@pytest.mark.parametrize("cx,ca,c0,f,T", [(2, 0, 8, 1, 1025), (2, 2, 8, 4, 4 * 257), (16, 0, 64, 1, 1025),
                                          (12, 4, 256, 2, 2 * 129), (32, 0, 256, 1, 257), (40, 0, 256, 1, 257)])
def test_stem_in_tail_guarded(ops, cx, ca, c0, f, T):
    """The narrow (<= 32 inputs per output position) and wide routes at T one past a tile, B = 3;
    c0 = 256 at 32 inputs per position once failed to launch (the narrow route's shared memory passed
    the 48 KiB default without the opt-in)."""
    B = 3
    with lc.Shadow(guard=True) as sh:
        ops.stem_in(_rnd(B, cx, T, seed=1), _rnd(c0, cx + ca, f, seed=2, scale=((cx + ca) * f) ** -0.5),
                    _rnd(c0, seed=3), torch.empty(B, T // f, c0, dtype=torch.bfloat16, device=DEV), f,
                    append=_rnd(B, ca, T, seed=4) if ca else None,
                    noise=_rnd(B, cx, T, seed=5), alpha=torch.rand(B, device=DEV), beta=torch.rand(B, device=DEV),
                    stats=torch.zeros(B, 8, 2, dtype=torch.float64, device=DEV), groups=8)
    assert sh.n_guarded == sh.n_launch == 1


@pytest.mark.parametrize("cx,ca,co,c0,f,T", [(2, 0, 2, 8, 1, 1025), (1, 1, 1, 32, 4, 4 * 257),
                                             (16, 0, 16, 64, 1, 1025), (12, 4, 6, 256, 2, 2 * 129)])
def test_stem_out_tail_guarded(ops, cx, ca, co, c0, f, T):
    """v, x_next and the loss outputs of the narrow and wide routes at T one past a tile, B = 3."""
    B = 3
    adapt = cx + ca != co
    x = _rnd(B, cx, T, seed=11)
    kw = dict(append=_rnd(B, ca, T, seed=12) if ca else None,
              w_adapt=_rnd(co, cx + ca, seed=13) if adapt else None, b_adapt=_rnd(co, seed=14) if adapt else None)
    args = (_rnd(B, T // f, c0, seed=15).bfloat16(), x, _rnd(co, c0, 3, seed=16, scale=(3 * c0) ** -0.5),
            _rnd(co, seed=17), _rnd(B, co, seed=18), f)
    with lc.Shadow(guard=True) as sh:
        ops.stem_out(*args, v_out=torch.empty(B, co, T, device=DEV), x_next=torch.empty(B, co, T, device=DEV),
                     ab=torch.tensor([0.8, 0.6, 0.9, 0.43589], device=DEV), **kw)
        if cx == co:                     # the v target alpha noise - beta x has the input's channels
            ops.stem_out(*args, v_out=torch.empty(B, co, T, device=DEV), noise=_rnd(B, cx, T, seed=19),
                         alpha=torch.rand(B, device=DEV), beta=torch.rand(B, device=DEV),
                         loss_sum=torch.zeros(1, dtype=torch.float64, device=DEV),
                         dv=torch.empty(B, co, T, device=DEV), **kw)
    assert sh.n_guarded == sh.n_launch == (2 if cx == co else 1)


@pytest.mark.parametrize("C,film,res,packed", [(8, False, False, False), (8, True, True, False),
                                               (32, True, True, True), (64, False, True, True), (64, True, False, False)])
def test_narrow_conv_tail_guarded(ops, C, film, res, packed):
    """The thin-level conv (narrow_conv; with host-packed weights, the mid_conv route) at T = 3001."""
    B, T, G = 3, 3001, 8
    x = (_rnd(B, T, C, seed=21) * 1.3 + 0.2).bfloat16()
    xg = x.double().reshape(B, T, G, C // G)
    stats_in = torch.stack([xg.sum(dim=(1, 3)), (xg * xg).sum(dim=(1, 3))], -1).contiguous()
    w = _rnd(C, C, 3, seed=22, scale=(3 * C) ** -0.5)
    with lc.Shadow(guard=True) as sh:
        ops.narrow_conv(x, torch.empty_like(x), stats_in, _rnd(C, seed=23) * 0.2 + 1.0, _rnd(C, seed=24) * 0.2, w,
                        _rnd(C, seed=25), G, residual=_rnd(B, T, C, seed=26).bfloat16() if res else None,
                        scale_shift=_rnd(B, 2 * C, seed=27) * 0.3 if film else None, ss_stride=2 * C,
                        stats_out=torch.zeros(B, G, 2, dtype=torch.float64, device=DEV),
                        w_packed=ops.pack_mid_conv(w) if packed else None)
    assert sh.n_guarded == sh.n_launch == 1


@pytest.mark.parametrize("n", [8 * 1024 + 8, 8 * 4096 + 1, 3 * 2 * 1001])
def test_rowwise_tail_guarded(ops, n):
    """sampler_step and silu_bf16 at element counts just past a multiple of a vector tile."""
    x, v = _rnd(n, seed=31), _rnd(n, seed=32)
    with lc.Shadow(guard=True) as sh:
        ops.sampler_step(x, v, torch.tensor([0.8, 0.6, 0.9, 0.43589], device=DEV), torch.empty_like(x))
        ops.silu_bf16(x, torch.empty(n, dtype=torch.bfloat16, device=DEV))        # fp32 in, bf16 out
    assert sh.n_guarded == sh.n_launch == 2


# ------------------------------------------------------------------ b. the STFT loss
def _stft_outputs(x):
    """acc, loss, dx and (bf16 signals) dx_bf16, as the loss's autograd function allocates them."""
    return (torch.empty(1, device=DEV, dtype=torch.float64), torch.empty((), device=DEV),
            torch.empty(x.shape, device=DEV), torch.empty_like(x) if x.dtype == torch.bfloat16 else None)


def _stft_launches(losses, x, y, res, w, go, acc, loss, dx, dx_bf16):
    """The loss's launches as its autograd function makes them: every resolution's forward, then
    every backward, dx rounded to bf16 on the last for bf16 signals."""
    scale = 1.0 / len(res)
    stats = [losses._fwd(x, y, r, w, 1e-8, scale, acc, loss, i > 0) for i, r in enumerate(res)]
    for i, (r, st) in enumerate(zip(res, stats)):
        losses._bwd(x, y, r, w, 1e-8, scale, st, go, dx, dx_bf16 if i == len(res) - 1 else None, i > 0)
    torch.cuda.synchronize()


STFT_CASES = [6, 4, 13]         # test_stft_loss_gpu.CASES rows: 441 = 3^2 7^2; 400 with silent rows, bf16; n_fft 8192


@pytest.mark.parametrize("case", STFT_CASES)
def test_stft_loss_guarded(adp, monkeypatch, case):
    import test_stft_loss_gpu as tsl
    from audio_diffusion_pytorch_b200 import losses
    res, rows, t, dtype, silent = tsl.CASES[case]
    x, y = tsl.signals(rows, t, case, dtype, silent)
    x, y = x.reshape(-1, t).contiguous(), y.reshape(-1, t).contiguous()
    w = (0.5, 2.0, 1.5)
    go = torch.ones(1, device=DEV)
    want = _stft_outputs(x)
    _stft_launches(losses, x, y, res, w, go, *want)
    g = lc.Guards()
    args = dict(zip(("acc", "loss", "dx", "dx_bf16"), _stft_outputs(x)), x=x, y=y, grad_out=go)
    r = g.relocate(args)
    monkeypatch.setattr(losses, "torch", g.torch_proxy())      # partials, stats and frame_grad between guards
    _stft_launches(losses, r["x"], r["y"], res, w, r["grad_out"], r["acc"], r["loss"], r["dx"], r["dx_bf16"])
    monkeypatch.undo()
    assert len(g.made) == 3 * len(res)

    def fail(msg):
        raise lc.CheckError(f"stft loss {res} rows {rows} T {t}: {msg}")
    g.check(fail)
    for name, a in zip(("acc", "loss", "dx", "dx_bf16"), want):
        if a is not None:
            assert torch.equal(lc._bits(r[name]), lc._bits(a)), f"{name} differs from the unguarded run"
    assert torch.equal(r["x"], x) and torch.equal(r["y"], y)


# ------------------------------------------------------------------ c. whole programs
class _GuardedShadow(lc.Shadow):
    """Shadow(guard=True), timed; every instance is kept so the test can read its counts."""
    made = []

    def __init__(self, **kw):
        super().__init__(guard=True, **kw)
        _GuardedShadow.made.append(self)

    def __enter__(self):
        self.t0 = time.perf_counter()
        return super().__enter__()

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.wall = time.perf_counter() - self.t0
        return super().__exit__(*exc)


@pytest.fixture
def guarded(monkeypatch):
    """The drivers of the other files, whose lc.Shadow() becomes Shadow(guard=True)."""
    _GuardedShadow.made = []
    monkeypatch.setattr(lc, "Shadow", _GuardedShadow)
    yield
    assert _GuardedShadow.made
    for sh in _GuardedShadow.made:
        print(f"guarded: {sh.n_guarded} of {sh.n_launch} launches, {sh.wall:.1f} s")
        assert sh.n_guarded == sh.n_checked == sh.n_launch > 0, sh.table()


def _small_cases():
    import test_lengths_gpu as tlg
    return tlg.SMALL


@pytest.mark.parametrize("case", _small_cases(), ids=lambda c: "-".join(map(str, c)))
def test_small_programs_guarded(adp, guarded, case):
    import test_lengths_gpu as tlg
    tlg.test_small_under_launch_checker(adp, case)


def test_full_size_readme_v_guarded(adp, guarded):
    import test_lengths_gpu as tlg
    tlg.test_full_size_readme_v(adp)


def test_full_size_cfg3_sample_guarded(adp, guarded):
    import test_lengths_gpu as tlg
    tlg.test_full_size_cfg3_sample(adp)


def test_full_size_readme_training_step_guarded(adp, guarded):
    """One README training step (fused v loss, backward) at B = 3, T = 239616."""
    import test_lengths_gpu as tlg
    tlg._room(16)
    torch.manual_seed(1234)
    model = adp.DiffusionModel(net_t=adp.UNetV0, **tlg.README).to(DEV)
    audio = torch.randn(3, 2, tlg.T_FULL, generator=torch.Generator().manual_seed(0)).to(DEV)

    def step():
        model.zero_grad(set_to_none=True)
        torch.manual_seed(77)
        loss = model(audio)
        loss.backward()
        return loss.detach().clone(), [p.grad.clone() for p in model.parameters()]
    try:
        sh = tlg._step_and_compare(model, step, f"README training step B=3 T={tlg.T_FULL}")
        assert any(lab.startswith("wgrad[M=") and f"M={3 * 3744} " in lab for lab in sh.labels)
    finally:
        tlg._free(model)


@pytest.mark.parametrize("program", ["test_cfg5_sample", "test_vocoder_training_step", "test_inpainter_readme",
                                     "test_autoregressive_readme"])
def test_frontend_programs_guarded(adp, guarded, program):
    import test_launch_check_frontends_gpu as tfe
    getattr(tfe, program)(adp)
