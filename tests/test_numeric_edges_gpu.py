"""Numerical edges on the bf16 path: inputs that real audio makes and randn-scaled data never does.

The launch checker (tests/launch_check.py) holds every launch to an fp64 restatement, but only on
well-conditioned activations.  Here the same checks run on the inputs where single-pass fp32
arithmetic is fragile:

  a. GroupNorm statistics, launch by launch: every bf16 statistics producer (gn_stats; conv_gemm on
     the 128- and 256-row tile plans, the narrow-group path at group sizes 1, 2 and 4, a deep level
     and an upsample phase; ln_film, stem_in, skip_gate and narrow_conv) writes groups with a chosen
     mean / std ratio R (0, 10, 100, 256, -256), an exactly constant group, an all-zero group and a
     tiny one (std 1e-4, var << eps), at B = 1 and T = 2^18 (the longest accumulation chains).
     Each runs under Shadow(probe=True) and Shadow(guard=True): the statistics meet STATS_TOL /
     VAR_TOL.  Each producer's statistics then feed a consumer (gn_silu, the conv GEMM's fused
     GroupNorm A transform, narrow_conv), whose output is compared with fp64 GroupNorm from a
     two-pass fp64 variance of the same bf16 input -- not from the kernel's statistics, which the
     launch checker's consumer checks start from and so cannot see a statistics error.  A second
     layout with every group at R = 1000 runs unchecked: its variance error is measured and printed.
  b. LayerNorm rows (ln_film: plain, FiLM, FiLM + y2) at C = 8 .. 2048 over the same R sweep; a
     constant row gives y = shift.
  c. attention and attention_bwd at the logit edges: a row maximum 40 or 80 above every earlier
     logit arriving in the last (ragged) key tile, all-equal logits, one key dominant by 30 among
     10^4, logits up to +-60 throughout; o, lse, dq, dk, dv against fp64 softmax.
  d. whole programs on audio at the edge (silence, a DC offset, a full-scale square wave, noise at
     1e-4): v at sigma 0, 1e-4, 0.5 and 1, a 3-step sample and one fused-loss training step with
     sigma 0 and 1, every launch under the checker, against the oracle in fp64, and the fp32
     verification mode (STORAGE_LIMITED and FP32_LIMITED name the cases that bf16, or fp32
     arithmetic itself, cannot carry).

tests/test_numeric_edges_cpu.py shows, without a GPU, that the checks of a and c fail on a
single-pass fp32 statistic and on an online softmax without its rescale.  Run with -s for the
statistics table (err/bound and var_rel per producer and group) and the per-case errors; DESIGN.md
quotes the H100 numbers."""
import inspect
import math
import time

import numpy as np
import pytest
import torch

import launch_check as lc
from audio_diffusion_pytorch_b200 import ops

pytestmark = pytest.mark.gpu

DEV = "cuda"
F64 = torch.float64
T_LONG = 1 << 18
G = 8
# one group each: R = |mean| / std; every group of this layout is held to the checker's bounds
KINDS = ["R0", "R10", "R100", "R256", "const", "zero", "tiny", "R256-"]
KINDS_1000 = ["R1000", "R1000-"] * 4              # measured and printed, no bound
CONST = 3.3                                       # the constant group's value (bf16 3.296875)
SIGS = {n: inspect.signature(getattr(ops, n)) for n in ("gn_silu", "conv_gemm", "narrow_conv")}
TABLE = []                                        # (producer, group kind, R, stats, var, var_rel, consumers)


# ------------------------------------------------------------------ group construction
def target(kind, g):
    """(mean, std) of group g of the given kind; std varies over 0.5, 1, 2 from group to group."""
    s = 2.0 ** (g % 3 - 1)
    if kind == "const":
        return CONST, 0.0
    if kind == "zero":
        return 0.0, 0.0
    if kind == "tiny":
        return 0.0, 1e-4
    r = float(kind[1:].rstrip("-"))
    return (-r if kind.endswith("-") else r) * s, s


def channel_targets(kinds, C):
    """(mu, sd) fp64 [C]: channel c takes its group's target (G groups of C / G channels)."""
    t = torch.tensor([target(k, g) for g, k in enumerate(kinds)], dtype=F64)
    rep = C // len(kinds)
    return t[:, 0].repeat_interleave(rep), t[:, 1].repeat_interleave(rep)


def _rnd(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g, dtype=F64) * scale


def _rows(n, k, seed, sd):
    """Weights [n, k] whose row c has L2 norm sd[c]: over unit-variance independent inputs,
    output channel c has std sd[c]."""
    w = _rnd(n, k, seed=seed)
    return w / w.norm(dim=1, keepdim=True) * sd[:, None]


def group_moments(y, groups):
    """Two-pass fp64 (mean, var) [B, groups] of a channels-last tensor."""
    B, T, C = y.shape
    yg = y.to(F64).reshape(B, T, groups, C // groups)
    mean = yg.mean(dim=(1, 3))
    var = ((yg - mean[:, None, :, None]) ** 2).mean(dim=(1, 3))
    return mean, var


def ideal_slots(y, groups):
    """The (sum, sumsq) slots of y [B, T, C] from a two-pass fp64 variance: GroupNorm from these is
    the exact GroupNorm of the stored tensor."""
    B, T, C = y.shape
    n = T * (C // groups)
    mean, var = group_moments(y, groups)
    return torch.stack([mean * n, (var + mean * mean) * n], dim=-1)


def fp32_sequential_slots(y, groups):
    """(sum, sumsq) of each group as ONE single-pass fp32 running sum over the whole group, in
    (t, c) order (numpy's add.accumulate rounds every partial sum to fp32)."""
    B, T, C = y.shape
    yg = y.float().reshape(B, T, groups, C // groups).permute(0, 2, 1, 3).reshape(B, groups, -1).cpu().numpy()
    out = np.zeros((B, groups, 2))
    for b in range(B):
        for g in range(groups):
            v = yg[b, g]
            out[b, g] = np.add.accumulate(v)[-1], np.add.accumulate(v * v)[-1]
    return torch.from_numpy(out).to(y.device)


def m_fp32_sequential(post, outs, pre):
    """The statistics slots replaced by a single-pass fp32 sequential sum over the whole group."""
    o = next((o for o in outs if isinstance(o, lc.Stat)), None)
    if o is None:
        return False
    o.view(post).copy_(o.view(pre) + fp32_sequential_slots(o.src(post), o.groups))


# ------------------------------------------------------------------ statistics: producer side
def producer_report(stats, y, groups):
    """Per group: (R, stats err/bound, variance err/bound, var_rel) as the launch checker measures
    them (STATS_TOL of sum|x| and sum x^2; VAR_TOL (var + eps) of the two-pass variance)."""
    B, T, C = y.shape
    yg = y.to(F64).reshape(B, T, groups, C // groups)
    ref = lc.stats_of(y, groups)
    scale = torch.stack([yg.abs().sum(dim=(1, 3)), (yg * yg).sum(dim=(1, 3))], dim=-1)
    err = (stats.to(F64) - ref).abs()
    sr = torch.where(scale > 0, err / (lc.STATS_TOL * scale).clamp_min(1e-300),
                     torch.where(err > 0, math.inf, 0.0)).amax(-1)
    n = float(T * (C // groups))
    mean = stats[..., 0].to(F64) / n
    var = stats[..., 1].to(F64) / n - mean * mean
    mu, var2 = group_moments(y, groups)
    vr = (var - var2).abs() / (lc.VAR_TOL * (var2 + lc.GN_EPS))
    rel = (var - var2).abs() / var2.clamp_min(1e-300)
    R = mu.abs() / var2.sqrt()
    return R.cpu(), sr.cpu(), vr.cpu(), rel.cpu()


# ------------------------------------------------------------------ statistics: consumer side
def _bind(kind, *args, **kw):
    b = SIGS[kind].bind(*args, **kw)
    b.apply_defaults()
    return dict(b.arguments)


def consumer_ratio(kind, a, groups_of_out=None):
    """err / bound of a consumer's stored output against fp64 GroupNorm from a two-pass fp64
    variance of its bf16 input (the statistics it was given replaced by ideal_slots), at the
    launch checker's bf16 bound.  Per output group when groups_of_out is given, else [1]."""
    a2 = dict(a)
    if kind == "conv_gemm":
        st, gg, gb, gG, geps = a["gn"]
        a2["gn"] = (ideal_slots(a["a"][..., :a["c_in"]], gG), gg, gb, gG, geps)
    elif kind == "gn_silu":
        a2["stats"] = ideal_slots(a["x"], a["groups"])
    else:
        a2["stats_in"] = ideal_slots(a["x"], a["groups"])
    o = next(o for o in lc.CHECKERS[kind](a2, None) if isinstance(o, lc.Val))
    got = o.view(a).to(F64)
    err = (got - o.ref).abs()
    bound = lc.BF16_REL * o.ref.abs() + o.tau * o.absref
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    ratio = torch.where(torch.isfinite(got), ratio, math.inf)
    if groups_of_out is None:
        return ratio.amax().reshape(1).cpu()
    B, T, C = ratio.shape
    return ratio.reshape(B, T, groups_of_out, C // groups_of_out).amax(dim=(1, 3)).cpu()


def _gn_params(C, seed):
    return ((1.0 + 0.2 * _rnd(C, seed=seed)).float().to(_dev()), (0.3 * _rnd(C, seed=seed + 1)).float().to(_dev()))


_DEVICE = [DEV]


def _dev():
    return _DEVICE[0]


def cons_gn_silu(y, stats, groups):
    gamma, beta = _gn_params(y.shape[-1], 101)
    out = torch.empty_like(y)
    ops.gn_silu(y, out, stats, gamma, beta, groups)
    return "gn_silu", _bind("gn_silu", y, out, stats, gamma, beta, groups), groups


def cons_conv_xf(y, stats, groups):
    """The conv GEMM with GroupNorm + SiLU fused into its A operand (c_in = the producer's width)."""
    B, T, C = y.shape
    n = 64
    w = ops.pack_conv(_rnd(n, C, 3, seed=111, scale=(3 * C) ** -0.5).to(torch.bfloat16).to(_dev()))
    gamma, beta = _gn_params(C, 112)
    out = torch.empty(B, T, n, dtype=torch.bfloat16, device=_dev())
    kw = dict(c_in=C, n_valid=n, taps=(-1, 0, 1), bias=(0.1 * _rnd(n, seed=113)).float().to(_dev()),
              gn=(stats, gamma, beta, groups, 1e-5))
    ops.conv_gemm(y, w, out, **kw)
    return "conv_gemm", _bind("conv_gemm", y, w, out, **kw), None


def cons_narrow(y, stats, groups):
    """narrow_conv (C = 8: stem.cu's ConvBlock; 32 / 64: mid_conv with host-packed weights)."""
    C = y.shape[-1]
    gamma, beta = _gn_params(C, 121)
    w = _rnd(C, C, 3, seed=122, scale=(3 * C) ** -0.5).float().to(_dev())
    out = torch.empty_like(y)
    kw = dict(w_packed=ops.pack_mid_conv(w) if C > 8 else None)
    bias = (0.1 * _rnd(C, seed=123)).float().to(_dev())
    ops.narrow_conv(y, out, stats, gamma, beta, w, bias, groups, **kw)
    return "narrow_conv", _bind("narrow_conv", y, out, stats, gamma, beta, w, bias, groups, **kw), None


# ------------------------------------------------------------------ statistics producers
def _debug_set(key, value):
    from audio_diffusion_pytorch_b200 import _lib
    _lib.check(_lib.lib().adp_debug_set(key, value), "adp_debug_set")


def _stats():
    return torch.zeros(1, G, 2, dtype=F64, device=_dev())


def p_gn_stats(kinds, T):
    C = 256
    mu, sd = channel_targets(kinds, C)
    x = (mu + sd * _rnd(1, T, C, seed=1)).to(torch.bfloat16).to(_dev())
    st = _stats()
    return (lambda: ops.gn_stats(x, st, G)), x, st, [cons_gn_silu]


def p_conv(kinds, T, c_in, n, kind="k3", plan=0, block_n=0):
    """out = conv(a, w) + bias: w's rows scaled by each channel's std, the bias its mean."""
    mu, sd = channel_targets(kinds, n)
    a = _rnd(1, T, c_in, seed=2).to(torch.bfloat16).to(_dev())
    up = int(kind[2:]) if kind.startswith("up") else 0
    taps = 3 if kind != "k1" else 1
    w = _rows(n, c_in * taps, 3, sd).reshape(n, c_in, taps).to(torch.bfloat16).to(_dev())
    wp = ops.pack_upsample_conv(w, up) if up else ops.pack_conv(w)
    phases = up or 1
    out = torch.empty(1, T * phases, n, dtype=torch.bfloat16, device=_dev())
    st = _stats()
    kw = dict(c_in=c_in, n_valid=n, taps=(-1, 0, 1) if kind == "k3" else (0,), up_factor=up,
              bias=mu.float().to(_dev()), stats=st, groups=G, block_n=block_n)

    def launch():
        if plan:
            _debug_set(4, plan)
        try:
            ops.conv_gemm(a, wp, out.view(1, T, phases * n), **kw)
        finally:
            if plan:
                _debug_set(4, 0)
    cons = [cons_gn_silu] + ([cons_conv_xf] if n % 16 == 0 and n >= 64 and not up else [])
    return launch, out, st, cons


def p_ln_film(kinds, T):
    """y = LN(x) (1 + s) + t with 1 + s = the channel's std, t its mean (s = -1: y = t exactly)."""
    C = 256
    mu, sd = channel_targets(kinds, C)
    x = _rnd(1, T, C, seed=4).to(torch.bfloat16).to(_dev())
    ss = torch.cat([sd - 1.0, mu])[None].float().to(_dev())
    y = torch.empty_like(x)
    st = _stats()
    return (lambda: ops.ln_film(x, y, ss, 2 * C, stats_out=st, groups=G)), y, st, [cons_gn_silu]


def p_stem_in(kinds, T, c0):
    mu, sd = channel_targets(kinds, c0)
    x = _rnd(1, 2, T, seed=5).float().to(_dev())
    w = _rows(c0, 2, 6, sd).reshape(c0, 2, 1).float().to(_dev())
    out = torch.empty(1, T, c0, dtype=torch.bfloat16, device=_dev())
    st = _stats()
    return (lambda: ops.stem_in(x, w, mu.float().to(_dev()), out, 1, stats=st, groups=G)), out, st, [cons_narrow]


def p_skip_gate(kinds, T):
    """out = skip + gate y: the skip carries the mean, the gate the std."""
    C = 256
    mu, sd = channel_targets(kinds, C)
    y = _rnd(1, T, C, seed=7).to(torch.bfloat16).to(_dev())
    skip = mu.expand(1, T, C).to(torch.bfloat16).to(_dev())
    gate = sd[None].float().to(_dev())
    out = torch.empty_like(y)
    st = _stats()
    return (lambda: ops.skip_gate(y, skip, gate, out, st, G)), out, st, [cons_gn_silu]


def p_narrow_conv(kinds, T, C):
    mu, sd = channel_targets(kinds, C)
    x = _rnd(1, T, C, seed=8).to(torch.bfloat16).to(_dev())
    stats_in = ideal_slots(x, G)
    gamma, beta = torch.ones(C, device=_dev()), torch.zeros(C, device=_dev())
    # silu of a unit normal has std ~0.6: the conv term has unit std before the row scaling
    w = _rows(C, 3 * C, 9, sd / 0.6).reshape(C, C, 3).float().to(_dev())
    y = torch.empty_like(x)
    st = _stats()
    kw = dict(w_packed=ops.pack_mid_conv(w) if C > 8 else None, stats_out=st)
    return (lambda: ops.narrow_conv(x, y, stats_in, gamma, beta, w, mu.float().to(_dev()), G, **kw)), y, st, \
        [cons_narrow]


PRODUCERS = {
    "gn_stats": p_gn_stats,
    "conv_k3_256w_128rows": lambda k, T: p_conv(k, T, 256, 256, plan=128),
    "conv_k3_256w_256rows": lambda k, T: p_conv(k, T, 256, 256, plan=256),
    "conv_narrow_group1": lambda k, T: p_conv(k, T, 64, 8),
    "conv_narrow_group2": lambda k, T: p_conv(k, T, 64, 16),
    "conv_narrow_group4": lambda k, T: p_conv(k, T, 64, 32),
    "conv_deep_512w": lambda k, T: p_conv(k, T // 8, 512, 512),       # 2^15 rows: ~16 tiles per CTA
    "conv_up2": lambda k, T: p_conv(k, T // 2, 256, 128, kind="up2"),
    "ln_film": p_ln_film,
    "stem_in_c8": lambda k, T: p_stem_in(k, T, 8),
    "stem_in_c64": lambda k, T: p_stem_in(k, T, 64),
    "skip_gate": p_skip_gate,
    "narrow_conv_c8": lambda k, T: p_narrow_conv(k, T, 8),
    "narrow_conv_c64": lambda k, T: p_narrow_conv(k, T, 64),
}


def stats_case(name, kinds, shadow, T=T_LONG, dev=DEV, slots=None, bounded=True):
    """One producer launch under shadow(), then each of its consumers under shadow() fed the
    statistics it made (or slots(y, G) in their place).  bounded: the statistics must meet the
    checker's bounds and every consumer its bf16 bound against the two-pass fp64 GroupNorm (a
    CheckError names the failing groups).  Returns the report rows."""
    _DEVICE[0] = dev
    launch, y, st, consumers = PRODUCERS[name](kinds, T)
    with shadow():
        launch()
    if dev != "cpu":
        torch.cuda.synchronize()
    made = st.clone()
    y3 = y.reshape(1, -1, y.shape[-1])
    R, sr, vr, rel = producer_report(made, y3, G)
    feed = made if slots is None else slots(y3, G).to(made.dtype)
    cons = {}
    for c in consumers:
        with shadow():
            kind, a, og = c(y3, feed.clone(), G)
        ratio = consumer_ratio(kind, a, og)
        cons[kind] = ratio.reshape(-1) if og is not None else ratio.expand(G)
    rows = [(name, kinds[g], float(R[0, g]), float(sr[0, g]), float(vr[0, g]), float(rel[0, g]),
             {k: float(v.reshape(-1)[g]) for k, v in cons.items()}) for g in range(G)]
    if bounded:
        bad = [f"{r[1]} (R {r[2]:.4g}): statistics {r[3]:.3g}, variance {r[4]:.3g}" for r in rows if max(r[3], r[4]) > 1]
        bad += [f"{k} on {kinds[g]}: err/bound {float(v[g]):.3g}" for k, v in cons.items() for g in range(G)
                if not float(v[g]) <= 1.0]
        if bad:
            raise lc.CheckError(f"{name}: " + "; ".join(bad))
    return rows


def format_rows(rows):
    lines = [f"{'producer':22s} {'group':7s} {'R':>9s} {'stats':>7s} {'var':>7s} {'var_rel':>9s}  consumers err/bound"]
    for name, kind, R, sr, vr, rel, cons in rows:
        c = " ".join(f"{k} {v:.3g}" for k, v in cons.items())
        lines.append(f"{name:22s} {kind:7s} {R:9.4g} {sr:7.3g} {vr:7.3g} {rel:9.3g}  {c}")
    return "\n".join(lines)


@pytest.fixture(autouse=True)
def release_memory():
    """Each test's tensors (fp64 references of 2^18-row launches, 10^4 x 10^4 score matrices) go
    back to the device when it ends, not to this process's allocator cache."""
    yield
    import gc
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def summary():
    yield
    if TABLE:
        print("\nstatistics conditioning (err/bound: <= 1 holds the checker's bound; R1000 unbounded)\n"
              + format_rows(TABLE))


# ------------------------------------------------------------------ a. statistics conditioning sweep
@pytest.fixture(scope="module")
def dev_ready():
    ops.device_check()
    print("\n" + torch.cuda.get_device_name(0))


@pytest.mark.parametrize("name", list(PRODUCERS))
def test_statistics_conditioning(dev_ready, name):
    """Layout KINDS under Shadow(probe=True) and Shadow(guard=True), held to the bounds; every
    group at R = 1000 measured and printed."""
    t0 = time.perf_counter()
    rows = stats_case(name, KINDS, lambda: lc.Shadow(probe=True))
    stats_case(name, KINDS, lambda: lc.Shadow(guard=True))
    rows_1000 = stats_case(name, KINDS_1000, lambda: _Bare(), bounded=False)
    TABLE.extend(rows + rows_1000)
    print(f"\n{name}: {time.perf_counter() - t0:.1f} s\n{format_rows(rows + rows_1000)}")
    for r in rows:                         # constant, zero and tiny groups: finite, and silu(beta) within the bound
        assert math.isfinite(r[4]) and all(math.isfinite(v) and v <= 1 for v in r[6].values()), r


class _Bare:
    """No checking (the R = 1000 layout is measured, not bounded)."""

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False


# ------------------------------------------------------------------ b. LayerNorm rows
ROW_KINDS = ["R0", "R10", "R100", "R256", "R1000", "const", "zero", "tiny"]


def ln_rows_case(C, film, dual, shadow, dev=DEV, rows_per_kind=32):
    """ln_film over rows of every kind (mean / std per row); constant and zero rows must give
    y = shift (FiLM) or 0 within the bf16 bound."""
    T = rows_per_kind * len(ROW_KINDS)
    t = torch.tensor([target(k, g) for g, k in enumerate(ROW_KINDS)], dtype=F64).repeat_interleave(rows_per_kind, 0)
    x = (t[:, :1] + t[:, 1:] * _rnd(T, C, seed=31))[None].to(torch.bfloat16).to(dev)
    ss = torch.cat([0.3 * _rnd(1, C, seed=32), _rnd(1, C, seed=33)], 1).float().to(dev) if film else None
    y = torch.empty_like(x)
    y2 = torch.empty_like(x) if dual else None
    with shadow() as sh:
        ops.ln_film(x, y, ss, 2 * C if film else 0, y2=y2)
    assert torch.isfinite(y.float()).all() and (y2 is None or torch.isfinite(y2.float()).all())
    shift = ss[0, C:].double() if film else torch.zeros(C, dtype=F64, device=dev)
    for k in ("const", "zero"):
        i = ROW_KINDS.index(k) * rows_per_kind
        err = (y[0, i:i + rows_per_kind].double() - shift).abs()
        bound = (lc.BF16_REL + lc.TAU_FP32_ACC) * shift.abs()
        assert bool((err <= bound).all()), \
            f"ln_film C={C}: {k} rows give y {float(err.amax()):.3g} away from the shift"
    return sh


@pytest.mark.parametrize("mode", ["probe", "guard"])
@pytest.mark.parametrize("C", [8, 64, 512, 2048])
@pytest.mark.parametrize("film,dual", [(False, False), (True, False), (True, True)], ids=["plain", "film", "film_y2"])
def test_layernorm_rows(dev_ready, C, film, dual, mode):
    sh = ln_rows_case(C, film, dual, lambda: lc.Shadow(**{mode: True}))
    assert sh.n_checked == sh.n_launch == 1
    print(f"\nln_film C={C} film={film} y2={dual} {mode}: " +
          ", ".join(f"{k} {r.worst:.3g}" for k, r in sorted(sh.records.items())))


# ------------------------------------------------------------------ c. attention logits at the edge
# (name, Tq = Tk, heads): Tk ragged against the 128-key tile
ATT_CASES = {"late40": (300, 2), "late80": (300, 2), "equal": (300, 2), "dominant30": (10000, 1), "wide60": (300, 2)}


def attention_inputs(case, D, dev):
    """q, k, v bf16 [1, T, H D] and the scale D^-1/2 for each case; logits q k scale."""
    T, H = ATT_CASES[case]
    scale = D ** -0.5
    q = 0.5 * _rnd(1, T, H, D, seed=41)
    k = 0.5 * _rnd(1, T, H, D, seed=42)
    v = _rnd(1, T, H, D, seed=43)
    if case.startswith("late") or case.startswith("dominant"):
        gap = float(case[4:] if case.startswith("late") else case[8:])
        jstar = T - 3 if case.startswith("late") else 7777        # the last key tile / mid-sequence
        q[..., 0] = 1.0
        k[..., 0] = 0.0
        # the base logits span about +-2: the key jstar is `gap` above every other one
        k[0, jstar, :, 0] = (gap + 2.0) / scale
    elif case == "equal":
        k[:] = k[:, :1]                                           # every key the same: equal logits per row
    elif case == "wide60":
        a = (12.0 ** 0.5)                                         # logit std 12: |logits| up to ~60
        q, k = q * 2 * a, k * 2 * a
    f = lambda t: t.reshape(1, T, H * D).to(torch.bfloat16).to(dev)
    return f(q), f(k), f(v), scale, H


def exact_forward(q, k, v, H, D, scale):
    """fp64 softmax attention: o [1, T, H D] and lse [1, H, T]."""
    B, Tq, Tk = q.shape[0], q.shape[1], k.shape[1]
    Q = q[0].to(F64).reshape(Tq, H, D).transpose(0, 1)
    K = k[0].to(F64).reshape(Tk, H, D).transpose(0, 1)
    V = v[0].to(F64).reshape(Tk, H, D).transpose(0, 1)
    S = (Q @ K.transpose(1, 2)) * scale
    lse = torch.logsumexp(S, -1)
    o = (torch.softmax(S, -1) @ V).transpose(0, 1).reshape(1, Tq, H * D)
    return o, lse[None], float(S.abs().amax())


def attention_case(case, D, shadow, dev=DEV, backward=True):
    q, k, v, scale, H = attention_inputs(case, D, dev)
    T, mid = q.shape[1], H * D
    o = torch.empty_like(q)
    lse = torch.empty(1, H, T, dtype=torch.float32, device=dev)
    with shadow() as sh:
        ops.attention(q, k, v, o, H, scale, lse=lse, head_dim=D)
        if backward:
            d_o = _rnd(1, T, mid, seed=44).to(torch.bfloat16).to(dev)
            dq, dk, dv = (torch.empty_like(q) for _ in range(3))
            delta = torch.empty(1, H, T, dtype=torch.float32, device=dev)
            ops.attention_bwd(q, k, v, o, d_o, lse, delta, dq, dk, dv, H, scale, head_dim=D)
    outs = [o, lse] + ([dq, dk, dv, delta] if backward else [])
    assert all(bool(torch.isfinite(t.float()).all()) for t in outs), f"{case} D={D}: NaN or Inf"
    o_ref, lse_ref, smax = exact_forward(q, k, v, H, D, scale)
    worst = {}
    if backward:
        # dq, dk, dv against the backward of the exact forward (fp64 o and lse), not the kernel's
        a = dict(q=q, k=k, v=v, o=o_ref, d_o=d_o, lse=lse_ref, delta=delta, dq=dq, dk=dk, dv=dv,
                 heads=H, scale=scale, head_dim=D)
        for val in lc.c_attention_bwd(a, None):
            if val.name == "delta":
                continue
            got = val.view(a).to(F64)
            bound = lc.BF16_REL * val.ref.abs() + val.tau * val.absref
            r = float(((got - val.ref).abs() / bound.clamp_min(1e-300)).amax())
            worst[val.name] = r
            assert r <= 1.0, f"{case} D={D}: {val.name} err/bound {r:.3g} against the exact backward"
    print(f"\nattention {case} D={D} T={T}: max |logit| {smax:.1f}; "
          + ", ".join(f"{k} {r.worst:.3g}" for k, r in sorted(sh.records.items()))
          + "".join(f", exact-bwd {k} {v:.3g}" for k, v in worst.items()))
    return sh


@pytest.mark.parametrize("mode", ["probe", "guard"])
@pytest.mark.parametrize("D", [32, 64, 128])
@pytest.mark.parametrize("case", list(ATT_CASES))
def test_attention_logit_edges(dev_ready, case, D, mode):
    sh = attention_case(case, D, lambda: lc.Shadow(**{mode: True}))
    assert sh.n_checked == sh.n_launch == 2


# ------------------------------------------------------------------ d. whole programs at the edge
SIGNALS = ["silence", "dc", "square", "quiet"]
SIGMAS = [0.0, 1e-4, 0.5, 1.0]


def signal(name, B, T):
    t = torch.arange(T, dtype=F64) / 48000.0
    if name == "silence":
        x = torch.zeros(T, dtype=F64)
    elif name == "dc":
        x = 0.5 + 0.01 * torch.sin(2 * math.pi * 440.0 * t)
    elif name == "square":
        x = torch.where(torch.sin(2 * math.pi * 100.0 * t) >= 0, 1.0, -1.0).to(F64)
    else:
        x = 1e-4 * _rnd(T, seed=51)
    return x.expand(B, 2, T).float().contiguous()


NET_T = 1 << 13


class _f64:
    """The oracle in fp64: tensors it makes itself (the sampler's sigmas) default to fp64 too."""

    def __enter__(self):
        self.saved = torch.get_default_dtype()
        torch.set_default_dtype(F64)

    def __exit__(self, *exc):
        torch.set_default_dtype(self.saved)


# Cases whose bf16 run may miss test_net_gpu.py's output bounds because bf16 storage cannot carry
# the signal; their fp32 verification run must meet the fp32 bound, every launch of both runs its
# own bound, and the bf16 errors are printed as measured.  Every other case meets the bf16 bounds.
STORAGE_LIMITED = {
    "dc": "0.5 + 0.01 sin: bf16 keeps 2^-9 of the 0.5 offset, a fifth of the detail, and the level-0 "
          "groups it makes are near-constant, so GroupNorm scales the rounding up with the detail",
    "quiet": "noise at 1e-4 under the O(0.1) stem biases: bf16 rounds the level-0 activations to the "
             "bias, the groups are near-constant and GroupNorm normalises their rounding",
    "silence": "no signal: the level-0 groups are the biases alone (constant), v is the branch only",
}
# The 3-step sample started from silent "noise" is ill-conditioned in fp32 arithmetic itself: the
# oracle run in fp32 misses the fp32 bound against the oracle in fp64 too (rel-L2 2.0e-3 tiny,
# 1.5e-3 README).  There the fp32 mode is held to twice the fp32 oracle's own error instead.
FP32_LIMITED = {("silence", "sample")}
FP32_TOL = dict(rtol=1e-3, atol=1e-4)           # test_net_gpu.py / test_lengths_gpu.py fp32 mode


def _edge_run(model, x4, sigma4, x1, x2, noise2, sigma2):
    """v at the four sigmas, a 3-step sample and one fused-loss step, every launch checked."""
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    with lc.Shadow() as sh:
        with torch.no_grad():
            v = model.net(x4.to(DEV), sigma4.to(DEV)).clone()
            s = model.sample(x1.to(DEV), num_steps=3).clone()
        model.zero_grad(set_to_none=True)
        loss = fused_v_loss(model.net, x2.to(DEV), noise2.to(DEV), sigma2.to(DEV))
        loss.backward()
    torch.cuda.synchronize()
    assert sh.n_checked == sh.n_launch > 0
    assert torch.isfinite(v).all() and torch.isfinite(s).all() and torch.isfinite(loss.detach())
    for n, p in model.net.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), f"gradient of {n}"
    return v.cpu(), s.cpu(), loss.detach().cpu(), sh


@pytest.mark.parametrize("sig", SIGNALS)
@pytest.mark.parametrize("net", ["tiny", "readme"])
def test_programs_on_edge_audio(dev_ready, oracle_port, net, sig):
    """Every launch of both modes within its own bound; outputs, loss and every parameter gradient
    finite; v and the sample against the oracle in fp64 at test_net_gpu.py's bounds (bf16) or
    STORAGE_LIMITED and the fp32 mode at the fp32 bound; the loss at the training tests' bounds.
    The gradients' errors against the oracle are printed: with silence or quiet noise many of them
    are sums that vanish analytically, whose fp32 residues the near-constant GroupNorm groups scale
    by up to 1 / sqrt(eps) (the oracle in fp32 is as far from the oracle in fp64 there)."""
    import test_lengths_gpu as tlg
    import audio_diffusion_pytorch_b200 as adp
    cfg = tlg.NETS[net]
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**cfg)
    model = adp.DiffusionModel(net_t=adp.UNetV0, **cfg).to(DEV)
    model.net.load_reference_parameters(ref.net)
    ref32 = None
    if any(k[0] == sig for k in FP32_LIMITED):
        torch.manual_seed(0)
        ref32 = oracle_port.DiffusionModelPort(**cfg)
    ref = ref.double()
    model.net.use_cuda_graph = False
    x1 = signal(sig, 1, NET_T)
    x4, sigma4 = x1.expand(4, 2, NET_T).contiguous(), torch.tensor(SIGMAS)
    x2, sigma2 = x1.expand(2, 2, NET_T).contiguous(), torch.tensor([0.0, 1.0])
    noise2 = torch.randn(2, 2, NET_T, generator=torch.Generator().manual_seed(52))
    try:
        with _f64():
            with torch.no_grad():
                v_ref = ref.net(x4.double(), sigma4.double())
                s_ref = ref.sample(x1.double(), num_steps=3)
            loss_ref = tlg._oracle_loss(ref.net, x2.double(), noise2.double(), sigma2.double())
            loss_ref.backward()
        runs = {}
        for mode in ("bf16", "fp32"):
            model.net.verify_fp32 = mode == "fp32"
            v, s, loss, sh = _edge_run(model, x4, sigma4, x1, x2, noise2, sigma2)
            worst, cos = tlg._grads(ref, model)
            runs[mode] = (v, s, loss, worst, cos)
            print(f"\n{net} {sig} {mode}:\n{sh.table()}")
        lines, missed = [], []
        v, s, loss, worst, cos = runs["bf16"]
        for b, sg in enumerate(SIGMAS):
            e_v = tlg.rel_l2(v[b], v_ref[b])
            e_b = tlg.rel_l2(v[b].double() - x4[b], v_ref[b] - x4[b].double())
            lines.append(f"bf16 v sigma={sg}: rel-L2 v {e_v:.2e} (bound {tlg.V_TOL}), branch {e_b:.2e} "
                         f"({tlg.BRANCH_TOL})")
            if e_v > tlg.V_TOL or e_b > tlg.BRANCH_TOL:
                missed.append(lines[-1])
        e_s = tlg.rel_l2(s, s_ref)
        rel = abs(float(loss) - float(loss_ref)) / abs(float(loss_ref))
        lines.append(f"bf16 3-step sample rel-L2 {e_s:.2e} ({tlg.SAMPLE_TOL}); loss rel {rel:.2e} (2e-3); "
                     f"gradients worst {worst:.2e} cos {cos:.6f}")
        if e_s > tlg.SAMPLE_TOL:
            missed.append(lines[-1])
        assert rel < 2e-3, lines[-1]
        v32, s32, loss32, worst32, _ = runs["fp32"]
        e_s32 = tlg.rel_l2(s32, s_ref)
        lines.append(f"fp32 v worst rel-L2 {max(tlg.rel_l2(v32[b], v_ref[b]) for b in range(4)):.2e}; 3-step sample "
                     f"{e_s32:.2e}; loss rel {abs(float(loss32) - float(loss_ref)) / abs(float(loss_ref)):.2e}; "
                     f"gradients worst {worst32:.2e}")
        for b in range(4):
            torch.testing.assert_close(v32[b].double(), v_ref[b], **FP32_TOL)
        torch.testing.assert_close(loss32.double(), loss_ref.detach(), **FP32_TOL)
        if (sig, "sample") in FP32_LIMITED:
            with torch.no_grad():
                e_o32 = tlg.rel_l2(ref32.sample(x1, num_steps=3), s_ref)
            lines.append(f"fp32 oracle 3-step sample rel-L2 {e_o32:.2e} against the oracle in fp64")
            assert e_s32 <= 2 * e_o32, lines[-2:]
        else:
            torch.testing.assert_close(s32.double(), s_ref, **FP32_TOL)
        print(f"\n{net} {sig} T={NET_T}:\n  " + "\n  ".join(lines))
        if missed:
            assert sig in STORAGE_LIMITED, f"{net} {sig}: bf16 run outside the suite's bounds:\n" + "\n".join(missed)
            print(f"  bf16 outside the output bounds ({STORAGE_LIMITED[sig]}); fp32 mode within them")
    finally:
        tlg._free(model)
