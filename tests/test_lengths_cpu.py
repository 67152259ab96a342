"""Clip lengths and batch sizes off the power-of-two grid, without a GPU (tests/test_lengths_gpu.py
runs the same shapes on the kernels).

  * the sweep of test_lengths_gpu.py, level by level from the net configs: it must hit every edge
    it is there for (a level of length 1, odd and ragged attention lengths, ragged 64-, 128- and
    256-row tiles, an odd batch, a single row under guidance), and the power-of-two grid the rest
    of the suite runs must miss every edge that is about raggedness;
  * the launch checker over a single key: attention at Tk = 1 reads neither q nor k unless it writes
    the lse rows, and at Tk = 2 the probe still requires both;
  * the inference, guidance, sampling and training programs at the sweep's small shapes, on fake
    kernels that write the checker's fp64 restatements, against the CPU oracle per batch row: this
    pins the host side (plans, pooled buffers, statistics slots, batch-offset views), so that a
    failure of the GPU file at these shapes is a kernel failure.
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
from test_lengths_gpu import FULL, NETS, SMALL, level_lengths

BF = torch.bfloat16
V_TOL, BRANCH_TOL, GRAD_TOL = 1e-4, 1.2e-2, 6e-2
CFG_V_TOL, CFG_BRANCH_TOL, SAMPLE_TOL = 3e-4, 2.5 * BRANCH_TOL, 5e-3
GUIDANCE = 5.0


# ------------------------------------------------------------------------------ the sweep's edges
def edges(cases):
    """The edges a list of (net, B, T) cases reaches."""
    hit = set()
    for name, B, T in cases:
        cfg = NETS[name]
        guided = bool(cfg.get("use_embedding_cfg"))
        if B % 2 and B > 1:
            hit.add("odd batch above 1")
        if guided and B == 1:
            hit.add("one row under guidance")
        for t, ch, att in zip(level_lengths(cfg, T), cfg["channels"], cfg.get("attentions", [0] * 99)):
            if t == 1:
                hit.add("level of length 1")
            if t % 64:
                hit.add("length not a multiple of 64 (wgrad chunks)")
            if ch % 64 == 0 and t >= 256 and t % 256:
                hit.add("ragged 256-row conv tile")
            if ch <= 64 and t % 128:
                hit.add("thin level ragged in 128-row tiles")
            if ch <= 64 and t % 128 == 0 and t % 256:
                hit.add("thin level ragged in 256-row tiles only")
            if att:
                if t % 2:
                    hit.add("odd attention length")
                if t < 128:
                    hit.add("attention length below 128")
                if t > 128 and t % 128:
                    hit.add("attention length above 128, not a multiple of it")
    return hit


EDGES = {"level of length 1", "length not a multiple of 64 (wgrad chunks)", "ragged 256-row conv tile",
         "thin level ragged in 128-row tiles", "thin level ragged in 256-row tiles only", "odd attention length",
         "attention length below 128", "attention length above 128, not a multiple of it", "odd batch above 1",
         "one row under guidance"}


def test_level_lengths_of_the_table():
    readme = NETS["readme"]
    assert level_lengths(readme, 2048) == [2048, 512, 128, 32, 16, 8, 4, 2, 1]
    assert level_lengths(readme, 6144) == [6144, 1536, 384, 96, 48, 24, 12, 6, 3]
    assert level_lengths(readme, 239616) == [239616, 59904, 14976, 3744, 1872, 936, 468, 234, 117]
    for name in ("tiny", "tiny_text"):
        assert level_lengths(NETS[name], 16) == [16, 4, 1]
        assert level_lengths(NETS[name], 4080) == [4080, 1020, 255]
    for name, _, T in SMALL + FULL:
        total = math.prod(NETS[name]["factors"])
        assert T % total == 0, (name, T)


def test_sweep_hits_every_edge():
    assert edges(SMALL + FULL) == EDGES
    assert edges(SMALL) == EDGES                 # the small sizes alone: oracle and checker (parts a, b)


def test_power_of_two_grid_misses_the_ragged_edges():
    """What the rest of the suite runs, T = 2^12 ... 2^18 and B in {1, 2, 4, 8, 16}, reaches only
    the edges that any deep level or a single row reaches."""
    grid = [(n, B, 2 ** k) for n in NETS for B in (1, 2, 4, 8, 16) for k in range(12, 19)]
    assert edges(grid) == {"attention length below 128", "length not a multiple of 64 (wgrad chunks)",
                           "one row under guidance"}


# ------------------------------------------------------------------------------ fake kernels
@pytest.fixture
def cpu_launches(monkeypatch):
    monkeypatch.setattr(ops, "device_check", lambda: None)
    monkeypatch.setattr(ops, "require_cuda", lambda x: None)

    def no_library():
        raise AssertionError("a launch reached the CUDA library")
    monkeypatch.setattr(_lib, "lib", no_library)


def _qkv(B, Tq, Tk, H=2, D=32, seed=3):
    g = torch.Generator().manual_seed(seed)
    mid = H * D
    return [torch.randn(B, t, mid, generator=g).to(BF) for t in (Tq, Tk, Tk)]


def _attention(Tq, Tk, with_lse, B=3, H=2, D=32):
    q, k, v = _qkv(B, Tq, Tk, H, D)
    ops.attention(q, k, v, torch.empty(B, Tq, H * D, dtype=BF), H, D ** -0.5,
                  lse=torch.empty(B, H, Tq) if with_lse else None, head_dim=D)


@pytest.mark.parametrize("Tq", [1, 5])
def test_single_key_attention_under_the_probe(cpu_launches, Tq):
    """The innermost level of length 1 (T = 16 in TINY, T = 2048 in README): one key.  The output
    is v; the lse rows, written for the backward, still read q and k, and so does attention_bwd."""
    B, H, D = 3, 2, 32
    with lc.Shadow(fake=True, probe=True) as sh:
        _attention(Tq, 1, with_lse=False)
        _attention(Tq, 1, with_lse=True)
        q, k, v = _qkv(B, Tq, 1, H, D, seed=4)
        S = torch.einsum("bqhd,bkhd->bhqk", q.double().reshape(B, Tq, H, D), k.double().reshape(B, 1, H, D)) * D ** -0.5
        o = v.expand(B, Tq, H * D).contiguous()
        d_o = torch.randn(B, Tq, H * D, generator=torch.Generator().manual_seed(5)).to(BF)
        ops.attention_bwd(q, k, v, o, d_o, torch.logsumexp(S, -1).float(), torch.zeros(2 * B * H * Tq),
                          torch.empty(B, Tq, H * D, dtype=BF), torch.empty(B, 1, H * D, dtype=BF),
                          torch.empty(B, 1, H * D, dtype=BF), H, D ** -0.5, head_dim=D)
    assert sh.n_checked == sh.n_launch == 3
    assert sorted(k for k, _ in sh.probed) == ["attention", "attention", "attention_bwd"]
    args = dict(q=q, k=k, lse=None)
    assert lc.NOT_READ["attention"](args) == {"q", "k"}
    assert lc.NOT_READ["attention"](dict(args, lse=torch.empty(B, H, Tq))) == set()
    assert "attention_bwd" not in lc.NOT_READ


@pytest.mark.parametrize("name", ["k", "q"])
def test_two_keys_still_require_q_and_k(cpu_launches, monkeypatch, name):
    """At Tk = 2 the exemption is gone: a restatement that ignores k (or q) is refused."""
    assert lc.NOT_READ["attention"](dict(k=torch.empty(3, 2, 64), lse=None)) == set()
    real = lc.CHECKERS["attention"]

    def ignores(a, ctx):
        return real(dict(a, **{name: torch.ones_like(a[name])}), ctx)
    monkeypatch.setitem(lc.CHECKERS, "attention", ignores)
    with lc.Shadow(fake=True, probe=True), pytest.raises(lc.CheckError, match=f"does not depend on `{name}`"):
        _attention(5, 2, with_lse=False)
    with lc.Shadow(fake=True, probe=True):      # and the real restatement passes there
        monkeypatch.setitem(lc.CHECKERS, "attention", real)
        _attention(5, 2, with_lse=False)


# ------------------------------------------------------------------------------ programs
def _pair(oracle_port, cfg):
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**cfg)
    model = DiffusionModel(net_t=UNetV0, **cfg)
    model.net.load_reference_parameters(ref.net)
    model.net.use_cuda_graph = False
    return ref, model.net


def _inputs(cfg, B, T, seed):
    g = torch.Generator().manual_seed(seed)
    x, noise, sigma = torch.randn(B, 2, T, generator=g), torch.randn(B, 2, T, generator=g), torch.rand(B, generator=g)
    emb = None
    if cfg.get("embedding_features"):
        emb = torch.randn(B, cfg["embedding_max_length"], cfg["embedding_features"], generator=g)
    return x, noise, sigma, emb


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def per_row(got, want, what, tol, skip=None, v_tol=None):
    """rel-L2 of every batch row; with `skip`, of v (<= v_tol) and of the branch v - skip (<= tol)."""
    errs = []
    for b in range(want.shape[0]):
        if skip is None:
            errs.append((rel_l2(got[b], want[b]),))
        else:
            errs.append((rel_l2(got[b], want[b]), rel_l2(got[b] - skip[b], want[b] - skip[b])))
    print(f"{what}: per row " + "  ".join("/".join(f"{e:.2e}" for e in row) for row in errs))
    for b, row in enumerate(errs):
        if skip is None:
            assert row[0] <= tol, f"{what}: row {b} error {row[0]:.3e} > {tol}"
        else:
            assert row[0] <= v_tol, f"{what}: row {b} v error {row[0]:.3e} > {v_tol}"
            assert row[1] <= tol, f"{what}: row {b} branch error {row[1]:.3e} > {tol}"


TINY_CASES = [c for c in SMALL if c[0] != "readme"]


def _id(case):
    return "-".join(map(str, case))


@pytest.mark.parametrize("case", TINY_CASES, ids=_id)
def test_tiny_programs_vs_oracle(cpu_launches, oracle_port, case):
    """v, guidance 5 (TINY_TEXT) and a 3-step sample, every launch checked and probed."""
    name, B, T = case
    cfg = NETS[name]
    ref, net = _pair(oracle_port, cfg)
    x, _, sigma, emb = _inputs(cfg, B, T, 1)
    kw = dict(embedding=emb) if emb is not None else {}
    what = f"{name} B={B} T={T}"
    with torch.no_grad(), lc.Shadow(fake=True, probe=True) as sh:
        per_row(net(x, sigma, embedding=emb), ref.net(x, sigma, **kw), f"{what} v/branch", BRANCH_TOL, x, V_TOL)
        scale = GUIDANCE if emb is not None else 1.0
        if emb is not None:
            per_row(net(x, sigma, embedding=emb, embedding_scale=scale), ref.net(x, sigma, embedding_scale=scale, **kw),
                    f"{what} guidance {scale}", CFG_BRANCH_TOL, x, CFG_V_TOL)
        want = ref.sample(x, num_steps=3, **(dict(kw, embedding_scale=scale) if kw else {}))
        per_row(VSampler(net=net)(x, num_steps=3, embedding=emb, embedding_scale=scale), want, f"{what} 3-step sample", SAMPLE_TOL)
    assert sh.n_checked == sh.n_launch > 0
    labels = " ".join(sh.labels)
    t_att = level_lengths(cfg, T)[-1]
    assert f"stem_in[{[B, 2, T]}" in labels.replace("(", "[").replace(")", "]")
    assert sh.records["attention.o"].count > 0 and {"step_select", "step_advance"} <= {k for k, _ in sh.probed}
    if t_att == 1:                                # the single-key exemption was used, and only there
        assert any(k == "attention" and "lse" not in args for k, args in sh.probed)


def _grads(ref_net, net):
    pairs = [(n, p, q) for (n, p), q in zip(ref_net.named_parameters(), net.parameters()) if p.grad is not None]
    norms = torch.stack([p.grad.double().norm() for _, p, _ in pairs])
    floor = max(0.1 * float(norms.median()), 1e-3 * float(norms.max()))
    worst, worst_name, dots, n1, n2 = 0.0, "", 0.0, 0.0, 0.0
    for name, p, q in pairs:
        assert q.grad is not None, f"no gradient for {name}"
        g_ref, g = p.grad.double(), q.grad.double()
        rel = float((g - g_ref).norm() / g_ref.norm().clamp_min(floor))
        if rel > worst:
            worst, worst_name = rel, name
        dots += float((g * g_ref).sum()); n1 += float((g * g).sum()); n2 += float((g_ref * g_ref).sum())
    cos = dots / math.sqrt(n1 * n2)
    print(f"worst per-parameter rel-L2 {worst:.3e} ({worst_name}); global cosine {cos:.6f}")
    return worst, cos


@pytest.mark.parametrize("case", [c for c in TINY_CASES if c[1] == 3], ids=_id)
def test_tiny_training_step_vs_oracle(cpu_launches, oracle_port, case):
    """Loss and every parameter gradient of one training step (split-K wgrad, cond_bwd, colsum and
    the attention backward at 255 and at one position)."""
    name, B, T = case
    cfg = NETS[name]
    ref, net = _pair(oracle_port, cfg)
    x, noise, sigma, emb = _inputs(cfg, B, T, 5)
    a, b = torch.cos(sigma * math.pi / 2)[:, None, None], torch.sin(sigma * math.pi / 2)[:, None, None]
    kw = dict(embedding=emb, embedding_mask_proba=0.0) if emb is not None else {}
    loss_ref = F.mse_loss(ref.net(a * x + b * noise, sigma, **kw), a * noise - b * x)
    loss_ref.backward()
    with lc.Shadow(fake=True) as sh:
        loss = training.fused_v_loss(net, x, noise, sigma, embedding=emb)
        loss.backward()
    assert sh.n_checked == sh.n_launch > 0
    assert {"wgrad", "cond_bwd", "attention_bwd", "stem_in_bwd"} <= {k.split(".")[0] for k in sh.records}
    t_att = level_lengths(cfg, T)[-1]
    assert f"attention_bwd[{[B, t_att, 128]}" in " ".join(sh.labels).replace("(", "[").replace(")", "]")
    loss, loss_ref = float(loss.detach()), float(loss_ref.detach())
    rel = abs(loss - loss_ref) / loss_ref
    print(f"{name} B={B} T={T}: loss {loss:.6f} vs oracle {loss_ref:.6f} (rel {rel:.2e})")
    assert rel < 2e-3
    worst, cos = _grads(ref.net, net)
    assert worst < GRAD_TOL and cos > 1 - 1e-3


@pytest.mark.parametrize("T", [2048, 2048 * 3])
def test_readme_v_program_vs_oracle(cpu_launches, oracle_port, T):
    """The README net at B = 3: an innermost level of 1 or 3 positions, attention at 8 ... 1 and
    24 ... 3, conv GEMMs at 96, 48, ... rows per batch element."""
    ref, net = _pair(oracle_port, NETS["readme"])
    x, _, sigma, _ = _inputs(NETS["readme"], 3, T, 2)
    with torch.no_grad(), lc.Shadow(fake=True) as sh:
        v = net(x, sigma)
        want = ref.net(x, sigma)
    assert sh.n_checked == sh.n_launch > 0
    per_row(v, want, f"README B=3 T={T} v/branch", BRANCH_TOL, x, V_TOL)


def test_groupnorm_backward_bound_of_a_one_row_group():
    """gn_silu_bwd at M = 1 (README, B = 1, T = 2048: the innermost level, 1024 channels): dgamma[c]
    is one product dz * xhat, and the kernel forms xhat = (x - mean) * rstd in fp32 from an fp32
    mean.  For an x next to its group's mean that rounding is relative to (|x| + |mean|) rstd, far
    above |xhat|: the checker's magnitude must carry it.  On an H100 a bound on |dz xhat| alone was
    exceeded there (err/bound 1.02), and so was one on |dz| rather than DSILU_MAX |da| (2.99: SiLU'
    crosses zero by cancellation)."""
    C, G = 24, 2
    g = torch.Generator().manual_seed(8)
    # group 0: pairs 48 +- d, one of them a bf16 step off, and 48 twice: its mean 48 + 2^-8 / 12 is
    # 3.3e-4 from x[11] = 48 and 85.33 fp32 steps above 48, so the fp32 mean is off by a third of a step
    group0 = [47, 49, 46, 50, 44, 52, 40, 56, 0.5 + 2 ** -8, 95.5, 48, 48]
    x = torch.cat([torch.tensor(group0), torch.randn(C - 12, generator=g)]).reshape(1, 1, C).to(BF)
    assert x[0, 0, :12].tolist() == group0
    stats = lc.stats_of(x, G)
    gamma, beta = torch.ones(C), torch.zeros(C)
    da = torch.randn(1, 1, C, generator=g).to(BF)
    outs = {o.name: o for o in lc.CHECKERS["gn_silu_bwd"](dict(
        da=da, x=x, stats=stats, gamma=gamma, beta=beta, dxh=None, dgamma=None, dbeta=None, S=None, groups=G,
        eps=1e-5), None)}
    ref, mag = outs["dgamma"].ref, outs["dgamma"].absref
    st = stats.double()[0]                                   # the kernel's coefficients (backward.cu gn_coeffs)
    n = C // G
    m64 = st[:, 0] / n
    var = (st[:, 1] / n - m64 * m64).float().clamp_min(0).repeat_interleave(n)
    m64 = m64.repeat_interleave(n)
    xh32 = (x.float()[0, 0] - m64.float()) * torch.rsqrt(var + 1e-5)
    z = xh32 * gamma + beta
    sg = torch.sigmoid(z)
    got = (da.float()[0, 0] * sg * (1 + z * (1 - sg)) * xh32).double()
    err = (got - ref).abs()
    assert (err <= lc.FP32_REL * ref.abs() + lc.FP32_TAU * mag).all()
    assert err[11] > (lc.FP32_REL + lc.FP32_TAU) * ref[11].abs(), "the case must need the wider magnitude"
