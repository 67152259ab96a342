"""Backward kernels against torch.autograd of the fp32 PyTorch restatement of each op
(same bf16-rounded inputs).  Gradient outputs that are bf16 get 2^-6 relative + small
absolute slack; fp32 parameter-gradient accumulators (sums over up to 10^5 terms of bf16
products) get 1e-2 relative to the largest entry."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def bf(t):
    return t.to(torch.bfloat16)


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def close(got, ref, rtol, atol_frac, what):
    got, ref = got.double(), ref.double()
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item()
    print(f"{what}: max abs err {err:.4e} (ref max {scale:.3e})")
    assert err <= rtol * scale + atol_frac * scale + 1e-12, f"{what}: {err} vs scale {scale}"


@pytest.fixture(scope="module")
def ops():
    from audio_diffusion_pytorch_b200 import ops
    ops.device_check()
    return ops


def group_ids(cases):
    """pytest ids of cases whose last entry is the GroupNorm group count; 8 groups (the default
    of UNetV0) is left out of the id."""
    return ["-".join(str(v) for v in c[:-1]) + ("" if c[-1] == 8 else f"-g{c[-1]}") for c in cases]


def stats_of(y, groups):
    B, T, Cc = y.shape
    yg = y.double().reshape(B, T, groups, Cc // groups)
    return torch.stack([yg.sum(dim=(1, 3)), (yg * yg).sum(dim=(1, 3))], dim=-1).contiguous()


@pytest.mark.parametrize("B,T,n,k,off", [(2, 256, 64, 64, 0), (2, 300, 128, 128, -1), (1, 128, 32, 32, 1),
                                         (2, 1000, 256, 256, 0), (1, 64, 1024, 512, 1),
                                         (3, 100, 8, 32, 0), (2, 4096, 64, 64, -1)])
def test_wgrad(ops, B, T, n, k, off):
    """The contract is dw += g^T x: the gradient arenas and the upsample per-phase slots rely on
    accumulation, so dw starts from non-zero values of the size of the product."""
    g = bf(rnd(B, T, n, seed=1))
    x = bf(rnd(B, T, k, seed=2))
    dw0 = rnd(n, k, scale=(B * T) ** 0.5, seed=3)
    dw = dw0.clone()
    ops.wgrad(g, x, dw, n=n, k=k, off=off)
    xs = torch.zeros_like(x.float())
    if off == 0:
        xs = x.float()
    elif off > 0:
        xs[:, :-off] = x.float()[:, off:]
    else:
        xs[:, -off:] = x.float()[:, :off]
    ref = dw0 + torch.einsum("btn,btk->nk", g.float(), xs)
    close(dw, ref, 2e-3, 1e-3, f"wgrad n{n} k{k} off{off}")


def test_wgrad_column_views(ops):
    """Phase views of the upsample conv: g is a column block of a wider row."""
    B, T, co, ci, f = 2, 256, 64, 128, 2
    g = bf(rnd(B, T, f * co, seed=3))
    x = bf(rnd(B, T, ci, seed=4))
    dw = torch.zeros(co, ci, device=DEV)
    ops.wgrad(g, x, dw, n=co, k=ci, off=0, g_col0=co)
    ref = torch.einsum("btn,btk->nk", g.float()[..., co:], x.float())
    close(dw, ref, 2e-3, 1e-3, "wgrad column view")


# the per-channel coefficients (gn_coeffs), the per-group S sums of gn_silu_bwd and their
# broadcast back to channels in gn_bwd_apply all index by channel / group size
_GN_BWD = [(2, 1000, 8, 8), (2, 512, 32, 8), (2, 300, 64, 8), (1, 256, 512, 8), (2, 128, 1024, 8),
           (2, 1000, 8, 1), (2, 1000, 8, 2), (2, 1000, 8, 4), (2, 512, 32, 2), (2, 512, 32, 16),
           (2, 300, 64, 1), (2, 300, 64, 4), (2, 300, 64, 16), (2, 300, 64, 64), (1, 256, 512, 2),
           (2, 128, 1024, 1), (2, 128, 1024, 4), (2, 128, 1024, 16), (2, 128, 1024, 64)]


@pytest.mark.parametrize("B,T,C,groups", _GN_BWD, ids=group_ids(_GN_BWD))
def test_gn_silu_backward(ops, B, T, C, groups):
    x = bf(rnd(B, T, C, seed=5) * 1.5 + 0.3)
    da = bf(rnd(B, T, C, seed=6))
    dres = bf(rnd(B, T, C, seed=7))
    gamma = (rnd(C, seed=8) * 0.2 + 1.0).requires_grad_()
    beta = (rnd(C, seed=9) * 0.2).requires_grad_()
    xr = x.float().requires_grad_()
    a = F.silu(F.group_norm(xr.transpose(1, 2), groups, gamma, beta, 1e-5)).transpose(1, 2)
    a.backward(da.float())
    stats = stats_of(x, groups)
    dxh, dx = torch.empty_like(x), torch.empty_like(x)
    dg, db = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    S = torch.zeros(B, groups, 2, dtype=torch.float64, device=DEV)
    cs = torch.zeros(C, device=DEV)
    ops.gn_silu_bwd(da, x, stats, gamma.detach(), beta.detach(), dxh, dg, db, S, groups)
    ops.gn_bwd_apply(dxh, x, stats, S, dx, groups, dres=dres, colsum=cs)
    close(dx, xr.grad + dres.float(), 2 ** -6, 2e-3, f"gn bwd dx C{C} G{groups}")
    close(dg, gamma.grad, 1e-2, 2e-3, f"gn bwd dgamma C{C} G{groups}")
    close(db, beta.grad, 1e-2, 2e-3, f"gn bwd dbeta C{C} G{groups}")
    # the column sum is taken from the unrounded fp32 values (it feeds a bias gradient)
    close(cs, (xr.grad + dres.float()).sum(dim=(0, 1)), 2e-3, 2e-3, "gn bwd colsum")


@pytest.mark.parametrize("B,T,C", [(2, 1000, 8), (2, 512, 32), (2, 300, 64), (1, 256, 512), (2, 128, 1024)])
def test_ln_film_backward(ops, B, T, C):
    x = bf(rnd(B, T, C, seed=10) * 2.0 + 0.5)
    dy = bf(rnd(B, T, C, seed=11))
    ss = (rnd(B, 2 * C, seed=12) * 0.3).requires_grad_()
    xr = x.float().requires_grad_()
    y = F.layer_norm(xr, (C,), eps=1e-6) * (1 + ss[:, None, :C]) + ss[:, None, C:]
    y.backward(dy.float())
    dx = torch.empty_like(x)
    dss = torch.zeros(B, 2 * C, device=DEV)
    cs = torch.zeros(C, device=DEV)
    ops.ln_film_bwd(dy, x, ss.detach(), 2 * C, dx, dss=dss, dss_stride=2 * C, colsum=cs)
    close(dx, xr.grad, 2 ** -6, 2e-3, f"ln_film bwd dx C{C}")
    close(dss, ss.grad, 1e-2, 2e-3, f"ln_film bwd dss C{C}")
    close(cs, xr.grad.sum(dim=(0, 1)), 2e-3, 2e-3, "ln_film bwd colsum")


def _colsum_and_skip_gate(ops, C, groups):
    B, T = 2, 700
    y, skip, dout = bf(rnd(B, T, C, seed=13)), bf(rnd(B, T, C, seed=14)), bf(rnd(B, T, C, seed=15))
    gate = rnd(B, C + 8, seed=16)[:, :C]       # strided view, like a slice of ss_all
    out = torch.empty_like(y)
    stats = torch.zeros(B, groups, 2, dtype=torch.float64, device=DEV)
    ops.skip_gate(y, skip, gate, out, stats, groups)
    ref = skip.float() + gate[:, None, :] * y.float()
    close(out, ref, 2 ** -7, 1e-3, "skip_gate out")
    close(stats, stats_of(out, groups), 1e-4, 1e-6, f"skip_gate stats C{C} G{groups}")
    dys = torch.empty_like(y)
    dgate = torch.zeros(B, C + 8, device=DEV)
    ops.skip_gate_bwd(dout, y, gate, dys, dgate[:, :C])
    close(dys, gate[:, None, :] * dout.float(), 2 ** -7, 1e-3, "skip_gate_bwd dys")
    close(dgate[:, :C], (dout.float() * y.float()).sum(1), 1e-3, 1e-3, "skip_gate_bwd dgate")
    cs = torch.zeros(C, device=DEV)
    ops.colsum(dout, cs, gate)
    close(cs, (dout.float() * gate[:, None, :]).sum(dim=(0, 1)), 1e-3, 1e-3, "colsum gated")


def test_colsum_and_skip_gate(ops):
    _colsum_and_skip_gate(ops, 64, 8)


# the skip_gate statistics sum each group's per-channel sums: other group counts, also at C = 1024
@pytest.mark.parametrize("C,groups", [(64, 1), (64, 4), (64, 16), (64, 64), (1024, 8), (1024, 1), (1024, 4),
                                      (1024, 16), (1024, 64)])
def test_colsum_and_skip_gate_groups(ops, C, groups):
    _colsum_and_skip_gate(ops, C, groups)


@pytest.mark.parametrize("B,want_dcond", [(4, True), (8, True), (19, True), (4, False), (32, False),
                                          (40, False)])
def test_cond_bwd(ops, B, want_dcond):
    """In-graph call (with d cond, 8 rows per pass) and the data-parallel call on all-gathered rows
    (parameter gradients only, 32 rows per pass); batches beyond one pass accumulate."""
    N, K = 840, 1024
    dss = rnd(B, N + 8, seed=17)[:, :N]
    cond = bf(rnd(B, K, seed=18)).float()
    w = bf(rnd(N, K, seed=19) * 0.03)
    dw, dbias = torch.full((N, K), float("nan"), device=DEV), torch.full((N,), float("nan"), device=DEV)
    dcond = torch.zeros(B, K, device=DEV) if want_dcond else None
    ops.cond_bwd(dss, cond, w, dw, dbias, dcond, N)
    close(dw, dss.t() @ cond, 1e-4, 1e-5, "cond_bwd dw")
    close(dbias, dss.sum(0), 1e-4, 1e-5, "cond_bwd dbias")
    if want_dcond:
        close(dcond, dss @ w.float(), 1e-3, 1e-4, "cond_bwd dcond")


def _narrow_conv_backward(ops, groups):
    B, T, C = 2, 3000, 8
    x = bf(rnd(B, T, C, seed=20) * 1.3 + 0.2)
    dy = bf(rnd(B, T, C, seed=21))
    gamma = (rnd(C, seed=22) * 0.2 + 1.0).requires_grad_()
    beta = (rnd(C, seed=23) * 0.2).requires_grad_()
    w = rnd(C, C, 3, scale=(3 * C) ** -0.5, seed=24).requires_grad_()
    bias = rnd(C, seed=25).requires_grad_()
    xr = x.float().requires_grad_()
    a = F.silu(F.group_norm(xr.transpose(1, 2), groups, gamma, beta, 1e-5))
    y = F.conv1d(a, w, bias, padding=1).transpose(1, 2)
    y.backward(dy.float())
    stats = stats_of(x, groups)
    dxh, dx = torch.empty_like(x), torch.empty_like(x)
    dg, db = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    dw, dbias = torch.zeros(C, C, 3, device=DEV), torch.zeros(C, device=DEV)
    S = torch.zeros(B, groups, 2, dtype=torch.float64, device=DEV)
    ops.narrow_conv_bwd(dy, x, stats, gamma.detach(), beta.detach(), w.detach(), dxh, dg, db, S, dw,
                        dbias, groups)
    ops.gn_bwd_apply(dxh, x, stats, S, dx, groups)
    close(dx, xr.grad, 2 ** -6, 3e-3, f"narrow bwd dx G{groups}")
    close(dw, w.grad, 1e-2, 2e-3, "narrow bwd dw")
    close(dbias, bias.grad, 1e-3, 1e-3, "narrow bwd dbias")
    close(dg, gamma.grad, 1e-2, 2e-3, f"narrow bwd dgamma G{groups}")
    close(db, beta.grad, 1e-2, 2e-3, f"narrow bwd dbeta G{groups}")


def test_narrow_conv_backward(ops):
    _narrow_conv_backward(ops, 8)


# the C = 8 GroupNorm coefficients and the per-group S sums of narrow_conv_bwd at other group counts
@pytest.mark.parametrize("groups", [1, 2, 4])
def test_narrow_conv_backward_groups(ops, groups):
    _narrow_conv_backward(ops, groups)


@pytest.mark.parametrize("cx,ca,co,c0,f", [(2, 0, 2, 8, 1), (2, 2, 2, 8, 1), (1, 1, 1, 32, 4), (4, 4, 4, 8, 1)])
def test_stem_backward(ops, cx, ca, co, c0, f):
    B, T = 2, 1024
    cin = cx + ca
    h = bf(rnd(B, T // f, c0, seed=26))
    x = rnd(B, cx, T, seed=27)
    app = rnd(B, ca, T, seed=28) if ca else None
    noise = rnd(B, cx, T, seed=29)
    alpha, beta = torch.rand(B, device=DEV), torch.rand(B, device=DEV)
    w = rnd(co, c0, 3, scale=(3 * c0) ** -0.5, seed=30).requires_grad_()
    bias = rnd(co, seed=31).requires_grad_()
    gate = rnd(B, co, seed=32).requires_grad_()
    adapt = cin != co
    wa = rnd(co, cin, seed=33).requires_grad_() if adapt else None
    ba = rnd(co, seed=34).requires_grad_() if adapt else None
    dv = rnd(B, co, T, seed=35)
    hr = h.float().requires_grad_()
    xin = alpha[:, None, None] * x + beta[:, None, None] * noise
    xin_full = torch.cat([xin, app], 1) if ca else xin
    up = F.interpolate(hr.transpose(1, 2), scale_factor=f, mode="nearest")
    y = F.conv1d(up, w, bias, padding=1)
    skip = F.conv1d(xin_full, wa[:, :, None], ba) if adapt else xin_full
    v = skip + gate[:, :, None] * y
    v.backward(dv)
    dh = torch.empty_like(h)
    dw, db = torch.zeros(co, c0, 3, device=DEV), torch.zeros(co, device=DEV)
    dgate = torch.zeros(B, co, device=DEV)
    dwa = torch.zeros(co, cin, device=DEV) if adapt else None
    dba = torch.zeros(co, device=DEV) if adapt else None
    ops.stem_out_bwd(dv, h, x, w.detach(), bias.detach(), gate.detach(), f, dh, dw, db, dgate,
                     append=app, noise=noise, alpha=alpha, beta=beta,
                     w_adapt=wa.detach() if adapt else None, dw_adapt=dwa, db_adapt=dba)
    close(dh, hr.grad, 2 ** -6, 2e-3, "stem_out_bwd dh")
    close(dw, w.grad, 1e-3, 1e-3, "stem_out_bwd dw")
    close(db, bias.grad, 1e-3, 1e-3, "stem_out_bwd dbias")
    close(dgate, gate.grad, 1e-3, 1e-3, "stem_out_bwd dgate")
    if adapt:
        close(dwa, wa.grad, 1e-3, 1e-3, "stem_out_bwd dw_adapt")
        close(dba, ba.grad, 1e-3, 1e-3, "stem_out_bwd db_adapt")
    # stem_in backward
    w_in = rnd(c0, cin, f, seed=36).requires_grad_()
    b_in = rnd(c0, seed=37).requires_grad_()
    dout = bf(rnd(B, T // f, c0, seed=38))
    out = F.conv1d(xin_full, w_in, b_in, stride=f).transpose(1, 2)
    out.backward(dout.float())
    dwi, dbi = torch.zeros(c0, cin, f, device=DEV), torch.zeros(c0, device=DEV)
    ops.stem_in_bwd(dout, x, dwi, dbi, f, append=app, noise=noise, alpha=alpha, beta=beta)
    close(dwi, w_in.grad, 1e-3, 1e-3, "stem_in_bwd dw")
    close(dbi, b_in.grad, 1e-3, 1e-3, "stem_in_bwd dbias")


@pytest.mark.parametrize("B,H,Tq,Tk", [(2, 8, 256, 256), (1, 2, 128, 128), (2, 4, 200, 200),
                                       (2, 8, 512, 64), (1, 2, 300, 8), (1, 1, 64, 384),
                                       (1, 8, 1024, 1024)])
def test_attention_bwd(ops, B, H, Tq, Tk):
    """adp_attention (with its log-sum-exp output) + adp_attention_bwd against autograd through
    F.scaled_dot_product_attention on the same bf16 q/k/v, read out of packed projection rows."""
    mid = H * 64
    if Tq == Tk:
        qkv = bf(rnd(B, Tq, 3 * mid, seed=70))
        q, k, v = qkv[..., :mid], qkv[..., mid:2 * mid], qkv[..., 2 * mid:]
        dqkv = torch.full_like(qkv, float("nan"))
        dq, dk, dv = dqkv[..., :mid], dqkv[..., mid:2 * mid], dqkv[..., 2 * mid:]
    else:
        q = bf(rnd(B, Tq, mid, seed=71))
        kv = bf(rnd(B, Tk, 2 * mid, seed=72))
        k, v = kv[..., :mid], kv[..., mid:]
        dq = torch.full_like(q, float("nan"))
        dkv = torch.full_like(kv, float("nan"))
        dk, dv = dkv[..., :mid], dkv[..., mid:]
    d_o = bf(rnd(B, Tq, mid, seed=73))
    o = torch.empty(B, Tq, mid, dtype=torch.bfloat16, device=DEV)
    lse = torch.full((B, H, Tq), float("nan"), device=DEV)
    delta = torch.empty(B, H, Tq, device=DEV)
    ops.attention(q, k, v, o, H, 64 ** -0.5, lse=lse)
    ops.attention_bwd(q, k, v, o, d_o, lse, delta, dq, dk, dv, H, 64 ** -0.5)

    def heads(t):
        return t.float().reshape(B, -1, H, 64).transpose(1, 2)
    qf, kf, vf = (heads(t).detach().requires_grad_(True) for t in (q, k, v))
    ref = F.scaled_dot_product_attention(qf, kf, vf)
    ref.backward(heads(d_o))
    lse_ref = torch.logsumexp(qf.detach() @ kf.detach().transpose(-1, -2) * 64 ** -0.5, dim=-1)
    close(lse, lse_ref, 1e-3, 1e-3, "lse")

    def flat(t):
        return t.transpose(1, 2).reshape(B, -1, mid)
    close(dq, flat(qf.grad), 2 ** -6, 1.5e-2, f"dq B{B} H{H} Tq{Tq} Tk{Tk}")
    close(dk, flat(kf.grad), 2 ** -6, 1.5e-2, "dk")
    close(dv, flat(vf.grad), 2 ** -6, 1.5e-2, "dv")


@pytest.mark.parametrize("N,C", [(128, 64), (1536, 512), (256, 768), (1024, 1024)])
def test_ln_fold_bwd(ops, N, C):
    w, g, b = rnd(N, C, seed=80), rnd(C, seed=81) * 0.3 + 1.0, rnd(C, seed=82) * 0.3
    dwf, dbf = rnd(N, C, seed=83), rnd(N, seed=84)
    dw = torch.full((N, C), float("nan"), device=DEV)
    dg, db = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    ops.ln_fold_bwd(w, g, b, dwf, dbf, dw, dg, db)
    wr, gr, br = (t.double().detach().requires_grad_(True) for t in (w, g, b))
    ((wr * gr[None, :]) * dwf.double()).sum().backward(retain_graph=True)
    ((wr @ br) * dbf.double()).sum().backward()
    close(dw, wr.grad, 1e-5, 1e-5, "dW")
    close(dg, gr.grad, 1e-4, 1e-4, "dg")
    close(db, br.grad, 1e-4, 1e-4, "db")


def test_ln_bwd_with_residual_gradient(ops):
    """Affine-free LayerNorm backward + a gradient arriving on the residual path (attention)."""
    B, T, C = 2, 300, 256
    x, dy, dres = bf(rnd(B, T, C, seed=90)), bf(rnd(B, T, C, seed=91)), bf(rnd(B, T, C, seed=92))
    dx = torch.empty_like(x)
    ops.ln_film_bwd(dy, x, None, 0, dx, dres=dres, eps=1e-5)
    xr = x.float().requires_grad_(True)
    F.layer_norm(xr, (C,), eps=1e-5).backward(dy.float())
    close(dx, xr.grad + dres.float(), 2 ** -7, 1e-2, "ln bwd + dres")


@pytest.mark.parametrize("adapter", [False, True])
def test_stem_input_gradient(ops, adapter):
    """dxin of adp_stem_out_bwd (skip path, stored) + adp_stem_in_bwd (DownsampleItem path, added)
    against autograd of the same two ops."""
    B, T, f, c0 = 2, 1024, 1, 8
    cx, ca, co = (2, 2, 2) if adapter else (2, 0, 2)
    cin = cx + ca
    x, app = rnd(B, cx, T, seed=100), (rnd(B, ca, T, seed=101) if ca else None)
    w_dn, b_dn = rnd(c0, cin, f, seed=102) * 0.5, rnd(c0, seed=103)
    w_up, b_up = rnd(co, c0, 3, seed=104) * 0.3, rnd(co, seed=105)
    w_ad = rnd(co, cin, seed=106) * 0.5 if adapter else None
    b_ad = rnd(co, seed=107) if adapter else None
    gate = rnd(B, 8, seed=108)
    h = bf(rnd(B, T // f, c0, seed=109))
    dv = rnd(B, co, T, seed=110)
    dout = bf(rnd(B, T // f, c0, seed=111))
    dxin = torch.full((B, cin, T), float("nan"), device=DEV)
    dh = torch.empty_like(h)
    z = lambda *s: torch.zeros(*s, device=DEV)  # noqa: E731
    ops.stem_out_bwd(dv, h, x, w_up, b_up, gate, f, dh, z(co, c0, 3), z(co), z(B, 8), append=app,
                     w_adapt=w_ad, dw_adapt=z(co, cin) if adapter else None,
                     db_adapt=z(co) if adapter else None, dxin=dxin)
    ops.stem_in_bwd(dout, x, z(c0, cin, f), z(c0), f, append=app, w=w_dn, dxin=dxin)
    xin = (torch.cat([x, app], 1) if ca else x).detach().requires_grad_(True)
    skip = F.conv1d(xin, w_ad[:, :, None], b_ad) if adapter else xin
    down = F.conv1d(xin, w_dn, b_dn, stride=f)                      # [B, c0, T/f]
    ((skip * dv).sum() + (down * dout.float().transpose(1, 2)).sum()).backward()
    close(dxin, xin.grad, 1e-4, 1e-4, "dxin")


@pytest.mark.parametrize("B,T,n,k", [(2, 256, 64, 64), (2, 300, 128, 128), (1, 100, 32, 32), (4, 256, 1024, 1024),
                                     (3, 1000, 256, 512), (2, 4096, 8, 32), (1, 64, 512, 96)])
def test_wgrad_three_taps_fused(ops, B, T, n, k):
    """The three taps of a k=3 convolution in one launch (row-shifted views of one X box),
    accumulated into a non-zero dw."""
    g = bf(rnd(B, T, n, seed=11))
    x = bf(rnd(B, T, k, seed=12))
    dw0 = rnd(3, n, k, scale=(B * T) ** 0.5, seed=13)
    dw = dw0.clone()
    ops.wgrad(g, x, dw, n=n, k=k, off=-1, ntaps=3)
    xp = F.pad(x.float(), (0, 0, 1, 1))                      # zero rows at t = -1 and t = T
    for tap in range(3):
        ref = dw0[tap] + torch.einsum("btn,btk->nk", g.float(), xp[:, tap:tap + T])
        close(dw[tap], ref, 1e-2, 1e-3, f"fused wgrad tap {tap} B{B} T{T} n{n} k{k}")
