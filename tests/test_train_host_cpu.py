"""Host side of the training backward (training.py): the transposed / phase-folded dgrad packs,
the per-phase weight-gradient slots and folds, SkipCat and InjectChannels packs, the level-0
SkipCat unfold and the LayerNorm-folded projection packs.

The launch-sequence functions of training.py run here unchanged, with adp_conv_gemm, adp_wgrad
and adp_colsum replaced by float64 restatements of their contracts (rows outside [0, T) of each
batch element read as zero).  Every gradient is compared with torch.autograd of the PyTorch module
the composite replaces, in float64, to 1e-10 of its largest entry: the packing algebra is exact,
so any wrong tap, phase, slot, block or scale shows up far above round-off."""
import pytest
import torch
import torch.nn.functional as F

from audio_diffusion_pytorch_b200 import ops, training

D = torch.float64
TOL = 1e-10


def close(got, ref, what):
    err = float((got.double() - ref.double()).abs().max())
    scale = float(ref.double().abs().max())
    assert err <= TOL * scale, f"{what}: max abs err {err:.3e} vs ref max {scale:.3e}"


def rnd(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=D)


def shift_rows(x, off):
    """Row t of the result is x[:, t + off], zero outside [0, T) of each batch element."""
    T = x.shape[1]
    out = torch.zeros_like(x)
    if abs(off) < T:
        if off >= 0:
            out[:, :T - off] = x[:, off:]
        else:
            out[:, -off:] = x[:, :T + off]
    return out


def conv_gemm_f64(a, w, out, *, c_in, n_valid, taps=(0,), up_factor=0, bias=None, residual=None,
                  gate=None, stats=None, groups=8, block_n=0, gn=None):
    """adp_conv_gemm without the forward-only options: out[..., :n_valid] = sum_j
    a[t + taps[j], :c_in] @ W_j^T (+ bias) (+ residual); W_j = columns [j*c_in, (j+1)*c_in)."""
    assert up_factor <= 1 and gate is None and stats is None and gn is None
    assert w.shape[1] == len(taps) * c_in and n_valid <= w.shape[0]
    assert torch.count_nonzero(w[n_valid:]) == 0, "pack rows beyond n_valid must be zero padding"
    acc = sum(shift_rows(a[..., :c_in].double(), off) @ w[:n_valid, j * c_in:(j + 1) * c_in].double().t()
              for j, off in enumerate(taps))
    if bias is not None:
        acc = acc + bias.double()
    if residual is not None:              # may be `out` itself: read before the write
        acc = acc + residual[..., :n_valid].double()
    out[..., :n_valid] = acc.to(out.dtype)
    return out


def wgrad_f64(g, x, dw, *, n, k, off=0, g_col0=0, x_col0=0, ntaps=1):
    """adp_wgrad: dw[j] += sum_{b,t} g[b, t, g_col0 + n_] x[b, t + off + j, x_col0 + k_]."""
    assert g.shape[:2] == x.shape[:2]
    gs = g[..., g_col0:g_col0 + n].double()
    for j in range(ntaps):
        xs = shift_rows(x[..., x_col0:x_col0 + k].double(), off + j)
        (dw[j] if ntaps == 3 else dw).add_(torch.einsum("btn,btk->nk", gs, xs).to(dw.dtype))
    return dw


def colsum_f64(x, out, gate=None):
    assert gate is None
    out.add_(x.double().sum(dim=(0, 1)).to(out.dtype))
    return out


@pytest.fixture(autouse=True)
def f64_kernels(monkeypatch):
    monkeypatch.setattr(ops, "conv_gemm", conv_gemm_f64)
    monkeypatch.setattr(ops, "wgrad", wgrad_f64)
    monkeypatch.setattr(ops, "colsum", colsum_f64)
    with ops.pack_dtype(D):
        yield


def cl(t):
    """[B, C, T] -> channels-last [B, T, C]."""
    return t.transpose(1, 2).contiguous()


# ----------------------------------------------------------------------------- upsample
@pytest.mark.parametrize("f", [2, 3, 4, 8])
@pytest.mark.parametrize("B,Tl", [(2, 1), (2, 2), (3, 5)])
def test_upsample_backward(f, B, Tl):
    """Nearest-upsample(f) -> Conv1d(k=3, p=1), C != Co: dgrad through pack_upsample_dgrad, the
    per-phase wgrad slots, fold_upsample_wgrad and the bias column sum.  At Tl <= 2 every
    low-res row is a boundary row; f = 3 and 8 have interior phases."""
    C, Co = 16, 8
    x = rnd(B, C, Tl, seed=1).requires_grad_()
    w = rnd(Co, C, 3, seed=2).requires_grad_()
    b = rnd(Co, seed=3).requires_grad_()
    dy = rnd(B, Co, Tl * f, seed=4)
    F.conv1d(F.interpolate(x, scale_factor=f, mode="nearest"), w, b, padding=1).backward(dy)
    gw, db = torch.zeros(f, 2, Co, C, dtype=D), torch.zeros(Co, dtype=D)
    dx = torch.full((B, Tl, C), float("nan"), dtype=D)
    training.upsample_bwd(cl(dy), cl(x.detach()), training.pack_upsample_dgrad(w, f), gw, db, dx, f)
    close(dx, cl(x.grad), "d x")
    close(training.fold_upsample_wgrad(gw, f), w.grad, "d weight")
    close(db, b.grad, "d bias")


@pytest.mark.parametrize("B,T", [(2, 1), (3, 7)])
def test_upsample_f1_backward(B, T):
    """f = 1 up conv (a plain k=3 conv, Co != C): pack_conv_dgrad + the fused 3-tap wgrad."""
    C, Co = 24, 40
    x = rnd(B, C, T, seed=5).requires_grad_()
    w = rnd(Co, C, 3, seed=6).requires_grad_()
    b = rnd(Co, seed=7).requires_grad_()
    dy = rnd(B, Co, T, seed=8)
    F.conv1d(x, w, b, padding=1).backward(dy)
    gw, db = torch.zeros(3, Co, C, dtype=D), torch.zeros(Co, dtype=D)
    dx = torch.full((B, T, C), float("nan"), dtype=D)
    training.upsample_bwd(cl(dy), cl(x.detach()), ops.pack_conv_dgrad(w.detach()), gw, db, dx, 1)
    close(dx, cl(x.grad), "d x")
    close(gw.permute(1, 2, 0), w.grad, "d weight")       # [tap][co][ci] -> PyTorch layout
    close(db, b.grad, "d bias")


# --------------------------------------------------------------------------- downsample
@pytest.mark.parametrize("f", [2, 4])
@pytest.mark.parametrize("ci", [8, 32])
@pytest.mark.parametrize("B,Tl", [(2, 1), (3, 5)])
def test_downsample_backward(f, ci, B, Tl):
    """Conv1d(ci, C, k = stride = f): pack_down_dgrad writes the [B, T/f, f*ci] view with the skip
    gradient as residual; the [co][tap][ci] weight-gradient accumulator maps to PyTorch layout."""
    C = 16
    x = rnd(B, ci, Tl * f, seed=9).requires_grad_()
    w = rnd(C, ci, f, seed=10).requires_grad_()
    b = rnd(C, seed=11).requires_grad_()
    dy = rnd(B, C, Tl, seed=12)
    d_skip = rnd(B, Tl * f, ci, seed=13)
    F.conv1d(x, w, b, stride=f).backward(dy)
    gw, db = torch.zeros(C, f * ci, dtype=D), torch.zeros(C, dtype=D)
    d_xin = torch.full((B, Tl * f, ci), float("nan"), dtype=D)
    calls = []
    training.downsample_bwd(cl(dy), cl(x.detach()), training.pack_down_dgrad(w), gw, db, d_xin, d_skip, f,
                            wgrad_done=lambda: calls.append(gw.clone()))
    close(d_xin, cl(x.grad) + d_skip, "d x + d skip")
    close(gw.view(C, f, ci).permute(0, 2, 1), w.grad, "d weight")
    close(db, b.grad, "d bias")
    assert len(calls) == 1 and torch.equal(calls[0], gw), "wgrad_done must follow the weight gradient"


# ------------------------------------------------------------------------------ SkipCat
@pytest.mark.parametrize("Co,rp", [(8, 2), (32, 1)])
@pytest.mark.parametrize("B,T", [(2, 2), (3, 10)])
def test_skipcat_backward(Co, rp, B, T):
    """out = Conv1d(2*Co, Co, 1)(cat([skip * 2^-0.5, y])) with rp positions per GEMM row:
    block-diagonal dgrad packs and the diagonal-block extraction of the weight gradient."""
    skip = rnd(B, Co, T, seed=14).requires_grad_()
    y = rnd(B, Co, T, seed=15).requires_grad_()
    w = rnd(Co, 2 * Co, 1, seed=16).requires_grad_()
    b = rnd(Co, seed=17).requires_grad_()
    d_out = rnd(B, Co, T, seed=18)
    F.conv1d(torch.cat([skip * 2 ** -0.5, y], 1), w, b).backward(d_out)
    wd_c1, wd_c2 = training.pack_skipcat_dgrad(w, rp)
    gw, db = torch.full((Co, 2 * Co), float("nan"), dtype=D), torch.zeros(Co, dtype=D)
    blk1, blk2 = torch.zeros(rp * Co, rp * Co, dtype=D), torch.zeros(rp * Co, rp * Co, dtype=D)
    dys, d_skip = torch.empty(B, T, Co, dtype=D), torch.empty(B, T, Co, dtype=D)
    training.skipcat_bwd(cl(d_out), cl(skip.detach()), cl(y.detach()), wd_c1, wd_c2, gw, db, blk1, blk2,
                         dys, d_skip, rp)
    close(gw, w.grad[:, :, 0], "d weight")
    close(db, b.grad, "d bias")
    close(dys, cl(y.grad), "d y")
    close(d_skip, cl(skip.grad), "d skip")


@pytest.mark.parametrize("adapter", [False, True])
def test_level0_skipcat_unfold(adapter):
    """Level-0 SkipCat: the stem kernels see the merge folded into the up conv and the skip
    adapter; the unfold turns the folded gradients into merge / up / adapter gradients, against
    autograd of merge(cat([adapter(x) * 2^-0.5, up(h)]))."""
    B, T, C, Co = 2, 9, 8, 2
    Ci = 3 if adapter else Co
    torch.manual_seed(19)
    merge = torch.nn.Conv1d(2 * Co, Co, 1).to(D)
    up = torch.nn.Conv1d(C, Co, 3, padding=1).to(D)
    ad = torch.nn.Conv1d(Ci, Co, 1).to(D) if adapter else None
    x, h, dv = rnd(B, Ci, T, seed=20), rnd(B, C, T, seed=21), rnd(B, Co, T, seed=22)
    skip = ad(x) if adapter else x
    merge(torch.cat([skip * 2 ** -0.5, up(h)], 1)).backward(dv)
    # the folded weights the stem kernels run (B200UNet._compute_packed), as autograd leaves
    wm = merge.weight.detach()[:, :, 0]
    wc1, wc2 = wm[:, :Co] * 2 ** -0.5, wm[:, Co:]
    fw_up = torch.einsum("om,mck->ock", wc2, up.weight.detach()).requires_grad_()
    fb_up = (wc2 @ up.bias.detach() + merge.bias.detach()).requires_grad_()
    fw_ad = (wc1 @ ad.weight.detach()[:, :, 0] if adapter else wc1).requires_grad_()
    fb_ad = (wc1 @ ad.bias.detach() if adapter else torch.zeros(Co, dtype=D)).requires_grad_()
    (F.conv1d(x, fw_ad[:, :, None], fb_ad) + F.conv1d(h, fw_up, fb_up, padding=1)).backward(dv)
    g = training.unfold_level0_grads(merge.weight, up.weight, up.bias, fw_up.grad, fb_up.grad, fw_ad.grad,
                                     fb_ad.grad, ad.weight if adapter else None, ad.bias if adapter else None)
    mods = {"merge": merge, "up": up, **({"adapter": ad} if adapter else {})}
    assert sorted(g) == sorted(f"{m}.{p}" for m in mods for p in ("weight", "bias"))
    for name, m in mods.items():
        close(g[name + ".weight"].reshape(m.weight.shape), m.weight.grad, name + ".weight")
        close(g[name + ".bias"], m.bias.grad, name + ".bias")


# ------------------------------------------------------------------------ InjectChannels
@pytest.mark.parametrize("n_ctx", [5, 20])
def test_inject_channels_backward(n_ctx):
    """out = Conv1d(C + n_ctx, C, 1)(cat([x, ctx])) + x with the context zero-padded to a
    multiple of 16 channels; the context gradient is ADDED to what dctx already holds."""
    B, T, C = 2, 6, 32
    ctx_pad = ops.round_up(n_ctx, 16)
    x = rnd(B, C, T, seed=23).requires_grad_()
    ctx = rnd(B, n_ctx, T, seed=24).requires_grad_()
    w = rnd(C, C + n_ctx, 1, seed=25).requires_grad_()
    b = rnd(C, seed=26).requires_grad_()
    d_out = rnd(B, C, T, seed=27)
    (F.conv1d(torch.cat([x, ctx], 1), w, b) + x).backward(d_out)
    ctxb = torch.zeros(B, T, ctx_pad, dtype=D)
    ctxb[..., :n_ctx] = cl(ctx.detach())
    prior = rnd(B, T, ctx_pad, seed=28)                 # gradients of the depth's earlier items
    dctxb = prior.clone()
    gw, db = torch.zeros(C, C + n_ctx, dtype=D), torch.zeros(C, dtype=D)
    dx = torch.full((B, T, C), float("nan"), dtype=D)
    wd_x, wd_c = training.pack_inject_dgrad(w, C, ctx_pad)
    training.inject_bwd(cl(d_out), cl(x.detach()), ctxb, dctxb, wd_x, wd_c, gw, db, dx, n_ctx)
    close(dx, cl(x.grad), "d x")
    close(dctxb[..., :n_ctx], prior[..., :n_ctx] + cl(ctx.grad), "d ctx (accumulated)")
    assert torch.equal(dctxb[..., n_ctx:], prior[..., n_ctx:]), "padding channels of d ctx changed"
    close(gw, w.grad[:, :, 0], "d weight")
    close(db, b.grad, "d bias")


# ---------------------------------------------------------------- LayerNorm-folded q / kv
@pytest.mark.parametrize("fused", [True, False])
def test_ln_folded_projection_dgrad(fused):
    """Attention projections run on xn = LayerNorm(x) without affine, the norms' gamma / beta
    folded into the weights: the dgrad packs must give d xn of q = (xn g1 + b1) Wq^T and
    kv = (xn g2 + b2) Wkv^T.  fused: self-attention's one [C, 3*mid] pack; else cross-attention's
    separate q and kv packs."""
    B, T, C, mid = 2, 5, 24, 32
    xn = rnd(B, T, C, seed=29).requires_grad_()
    wq, wkv = rnd(mid, C, seed=30), rnd(2 * mid, C, seed=31)
    g1, b1, g2, b2 = rnd(C, seed=32), rnd(C, seed=33), rnd(C, seed=34), rnd(C, seed=35)
    dq, dkv = rnd(B, T, mid, seed=36), rnd(B, T, 2 * mid, seed=37)
    q = (xn * g1 + b1) @ wq.t()
    kv = (xn * g2 + b2) @ wkv.t()
    ((q * dq).sum() + (kv * dkv).sum()).backward()
    dxn = torch.empty(B, T, C, dtype=D)
    if fused:
        wd = training.pack_ln_folded_dgrad((wq, g1), (wkv, g2))
        ops.conv_gemm(torch.cat([dq, dkv], -1), wd, dxn, c_in=3 * mid, n_valid=C)
    else:
        dxk = torch.empty(B, T, C, dtype=D)
        ops.conv_gemm(dq, training.pack_ln_folded_dgrad((wq, g1)), dxn, c_in=mid, n_valid=C)
        ops.conv_gemm(dkv, training.pack_ln_folded_dgrad((wkv, g2)), dxk, c_in=2 * mid, n_valid=C)
        dxn += dxk
    close(dxn, xn.grad, "d xn")
