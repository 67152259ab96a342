"""Stage tests of the training backward: each launch sequence of training.py (the code the
backward program runs) on random bf16 inputs, against torch.autograd of the fp32 PyTorch
restatement of the module it differentiates, on the same bf16-rounded inputs and weights.

Bounds as in test_bwd_ops_gpu.py: bf16 gradient outputs 2^-6 relative + 2e-3 of the largest
entry; fp32 parameter-gradient accumulators 1e-2 of the largest entry.  Every family runs at
README level shapes plus two edge shapes: a low-resolution length <= 8 with B >= 2 (boundary rows
carry a large share of every gradient) and a ragged length (not a multiple of the 128-row tile)
with B = 3 (tiles that span two batch elements)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

S_CAT = 2 ** -0.5


def bf(t):
    return t.to(torch.bfloat16)


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


class Checks:
    """Compares every output of a stage first, then fails with the list of violations."""

    def __init__(self, name):
        self.name, self.bad = name, []

    def _close(self, got, ref, rtol, atol_frac, what):
        got, ref = got.double(), ref.double()
        err = (got - ref).abs().max().item()
        scale = ref.abs().max().item()
        print(f"{self.name} {what}: max abs err {err:.4e} (ref max {scale:.3e}, "
              f"err/max {err / max(scale, 1e-30):.2e})")
        if not err <= rtol * scale + atol_frac * scale + 1e-12:
            self.bad.append(f"{what}: {err:.3e} vs ref max {scale:.3e}")

    def act(self, got, ref, what):        # bf16 gradient outputs
        self._close(got, ref, 2 ** -6, 2e-3, what)

    def acc(self, got, ref, what):        # fp32 parameter-gradient accumulators
        self._close(got, ref, 1e-2, 0.0, what)

    def done(self):
        assert not self.bad, f"{self.name}: " + "; ".join(self.bad)


def cl(t):
    """[B, C, T] -> channels-last [B, T, C]."""
    return t.transpose(1, 2).contiguous()


def leaf(t):
    return t.float().detach().requires_grad_(True)


@pytest.fixture(scope="module")
def tr():
    from audio_diffusion_pytorch_b200 import ops, training
    ops.device_check()
    return training


@pytest.fixture(scope="module")
def ops():
    from audio_diffusion_pytorch_b200 import ops
    return ops


def zeros(*shape, dtype=torch.float32):
    return torch.zeros(*shape, dtype=dtype, device=DEV)


def nan_act(*shape):
    return torch.full(shape, float("nan"), dtype=torch.bfloat16, device=DEV)


# ----------------------------------------------------------------------------- upsample
@pytest.mark.parametrize("B,Tl,C,Co,f", [
    (2, 256, 32, 8, 4), (2, 256, 64, 32, 4), (2, 128, 128, 64, 4), (2, 128, 256, 128, 2),
    (2, 64, 512, 512, 2), (2, 64, 1024, 512, 2),      # README levels
    (2, 128, 128, 64, 1),                             # f = 1 level
    (2, 3, 32, 8, 4), (2, 5, 512, 512, 2), (2, 6, 64, 32, 1),          # low-res length <= 8
    (3, 203, 32, 8, 4), (3, 141, 256, 128, 2), (3, 203, 128, 64, 1),   # ragged, B = 3
])
def test_upsample_stage(tr, ops, B, Tl, C, Co, f):
    """training.upsample_bwd against autograd of Conv1d(k=3, p=1)(Upsample(nearest, f)(x))."""
    x = bf(rnd(B, Tl, C, seed=1))
    w = bf(rnd(Co, C, 3, scale=(3 * C) ** -0.5, seed=2)).float()
    dys = bf(rnd(B, Tl * f, Co, seed=3))
    xr, wr, br = leaf(x), leaf(w), leaf(zeros(Co))
    up = F.interpolate(xr.transpose(1, 2), scale_factor=f, mode="nearest") if f > 1 else xr.transpose(1, 2)
    F.conv1d(up, wr, br, padding=1).backward(dys.float().transpose(1, 2))
    dx = nan_act(B, Tl, C)
    db = zeros(Co)
    if f > 1:
        gw = zeros(f, 2, Co, C)
        tr.upsample_bwd(dys, x, tr.pack_upsample_dgrad(w, f), gw, db, dx, f)
        dw = tr.fold_upsample_wgrad(gw, f)
    else:
        gw = zeros(3, Co, C)
        tr.upsample_bwd(dys, x, ops.pack_conv_dgrad(w), gw, db, dx, f)
        dw = gw.permute(1, 2, 0)
    ck = Checks(f"up B{B} Tl{Tl} C{C} Co{Co} f{f}")
    ck.act(dx, xr.grad, "dx")
    ck.acc(dw, wr.grad, "dw")
    ck.acc(db, br.grad, "db")
    ck.done()


# --------------------------------------------------------------------------- downsample
@pytest.mark.parametrize("B,Tl,ci,C,f", [
    (2, 256, 8, 32, 4), (2, 256, 32, 64, 4), (2, 128, 64, 128, 4), (2, 64, 512, 512, 2),
    (2, 64, 1024, 1024, 2),                           # kdim = f * ci: 32, 128, 256, 1024, 2048
    (2, 3, 8, 32, 4), (2, 5, 512, 512, 2),            # low-res length <= 8
    (3, 203, 8, 32, 4), (3, 141, 512, 512, 2),        # ragged, B = 3
])
def test_downsample_stage(tr, B, Tl, ci, C, f):
    """training.downsample_bwd against autograd of Conv1d(ci, C, k = stride = f); the level
    input's gradient adds the skip path's gradient through the dgrad GEMM's residual."""
    x = bf(rnd(B, Tl * f, ci, seed=4))
    w = bf(rnd(C, ci, f, scale=(f * ci) ** -0.5, seed=5)).float()
    d = bf(rnd(B, Tl, C, seed=6))
    d_skip = bf(rnd(B, Tl * f, ci, seed=7))
    xr, wr, br = leaf(x), leaf(w), leaf(zeros(C))
    F.conv1d(xr.transpose(1, 2), wr, br, stride=f).backward(d.float().transpose(1, 2))
    gw, db = zeros(C, f * ci), zeros(C)
    d_xin = nan_act(B, Tl * f, ci)
    tr.downsample_bwd(d, x, tr.pack_down_dgrad(w), gw, db, d_xin, d_skip, f)
    ck = Checks(f"down B{B} Tl{Tl} kdim{f * ci} C{C}")
    ck.act(d_xin, xr.grad + d_skip.float(), "dx + dskip")
    ck.acc(gw.view(C, f, ci).permute(0, 2, 1), wr.grad, "dw")
    ck.acc(db, br.grad, "db")
    ck.done()


# ------------------------------------------------------------------------------ SkipCat
@pytest.mark.parametrize("B,T,Co", [
    (2, 1024, 8), (2, 512, 32), (2, 256, 64),         # rp = 2, 1, 1
    (2, 4, 8), (2, 6, 64),                            # length <= 8
    (3, 406, 8), (3, 203, 32),                        # ragged, B = 3
])
def test_skipcat_stage(tr, B, T, Co):
    """training.skipcat_bwd against autograd of Conv1d(2 Co, Co, 1)(cat([skip * 2^-0.5, y]))."""
    rp = max(1, 16 // Co)
    skip, y = bf(rnd(B, T, Co, seed=8)), bf(rnd(B, T, Co, seed=9))
    w = bf(rnd(Co, 2 * Co, 1, scale=(2 * Co) ** -0.5, seed=10)).float()
    d_out = bf(rnd(B, T, Co, seed=11))
    sr, yr, wr, br = leaf(skip), leaf(y), leaf(w), leaf(zeros(Co))
    F.conv1d(torch.cat([sr * S_CAT, yr], 2).transpose(1, 2), wr, br).backward(d_out.float().transpose(1, 2))
    wd_c1, wd_c2 = tr.pack_skipcat_dgrad(w, rp)
    gw, db = torch.full((Co, 2 * Co), float("nan"), device=DEV), zeros(Co)
    blk1, blk2 = zeros(rp * Co, rp * Co), zeros(rp * Co, rp * Co)
    dys, d_skip = nan_act(B, T, Co), nan_act(B, T, Co)
    tr.skipcat_bwd(d_out, skip, y, wd_c1, wd_c2, gw, db, blk1, blk2, dys, d_skip, rp)
    ck = Checks(f"skipcat B{B} T{T} Co{Co} rp{rp}")
    ck.act(dys, yr.grad, "dy")
    ck.act(d_skip, sr.grad, "dskip")
    ck.acc(gw, wr.grad[:, :, 0], "dw")
    ck.acc(db, br.grad, "db")
    ck.done()


# ------------------------------------------------------------------------ InjectChannels
@pytest.mark.parametrize("B,T,C,n_ctx", [
    (2, 512, 64, 20), (2, 256, 512, 16),
    (2, 5, 64, 20),                                   # length <= 8
    (3, 203, 128, 24),                                # ragged, B = 3
])
def test_inject_stage(tr, ops, B, T, C, n_ctx):
    """training.inject_bwd against autograd of Conv1d(C + n_ctx, C, 1)(cat([x, ctx])) + x.  The
    context gradient buffer starts pre-filled (the gradients of the depth's earlier items): the
    dgrad GEMM adds into it in place (its residual is its output)."""
    ctx_pad = ops.round_up(n_ctx, 16)
    x = bf(rnd(B, T, C, seed=12))
    ctxb = torch.zeros(B, T, ctx_pad, dtype=torch.bfloat16, device=DEV)
    ctxb[..., :n_ctx] = bf(rnd(B, T, n_ctx, seed=13))
    w = bf(rnd(C, C + n_ctx, 1, scale=(C + n_ctx) ** -0.5, seed=14)).float()
    d_out = bf(rnd(B, T, C, seed=15))
    prior = bf(rnd(B, T, ctx_pad, seed=16))
    xr, cr, wr, br = leaf(x), leaf(ctxb[..., :n_ctx]), leaf(w), leaf(zeros(C))
    y = F.conv1d(torch.cat([xr, cr], 2).transpose(1, 2), wr, br).transpose(1, 2) + xr
    y.backward(d_out.float())
    dctxb = prior.clone()
    gw, db = zeros(C, C + n_ctx), zeros(C)
    dx = nan_act(B, T, C)
    wd_x, wd_c = tr.pack_inject_dgrad(w, C, ctx_pad)
    tr.inject_bwd(d_out, x, ctxb, dctxb, wd_x, wd_c, gw, db, dx, n_ctx)
    ck = Checks(f"inject B{B} T{T} C{C} n_ctx{n_ctx}")
    ck.act(dx, xr.grad, "dx")
    ck.act(dctxb[..., :n_ctx], prior[..., :n_ctx].float() + cr.grad, "dctx (accumulated)")
    ck.acc(gw, wr.grad[:, :, 0], "dw")
    ck.acc(db, br.grad, "db")
    ck.done()
    assert torch.equal(dctxb[..., n_ctx:], prior[..., n_ctx:]), "padding channels of d ctx changed"


# ----------------------------------------------------------- ResnetItem + ModulationItem
def stats_of(y, groups):
    B, T, Cc = y.shape
    yg = y.double().reshape(B, T, groups, Cc // groups)
    return torch.stack([yg.sum(dim=(1, 3)), (yg * yg).sum(dim=(1, 3))], dim=-1).contiguous()


_ITEM = [(2, 512, 64, 8), (2, 256, 512, 8), (2, 5, 64, 8), (3, 203, 512, 8),
         (2, 512, 64, 1), (2, 512, 64, 4), (3, 203, 512, 1), (3, 203, 512, 4)]


@pytest.mark.parametrize("mod", [False, True])
@pytest.mark.parametrize("B,T,C,G", _ITEM,
                         ids=["-".join(str(v) for v in c[:3]) + ("" if c[3] == 8 else f"-g{c[3]}") for c in _ITEM])
def test_resnet_item_stage(tr, ops, B, T, C, G, mod):
    """training.resnet_item_bwd (the C >= 32 item path) against autograd of
    GroupNorm -> SiLU -> conv3 -> GroupNorm -> SiLU -> conv3 + x (-> LayerNorm (1 + scale) + shift).
    The saved activations (a1, h, a2, rr) are the bf16-rounded values of that fp32 forward, as
    the training forward stores them."""
    gn_eps, ln_eps = 1e-5, 1e-6
    x = bf(rnd(B, T, C, seed=17) * 1.5 + 0.3)
    w1 = bf(rnd(C, C, 3, scale=(3 * C) ** -0.5, seed=18)).float()
    w2 = bf(rnd(C, C, 3, scale=(3 * C) ** -0.5, seed=19)).float()
    b1, b2 = rnd(C, seed=20) * 0.1, rnd(C, seed=21) * 0.1
    g1, be1 = rnd(C, seed=22) * 0.2 + 1.0, rnd(C, seed=23) * 0.2
    g2, be2 = rnd(C, seed=24) * 0.2 + 1.0, rnd(C, seed=25) * 0.2
    ss = rnd(B, 2 * C, seed=26) * 0.3
    dy = bf(rnd(B, T, C, seed=27))

    def gn_silu(t, g, b):
        return F.silu(F.group_norm(t.transpose(1, 2), G, g, b, gn_eps))          # [B, C, T]

    def conv(a, w, b):
        return F.conv1d(a, w, b, padding=1).transpose(1, 2)                      # [B, T, C]

    # reference: one fp32 autograd graph through the whole item
    P = [leaf(t) for t in (x, w1, w2, b1, b2, g1, be1, g2, be2, ss)]
    xr, w1r, w2r, b1r, b2r, g1r, be1r, g2r, be2r, ssr = P
    hr = conv(gn_silu(xr, g1r, be1r), w1r, b1r)
    rrr = conv(gn_silu(hr, g2r, be2r), w2r, b2r) + xr
    out = F.layer_norm(rrr, (C,), eps=ln_eps) * (1 + ssr[:, None, :C]) + ssr[:, None, C:] if mod else rrr
    out.backward(dy.float())
    # the bf16 activations the forward saves (channels-last, contiguous)
    with torch.no_grad():
        a1 = bf(gn_silu(x.float(), g1, be1)).transpose(1, 2).contiguous()
        h = bf(conv(a1.float().transpose(1, 2), w1, b1)).contiguous()
        a2 = bf(gn_silu(h.float(), g2, be2)).transpose(1, 2).contiguous()
        rr = bf(conv(a2.float().transpose(1, 2), w2, b2) + x.float()).contiguous()
    gw1, gw2 = zeros(3, C, C), zeros(3, C, C)
    dgn1, dgn2 = (zeros(C), zeros(C)), (zeros(C), zeros(C))
    db1, db2 = zeros(C), zeros(C)
    S1, S2 = zeros(B, G, 2, dtype=torch.float64), zeros(B, G, 2, dtype=torch.float64)
    work = tuple(nan_act(B, T, C) for _ in range(5))
    dss = zeros(B, 2 * C)
    film = (ss, dss, 2 * C, ln_eps) if mod else None
    dx = tr.resnet_item_bwd(dy, x, h, rr, a1, a2, stats_of(x, G), stats_of(h, G), (g1, be1), (g2, be2),
                            ops.pack_conv_dgrad(w1), ops.pack_conv_dgrad(w2), gw1, gw2, dgn1, dgn2, db1, db2,
                            S1, S2, work, G, film=film)
    ck = Checks(f"item B{B} T{T} C{C} G{G} mod{int(mod)}")
    ck.act(dx, xr.grad, "dx")
    ck.acc(gw1.permute(1, 2, 0), w1r.grad, "dw1")
    ck.acc(gw2.permute(1, 2, 0), w2r.grad, "dw2")
    ck.acc(db1, b1r.grad, "db1")
    ck.acc(db2, b2r.grad, "db2")
    ck.acc(dgn1[0], g1r.grad, "dgamma1")
    ck.acc(dgn1[1], be1r.grad, "dbeta1")
    ck.acc(dgn2[0], g2r.grad, "dgamma2")
    ck.acc(dgn2[1], be2r.grad, "dbeta2")
    if mod:
        ck.acc(dss, ssr.grad, "d scale/shift")
    ck.done()
