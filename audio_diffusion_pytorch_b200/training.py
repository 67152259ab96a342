"""Differentiable execution of the CUDA U-Net: the training step of the hot path
(reference diffusion.py:82-95, `loss = model(x); loss.backward()`) and the generic
`v = net(x, sigma, ...)` with autograd support (custom `loss_fn` / `diffusion_t`,
reference models.py:28,37 and tests/testcustomloss.py:28).

Two entry points, ONE hand-written backward program:

* `fused_v_loss`  -- `F.mse_loss(net(alpha*x + beta*noise, sigma), alpha*noise - beta*x)` with the
  noising fused into the first kernel and the MSE + dL/dv into the last one.
* `differentiable_forward` -- returns v wired into autograd; backward receives dL/dv.

The backward program = data-gradient GEMMs (adp_conv_gemm on transposed packed weights),
weight-gradient GEMMs (adp_wgrad), GroupNorm / LayerNorm-FiLM / stem backward kernels, and for
AttentionItem / CrossAttentionItem the flash-attention backward (adp_attention_bwd) plus the
LayerNorm-folded projection backward (adp_ln_fold_bwd).  Every parameter receives its fp32
gradient in PyTorch layout, so optimizers, gradient clipping and DistributedDataParallel work
unchanged; gradients w.r.t. `append_channels` (DiffusionVocoder's `to_flat`), `embedding` (the
classifier-free-guidance mask embedding) and `x` flow back as well.

Only the 3 tiny time-embedding linears run as PyTorch ops (their autograd supplies d(features);
[B,1024] matrices, < 0.1 % of the step).

One plan (static activation buffers + two CUDA graphs) exists per input shape: a second forward
on the same shape before the first one's backward would overwrite the saved activations, so each
forward stamps a generation number and a stale backward raises instead of returning the wrong
gradients.
"""
from math import pi
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F
from torch import Tensor

from . import ops
from .unet import B200UNet, _ForwardWalk, _Graphed, _Plan, _refreshed


class _TrainPlan:
    def __init__(self):
        self.forward = _Plan(early_weights=False)
        self.fwd = self.forward.prog     # the forward's launch list (the same list object)
        self.backward = _Graphed(lambda: self.backward_program(), early_weights=False)
        self.refresh_graph = None
        self.generation = 0
        self.on_mark = None          # callable(interval) while a gradient all-reduce is overlapped
        self.seg_graphs = None       # backward captured as segments cut at the flush marks
        self.mark_log: List = []     # intervals in execution order (recorded on the eager run)

    def mark(self, interval) -> None:
        """A contiguous range [start, end) of the gradient arena is final (see level())."""
        if self.on_mark is not None:
            self.on_mark(interval)


def _zeros(shape, dev, dtype=torch.float32):
    return torch.zeros(shape, device=dev, dtype=dtype)


S_CAT = 2 ** -0.5          # SkipCat scales the skip branch before the 1x1 merge conv


def _master(w: Tensor) -> Tensor:
    """fp32 copy of a weight for the host-side packers (an fp64 weight stays fp64, so the
    packing algebra can be checked exactly on the CPU)."""
    w = w.detach()
    return w if w.dtype == torch.float64 else w.float()


# ------------------------------------------------------------------ host packers and folds
def pack_ln_folded_dgrad(*pairs) -> Tensor:
    """Data-gradient pack of projections run with their input LayerNorm's affine folded in:
    pairs (W_i [N_i, C], gamma_i [C]) -> pack of cat_i(W_i diag(gamma_i))^T, [C, sum N_i]."""
    wf = torch.cat([_master(w) * _master(g)[None, :] for w, g in pairs], 0)
    return ops.pack_linear(wf.t().contiguous())


def pack_upsample_dgrad(w: Tensor, f: int) -> Tensor:
    """Upsample conv (nearest x f, then Conv1d k=3 p=1, w [Co, C, 3]) backward w.r.t. its low-res
    input: one 3-tap GEMM over the [B, T, f*Co] view of the output gradient.  Tap j reads
    low-res row q + j - 1; column block p holds the transposed phase-p weights."""
    Co, C = w.shape[0], w.shape[1]
    w = _master(w)
    w0, w1, w2 = w[:, :, 0], w[:, :, 1], w[:, :, 2]
    wd = torch.zeros(3, C, f * Co, dtype=w.dtype, device=w.device)
    wd[2, :, 0:Co] = w0.t()                          # forward off -1 (phase 0, slot 0)
    wd[1, :, 0:Co] = (w1 + w2).t()
    wd[1, :, (f - 1) * Co:f * Co] = (w0 + w1).t()
    wd[0, :, (f - 1) * Co:f * Co] = w2.t()          # forward off +1 (last phase, slot 1)
    for p_ in range(1, f - 1):
        wd[1, :, p_ * Co:(p_ + 1) * Co] = (w0 + w1 + w2).t()
    return ops._pad_rows(wd.permute(1, 0, 2).reshape(C, 3 * f * Co), ops.round_up(C, 16))


def upsample_wgrad_slots(f: int):
    """[(phase, slot, row offset)] of the per-phase weight-gradient GEMMs of an upsample conv
    (f >= 2): slot s of phase p multiplies the same low-res input rows as the forward phase
    weights in slot s (see ops.pack_upsample_conv)."""
    out = []
    for p_ in range(f):
        slots = [(0, -1), (1, 0)] if p_ == 0 else ([(0, 0), (1, 1)] if p_ == f - 1 else [(0, 0)])
        out += [(p_, s_, off) for s_, off in slots]
    return out


def fold_upsample_wgrad(gwc: Tensor, f: int) -> Tensor:
    """Per-phase, per-slot gradients gwc [f, 2, Co, C] -> the conv's weight gradient [Co, C, 3]."""
    g0 = gwc[0, 0] + gwc[f - 1, 0]
    g1 = gwc[0, 1] + gwc[f - 1, 0]
    g2 = gwc[0, 1] + gwc[f - 1, 1]
    for p_ in range(1, f - 1):
        g0, g1, g2 = g0 + gwc[p_, 0], g1 + gwc[p_, 0], g2 + gwc[p_, 0]
    return torch.stack([g0, g1, g2], dim=-1)


def pack_down_dgrad(w: Tensor) -> Tensor:
    """Downsample conv (k = stride = f, w [C, ci, f]) backward w.r.t. its input: a linear GEMM
    writing the [B, T/f, f*ci] view; pack rows are ordered [tap][ci]."""
    C, ci, f = w.shape
    return ops.pack_linear(w.detach().permute(0, 2, 1).reshape(C, f * ci).t().contiguous())


def pack_skipcat_dgrad(w_merge: Tensor, rp: int):
    """SkipCat merge (1x1 conv over cat([skip * S_CAT, y]), w_merge [Co, 2*Co, 1]) backward:
    (pack for d skip, pack for d y), block-diagonal over rp positions per row."""
    Co = w_merge.shape[0]
    wm = _master(w_merge)[:, :, 0]
    wd_c1 = ops.pack_linear(torch.block_diag(*[wm[:, :Co].t() * S_CAT] * rp).contiguous())
    wd_c2 = ops.pack_linear(torch.block_diag(*[wm[:, Co:].t()] * rp).contiguous())
    return wd_c1, wd_c2


def skipcat_weight_grad(blk1: Tensor, blk2: Tensor, rp: int, Co: int) -> Tensor:
    """Weight gradients of the paired-position merge GEMMs [rp*Co, rp*Co] -> the merge conv's
    [Co, 2*Co]: the diagonal blocks (same position in and out) sum to the 1x1 conv's gradient."""
    g1 = blk1.view(rp, Co, rp, Co).diagonal(dim1=0, dim2=2).sum(-1) * S_CAT
    g2 = blk2.view(rp, Co, rp, Co).diagonal(dim1=0, dim2=2).sum(-1)
    return torch.cat([g1, g2], dim=1)


def unfold_level0_grads(w_merge: Tensor, w_up: Tensor, b_up: Tensor, dw_up: Tensor, db_up: Tensor,
                        dwa: Tensor, dba: Tensor, w_ad: Optional[Tensor] = None,
                        b_ad: Optional[Tensor] = None) -> Dict[str, Tensor]:
    """Level-0 SkipCat runs in the stem kernels with the merge conv folded into the upsample conv
    (Wc2 W_up, Wc2 b_up + b_merge) and the skip adapter (S_CAT Wc1 W_ad, ...).  From the
    gradients of the folded weights (dw_up [Co, C, 3], db_up, dwa [Co, Ci], dba) recover those of
    merge / up / adapter, keyed by module and parameter name."""
    Co = w_merge.shape[0]
    wm = _master(w_merge)[:, :, 0]
    wc1, wc2 = wm[:, :Co], wm[:, Co:]
    w_up, b_up = _master(w_up), _master(b_up)
    g = {"up.weight": torch.einsum("om,ock->mck", wc2, dw_up), "up.bias": wc2.t() @ db_up}
    d_wc2 = torch.einsum("ock,mck->om", dw_up, w_up) + torch.outer(db_up, b_up)
    if w_ad is not None:
        w_ad, b_ad = _master(w_ad)[:, :, 0], _master(b_ad)
        g["adapter.weight"] = S_CAT * (wc1.t() @ dwa)
        g["adapter.bias"] = S_CAT * (wc1.t() @ dba)
        d_wc1 = S_CAT * (dwa @ w_ad.t() + torch.outer(dba, b_ad))
    else:
        d_wc1 = S_CAT * dwa
    g["merge.weight"] = torch.cat([d_wc1, d_wc2], dim=1)
    g["merge.bias"] = db_up.clone()
    return g


def pack_inject_dgrad(w: Tensor, C: int, ctx_pad: int):
    """InjectChannelsItem (1x1 conv over cat([x, ctx]), w [C, C + n_ctx, 1]) backward:
    (pack for d x, pack for d ctx with the context channels zero-padded to ctx_pad)."""
    n_ctx = w.shape[1] - C
    wd_x = ops.pack_linear(w.detach()[:, :C, 0].t().contiguous())
    wc = _master(w)[:, C:, 0].t()
    wpad = torch.zeros(ctx_pad, C, dtype=wc.dtype, device=w.device)
    wpad[:n_ctx] = wc
    return wd_x, ops.pack_linear(wpad)


# ------------------------------------------------------------------------ launch sequences
def conv3_bwd(dy: Tensor, a_in: Tensor, gw: Tensor, da: Tensor, wd: Tensor, C: int):
    """dy: grad of the conv output; a_in: its input; writes da, accumulates dW (3 taps)."""
    ops.wgrad(dy, a_in, gw, n=C, k=C, off=-1, ntaps=3)
    ops.conv_gemm(dy, wd, da, c_in=C, n_valid=C, taps=(-1, 0, 1))


def upsample_bwd(dys: Tensor, x_last: Tensor, wd_up: Tensor, gw: Tensor, db: Tensor, dx_last: Tensor,
                 f: int) -> None:
    """Backward of the up conv x_last [B, Tl, C] -> y [B, f*Tl, Co], given dys = dL/dy.
    f >= 2: gw is the per-phase accumulator [f, 2, Co, C] (fold_upsample_wgrad), wd_up from
    pack_upsample_dgrad.  f = 1: a plain k=3 conv, gw [3, Co, C], wd_up = ops.pack_conv_dgrad.
    Accumulates gw and db (bias), writes dx_last."""
    B, Tl, C = x_last.shape
    Co = dys.shape[-1]
    ops.colsum(dys, db)
    if f > 1:
        for p_, s_, off in upsample_wgrad_slots(f):
            ops.wgrad(dys.view(B, Tl, f * Co), x_last, gw[p_, s_], n=Co, k=C, off=off, g_col0=p_ * Co)
        ops.conv_gemm(dys.view(B, Tl, f * Co), wd_up, dx_last, c_in=f * Co, n_valid=C, taps=(-1, 0, 1))
    else:
        ops.wgrad(dys, x_last, gw, n=Co, k=C, off=-1, ntaps=3)
        ops.conv_gemm(dys, wd_up, dx_last, c_in=Co, n_valid=C, taps=(-1, 0, 1))


def downsample_bwd(d: Tensor, x_in: Tensor, wd_down: Tensor, gw_down: Tensor, db_down: Tensor,
                   d_xin: Tensor, d_skip: Tensor, f: int, wgrad_done=None) -> None:
    """Backward of the down conv x_in [B, T, ci] -> [B, T/f, C] (k = stride = f), given d = its
    output gradient.  Accumulates gw_down ([C, f*ci], [co][tap][ci]) and db_down; writes
    d_xin = dgrad + d_skip (the gradient reaching the level input through the skip path).
    wgrad_done() runs once the weight gradients are complete."""
    B, Tl, C = d.shape
    kdim = f * x_in.shape[-1]
    ops.colsum(d, db_down)
    ops.wgrad(d, x_in.view(B, Tl, kdim), gw_down, n=C, k=kdim, off=0)
    if wgrad_done is not None:
        wgrad_done()
    ops.conv_gemm(d, wd_down, d_xin.view(B, Tl, kdim), c_in=C, n_valid=kdim,
                  residual=d_skip.view(B, Tl, kdim))


def skipcat_bwd(d_out: Tensor, skip: Tensor, y_up: Tensor, wd_c1: Tensor, wd_c2: Tensor, gw_cat: Tensor,
                db_cat: Tensor, blk1: Tensor, blk2: Tensor, dys: Tensor, d_skip: Tensor, rp: int) -> None:
    """Backward of out = merge(cat([skip * S_CAT, y_up])) on [B, T, Co] tensors, rp positions per
    GEMM row.  Accumulates db_cat and the block products blk1 / blk2 [rp*Co, rp*Co], writes
    gw_cat [Co, 2*Co] (from blk1 / blk2), dys and d_skip."""
    B, T, Co = d_out.shape

    def rows(t):
        return t.view(B, T // rp, rp * Co)
    ops.colsum(d_out, db_cat)
    ops.wgrad(rows(d_out), rows(skip), blk1, n=rp * Co, k=rp * Co)
    ops.wgrad(rows(d_out), rows(y_up), blk2, n=rp * Co, k=rp * Co)
    gw_cat.copy_(skipcat_weight_grad(blk1, blk2, rp, Co))
    ops.conv_gemm(rows(d_out), wd_c2, rows(dys), c_in=rp * Co, n_valid=rp * Co)
    ops.conv_gemm(rows(d_out), wd_c1, rows(d_skip), c_in=rp * Co, n_valid=rp * Co)


def inject_bwd(d_out: Tensor, x: Tensor, ctxb: Tensor, dctxb: Tensor, wd_x: Tensor, wd_c: Tensor,
               gw: Tensor, db: Tensor, dx: Tensor, n_ctx: int) -> Tensor:
    """Backward of out = conv1x1(cat([x, ctx])) + x (InjectChannelsItem).  ctxb / dctxb: the
    context and its gradient [B, T, ctx_pad]; dctxb is ACCUMULATED in place (the items of one
    depth share it).  Accumulates gw [C, C + n_ctx] and db; writes and returns dx."""
    C = x.shape[-1]
    ops.colsum(d_out, db)
    ops.wgrad(d_out, x, gw[:, :C], n=C, k=C)
    ops.wgrad(d_out, ctxb, gw[:, C:], n=C, k=n_ctx)
    ops.conv_gemm(d_out, wd_c, dctxb, c_in=C, n_valid=ctxb.shape[-1], residual=dctxb)
    ops.conv_gemm(d_out, wd_x, dx, c_in=C, n_valid=C, residual=d_out)   # + the identity path
    return dx


def resnet_item_bwd(dy: Tensor, x: Tensor, h: Tensor, rr: Tensor, a1: Tensor, a2: Tensor, x_stats: Tensor,
                    h_stats: Tensor, gn1, gn2, wd1: Tensor, wd2: Tensor, gw1: Tensor, gw2: Tensor, dgn1, dgn2,
                    db1: Tensor, db2: Tensor, S1: Tensor, S2: Tensor, work, groups: int, film=None) -> Tensor:
    """Backward of a ResnetItem (C >= 32) and its ModulationItem:
        h = conv1(SiLU(GN1(x))), rr = conv2(SiLU(GN2(h))) + x, y = LN(rr) (1 + scale) + shift.
    Saved forward tensors: a1 = SiLU(GN1(x)), a2 = SiLU(GN2(h)), GroupNorm statistics x_stats,
    h_stats.  gn1 / gn2 = (gamma, beta); wd1 / wd2 = ops.pack_conv_dgrad packs.  Accumulates the
    parameter gradients gw1 / gw2 ([3, C, C] tap-major), dgn1 / dgn2 = (dgamma, dbeta), db1 / db2;
    S1 / S2 are the GroupNorm backward sums.  work = (dr, dh, dx, dxh, da) activation-dtype
    [B, T, C] buffers.  film = (scale_shift, d scale_shift, row stride, eps) of the ModulationItem, or None
    without one (dy is then dL/drr).  Returns dx."""
    dr, dh, dx, dxh, da = work
    C = x.shape[-1]
    if film is not None:
        ss, dss, ss_stride, eps = film
        ops.ln_film_bwd(dy, rr, ss, ss_stride, dr, dss=dss, dss_stride=ss_stride, colsum=db2, eps=eps)
    else:
        dr = dy
        ops.colsum(dy, db2)
    conv3_bwd(dr, a2, gw2, da, wd2, C)
    ops.gn_silu_bwd(da, h, h_stats, gn2[0], gn2[1], dxh, dgn2[0], dgn2[1], S2, groups)
    ops.gn_bwd_apply(dxh, h, h_stats, S2, dh, groups, colsum=db1)
    conv3_bwd(dh, a1, gw1, da, wd1, C)
    ops.gn_silu_bwd(da, x, x_stats, gn1[0], gn1[1], dxh, dgn1[0], dgn1[1], S1, groups)
    ops.gn_bwd_apply(dxh, x, x_stats, S1, dx, groups, dres=dr)
    return dx


def build_train_plan(net: B200UNet, B: int, T: int, M: int, mode: str, want_dxin: bool) -> _TrainPlan:
    """mode 'loss': noising + MSE fused (VDiffusion); 'v': plain net forward, backward from dL/dv.
    M = embedding tokens (0 without CrossAttentionItems)."""
    dev = net.net.down.weight.device
    P = net.packed()
    plan = _TrainPlan()
    G, Fm = net.groups, net.features
    levels = net.levels()
    adt = net._act_dtype()         # bf16, or fp32 in the verification mode (B200UNet.verify_fp32)
    loss_mode = mode == "loss"
    heads = net.heads or 0
    D = net.head_features or 64
    mid = heads * D
    att_scale = D ** -0.5

    def act(*shape):
        return torch.empty(*shape, dtype=adt, device=dev)

    # ---- static I/O
    cin = net.x_channels + net.append_channels
    net._static_io(plan, B, B, T, M)
    plan.noise = _zeros((B, net.x_channels, T), dev) if loss_mode else None
    plan.alpha = _zeros((B,), dev) if loss_mode else None
    plan.beta = _zeros((B,), dev) if loss_mode else None
    plan.cond = _zeros((B, Fm), dev)                      # SiLU(features), fp32 master
    plan.cond_bf = torch.zeros(1, B, Fm, dtype=adt, device=dev)
    plan.loss_sum = torch.zeros(1, dtype=torch.float64, device=dev)
    plan.dv = _zeros((B, net.out_channels, T), dev)
    plan.v = None if loss_mode else _zeros((B, net.out_channels, T), dev)
    plan.gscale = torch.ones(1, device=dev)
    plan.dcond = _zeros((B, Fm), dev)
    plan.dxin = _zeros((B, cin, T), dev) if want_dxin else None
    E = net.embedding_features
    plan.demb = torch.zeros(B, M, E, dtype=adt, device=dev) if M else None
    plan.dctx = {i: torch.zeros_like(c) for i, c in plan.ctx.items()}     # d InjectChannelsItem context

    # ---- statistics + gradient arenas
    n_items = sum(len(lv.items_down) + len(lv.items_up) for lv in levels)
    arena = torch.zeros(7 * n_items + 4 * len(levels) + 8, B, G, 2, dtype=torch.float64, device=dev)
    add = plan.forward.add
    add(lambda: (arena.zero_(), plan.loss_sum.zero_()))
    refreshers: List = []                  # re-pack the dgrad weights in place after a weight update

    def packed_dgrad(make_any):
        """make() -> one pack or a tuple of packs, re-made in place by the refreshers; packed in the
        activation dtype (the forward packs' B200UNet._compute_packed does the same)."""
        def make():
            with ops.pack_dtype(adt):
                return make_any()
        t = make()
        if isinstance(t, tuple):
            refreshers.append(lambda t=t, make=make: [a.copy_(b) for a, b in zip(t, make())])
        else:
            refreshers.append(lambda t=t, make=make: t.copy_(make()))
        return t

    grads: Dict[int, Tensor] = {}          # id(param) -> fp32 gradient (PyTorch layout / packed)
    finals: List = []                      # closures turning packed grads into PyTorch layout
    # one flat fp32 arena for every gradient accumulator: a single memset per backward
    n_param = sum(p.numel() for p in net.parameters())
    # every attention item adds a projection-gradient scratch smaller than its parameters on top of
    # its gradients; the margin below covers the first AttentionItem and CrossAttentionItem after each
    # ResnetItem (one UNetV0 repetition), every further one adds its parameters, and so does every
    # attention item ahead of a chain's first ResnetItem (no ResnetItem pays for its scratch)
    def extra_attention(chain):
        seen = {"att", "cross"}
        for kind, m in chain:
            if kind == "resnet":
                seen.clear()
            elif kind in ("att", "cross"):
                if kind in seen:
                    yield m
                seen.add(kind)
    n_extra = sum(p.numel() for lv in levels for up in (False, True) for am in extra_attention(lv.chain(up))
                  for p in am.parameters())
    flat = torch.zeros(int(1.25 * n_param) + n_extra + 64 * (4 * n_param // 1000 + 4096), device=dev)
    cursor = [0]

    specs: Dict[int, tuple] = {}           # id(param) -> (arena start, numel, view shape, permutation)

    def gbuf(shape):
        n = 1
        for d in shape:
            n *= d
        start = cursor[0]
        cursor[0] = start + (n + 63) // 64 * 64
        assert cursor[0] <= flat.numel(), "gradient arena too small"
        gbuf.last = start
        return flat[start:start + n].view(*shape)

    def grad_for(param, shape=None, perm=None):
        """Arena accumulator for `param`'s gradient: stored as `shape` (default: the parameter's),
        handed to autograd as `.view(shape).permute(perm)` of a per-backward copy of the arena."""
        shape = tuple(param.shape) if shape is None else tuple(shape)
        t = gbuf(shape)
        specs[id(param)] = (gbuf.last, t.numel(), shape, perm)
        return t

    n_tot = P["cond_n"]
    mod = net.use_modulation       # False: no conditioning projection (no ModulationItem, no SkipModulate)
    ss_all = net._ss_all(P, B)
    dss_all = gbuf(ss_all.shape)
    ss_stride = ss_all.shape[1]
    if mod:
        add(lambda: plan.cond_bf.copy_(plan.cond.view(1, B, Fm)))
        net._project_conditioning(add, P, plan.cond_bf, ss_all)

    # ---- cross-attention context: LayerNorm(embedding) once per forward (the per-item
    # norm_context affines are folded into each item's to_kv weights)
    en = den = None
    if M:
        en, den = act(B, M, E), torch.zeros(B, M, E, dtype=adt, device=dev)
        add(lambda: ops.ln_film(plan.embedding, en, None, 0, None, G, net.ATT_LN_EPS))
    # the forward launches; every intermediate the backward reads stays live
    walk = _ForwardWalk(net, P, plan, add, B, arena, ss_all, keep=True, add_ctx=add, en=en)
    trunk = walk.trunk(lambda: dict(loss_sum=plan.loss_sum if loss_mode else None,
                                    dv=plan.dv if loss_mode else None, v_out=plan.v),
                       noise=plan.noise, alpha=plan.alpha, beta=plan.beta)
    new_stats = walk.new_stats
    delta_ws = [None]    # shared fp32 workspace of adp_attention_bwd, sized for the largest item

    def delta_for(Tl: int) -> Tensor:
        if delta_ws[0] is None or delta_ws[0].numel() < B * heads * Tl:
            delta_ws[0] = _zeros((B * heads * Tl,), dev)
        return delta_ws[0]

    # ---- AttentionItem / CrossAttentionItem (a_unet): y = x + to_out(softmax(q k^T / sqrt(D)) v)
    def attention_backward(a: Dict, am, cross: bool, Tl: int, C: int):
        """a: the tensors of the walk's forward (x, xn = LayerNorm(x) with the affine folded into the
        projections, q / k / v, o, lse).  Returns the backward closure dy -> dx."""
        x, xn, q, k, v, o, lse = a["x"], a["xn"], a["q"], a["k"], a["v"], a["o"], a["lse"]
        delta_for(Tl)
        wo = am.to_out.weight
        wd_out = packed_dgrad(lambda: ops.pack_linear(wo.detach().t().contiguous()))
        gw_out = grad_for(wo)
        d_o, dxn, dx = act(B, Tl, mid), act(B, Tl, C), act(B, Tl, C)
        g1, b1 = am.norm.weight, am.norm.bias
        g2, b2 = am.norm_context.weight, am.norm_context.bias
        dWq, dWkv = grad_for(am.to_q.weight), grad_for(am.to_kv.weight)
        dg1, db1, dg2, db2 = grad_for(g1), grad_for(b1), grad_for(g2), grad_for(b2)
        if not cross:
            dqkv = act(B, Tl, 3 * mid)
            wd_qkv = packed_dgrad(lambda: pack_ln_folded_dgrad((am.to_q.weight, g1),
                                                               (am.to_kv.weight, g2)))   # [C, 3*mid]
            gwf, dbf = gbuf((3 * mid, C)), gbuf((3 * mid,))

            def bwd(dy2: Tensor) -> Tensor:
                ops.conv_gemm(dy2, wd_out, d_o, c_in=C, n_valid=mid)
                ops.wgrad(dy2, o, gw_out, n=C, k=mid)
                ops.attention_bwd(q, k, v, o, d_o, lse, delta_ws[0], dqkv[..., :mid],
                                  dqkv[..., mid:2 * mid], dqkv[..., 2 * mid:], heads, att_scale,
                                  head_dim=D)
                ops.conv_gemm(dqkv, wd_qkv, dxn, c_in=3 * mid, n_valid=C)
                ops.wgrad(dqkv, xn, gwf, n=3 * mid, k=C)
                ops.colsum(dqkv, dbf)
                ops.ln_fold_bwd(am.to_q.weight, g1, b1, gwf[:mid], dbf[:mid], dWq, dg1, db1)
                ops.ln_fold_bwd(am.to_kv.weight, g2, b2, gwf[mid:], dbf[mid:], dWkv, dg2, db2)
                ops.ln_film_bwd(dxn, x, None, 0, dx, dres=dy2, eps=net.ATT_LN_EPS)
                return dx
        else:
            dq, dkv = act(B, Tl, mid), act(B, M, 2 * mid)
            wd_q = packed_dgrad(lambda: pack_ln_folded_dgrad((am.to_q.weight, g1)))
            wd_kv = packed_dgrad(lambda: pack_ln_folded_dgrad((am.to_kv.weight, g2)))
            gwq, dbq = gbuf((mid, C)), gbuf((mid,))
            gwkv, dbkv = gbuf((2 * mid, E)), gbuf((2 * mid,))

            def bwd(dy2: Tensor) -> Tensor:
                ops.conv_gemm(dy2, wd_out, d_o, c_in=C, n_valid=mid)
                ops.wgrad(dy2, o, gw_out, n=C, k=mid)
                ops.attention_bwd(q, k, v, o, d_o, lse, delta_ws[0], dq,
                                  dkv[..., :mid], dkv[..., mid:], heads, att_scale, head_dim=D)
                ops.conv_gemm(dq, wd_q, dxn, c_in=mid, n_valid=C)
                ops.wgrad(dq, xn, gwq, n=mid, k=C)
                ops.colsum(dq, dbq)
                # d LayerNorm(embedding), summed over the cross-attention items (in place)
                ops.conv_gemm(dkv, wd_kv, den, c_in=2 * mid, n_valid=E, residual=den)
                ops.wgrad(dkv, en, gwkv, n=2 * mid, k=E)
                ops.colsum(dkv, dbkv)
                ops.ln_fold_bwd(am.to_q.weight, g1, b1, gwq, dbq, dWq, dg1, db1)
                ops.ln_fold_bwd(am.to_kv.weight, g2, b2, gwkv, dbkv, dWkv, dg2, db2)
                ops.ln_film_bwd(dxn, x, None, 0, dx, dres=dy2, eps=net.ATT_LN_EPS)
                return dx
        return bwd

    def cond_grads(mm, off: int, n: int) -> None:
        """A ModulationItem's or SkipModulate's Linear is one slice of the conditioning projection."""
        grads[id(mm.proj.weight if hasattr(mm, "proj") else mm.weight)] = ("cond_w", off, n)
        grads[id(mm.proj.bias if hasattr(mm, "proj") else mm.bias)] = ("cond_b", off, n)

    # ---- backward of a ResnetItem and the ModulationItem the walk fused into it (mm: its module)
    def resnet_backward(res: Dict, ip: Dict, r_, mm, mp: Optional[Dict], C: int, Tl: int):
        x, h, rr, ss = res["x"], res["h"], res["r"], res["ss"]
        xs, hs = res["x_stats"], res["h_stats"]
        mod = mp is not None
        dss = dss_all[:, mp["ss_off"]:] if mod else None
        S1, S2 = new_stats(), new_stats()
        dgn1 = (grad_for(r_.gn1.weight), grad_for(r_.gn1.bias))
        dgn2 = (grad_for(r_.gn2.weight), grad_for(r_.gn2.bias))
        db1, db2 = grad_for(r_.conv1.bias), grad_for(r_.conv2.bias)
        dr, dh, dx, dxh = act(B, Tl, C), act(B, Tl, C), act(B, Tl, C), act(B, Tl, C)
        if res["a1"] is None:      # the forward ran the C = 8 ConvBlocks as adp_narrow_conv
            dw1, dw2 = grad_for(r_.conv1.weight), grad_for(r_.conv2.weight)
            db_scratch = gbuf((C,))

            def bwd(dy):
                if mod:
                    ops.ln_film_bwd(dy, rr, ss, ss_stride, dr, dss=dss, dss_stride=ss_stride, eps=net.MOD_LN_EPS)
                d_r = dr if mod else dy
                ops.narrow_conv_bwd(d_r, h, hs, ip["gn2"][0], ip["gn2"][1], ip["w2"], dxh, dgn2[0],
                                    dgn2[1], S2, dw2, db2, G)
                ops.gn_bwd_apply(dxh, h, hs, S2, dh, G, colsum=db1)   # fp32 sum, pre-rounding
                ops.narrow_conv_bwd(dh, x, xs, ip["gn1"][0], ip["gn1"][1], ip["w1"], dxh, dgn1[0],
                                    dgn1[1], S1, dw1, db_scratch, G)
                ops.gn_bwd_apply(dxh, x, xs, S1, dx, G, dres=d_r)
                return dx
        else:
            a1, a2 = res["a1"], res["a2"]
            wd1 = packed_dgrad(lambda: ops.pack_conv_dgrad(r_.conv1.weight.detach()))
            wd2 = packed_dgrad(lambda: ops.pack_conv_dgrad(r_.conv2.weight.detach()))
            work = (dr, dh, dx, dxh, act(B, Tl, C))
            # [tap][co][ci] accumulators of the fused 3-tap wgrad -> PyTorch [co][ci][tap]
            gw1 = grad_for(r_.conv1.weight, (3, C, C), (1, 2, 0))
            gw2 = grad_for(r_.conv2.weight, (3, C, C), (1, 2, 0))
            if C == 8:
                # a C = 8 ConvBlock of the fp32 verification mode: the slot of the narrow branch's
                # bias scratch stays reserved, so every later parameter keeps its arena offset
                gbuf((C,))
            film = (ss, dss, ss_stride, net.MOD_LN_EPS) if mod else None

            def bwd(dy):
                return resnet_item_bwd(dy, x, h, rr, a1, a2, xs, hs, ip["gn1"], ip["gn2"], wd1, wd2, gw1, gw2,
                                       dgn1, dgn2, db1, db2, S1, S2, work, G, film=film)
        if mod:
            cond_grads(mm, mp["ss_off"], 2 * C)
        return bwd

    # ---- backward of a ModulationItem that runs as its own ln_film pass
    def modulation_backward(rec: Dict, mm, mp: Dict, C: int, Tl: int):
        dx, dss = act(B, Tl, C), dss_all[:, mp["ss_off"]:]
        cond_grads(mm, mp["ss_off"], 2 * C)

        def bwd(dy):
            ops.ln_film_bwd(dy, rec["x"], rec["ss"], ss_stride, dx, dss=dss, dss_stride=ss_stride,
                            eps=net.MOD_LN_EPS)
            return dx
        return bwd

    # ---- backward of an InjectChannelsItem: a_unet's conv1x1(cat([x, ctx])) + x, W = [W_x | W_c]
    def inject_backward(inj: Dict, conv, C: int, Tl: int, li: int):
        ctxb, dctxb = inj["ctx"], plan.dctx[li]
        n_ctx, ctx_pad = conv.weight.shape[1] - C, ctxb.shape[-1]
        dyi = act(B, Tl, C)
        gw_inj = grad_for(conv.weight, (C, C + n_ctx, 1)).view(C, C + n_ctx)
        db_inj = grad_for(conv.bias)
        wd_x, wd_c = packed_dgrad(lambda: pack_inject_dgrad(conv.weight, C, ctx_pad))
        # d context is summed over the items of this depth (in place through the residual)
        return lambda d_out: inject_bwd(d_out, inj["x"], ctxb, dctxb, wd_x, wd_c, gw_inj, db_inj, dyi, n_ctx)

    # ---- one backward closure per unit of an item chain, built from the walk's records
    def chain_backward(recs: List, items_p: List, chain_m: List, C: int, Tl: int, li: int) -> List:
        bwds = []
        for kind, i, width, rec in recs:
            m, pk = chain_m[i][1], items_p[i][1]
            if kind == "resnet":
                mm, mp = (chain_m[i + 1][1], items_p[i + 1][1]) if width == 2 else (None, None)
                bwds.append(resnet_backward(rec, pk, m, mm, mp, C, Tl))
            elif kind == "mod":
                bwds.append(modulation_backward(rec, m, pk, C, Tl))
            elif kind == "inj":
                bwds.append(inject_backward(rec, m, C, Tl, li))
            else:
                bwds.append(attention_backward(rec, m, kind == "cross", Tl, C))
        return bwds

    # ---- backward of one level from the walk's record (_ForwardWalk.trunk); level 0's closure
    # takes no argument, that of a level >= 1 maps d(its output) to d(its input)
    def level(rec: Dict):
        i, lv, Lp, Tl, T_in = rec["i"], rec["lv"], rec["Lp"], rec["Tl"], rec["T_in"]
        x_in, x_last, gate, C = rec["x_in"], rec["x"], rec["gate"], lv.ch
        # gradient-arena cursor at the level's sequence points: the arena is laid out in FORWARD
        # build order, so "down part", "inner levels" and "up part" of a level are three
        # contiguous ranges; the backward finishes them in the order up, inner, down and
        # announces each range through plan.mark (overlapped gradient all-reduce, parallel.py)
        cur = {"entry": cursor[0]}
        db_down = grad_for(lv.down.bias)
        if i == 0:
            dw_down = grad_for(lv.down.weight)
        else:
            wd_down = packed_dgrad(lambda: pack_down_dgrad(lv.down.weight))
            # [co][tap][ci] (the [B, T/f, f*C] view) -> PyTorch [co][ci][tap]
            gw_down = grad_for(lv.down.weight, (C, lv.factor, lv.in_ch), (0, 2, 1)).view(C, lv.factor * lv.in_ch)
        items_down_bwd = chain_backward(rec["down"], Lp["items_down"], lv.chain(up=False), C, Tl, i)
        cur["down_end"] = cursor[0]
        inner = level(rec["inner"]) if rec["inner"] is not None else None
        cur["inner_end"] = cursor[0]
        items_up_bwd = chain_backward(rec["up"], Lp["items_up"], lv.chain(up=True), C, Tl, i)

        def chains(d: Tensor) -> Tensor:
            """d(up chain output) -> d(down chain input), through the inner level."""
            for b_ in reversed(items_up_bwd):
                d = b_(d)
            if inner is not None:
                plan.mark((cur["inner_end"], cur["exit"]))
                d = inner(d)
            for b_ in reversed(items_down_bwd):
                d = b_(d)
            return d

        def mark_down() -> None:
            plan.mark((cur["entry"], cur["down_end"] if inner is not None else cur["exit"]))

        merge = net.merge
        if merge == "modulate":
            dgate = dss_all[:, Lp["gate_off"]:]
            cond_grads(lv.merge, Lp["gate_off"], lv.out_ch)
        elif i == 0:
            # SkipAdd and SkipCat at level 0: the stem epilogue with a unit gate, whose gradient is not used
            dgate = gbuf(gate.shape)
        if i == 0 and merge == "cat":
            # SkipCat at level 0 runs in the stem kernels with the 1x1 merge conv folded into both
            # branches (B200UNet._compute_packed): they produce the gradients of the FOLDED
            # weights, unfolded below (a few hundred numbers) into merge / up / adapter gradients
            Co, Ci = lv.out_ch, lv.in_ch
            dw_up, db_up = gbuf((Co, C, 3)), gbuf((Co,))
            dwa, dba = gbuf((Co, Ci)), gbuf((Co,))

            def unfold_level0():
                ad = lv.adapter
                g = unfold_level0_grads(lv.merge.weight, lv.up.weight, lv.up.bias, dw_up, db_up, dwa, dba,
                                        ad.weight if ad is not None else None,
                                        ad.bias if ad is not None else None)
                for mod_name, m in (("up", lv.up), ("merge", lv.merge), ("adapter", ad)):
                    if m is not None:
                        grads[id(m.weight)] = g[mod_name + ".weight"]
                        grads[id(m.bias)] = g[mod_name + ".bias"]
            finals.append(unfold_level0)
        else:
            db_up = grad_for(lv.up.bias)
        if i == 0:
            if merge != "cat":
                dw_up = grad_for(lv.up.weight)
                dwa = (grad_for(lv.adapter.weight, (lv.out_ch, lv.in_ch, 1)).view(lv.out_ch, lv.in_ch)
                       if lv.adapter is not None else None)
                dba = grad_for(lv.adapter.bias) if lv.adapter is not None else None
            dh0 = act(B, Tl, C)

            def backward_level0():
                ops.stem_out_bwd(plan.dv, x_last, plan.x, Lp["up_w"], Lp["up_b"], gate, lv.factor, dh0,
                                 dw_up, db_up, dgate, gscale=plan.gscale, append=plan.append,
                                 noise=plan.noise, alpha=plan.alpha, beta=plan.beta,
                                 w_adapt=Lp.get("adapt_w"), dw_adapt=dwa, db_adapt=dba, dxin=plan.dxin)
                d = chains(dh0)
                ops.stem_in_bwd(d, plan.x, dw_down, db_down, lv.factor, append=plan.append,
                                noise=plan.noise, alpha=plan.alpha, beta=plan.beta,
                                w=Lp["down_w"], dxin=plan.dxin)
                mark_down()
            cur["exit"] = cursor[0]
            return backward_level0

        # levels >= 1: the up conv wrote y_up (pre-gate), the merge combined it with the level's input
        f, Co, y_up = lv.factor, lv.out_ch, rec["y_up"]
        dys, dx_last, d_xin = act(B, T_in, Co), act(B, Tl, C), act(B, T_in, lv.in_ch)
        if f > 1:
            wd_up = packed_dgrad(lambda: pack_upsample_dgrad(lv.up.weight, f))
            gw_up = gbuf((f, 2, Co, C))

            def up_final():
                grads[id(lv.up.weight)] = fold_upsample_wgrad(gw_up, f)
            finals.append(up_final)
        else:
            wd_up = packed_dgrad(lambda: ops.pack_conv_dgrad(lv.up.weight.detach()))
            gw_up = grad_for(lv.up.weight, (3, Co, C), (1, 2, 0))
        if merge == "add":
            d_skip_of = lambda d_out: d_out      # noqa: E731
            merge_bwd = lambda d_out: d_out      # noqa: E731  (out = x_in + y_up: both gradients are d_out)
        elif merge == "modulate":
            d_skip_of = lambda d_out: d_out      # noqa: E731  (the skip path's gradient is d_out itself)

            def merge_bwd(d_out: Tensor) -> Tensor:
                ops.skip_gate_bwd(d_out, y_up, gate, dys, dgate)
                return dys
        else:
            rp = max(1, 16 // Co)                # positions per GEMM row of the SkipCat merge
            d_skip = act(B, T_in, Co)
            wm_ = lv.merge.weight
            wd_c1, wd_c2 = packed_dgrad(lambda: pack_skipcat_dgrad(wm_, rp))
            gw_cat = grad_for(wm_, (Co, 2 * Co, 1)).view(Co, 2 * Co)
            db_cat = grad_for(lv.merge.bias)
            blk1, blk2 = gbuf((rp * Co, rp * Co)), gbuf((rp * Co, rp * Co))
            d_skip_of = lambda d_out: d_skip     # noqa: E731

            def merge_bwd(d_out: Tensor) -> Tensor:
                skipcat_bwd(d_out, x_in, y_up, wd_c1, wd_c2, gw_cat, db_cat, blk1, blk2, dys, d_skip, rp)
                return dys

        def backward_level(d_out: Tensor) -> Tensor:
            upsample_bwd(merge_bwd(d_out), x_last, wd_up, gw_up, db_up, dx_last, f)
            d = chains(dx_last)
            # gradient w.r.t. the level input = dgrad(down conv) + the skip path
            downsample_bwd(d, x_in, wd_down, gw_down, db_down, d_xin, d_skip_of(d_out), lv.factor,
                           wgrad_done=mark_down)
            return d_xin

        cur["exit"] = cursor[0]
        return backward_level

    backward0 = level(trunk)
    plan.flat = flat
    plan.refreshers, plan.version = refreshers, net._version()
    plan.grads, plan.finals, plan.specs = grads, finals, specs
    plan.ss_all, plan.dss_all = ss_all, dss_all
    # conditioning projection backward
    plan.dw_all = _zeros((n_tot, Fm), dev)
    plan.dbias_all = _zeros((n_tot,), dev)
    plan.n_tot = n_tot

    def backward_program():
        flat.zero_()
        if den is not None:
            den.zero_()
        for d_ in plan.dctx.values():
            d_.zero_()
        backward0()
        if den is not None:      # d embedding = LayerNorm backward of the summed context gradients
            ops.ln_film_bwd(den, plan.embedding, None, 0, plan.demb, eps=net.ATT_LN_EPS)
        plan.dcond.zero_()
        if mod:
            ops.cond_bwd(dss_all, plan.cond_bf.view(B, Fm).float(), P["cond_w"], plan.dw_all,
                         plan.dbias_all, plan.dcond, n_tot)
    plan.backward_program = backward_program
    plan.P, plan.n_dss = P, dss_all.numel()
    return plan


@torch.no_grad()
def _refresh_dgrad_packs(plan: _TrainPlan, net: B200UNet) -> None:
    """Transposed / tap-reversed weight packs of the data-gradient GEMMs after a weight update:
    captured into a CUDA graph on first use (same reasoning as B200UNet._repack)."""
    def refresh():
        for r in plan.refreshers:
            r()
    plan.refresh_graph = _refreshed(plan.refresh_graph, refresh, net.use_cuda_graph)


def _run_backward_synced(plan: _TrainPlan, net: B200UNet, sync) -> None:
    """Data-parallel backward: the program runs as graph SEGMENTS cut where a bucket of the
    gradient arena is complete; the bucket's all-reduce (NCCL, async on its own stream) is issued
    right after the segment's replay and overlaps the remaining segments.  The gradients of the
    concatenated conditioning projection (48 M of the 175 M parameters of the 9-level net, final
    only at the very end) are not all-reduced at all: dW = sum_ranks dss_r^T cond_r is recomputed
    from the all-gathered [world*B, .] factors (a few MB)."""
    works: List = []
    flush = sync.flush_schedule(plan)            # {mark index: [intervals to reduce now]}
    counter = [0]

    def reduce_now(intervals):
        for a, b in intervals:
            works.append(sync.all_reduce_async(plan.flat[a:b]))

    record = flush is None                       # no synced backward of this plan has run yet
    if not net.use_cuda_graph or record:
        def on_mark(iv):
            if record:
                plan.mark_log.append(iv)
            todo = flush.get(counter[0]) if flush is not None else None
            counter[0] += 1
            if todo:
                reduce_now(todo)
        plan.on_mark = on_mark
        plan.backward_program()
        plan.on_mark = None
        if record:                               # the mark sequence was just recorded
            flush = sync.flush_schedule(plan)
            reduce_now([iv for ivs in flush.values() for iv in ivs])
    else:
        if plan.seg_graphs is None:
            segs: List = []
            pool = torch.cuda.graph_pool_handle()
            torch.cuda.synchronize()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                state = {"g": torch.cuda.CUDAGraph()}
                state["g"].capture_begin(pool=pool)

                def on_mark(iv):
                    todo = flush.get(counter[0])
                    counter[0] += 1
                    if todo:
                        state["g"].capture_end()
                        segs.append((state["g"], todo))
                        state["g"] = torch.cuda.CUDAGraph()
                        state["g"].capture_begin(pool=pool)
                plan.on_mark = on_mark
                plan.backward_program()
                plan.on_mark = None
                state["g"].capture_end()
                segs.append((state["g"], None))
            torch.cuda.current_stream().wait_stream(side)
            plan.seg_graphs = segs
        for g, todo in plan.seg_graphs:
            g.replay()
            if todo:
                reduce_now(todo)
    plan.backward.runs += 1
    sync.conditioning_gradients(plan)
    for w in works:
        w.wait()


class _UNetFn(torch.autograd.Function):
    """mode 'loss' -> scalar MSE loss; mode 'v' / 'v1' -> v [B, out, T] ('v1' = a second plan of
    the same shape, for the masked pass of classifier-free guidance under autograd).  Inputs that
    may receive a gradient: x, append, cond (SiLU of the time features), embedding, and every
    parameter."""

    @staticmethod
    def forward(ctx, net: B200UNet, mode: str, x, noise, sigmas, append, cond, embedding, ctx_depths,
                *rest):
        context, params = rest[:len(ctx_depths)], rest[len(ctx_depths):]
        if net.verify_fp32 and getattr(net, "_grad_sync", None) is not None:
            raise NotImplementedError("OverlappedDataParallel does not support B200UNet.verify_fp32; train the "
                                      "verification mode in one process or under torch DistributedDataParallel")
        B, _, T = x.shape
        M = embedding.shape[1] if (embedding is not None and any(net.cross_attentions)) else 0
        need = ctx.needs_input_grad       # (net, mode, x, noise, sigmas, append, cond, embedding, ...)
        want_dxin = bool(need[2] or need[5])
        key = ("train", B, T, M, mode, want_dxin)
        slot, mode = mode, ("loss" if mode == "loss" else "v")
        net.packed()                         # in-place refresh of the forward packs
        plan = net._plans.get(key)
        if plan is None:
            ops.device_check()
            plan = net._plans[key] = build_train_plan(net, B, T, M, mode, want_dxin)
        elif plan.version != net._version():
            _refresh_dgrad_packs(plan, net)
            plan.version = net._version()
        plan.x.copy_(x)
        if net.append_channels:
            assert append is not None, "append_channels is required (AppendChannelsPlugin)"
            plan.append.copy_(append)
        if mode == "loss":
            plan.noise.copy_(noise)
            angle = sigmas.float() * pi / 2
            plan.alpha.copy_(torch.cos(angle))
            plan.beta.copy_(torch.sin(angle))
        if M:
            plan.embedding.copy_(embedding)
        for d_, c_ in zip(ctx_depths, context):      # [B, ctx, T_d] -> channels-last
            plan.ctx[d_][:, :, : c_.shape[1]].copy_(c_.transpose(1, 2))
        plan.cond.copy_(cond)
        plan.forward(net.use_cuda_graph)
        plan.generation += 1
        ctx.plan, ctx.net, ctx.mode, ctx.generation = plan, net, mode, plan.generation
        ctx.params = params
        ctx.ctx_depths = ctx_depths
        ctx.ctx_channels = [c_.shape[1] for c_ in context]
        ctx.has_emb = M > 0
        ctx.x_dtype = x.dtype
        if mode == "loss":
            return (plan.loss_sum / plan.dv.numel()).float().reshape(())
        return plan.v.clone()

    @staticmethod
    def backward(ctx, grad_out):
        plan, net = ctx.plan, ctx.net
        if plan.generation != ctx.generation:
            raise RuntimeError(
                "B200UNet: another forward ran on the same input shape before this backward; its "
                "saved activations were overwritten (one static plan per shape).  Call backward() "
                "before the next forward of that shape.")
        if ctx.mode == "loss":
            plan.gscale.copy_(grad_out.reshape(1))
        else:
            plan.dv.copy_(grad_out)
        sync = getattr(net, "_grad_sync", None)
        if sync is None:
            plan.backward(net.use_cuda_graph)
        else:
            _run_backward_synced(plan, net, sync)
        for fin in plan.finals:
            fin()
        # .grad must never alias the plan's arenas (they are rewritten by the next backward): ONE copy
        # of the arena per backward, the gradients are views of that copy
        fresh = plan.flat.clone()
        cond_w, cond_b = plan.dw_all.clone(), plan.dbias_all.clone()
        out = []
        for p in ctx.params:
            spec = plan.specs.get(id(p))
            if spec is not None:
                start, n, shape, perm = spec
                g = fresh[start:start + n].view(shape)
                g = g.permute(perm) if perm is not None else g
            else:
                g = plan.grads.get(id(p))
                if isinstance(g, tuple):
                    kind, off, n = g
                    g = cond_w[off:off + n] if kind == "cond_w" else cond_b[off:off + n]
                elif g is not None:
                    g = g.reshape(p.shape).clone()       # computed by a `final` (upsample conv folds)
            out.append(None if g is None else (g if g.dtype == p.dtype else g.to(p.dtype)))
        dx = d_append = d_emb = None
        need = ctx.needs_input_grad        # (net, mode, x, noise, sigmas, append, cond, embedding, depths, ...)
        if plan.dxin is not None:
            cx = net.x_channels
            if need[2]:
                dx = plan.dxin[:, :cx]
                if ctx.mode == "loss":     # x enters through x_noisy (alpha) and the target (beta)
                    a, b = plan.alpha.view(-1, 1, 1), plan.beta.view(-1, 1, 1)
                    dx = a * dx + b * plan.dv * plan.gscale
                dx = dx.to(ctx.x_dtype).clone()
            if need[5] and net.append_channels:
                d_append = plan.dxin[:, cx:].clone()
        if ctx.has_emb and need[7]:
            d_emb = plan.demb.float()
        d_ctx = [plan.dctx[d_][:, :, :n_].transpose(1, 2).float() if need[9 + j] else None
                 for j, (d_, n_) in enumerate(zip(ctx.ctx_depths, ctx.ctx_channels))]
        return (None, None, dx, None, None, d_append, plan.dcond.clone(), d_emb, None, *d_ctx, *out)


def _time_cond(net: B200UNet, sigmas: Optional[Tensor], features: Optional[Tensor]) -> Tensor:
    """SiLU(f), f = MLP(GELU(NumberEmbedder(sigma))) (+features): a_unet TimeConditioningPlugin, as
    PyTorch ops so that autograd provides the gradients of its three [B,1024] linears."""
    if net.time is not None:
        assert sigmas is not None, "time conditioning requires the time argument"
    if not net.use_modulation:
        # no ModulationItem and no SkipModulate: nothing consumes the features.  An XUNet may still
        # carry the time plugin (a_unet ignores its output then); its MLP gets no gradient
        ref = next(net.parameters())
        return torch.zeros(1, net.features, device=ref.device)
    if net.time is not None:
        t = net.time
        s = sigmas.float().reshape(-1, 1)
        fr = s * t.weights * 2 * pi
        emb = t.to_out(torch.cat([s, fr.sin(), fr.cos()], dim=-1))
        f = F.gelu(t.mlp(F.gelu(t.mlp(F.gelu(emb)))))
        if features is not None:
            f = f + features
    else:
        assert features is not None, "use_time_conditioning=False needs features="
        f = features
    return F.silu(f)


def _train_embedding(net: B200UNet, B: int, embedding: Optional[Tensor],
                     embedding_mask_proba: float):
    """a_unet ClassifierFreeGuidancePlugin at training time: per-sample Bernoulli swap with the
    learned mask embedding (PyTorch ops, so its gradient reaches `fixed_embedding`).
    Returns (embedding fed to the net, the mask embedding or None)."""
    fixed = None
    if net.use_embedding_cfg:
        assert embedding is not None, "ClassiferFreeGuidancePlugin requires embedding"
        fixed = net.fixed_embedding.weight[: embedding.shape[1]].unsqueeze(0).expand_as(embedding)
        if embedding_mask_proba > 0.0:
            mask = torch.bernoulli(torch.full((B, 1, 1), float(embedding_mask_proba),
                                              device=embedding.device)).to(torch.bool)
            embedding = torch.where(mask, fixed, embedding)
    if any(net.cross_attentions):
        assert embedding is not None, "CrossAttentionItem requires embedding"
        return embedding.float(), (None if fixed is None else fixed.float())
    return None, None


def _context(net: B200UNet, channels):
    """(depths, tensors) of the InjectChannelsItem contexts, validated like a_unet does."""
    depths = tuple(i for i, c in enumerate(net.context_channels) if c > 0)
    tensors = []
    for d in depths:
        assert channels is not None and len(channels) > d and channels[d] is not None, \
            f"context `channels[{d}]` is required (context_channels[{d}] > 0)"
        assert channels[d].shape[1] == net.context_channels[d], \
            "context `channels` at depth must match resolution and context_channels"
        tensors.append(channels[d])
    return depths, tensors


def _net_params(net: B200UNet):
    time_ids = {id(p) for p in (net.time.parameters() if net.time is not None else [])}
    fixed_ids = {id(p) for p in (net.fixed_embedding.parameters() if net.fixed_embedding is not None else [])}
    return [p for p in net.parameters() if id(p) not in time_ids and id(p) not in fixed_ids]


def fused_v_loss(net: B200UNet, x: Tensor, noise: Tensor, sigmas: Tensor, *,
                 append_channels: Optional[Tensor] = None, features: Optional[Tensor] = None,
                 embedding: Optional[Tensor] = None, embedding_scale: float = 1.0,
                 embedding_mask_proba: float = 0.0, channels=None) -> Tensor:
    """mse(net(alpha*x + beta*noise, sigma), alpha*noise - beta*x)  (reference diffusion.py:90-95)."""
    ops.require_cuda(x)
    if net.use_embedding_cfg and embedding_scale != 1.0:
        # guidance inside the training objective = two differentiable evaluations (a_unet CFG
        # plugin); no fused-loss form: take the generic route
        sig_b = sigmas.view(-1, 1, 1)
        alphas, betas = torch.cos(sig_b * pi / 2), torch.sin(sig_b * pi / 2)
        v = differentiable_forward(net, alphas * x + betas * noise, sigmas, features=features,
                                   embedding=embedding, embedding_scale=embedding_scale,
                                   embedding_mask_proba=embedding_mask_proba,
                                   append_channels=append_channels, channels=channels)
        return F.mse_loss(v, alphas * noise - betas * x)
    cond = _time_cond(net, sigmas, features)
    emb, _ = _train_embedding(net, x.shape[0], embedding, embedding_mask_proba)
    depths, context = _context(net, channels)
    return _UNetFn.apply(net, "loss", x.float(), noise.float(), sigmas, append_channels, cond, emb, depths,
                         *context, *_net_params(net))


def differentiable_forward(net: B200UNet, x: Tensor, time: Optional[Tensor], *,
                           features: Optional[Tensor] = None, embedding: Optional[Tensor] = None,
                           embedding_scale: float = 1.0, embedding_mask_proba: float = 0.0,
                           append_channels: Optional[Tensor] = None, channels=None) -> Tensor:
    """v = net(x, time, ...) with autograd support (custom loss_fn / diffusion_t)."""
    ops.require_cuda(x)
    cond = _time_cond(net, time, features)
    emb, fixed = _train_embedding(net, x.shape[0], embedding, embedding_mask_proba)
    params = _net_params(net)
    depths, context = _context(net, channels)
    v = _UNetFn.apply(net, "v", x.float(), None, time, append_channels, cond, emb, depths, *context, *params)
    if net.use_embedding_cfg and embedding_scale != 1.0:
        # a_unet ClassifierFreeGuidancePlugin: out_masked + (out - out_masked) * scale, both passes
        # differentiable (a second plan of the same shape keeps the first one's activations alive)
        v_m = _UNetFn.apply(net, "v1", x.float(), None, time, append_channels, cond, fixed, depths, *context,
                            *params)
        v = v_m + (v - v_m) * embedding_scale
    return v.to(x.dtype)
