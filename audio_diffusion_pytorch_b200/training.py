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
from .unet import B200UNet, LevelParams, _pad_to


class _TrainPlan:
    def __init__(self):
        self.fwd: List = []
        self.graph_f = self.graph_b = None
        self.runs_f = self.runs_b = 0
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


def build_train_plan(net: B200UNet, B: int, T: int, M: int, mode: str, want_dxin: bool) -> _TrainPlan:
    """mode 'loss': noising + MSE fused (VDiffusion); 'v': plain net forward, backward from dL/dv.
    M = embedding tokens (0 without CrossAttentionItems)."""
    dev = net.net.down.weight.device
    P = net.packed()
    plan = _TrainPlan()
    G, Fm = net.groups, net.features
    levels = net.levels()
    bf16 = torch.bfloat16
    loss_mode = mode == "loss"
    heads = net.heads or 0
    mid = heads * 64
    att_scale = 64 ** -0.5

    def act(*shape):
        return torch.empty(*shape, dtype=bf16, device=dev)

    # ---- static I/O
    cin = net.x_channels + net.append_channels
    plan.x = _zeros((B, net.x_channels, T), dev)
    plan.noise = _zeros((B, net.x_channels, T), dev) if loss_mode else None
    plan.append = _zeros((B, net.append_channels, T), dev) if net.append_channels else None
    plan.alpha = _zeros((B,), dev) if loss_mode else None
    plan.beta = _zeros((B,), dev) if loss_mode else None
    plan.cond = _zeros((B, Fm), dev)                      # SiLU(features), fp32 master
    plan.cond_bf = torch.zeros(1, B, Fm, dtype=bf16, device=dev)
    plan.loss_sum = torch.zeros(1, dtype=torch.float64, device=dev)
    plan.dv = _zeros((B, net.out_channels, T), dev)
    plan.v = None if loss_mode else _zeros((B, net.out_channels, T), dev)
    plan.gscale = torch.ones(1, device=dev)
    plan.dcond = _zeros((B, Fm), dev)
    plan.dxin = _zeros((B, cin, T), dev) if want_dxin else None
    E = net.embedding_features
    plan.embedding = torch.zeros(B, M, E, dtype=bf16, device=dev) if M else None
    plan.demb = torch.zeros(B, M, E, dtype=bf16, device=dev) if M else None
    # InjectChannelsItem context per depth (channels-last bf16, channels zero-padded to 16) + gradient
    plan.ctx, plan.dctx, t_l = {}, {}, T
    for i, c in enumerate(net.context_channels):
        t_l //= net.factors[i]
        if c > 0:
            plan.ctx[i] = torch.zeros(B, t_l, ops.round_up(c, 16), dtype=bf16, device=dev)
            plan.dctx[i] = torch.zeros(B, t_l, ops.round_up(c, 16), dtype=bf16, device=dev)

    # ---- statistics + gradient arenas
    n_items = sum(len(lv.items_down) + len(lv.items_up) for lv in levels)
    arena = torch.zeros(7 * n_items + 4 * len(levels) + 8, B, G, 2, dtype=torch.float64, device=dev)
    slot = [0]

    def new_stats():
        s = arena[slot[0]]
        slot[0] += 1
        return s

    plan.fwd.append(lambda: (arena.zero_(), plan.loss_sum.zero_()))
    refreshers: List = []                  # re-pack the dgrad weights in place after a weight update

    def packed_dgrad(make):
        t = make()
        refreshers.append(lambda t=t, make=make: t.copy_(make()))
        return t

    grads: Dict[int, Tensor] = {}          # id(param) -> fp32 gradient (PyTorch layout / packed)
    finals: List = []                      # closures turning packed grads into PyTorch layout
    # one flat fp32 arena for every gradient accumulator: a single memset per backward
    n_param = sum(p.numel() for p in net.parameters())
    flat = torch.zeros(int(1.25 * n_param) + 64 * (4 * n_param // 1000 + 4096), device=dev)
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
    mod = net.use_modulation       # False: no ModulationItems, SkipCat merges (reference components.py:90,99)
    ss_all = _zeros((B, max(8, ops.round_up(n_tot, 8))), dev)
    dss_all = gbuf(ss_all.shape)
    ss_stride = ss_all.shape[1]
    if mod:
        cond_bias = _pad_to(P["cond_b"], ss_all.shape[1])
        plan.fwd.append(lambda: plan.cond_bf.copy_(plan.cond.view(1, B, Fm)))
        plan.fwd.append(lambda: ops.conv_gemm(plan.cond_bf, P["cond_w"], ss_all.view(1, B, -1), c_in=Fm,
                                              n_valid=ss_all.shape[1], bias=cond_bias))

    # ---- cross-attention context: LayerNorm(embedding) once per forward (the per-item
    # norm_context affines are folded into each item's to_kv weights)
    en = den = None
    if M:
        en, den = act(B, M, E), torch.zeros(B, M, E, dtype=bf16, device=dev)
        plan.fwd.append(lambda: ops.ln_film(plan.embedding, en, None, 0, None, G, net.ATT_LN_EPS))
    delta_ws = [None]    # shared fp32 workspace of adp_attention_bwd, sized for the largest item

    def delta_for(Tl: int) -> Tensor:
        if delta_ws[0] is None or delta_ws[0].numel() < B * heads * Tl:
            delta_ws[0] = _zeros((B * heads * Tl,), dev)
        return delta_ws[0]

    def conv3_bwd(dy: Tensor, a_in: Tensor, gw: Tensor, da: Tensor, wd: Tensor, C: int):
        """dy: grad of the conv output; a_in: its input; writes da, accumulates dW (3 taps)."""
        ops.wgrad(dy, a_in, gw, n=C, k=C, off=-1, ntaps=3)
        ops.conv_gemm(dy, wd, da, c_in=C, n_valid=C, taps=(-1, 0, 1))

    # ---- AttentionItem / CrossAttentionItem (a_unet): x + to_out(softmax(q k^T / 8) v)
    def attention_block(x: Tensor, xn: Tensor, ap: Dict, am, cross: bool, Tl: int, C: int,
                        out_stats: Optional[Tensor]):
        """x: the item's input (residual); xn = LayerNorm(x) (affine folded into the projections).
        Appends the forward launches; returns (y2, backward closure dy2 -> dx)."""
        o, y2 = act(B, Tl, mid), act(B, Tl, C)
        lse = _zeros((B, heads, Tl), dev)
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
            qkv, dqkv = act(B, Tl, 3 * mid), act(B, Tl, 3 * mid)
            q, k, v = qkv[..., :mid], qkv[..., mid:2 * mid], qkv[..., 2 * mid:]
            plan.fwd.append(lambda: ops.conv_gemm(xn, ap["w_qkv"], qkv, c_in=C, n_valid=3 * mid,
                                                  bias=ap["b_qkv"]))
            plan.fwd.append(lambda: ops.attention(q, k, v, o, heads, att_scale, lse=lse))

            def make_wd():
                wf = torch.cat([am.to_q.weight.detach().float() * g1.detach().float()[None, :],
                                am.to_kv.weight.detach().float() * g2.detach().float()[None, :]], 0)
                return ops.pack_linear(wf.t().contiguous())          # [C, 3*mid]
            wd_qkv = packed_dgrad(make_wd)
            gwf, dbf = gbuf((3 * mid, C)), gbuf((3 * mid,))

            def bwd(dy2: Tensor) -> Tensor:
                ops.conv_gemm(dy2, wd_out, d_o, c_in=C, n_valid=mid)
                ops.wgrad(dy2, o, gw_out, n=C, k=mid)
                ops.attention_bwd(q, k, v, o, d_o, lse, delta_ws[0], dqkv[..., :mid],
                                  dqkv[..., mid:2 * mid], dqkv[..., 2 * mid:], heads, att_scale)
                ops.conv_gemm(dqkv, wd_qkv, dxn, c_in=3 * mid, n_valid=C)
                ops.wgrad(dqkv, xn, gwf, n=3 * mid, k=C)
                ops.colsum(dqkv, dbf)
                ops.ln_fold_bwd(am.to_q.weight, g1, b1, gwf[:mid], dbf[:mid], dWq, dg1, db1)
                ops.ln_fold_bwd(am.to_kv.weight, g2, b2, gwf[mid:], dbf[mid:], dWkv, dg2, db2)
                ops.ln_film_bwd(dxn, x, None, 0, dx, dres=dy2, eps=net.ATT_LN_EPS)
                return dx
        else:
            q, kv = act(B, Tl, mid), act(B, M, 2 * mid)
            dq, dkv = act(B, Tl, mid), act(B, M, 2 * mid)
            plan.fwd.append(lambda: ops.conv_gemm(en, ap["w_kv"], kv, c_in=E, n_valid=2 * mid,
                                                  bias=ap["b_kv"]))
            plan.fwd.append(lambda: ops.conv_gemm(xn, ap["w_q"], q, c_in=C, n_valid=mid, bias=ap["b_q"]))
            plan.fwd.append(lambda: ops.attention(q, kv[..., :mid], kv[..., mid:], o, heads, att_scale,
                                                  lse=lse))
            wd_q = packed_dgrad(lambda: ops.pack_linear(
                (am.to_q.weight.detach().float() * g1.detach().float()[None, :]).t().contiguous()))
            wd_kv = packed_dgrad(lambda: ops.pack_linear(
                (am.to_kv.weight.detach().float() * g2.detach().float()[None, :]).t().contiguous()))
            gwq, dbq = gbuf((mid, C)), gbuf((mid,))
            gwkv, dbkv = gbuf((2 * mid, E)), gbuf((2 * mid,))

            def bwd(dy2: Tensor) -> Tensor:
                ops.conv_gemm(dy2, wd_out, d_o, c_in=C, n_valid=mid)
                ops.wgrad(dy2, o, gw_out, n=C, k=mid)
                ops.attention_bwd(q, kv[..., :mid], kv[..., mid:], o, d_o, lse, delta_ws[0], dq,
                                  dkv[..., :mid], dkv[..., mid:], heads, att_scale)
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
        plan.fwd.append(lambda: ops.conv_gemm(o, ap["w_out"], y2, c_in=mid, n_valid=C, residual=x,
                                              stats=out_stats, groups=G))
        return y2, bwd

    # ---- one chain of [ResnetItem, ModulationItem, AttentionItem?, CrossAttentionItem?]
    def run_items(x: Tensor, x_stats: Tensor, items_p: List[Dict], items_m, lv: LevelParams, Tl: int,
                  li: int = 0):
        C = lv.ch
        narrow = C == 8
        bwds: List = []
        for ip, im in zip(items_p, items_m):
            r_ = im.resnet
            ss = ss_all[:, ip["ss_off"]:] if mod else None
            dss = dss_all[:, ip["ss_off"]:] if mod else None
            has_att, has_cross, has_inj = im.attention is not None, im.cross is not None, im.inject is not None
            h_stats = new_stats()
            y_stats = None if (has_att or has_cross or has_inj) else new_stats()
            S1, S2 = new_stats(), new_stats()
            h, rr = act(B, Tl, C), act(B, Tl, C)
            # without a ModulationItem the ResnetItem's output is the item's output: conv2 writes
            # it (and its GroupNorm statistics) directly
            y = act(B, Tl, C) if mod else rr
            rs = None if mod else y_stats
            xn_first = act(B, Tl, C) if ((has_att or has_cross) and not has_inj and mod) else None
            dgn1 = (grad_for(r_.gn1.weight), grad_for(r_.gn1.bias))
            dgn2 = (grad_for(r_.gn2.weight), grad_for(r_.gn2.bias))
            db1, db2 = grad_for(r_.conv1.bias), grad_for(r_.conv2.bias)
            dr, dh, dx, dxh = act(B, Tl, C), act(B, Tl, C), act(B, Tl, C), act(B, Tl, C)

            def modulation_fwd(rr=rr, y=y, ss=ss, ys=y_stats, xn=xn_first):
                ops.ln_film(rr, y, ss, ss_stride, ys, G, net.MOD_LN_EPS, y2=xn, eps2=net.ATT_LN_EPS)
            if narrow:
                dw1, dw2 = grad_for(r_.conv1.weight), grad_for(r_.conv2.weight)
                db_scratch = gbuf((C,))
                plan.fwd.append(lambda x=x, h=h, s=x_stats, hs=h_stats, ip=ip: ops.narrow_conv(
                    x, h, s, ip["gn1"][0], ip["gn1"][1], ip["w1"], ip["b1"], G, stats_out=hs))
                plan.fwd.append(lambda x=x, h=h, rr=rr, hs=h_stats, ip=ip, rs=rs: ops.narrow_conv(
                    h, rr, hs, ip["gn2"][0], ip["gn2"][1], ip["w2"], ip["b2"], G, residual=x, stats_out=rs))
                if mod:
                    plan.fwd.append(modulation_fwd)

                def bwd(dy, x=x, h=h, rr=rr, ss=ss, dss=dss, xs=x_stats, hs=h_stats, ip=ip, dr=dr,
                        dh=dh, dx=dx, dxh=dxh, S1=S1, S2=S2, dgn1=dgn1, dgn2=dgn2, dw1=dw1, dw2=dw2,
                        db1=db1, db2=db2, db_scratch=db_scratch):
                    if mod:
                        ops.ln_film_bwd(dy, rr, ss, ss_stride, dr, dss=dss, dss_stride=ss_stride,
                                        eps=net.MOD_LN_EPS)
                    else:
                        dr = dy
                    ops.narrow_conv_bwd(dr, h, hs, ip["gn2"][0], ip["gn2"][1], ip["w2"], dxh, dgn2[0],
                                        dgn2[1], S2, dw2, db2, G)
                    ops.gn_bwd_apply(dxh, h, hs, S2, dh, G, colsum=db1)   # fp32 sum, pre-rounding
                    ops.narrow_conv_bwd(dh, x, xs, ip["gn1"][0], ip["gn1"][1], ip["w1"], dxh, dgn1[0],
                                        dgn1[1], S1, dw1, db_scratch, G)
                    ops.gn_bwd_apply(dxh, x, xs, S1, dx, G, dres=dr)
                    return dx
            else:
                a1, a2 = act(B, Tl, C), act(B, Tl, C)
                wd1 = packed_dgrad(lambda r_=r_: ops.pack_conv_dgrad(r_.conv1.weight.detach()))
                wd2 = packed_dgrad(lambda r_=r_: ops.pack_conv_dgrad(r_.conv2.weight.detach()))
                plan.fwd.append(lambda x=x, a1=a1, s=x_stats, ip=ip: ops.gn_silu(
                    x, a1, s, ip["gn1"][0], ip["gn1"][1], G, net.GN_EPS))
                plan.fwd.append(lambda a1=a1, h=h, hs=h_stats, ip=ip: ops.conv_gemm(
                    a1, ip["w1"], h, c_in=C, n_valid=C, taps=(-1, 0, 1), bias=ip["b1"], stats=hs, groups=G))
                plan.fwd.append(lambda a2=a2, h=h, hs=h_stats, ip=ip: ops.gn_silu(
                    h, a2, hs, ip["gn2"][0], ip["gn2"][1], G, net.GN_EPS))
                plan.fwd.append(lambda x=x, a2=a2, rr=rr, ip=ip, rs=rs: ops.conv_gemm(
                    a2, ip["w2"], rr, c_in=C, n_valid=C, taps=(-1, 0, 1), bias=ip["b2"], residual=x,
                    stats=rs, groups=G))
                if mod:
                    plan.fwd.append(modulation_fwd)
                da = act(B, Tl, C)
                # [tap][co][ci] accumulators of the fused 3-tap wgrad -> PyTorch [co][ci][tap]
                gw = {"w1": grad_for(r_.conv1.weight, (3, C, C), (1, 2, 0)),
                      "w2": grad_for(r_.conv2.weight, (3, C, C), (1, 2, 0))}

                def bwd(dy, x=x, h=h, rr=rr, a1=a1, a2=a2, ss=ss, dss=dss, xs=x_stats, hs=h_stats,
                        ip=ip, dr=dr, dh=dh, dx=dx, dxh=dxh, da=da, S1=S1, S2=S2, dgn1=dgn1,
                        dgn2=dgn2, db1=db1, db2=db2, wd1=wd1, wd2=wd2, gw=gw, C=C):
                    if mod:
                        ops.ln_film_bwd(dy, rr, ss, ss_stride, dr, dss=dss, dss_stride=ss_stride,
                                        colsum=db2, eps=net.MOD_LN_EPS)
                    else:
                        dr = dy
                        ops.colsum(dy, db2)
                    conv3_bwd(dr, a2, gw["w2"], da, wd2, C)
                    ops.gn_silu_bwd(da, h, hs, ip["gn2"][0], ip["gn2"][1], dxh, dgn2[0], dgn2[1], S2, G)
                    ops.gn_bwd_apply(dxh, h, hs, S2, dh, G, colsum=db1)
                    conv3_bwd(dh, a1, gw["w1"], da, wd1, C)
                    ops.gn_silu_bwd(da, x, xs, ip["gn1"][0], ip["gn1"][1], dxh, dgn1[0], dgn1[1], S1, G)
                    ops.gn_bwd_apply(dxh, x, xs, S1, dx, G, dres=dr)
                    return dx
            if mod:
                grads[id(im.modulation.proj.weight)] = ("cond_w", ip["ss_off"], 2 * C)
                grads[id(im.modulation.proj.bias)] = ("cond_b", ip["ss_off"], 2 * C)
            chain = [bwd]
            x, x_stats = y, y_stats
            xn = xn_first
            if has_inj:
                # a_unet InjectChannelsItem: conv1x1(cat([x, ctx])) + x, W = [W_x | W_c]
                jp, conv = ip["inj"], im.inject
                ctxb, dctxb = plan.ctx[li], plan.dctx[li]
                n_ctx, ctx_pad = conv.weight.shape[1] - C, ctxb.shape[-1]
                tmp, yi, dyi = act(B, Tl, C), act(B, Tl, C), act(B, Tl, C)
                inj_stats = None if (has_att or has_cross) else new_stats()
                plan.fwd.append(lambda ctxb=ctxb, jp=jp, tmp=tmp, x=x: ops.conv_gemm(
                    ctxb, jp["w_c"], tmp, c_in=ctxb.shape[-1], n_valid=C, bias=jp["b"], residual=x))
                plan.fwd.append(lambda x=x, jp=jp, tmp=tmp, yi=yi, st=inj_stats: ops.conv_gemm(
                    x, jp["w_x"], yi, c_in=C, n_valid=C, residual=tmp, stats=st, groups=G))
                gw_inj = grad_for(conv.weight, (C, C + n_ctx, 1)).view(C, C + n_ctx)
                db_inj = grad_for(conv.bias)
                wd_x = packed_dgrad(lambda conv=conv, C=C: ops.pack_linear(
                    conv.weight.detach()[:, :C, 0].t().contiguous()))

                def make_wd_c(conv=conv, C=C, ctx_pad=ctx_pad, n_ctx=n_ctx):
                    w = torch.zeros(ctx_pad, C, device=dev)
                    w[:n_ctx] = conv.weight.detach().float()[:, C:, 0].t()
                    return ops.pack_linear(w)
                wd_c = packed_dgrad(make_wd_c)

                def inj_bwd(d_out, x=x, ctxb=ctxb, dctxb=dctxb, gw_inj=gw_inj, db_inj=db_inj, wd_x=wd_x,
                            wd_c=wd_c, dyi=dyi, C=C, n_ctx=n_ctx, ctx_pad=ctx_pad):
                    ops.colsum(d_out, db_inj)
                    ops.wgrad(d_out, x, gw_inj[:, :C], n=C, k=C)
                    ops.wgrad(d_out, ctxb, gw_inj[:, C:], n=C, k=n_ctx)
                    # d context, summed over the items of this depth (in place through the residual)
                    ops.conv_gemm(d_out, wd_c, dctxb, c_in=C, n_valid=ctx_pad, residual=dctxb)
                    ops.conv_gemm(d_out, wd_x, dyi, c_in=C, n_valid=C, residual=d_out)   # + the identity path
                    return dyi
                chain.append(inj_bwd)
                x, x_stats = yi, inj_stats
            for kind, am in (("att", im.attention), ("cross", im.cross)):
                if am is None:
                    continue
                last = kind == "cross" or not has_cross
                ost = new_stats() if last else None
                if xn is None:                       # second attention of the item: its own pre-norm
                    xn = act(B, Tl, C)
                    plan.fwd.append(lambda x=x, xn=xn: ops.ln_film(x, xn, None, 0, None, G, net.ATT_LN_EPS))
                x, att_bwd = attention_block(x, xn, ip[kind], am, kind == "cross", Tl, C, ost)
                x_stats, xn = ost, None
                chain.append(att_bwd)

            def item_bwd(dy, chain=chain):
                for fn in reversed(chain):
                    dy = fn(dy)
                return dy
            bwds.append(item_bwd)
        return x, x_stats, bwds

    # ---- recursive level walk; returns (output tensor, its stats, backward closure)
    def level(i: int, x_in: Optional[Tensor], T_in: int):
        lv, Lp = levels[i], P["levels"][i]
        Tl, C = T_in // lv.factor, lv.ch
        innermost = i == len(levels) - 1
        # gradient-arena cursor at the level's sequence points: the arena is laid out in FORWARD
        # build order, so "down part", "inner levels" and "up part" of a level are three
        # contiguous ranges; the backward finishes them in the order up, inner, down and
        # announces each range through plan.mark (overlapped gradient all-reduce, parallel.py)
        cur = {"entry": cursor[0]}
        x0, st0 = act(B, Tl, C), new_stats()
        db_down = grad_for(lv.down.bias)
        if i == 0:
            dw_down = grad_for(lv.down.weight)
            plan.fwd.append(lambda: ops.stem_in(plan.x, Lp["down_w"], Lp["down_b"], x0, lv.factor,
                                                append=plan.append, noise=plan.noise, alpha=plan.alpha,
                                                beta=plan.beta, stats=st0, groups=G))
        else:
            kdim = lv.factor * lv.in_ch
            plan.fwd.append(lambda: ops.conv_gemm(x_in.view(B, Tl, kdim), Lp["down_w"], x0, c_in=kdim,
                                                  n_valid=C, bias=Lp["down_b"], stats=st0, groups=G))
            wd_down = packed_dgrad(lambda: ops.pack_linear(
                lv.down.weight.detach().permute(0, 2, 1).reshape(C, kdim).t().contiguous()))
            # [co][tap][ci] (the [B, T/f, f*C] view) -> PyTorch [co][ci][tap]
            gw_down = grad_for(lv.down.weight, (C, lv.factor, lv.in_ch), (0, 2, 1)).view(C, kdim)
        x, st, items_down_bwd = run_items(x0, st0, Lp["items_down"], lv.items_down, lv, Tl, li=i)
        cur["down_end"] = cursor[0]
        inner = None
        skip = x
        if not innermost:
            x, st, inner = level(i + 1, skip, Tl)
        cur["inner_end"] = cursor[0]
        x, st, items_up_bwd = run_items(x, st, Lp["items_up"], lv.items_up, lv, Tl, li=i)
        s_cat = 2 ** -0.5
        if mod:
            gate = ss_all[:, Lp["gate_off"]:]
            dgate = dss_all[:, Lp["gate_off"]:]
            grads[id(lv.merge.weight)] = ("cond_w", Lp["gate_off"], lv.out_ch)
            grads[id(lv.merge.bias)] = ("cond_b", Lp["gate_off"], lv.out_ch)
        x_last = x
        if i == 0 and not mod:
            # SkipCat at level 0 runs in the stem kernels with the 1x1 merge conv folded into both
            # branches (B200UNet._compute_packed): they produce the gradients of the FOLDED
            # weights, unfolded below (a few hundred numbers) into merge / up / adapter gradients
            Co, Ci = lv.out_ch, lv.in_ch
            gate, dgate = torch.ones(B, 8, device=dev), gbuf((B, 8))
            dw_up, db_up = gbuf((Co, C, 3)), gbuf((Co,))
            dwa, dba = gbuf((Co, Ci)), gbuf((Co,))

            def unfold_level0():
                wm = lv.merge.weight.detach().float()[:, :, 0]
                wc1, wc2 = wm[:, :Co], wm[:, Co:]
                w_up, b_up = lv.up.weight.detach().float(), lv.up.bias.detach().float()
                grads[id(lv.up.weight)] = torch.einsum("om,ock->mck", wc2, dw_up)
                grads[id(lv.up.bias)] = wc2.t() @ db_up
                d_wc2 = torch.einsum("ock,mck->om", dw_up, w_up) + torch.outer(db_up, b_up)
                if lv.adapter is not None:
                    w_ad = lv.adapter.weight.detach().float()[:, :, 0]
                    b_ad = lv.adapter.bias.detach().float()
                    grads[id(lv.adapter.weight)] = s_cat * (wc1.t() @ dwa)
                    grads[id(lv.adapter.bias)] = s_cat * (wc1.t() @ dba)
                    d_wc1 = s_cat * (dwa @ w_ad.t() + torch.outer(dba, b_ad))
                else:
                    d_wc1 = s_cat * dwa
                grads[id(lv.merge.weight)] = torch.cat([d_wc1, d_wc2], dim=1)
                grads[id(lv.merge.bias)] = db_up.clone()
            finals.append(unfold_level0)
        else:
            db_up = grad_for(lv.up.bias)
        if i == 0:
            if mod:
                dw_up = grad_for(lv.up.weight)
                dwa = (grad_for(lv.adapter.weight, (lv.out_ch, lv.in_ch, 1)).view(lv.out_ch, lv.in_ch)
                       if lv.adapter is not None else None)
                dba = grad_for(lv.adapter.bias) if lv.adapter is not None else None
            dh0 = act(B, Tl, C)
            plan.fwd.append(lambda: ops.stem_out(
                x_last, plan.x, Lp["up_w"], Lp["up_b"], gate, lv.factor, append=plan.append,
                w_adapt=Lp.get("adapt_w"), b_adapt=Lp.get("adapt_b"), noise=plan.noise,
                alpha=plan.alpha, beta=plan.beta, loss_sum=plan.loss_sum if loss_mode else None,
                dv=plan.dv if loss_mode else None, v_out=plan.v))

            def backward_level0():
                ops.stem_out_bwd(plan.dv, x_last, plan.x, Lp["up_w"], Lp["up_b"], gate, lv.factor, dh0,
                                 dw_up, db_up, dgate, gscale=plan.gscale, append=plan.append,
                                 noise=plan.noise, alpha=plan.alpha, beta=plan.beta,
                                 w_adapt=Lp.get("adapt_w"), dw_adapt=dwa, db_adapt=dba, dxin=plan.dxin)
                d = dh0
                for b_ in reversed(items_up_bwd):
                    d = b_(d)
                if inner is not None:
                    plan.mark((cur["inner_end"], cur["exit"]))
                    d = inner(d)
                for b_ in reversed(items_down_bwd):
                    d = b_(d)
                ops.stem_in_bwd(d, plan.x, dw_down, db_down, lv.factor, append=plan.append,
                                noise=plan.noise, alpha=plan.alpha, beta=plan.beta,
                                w=Lp["down_w"], dxin=plan.dxin)
                plan.mark((cur["entry"], cur["down_end"] if inner is not None else cur["exit"]))
            cur["exit"] = cursor[0]
            return None, None, backward_level0

        # levels >= 1: up conv writes y (pre-gate), skip_gate merges with the level's input
        f, Co = lv.factor, lv.out_ch
        y_up, out, ost = act(B, T_in, Co), act(B, T_in, Co), new_stats()
        dys, dx_last, d_xin = act(B, T_in, Co), act(B, Tl, C), act(B, T_in, lv.in_ch)
        if f > 1:
            plan.fwd.append(lambda: ops.conv_gemm(x_last, Lp["up_w"], y_up.view(B, Tl, f * Co), c_in=C,
                                                  n_valid=Co, up_factor=f, bias=Lp["up_b"]))

            def make_wd_up():
                w = lv.up.weight.detach().float()
                w0, w1, w2 = w[:, :, 0], w[:, :, 1], w[:, :, 2]
                wd = torch.zeros(3, C, f * Co, device=dev)      # taps read dys rows q-1, q, q+1
                wd[2, :, 0:Co] = w0.t()                          # forward off -1 (phase 0, slot 0)
                wd[1, :, 0:Co] = (w1 + w2).t()
                wd[1, :, (f - 1) * Co:f * Co] = (w0 + w1).t()
                wd[0, :, (f - 1) * Co:f * Co] = w2.t()          # forward off +1 (last phase, slot 1)
                for p_ in range(1, f - 1):
                    wd[1, :, p_ * Co:(p_ + 1) * Co] = (w0 + w1 + w2).t()
                return ops._pad_rows(wd.permute(1, 0, 2).reshape(C, 3 * f * Co), ops.round_up(C, 16))
            wd_up = packed_dgrad(make_wd_up)
            gwc = gbuf((f, 2, Co, C))

            def up_wgrad():
                for p_ in range(f):
                    slots = [(0, -1), (1, 0)] if p_ == 0 else ([(0, 0), (1, 1)] if p_ == f - 1 else [(0, 0)])
                    for s_, off in slots:
                        ops.wgrad(dys.view(B, Tl, f * Co), x_last, gwc[p_, s_], n=Co, k=C, off=off,
                                  g_col0=p_ * Co)

            def up_final():
                g0 = gwc[0, 0] + gwc[f - 1, 0]
                g1 = gwc[0, 1] + gwc[f - 1, 0]
                g2 = gwc[0, 1] + gwc[f - 1, 1]
                for p_ in range(1, f - 1):
                    g0, g1, g2 = g0 + gwc[p_, 0], g1 + gwc[p_, 0], g2 + gwc[p_, 0]
                grads[id(lv.up.weight)] = torch.stack([g0, g1, g2], dim=-1)
            finals.append(up_final)

            def up_dgrad():
                ops.conv_gemm(dys.view(B, Tl, f * Co), wd_up, dx_last, c_in=f * Co, n_valid=C,
                              taps=(-1, 0, 1))
        else:
            plan.fwd.append(lambda: ops.conv_gemm(x_last, Lp["up_w"], y_up, c_in=C, n_valid=Co,
                                                  taps=(-1, 0, 1), bias=Lp["up_b"]))
            wd_up = packed_dgrad(lambda: ops.pack_conv_dgrad(lv.up.weight.detach()))
            gw3 = grad_for(lv.up.weight, (3, Co, C), (1, 2, 0))

            def up_wgrad():
                ops.wgrad(dys, x_last, gw3, n=Co, k=C, off=-1, ntaps=3)

            def up_dgrad():
                ops.conv_gemm(dys, wd_up, dx_last, c_in=Co, n_valid=C, taps=(-1, 0, 1))
        if mod:
            plan.fwd.append(lambda: ops.skip_gate(y_up, x_in, gate, out, ost, G))
            d_skip_of = lambda d_out: d_out      # noqa: E731  (the skip path's gradient is d_out itself)

            def merge_bwd(d_out: Tensor) -> None:
                ops.skip_gate_bwd(d_out, y_up, gate, dys, dgate)
        else:
            # SkipCat: out = (s Wc1) skip + Wc2 y_up + bc as two accumulating GEMMs; an 8-channel
            # level is processed two positions per row against block-diagonal weights (K >= 16)
            rp = max(1, 16 // Co)
            assert T_in % rp == 0, "SkipCat merge of an 8-channel level needs an even length"

            def rows(t):
                return t.view(B, T_in // rp, rp * Co)
            tmp, d_skip = act(B, T_in, Co), act(B, T_in, Co)
            plan.fwd.append(lambda: ops.conv_gemm(rows(x_in), Lp["cat_w1"], rows(tmp), c_in=rp * Co,
                                                  n_valid=rp * Co, bias=Lp["cat_b"]))
            plan.fwd.append(lambda: ops.conv_gemm(rows(y_up), Lp["cat_w2"], rows(out), c_in=rp * Co,
                                                  n_valid=rp * Co, residual=rows(tmp),
                                                  stats=ost if rp == 1 else None, groups=G))
            if rp > 1:
                plan.fwd.append(lambda: ops.gn_stats(out, ost, G))
            wm_ = lv.merge.weight
            wd_c1 = packed_dgrad(lambda: ops.pack_linear(torch.block_diag(
                *[wm_.detach().float()[:, :Co, 0].t() * s_cat] * rp).contiguous()))
            wd_c2 = packed_dgrad(lambda: ops.pack_linear(torch.block_diag(
                *[wm_.detach().float()[:, Co:, 0].t()] * rp).contiguous()))
            gw_cat = grad_for(wm_, (Co, 2 * Co, 1)).view(Co, 2 * Co)
            db_cat = grad_for(lv.merge.bias)
            blk1, blk2 = gbuf((rp * Co, rp * Co)), gbuf((rp * Co, rp * Co))
            d_skip_of = lambda d_out: d_skip     # noqa: E731

            def merge_bwd(d_out: Tensor) -> None:
                ops.colsum(d_out, db_cat)
                ops.wgrad(rows(d_out), rows(x_in), blk1, n=rp * Co, k=rp * Co)
                ops.wgrad(rows(d_out), rows(y_up), blk2, n=rp * Co, k=rp * Co)
                # the diagonal blocks of the paired-position products sum to the 1x1 conv's gradient
                gw_cat[:, :Co].copy_(blk1.view(rp, Co, rp, Co).diagonal(dim1=0, dim2=2).sum(-1) * s_cat)
                gw_cat[:, Co:].copy_(blk2.view(rp, Co, rp, Co).diagonal(dim1=0, dim2=2).sum(-1))
                ops.conv_gemm(rows(d_out), wd_c2, rows(dys), c_in=rp * Co, n_valid=rp * Co)
                ops.conv_gemm(rows(d_out), wd_c1, rows(d_skip), c_in=rp * Co, n_valid=rp * Co)

        def backward_level(d_out: Tensor) -> Tensor:
            merge_bwd(d_out)
            ops.colsum(dys, db_up)
            up_wgrad()
            up_dgrad()
            d = dx_last
            for b_ in reversed(items_up_bwd):
                d = b_(d)
            if inner is not None:
                plan.mark((cur["inner_end"], cur["exit"]))
                d = inner(d)
            for b_ in reversed(items_down_bwd):
                d = b_(d)
            ops.colsum(d, db_down)
            kdim = lv.factor * lv.in_ch
            ops.wgrad(d, x_in.view(B, Tl, kdim), gw_down, n=C, k=kdim, off=0)
            plan.mark((cur["entry"], cur["down_end"] if inner is not None else cur["exit"]))
            # gradient w.r.t. the level input = dgrad(down conv) + the skip path (d_out)
            ops.conv_gemm(d, wd_down, d_xin.view(B, Tl, kdim), c_in=C, n_valid=kdim,
                          residual=d_skip_of(d_out).view(B, Tl, kdim))
            return d_xin

        cur["exit"] = cursor[0]
        return out, ost, backward_level

    _, _, backward0 = level(0, None, T)
    assert slot[0] <= arena.shape[0]
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
    if not net.use_cuda_graph:
        for r in plan.refreshers:
            r()
        return
    if getattr(plan, "refresh_graph", None) is None:
        for r in plan.refreshers:
            r()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for r in plan.refreshers:
                r()
        plan.refresh_graph = g
    else:
        plan.refresh_graph.replay()


def _run(plan: _TrainPlan, which: str, use_graph: bool) -> None:
    """Eager on the first call, captured on the second, replayed afterwards."""
    prog = (lambda: [f() for f in plan.fwd]) if which == "f" else plan.backward_program
    runs = plan.runs_f if which == "f" else plan.runs_b
    graph = plan.graph_f if which == "f" else plan.graph_b
    if not use_graph or runs == 0:
        prog()
    elif graph is None:
        g = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        with torch.cuda.graph(g):
            prog()
        if which == "f":
            plan.graph_f = g
        else:
            plan.graph_b = g
        g.replay()
    else:
        graph.replay()
    if which == "f":
        plan.runs_f += 1
    else:
        plan.runs_b += 1


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
    plan.runs_b += 1
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
        if net.verify_fp32:
            raise NotImplementedError("B200UNet.verify_fp32 covers inference and sampling; run it under "
                                      "torch.no_grad() (the differentiable program is bf16 only)")
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
        for d_, c_ in zip(ctx_depths, context):      # [B, ctx, T_d] -> channels-last bf16
            plan.ctx[d_][:, :, : c_.shape[1]].copy_(c_.transpose(1, 2))
        plan.cond.copy_(cond)
        _run(plan, "f", net.use_cuda_graph)
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
            _run(plan, "b", net.use_cuda_graph)
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
        t = net.time
        s = sigmas.float().reshape(-1, 1)
        fr = s * t.weights * 2 * pi
        emb = t.to_out(torch.cat([s, fr.sin(), fr.cos()], dim=-1))
        f = F.gelu(t.mlp(F.gelu(t.mlp(F.gelu(emb)))))
        if features is not None:
            f = f + features
    elif not net.use_modulation:         # no ModulationItems: nothing consumes the features
        ref = next(net.parameters())
        return torch.zeros(1, net.features, device=ref.device)
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
    assert x.is_cuda, "the CUDA path runs on a CUDA device only (no CPU fallback)"
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
    assert x.is_cuda, "the CUDA path runs on a CUDA device only (no CPU fallback)"
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
