"""UNetV0 on H100: the reference's `net_t` plugin slot (reference components.py:34-105),
rebuilt over the sm_90a kernels of libadp_b200.so.

`UNetV0(dim=1, in_channels=..., channels=[...], ...)` takes the reference's kwargs verbatim
and returns an nn.Module with the reference's call signature

    net(x[B,Cin,T], time[B], *, features=None, embedding=None, embedding_scale=1.0,
        embedding_mask_proba=0.0, channels=None[, append_channels]) -> [B,Cout,T]

Parameters keep PyTorch shapes (Conv1d [co,ci,k], Linear [out,in]) and are registered in
the same order as the a_unet module tree, so `load_reference_parameters` copies a reference
model's weights positionally.  The forward pass is a flat *program*: a list of kernel
launches over pre-allocated channels-last bf16 buffers, captured into one CUDA graph per
(batch, length) shape; nothing in it falls back to PyTorch ops or to the CPU.
"""
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor, nn
from torch.optim.optimizer import register_optimizer_step_post_hook

from . import _lib, ops


def exists(v) -> bool:
    return v is not None


def default(v, d):
    return v if exists(v) else d


# ----------------------------------------------------------------------------- parameters
class ResnetParams(nn.Module):
    """a_unet ResnetBlock: (GroupNorm, SiLU, Conv1d k3) x 2 + identity shortcut."""

    def __init__(self, channels: int, groups: int):
        super().__init__()
        self.gn1 = nn.GroupNorm(groups, channels)
        self.conv1 = nn.Conv1d(channels, channels, 3, padding=1)
        self.gn2 = nn.GroupNorm(groups, channels)
        self.conv2 = nn.Conv1d(channels, channels, 3, padding=1)


class ModulationParams(nn.Module):
    """a_unet Modulation: Linear(SiLU(features)) -> (scale, shift); LayerNorm has no params."""

    def __init__(self, channels: int, features: int):
        super().__init__()
        self.proj = nn.Linear(features, 2 * channels)


class AttentionParams(nn.Module):
    """a_unet Attention: norm, norm_context, to_q, to_kv, to_out (no biases)."""

    def __init__(self, channels: int, head_features: int, heads: int,
                 context_features: Optional[int] = None):
        super().__init__()
        mid = head_features * heads
        ctx = default(context_features, channels)
        self.norm = nn.LayerNorm(channels)
        self.norm_context = nn.LayerNorm(ctx)
        self.to_q = nn.Linear(channels, mid, bias=False)
        self.to_kv = nn.Linear(ctx, 2 * mid, bias=False)
        self.to_out = nn.Linear(mid, channels, bias=False)


class ItemParams(nn.Module):
    """One repetition of [ResnetItem, ModulationItem?, InjectChannelsItem?] + [AttentionItem] * att
    + [CrossAttentionItem] * cross (reference components.py:89-95).  The first attention and
    cross-attention are `attention` / `cross`; further ones follow each in `extra_attention` /
    `extra_cross`, registered only when a count exceeds 1 (a net with counts <= 1 keeps the
    state_dict keys it always had)."""

    def __init__(self, channels: int, groups: int, features: int, att: int, cross: int,
                 head_features: Optional[int], heads: Optional[int],
                 embedding_features: Optional[int], context: int = 0, modulation: bool = True):
        super().__init__()
        self.resnet = ResnetParams(channels, groups)
        self.modulation = ModulationParams(channels, features) if modulation else None
        # a_unet InjectChannelsItem: Conv1d(C + ctx -> C, k=1) over cat([x, channels[depth]]), + x
        self.inject = nn.Conv1d(channels + context, channels, 1) if context > 0 else None
        self.attention = AttentionParams(channels, head_features, heads) if att > 0 else None
        if att > 1:
            self.extra_attention = nn.ModuleList(
                [AttentionParams(channels, head_features, heads) for _ in range(att - 1)])
        self.cross = (AttentionParams(channels, head_features, heads, embedding_features)
                      if cross > 0 else None)
        if cross > 1:
            self.extra_cross = nn.ModuleList(
                [AttentionParams(channels, head_features, heads, embedding_features) for _ in range(cross - 1)])

    def attentions(self) -> List[AttentionParams]:
        """The item's AttentionItems in a_unet order."""
        first = [self.attention] if self.attention is not None else []
        return first + list(getattr(self, "extra_attention", []))

    def crosses(self) -> List[AttentionParams]:
        """The item's CrossAttentionItems in a_unet order (after every AttentionItem)."""
        first = [self.cross] if self.cross is not None else []
        return first + list(getattr(self, "extra_cross", []))


# the a_unet item types a chain may hold, by the name the program builder knows them under
ITEM_KINDS = ("resnet", "mod", "inj", "att", "cross")


class LevelParams(nn.Module):
    """a_unet Block: registration order = skip_adapter, (down, items, inner, items_up, up), merge."""

    def __init__(self, in_ch: int, out_ch: int, ch: int, factor: int, n_items: int, inner,
                 **item_kw):
        super().__init__()
        self.adapter = nn.Conv1d(in_ch, out_ch, 1) if in_ch != out_ch else None
        self.down = nn.Conv1d(in_ch, ch, factor, stride=factor)
        self.items_down = nn.ModuleList([ItemParams(ch, **item_kw) for _ in range(n_items)])
        self.inner = inner
        self.items_up = nn.ModuleList([ItemParams(ch, **item_kw) for _ in range(n_items)])
        self.up = nn.Conv1d(ch, out_ch, 3, padding=1)
        # a_unet SkipModulate (MergeModulate: Linear(features -> out)) or, with use_modulation=False,
        # SkipCat (MergeCat: Conv1d(2*out -> out, k=1) over cat([skip * 2^-0.5, y]))
        self.merge = (nn.Linear(item_kw["features"], out_ch) if item_kw.get("modulation", True)
                      else nn.Conv1d(2 * out_ch, out_ch, 1))
        self.in_ch, self.out_ch, self.ch, self.factor = in_ch, out_ch, ch, factor

    def chain(self, up: bool) -> List[Tuple[str, nn.Module]]:
        """The down (up=False) or up item chain as (kind, module) per a_unet item, in order."""
        out = []
        for it in (self.items_up if up else self.items_down):
            out.append(("resnet", it.resnet))
            if it.modulation is not None:
                out.append(("mod", it.modulation))
            if it.inject is not None:
                out.append(("inj", it.inject))
            out += [("att", a) for a in it.attentions()] + [("cross", a) for a in it.crosses()]
        return out


class TimeParams(nn.Module):
    """a_unet TimeConditioningPlugin: NumberEmbedder + (Linear, GELU) applied twice (shared)."""

    def __init__(self, features: int, dim: int = 256):
        super().__init__()
        self.weights = nn.Parameter(torch.randn(dim // 2))
        self.to_out = nn.Linear(dim + 1, features)
        self.mlp = nn.Linear(features, features)


# -------------------------------------------------------------------------------- program
class _Pool:
    """Reuses activation buffers whose value is dead (better L2 residency than fresh ones)."""

    def __init__(self, device, reuse: bool, dtype=torch.bfloat16):
        self.device, self.reuse, self.dtype = device, reuse, dtype
        self.free: Dict[Tuple, List[Tensor]] = {}
        self.total_bytes = 0

    def get(self, *shape, dtype=None) -> Tensor:
        dtype = self.dtype if dtype is None else dtype
        key = (tuple(shape), dtype)
        lst = self.free.get(key)
        if self.reuse and lst:
            return lst.pop()
        t = torch.empty(*shape, dtype=dtype, device=self.device)
        self.total_bytes += t.numel() * t.element_size()
        return t

    def put(self, t: Optional[Tensor]) -> None:
        if t is not None and self.reuse:
            self.free.setdefault((tuple(t.shape), t.dtype), []).append(t)


class _Graphed:
    """A program that runs eagerly on its first call (every launch is validated), is captured into a
    CUDA graph on the second and replayed from then on.  With use_graph False it runs eagerly."""

    def __init__(self, run: Callable[[], None], early_weights: bool):
        self.run, self.early_weights = run, early_weights
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.runs = 0

    def __call__(self, use_graph: bool) -> None:
        if not use_graph or self.runs == 0:
            self.run()
        else:
            if self.graph is None:
                self.graph = _capture(self.run, self.early_weights)
            self.graph.replay()
        self.runs += 1


class _Plan(_Graphed):
    """A launch list and (after warm-up) its CUDA graph; an inference or sampling plan also holds
    everything tied to its input shape: static I/O buffers and workspaces.  early_weights: see
    _capture; the training forward is captured without it."""

    def __init__(self, early_weights: bool = True):
        super().__init__(self.run_eager, early_weights)
        self.prog: List[Callable[[], None]] = []
        self.n_launches = 0
        self.n_kernels = 0

    def add(self, fn: Callable[[], None]) -> None:
        self.prog.append(fn)
        self.n_launches += 1

    def run_eager(self) -> None:
        for fn in self.prog:
            fn()


def _refreshed(graph: Optional[torch.cuda.CUDAGraph], run: Callable[[], None],
               use_graph: bool) -> Optional[torch.cuda.CUDAGraph]:
    """One in-place refresh of packed weights; returns the graph to keep for the next one.  The
    first refresh runs eagerly (the allocator warms up) and is then captured without a replay;
    later ones replay that graph.  With use_graph False it runs eagerly."""
    if not use_graph:
        run()
    elif graph is None:
        run()
        graph = _capture(run)
    else:
        graph.replay()
    return graph


def _capture(run: Callable[[], None], early_weights: bool = False) -> torch.cuda.CUDAGraph:
    """run() captured into a CUDA graph (not executed).  early_weights: no kernel in the graph
    writes the packed weights, so the GEMMs may fetch them before their programmatic-dependency
    wait (conv_gemm.cu, early_w)."""
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    if early_weights:
        _lib.lib().adp_debug_set(2, 1)
    try:
        with torch.cuda.graph(g):
            run()
    finally:
        if early_weights:
            _lib.lib().adp_debug_set(2, 0)
    return g


class _ForwardWalk:
    """Emits the trunk's forward launches, shared by the inference / sampling plans
    (B200UNet._build_plan) and the training plan (training.build_train_plan): `trunk` walks the
    levels and emits the level-0 stems, the item chains, the down conv of levels >= 1 and their up
    conv + merge.  The callers own the conditioning, the statistics arena and the static I/O (`io`:
    x, append, embedding, ctx, from B200UNet._static_io), and pass the stems their mode's inputs and
    outputs.  Every emitter returns the tensors it used; the training plan builds its backward from
    them.

    keep=False: dead activations are reused, and the fusions that never write a tensor are used
    (FiLM in the narrow / thin-level conv, the thin-level kernel, the GroupNorm A-transform, the
    merge gate in the up-conv epilogue); only the innermost down chain ends with GroupNorm
    statistics (the next level's ResnetItem reads them).  keep=True: every buffer stays live, every
    tensor the backward reads is written, every chain end writes its statistics and attention keeps
    its log-sum-exp."""

    def __init__(self, net: "B200UNet", P: Dict, io, add: Callable, Bh: int, stats: Tensor, ss_all: Tensor,
                 keep: bool, add_ctx: Callable, en: Optional[Tensor] = None):
        self.net, self.P, self.io, self.add, self.Bh, self.keep = net, P, io, add, Bh, keep
        self.pool = _Pool(net.net.down.weight.device, reuse=not keep, dtype=net._act_dtype())
        self.stats, self.n_stats = stats, 0
        self.ss_all, self.ss_stride = ss_all, ss_all.shape[1]
        self.add_ctx = add_ctx
        self.en = en         # LayerNorm(embedding), shared by all cross-attentions; made on first use
        self.G = net.groups
        self.D = net.head_features or 64
        self.mid = (net.heads or 0) * self.D

    def new_stats(self) -> Tensor:
        s = self.stats[self.n_stats]
        self.n_stats += 1
        return s

    def trunk(self, outputs: Callable[[], Dict], **noising) -> Dict:
        """The whole trunk: stem_in (once per half of the rows under classifier-free guidance), the
        levels' chains, down and up convs, and stem_out.  noising: the fused loss's noise, alpha and
        beta, for both stems; outputs() -> stem_out's output arguments, called when the launch runs
        (a plan's cfg_scale is set after it is built).  Returns level 0's record: the level (i, lv,
        Lp), Tl, T_in, its input x_in, the unit records of its "down" and "up" chains, the "inner"
        level's record, the up chain's output x, the merge gate and, for levels >= 1, up_merge's
        out, ost and y_up."""
        io, G, Bh, levels = self.io, self.G, self.Bh, self.net.levels()
        B, _, T = io.x.shape

        def level(i: int, x_in: Optional[Tensor], T_in: int) -> Dict:
            lv, Lp = levels[i], self.P["levels"][i]
            Tl, innermost = T_in // lv.factor, i == len(levels) - 1
            rec = dict(i=i, lv=lv, Lp=Lp, Tl=Tl, T_in=T_in, x_in=x_in, inner=None)
            if i == 0:
                x, st = self.pool.get(Bh, Tl, lv.ch), self.new_stats()
                for h in range(Bh // B):
                    self.add(lambda x=x[h * B:(h + 1) * B], st=st[h * B:(h + 1) * B]: ops.stem_in(
                        io.x, Lp["down_w"], Lp["down_b"], x, lv.factor, append=io.append, stats=st, groups=G,
                        **noising))
            else:
                x, st = self.down(lv, Lp, x_in, Tl)
            x, st, rec["down"] = self.items(x, st, Lp["items_down"], lv.ch, Tl, i,
                                            last_needs_stats=self.keep or innermost)
            if not innermost:
                skip = x
                rec["inner"] = level(i + 1, skip, Tl)
                x, st = rec["inner"]["out"], rec["inner"]["ost"]
                self.pool.put(skip)
            x, st, rec["up"] = self.items(x, st, Lp["items_up"], lv.ch, Tl, i, last_needs_stats=self.keep)
            gate = self.ss_all[:, Lp["gate_off"]:] if self.net.merge == "modulate" else None
            if i == 0 and gate is None:
                # SkipCat (folded into the stem's weights) and SkipAdd run the stem epilogue with a unit gate
                gate = torch.ones(Bh, max(8, lv.out_ch), device=x.device)
            rec.update(x=x, gate=gate)
            if i > 0:
                rec["out"], rec["ost"], rec["y_up"] = self.up_merge(lv, Lp, x, x_in, Tl, T_in, gate)
            else:
                self.add(lambda: ops.stem_out(x, io.x, Lp["up_w"], Lp["up_b"], gate, lv.factor, append=io.append,
                                              w_adapt=Lp.get("adapt_w"), b_adapt=Lp.get("adapt_b"), **noising,
                                              **outputs()))
            return rec
        return level(0, None, T)

    def items(self, x: Tensor, x_stats: Tensor, chain: List[Tuple[str, Dict]], C: int, Tl: int, li: int,
              last_needs_stats: bool):
        """One item chain of level li: `chain` holds (kind, pack) per a_unet item, in order, kind in
        ITEM_KINDS.  Returns (output, its statistics, one record per emitted unit).

        The items are emitted in order, with these fusions wherever their pattern occurs: a
        ModulationItem right after a ResnetItem runs in that ResnetItem's epilogue or its ln_film
        pass, and that pass also writes the LayerNorm of an attention item right after it.  A unit
        writes the GroupNorm statistics of its output only when a ResnetItem reads them (the next
        item, or for the last one the caller's last_needs_stats).  Each record is (kind, index of
        its first item in the chain, number of items it covers, its tensors)."""
        recs, xn, i, n = [], None, 0, len(chain)
        while i < n:
            kind, pk = chain[i]
            width = 2 if (kind == "resnet" and i + 1 < n and chain[i + 1][0] == "mod") else 1
            j = i + width
            want_stats = chain[j][0] == "resnet" if j < n else last_needs_stats
            pre_norm = j < n and chain[j][0] in ("att", "cross")
            y_stats = self.new_stats() if want_stats else None
            if kind == "resnet":
                rec = self._resnet(x, x_stats, pk, chain[i + 1][1] if width == 2 else None, C, Tl, y_stats,
                                   pre_norm)
            elif kind == "mod":
                rec = self._modulation(x, pk, C, Tl, y_stats, pre_norm)
            elif kind == "inj":
                rec = self._inject(x, pk, C, Tl, li, y_stats)
            else:
                rec = self._attention(x, xn, pk, kind == "cross", C, Tl, y_stats)
            x, x_stats, xn = rec["y"], y_stats, rec.get("xn") if kind in ("resnet", "mod") else None
            recs.append((kind, i, width, rec))
            i = j
        return x, x_stats, recs

    def _resnet(self, x: Tensor, x_stats: Tensor, ip: Dict, mp: Optional[Dict], C: int, Tl: int,
                y_stats: Optional[Tensor], pre_norm: bool) -> Dict:
        """ResnetItem, and the ModulationItem right after it when mp (its pack) is given.  pre_norm:
        the Modulation pass also writes the following attention's LayerNorm (xn) when it runs as its
        own kernel."""
        net, pool, add, G, Bh, mod = self.net, self.pool, self.add, self.G, self.Bh, mp is not None
        narrow = C == 8 and not net.verify_fp32
        # thin levels (C = 32, 64) are HBM-bound: one fused ConvBlock kernel (mid_conv.cu)
        # instead of gn_silu -> conv_gemm (-> ln_film)
        fused = not self.keep and (narrow or (net.fuse_thin_levels and C in (32, 64) and not net.verify_fp32))
        ss = self.ss_all[:, mp["ss_off"]:] if mod else None
        (g1, be1), (g2, be2) = ip["gn1"], ip["gn2"]
        h_stats = self.new_stats()
        h = pool.get(Bh, Tl, C)
        r = a1 = a2 = xn = None
        if narrow or fused:
            w1, w2 = (ip["w1"], ip["w2"]) if narrow else (ip["w1_raw"], ip["w2_raw"])
            p1, p2 = (None, None) if narrow else (ip["w1_mid"], ip["w2_mid"])
            add(lambda: ops.narrow_conv(x, h, x_stats, g1, be1, w1, ip["b1"], G, stats_out=h_stats,
                                        gn_eps=net.GN_EPS, w_packed=p1))
        if fused:               # the Modulation runs in conv2's epilogue
            y = pool.get(Bh, Tl, C)
            add(lambda: ops.narrow_conv(h, y, h_stats, g2, be2, w2, ip["b2"], G, residual=x, scale_shift=ss,
                                        ss_stride=self.ss_stride, stats_out=y_stats, gn_eps=net.GN_EPS,
                                        ln_eps=net.MOD_LN_EPS, w_packed=p2))
        else:
            r = pool.get(Bh, Tl, C)
            y = pool.get(Bh, Tl, C) if mod else r
            # no ModulationItem: the ResnetItem's output IS the unit's output, so its
            # GroupNorm statistics come out of conv2's epilogue
            rs = None if mod else y_stats
            if narrow:
                add(lambda: ops.narrow_conv(h, r, h_stats, g2, be2, w2, ip["b2"], G, residual=x, stats_out=rs))
            elif net.fuse_groupnorm and not self.keep and C <= net.MAX_FUSED_GN_C:
                # ConvBlock = ONE kernel: GroupNorm+SiLU applied to the smem A tile
                add(lambda: ops.conv_gemm(x, ip["w1"], h, c_in=C, n_valid=C, taps=(-1, 0, 1), bias=ip["b1"],
                                          stats=h_stats, groups=G, gn=(x_stats, g1, be1, G, net.GN_EPS)))
                add(lambda: ops.conv_gemm(h, ip["w2"], r, c_in=C, n_valid=C, taps=(-1, 0, 1), bias=ip["b2"],
                                          residual=x, stats=rs, groups=G, gn=(h_stats, g2, be2, G, net.GN_EPS)))
            else:
                a1 = pool.get(Bh, Tl, C)
                add(lambda: ops.gn_silu(x, a1, x_stats, g1, be1, G, net.GN_EPS))
                add(lambda: ops.conv_gemm(a1, ip["w1"], h, c_in=C, n_valid=C, taps=(-1, 0, 1), bias=ip["b1"],
                                          stats=h_stats, groups=G))
                pool.put(a1)
                a2 = pool.get(Bh, Tl, C)
                add(lambda: ops.gn_silu(h, a2, h_stats, g2, be2, G, net.GN_EPS))
                add(lambda: ops.conv_gemm(a2, ip["w2"], r, c_in=C, n_valid=C, taps=(-1, 0, 1), bias=ip["b2"],
                                          residual=x, stats=rs, groups=G))
                pool.put(a2)
            if mod:
                xn = pool.get(Bh, Tl, C) if pre_norm else None
                # Modulation and the following attention pre-norm in ONE pass over the rows
                add(lambda: ops.ln_film(r, y, ss, self.ss_stride, y_stats, G, net.MOD_LN_EPS, y2=xn,
                                        eps2=net.ATT_LN_EPS))
                pool.put(r)
        pool.put(h)
        pool.put(x)             # a level's skip is the chain's *output*, never an item input
        return dict(x=x, x_stats=x_stats, h=h, h_stats=h_stats, r=r, a1=a1, a2=a2, y=y, ss=ss, xn=xn)

    def _modulation(self, x: Tensor, mp: Dict, C: int, Tl: int, y_stats: Optional[Tensor], pre_norm: bool) -> Dict:
        """A ModulationItem that does not follow a ResnetItem: y = LN(x) (1 + scale) + shift in one
        ln_film pass, which also writes the following attention's LayerNorm when pre_norm."""
        net, pool = self.net, self.pool
        ss = self.ss_all[:, mp["ss_off"]:]
        y = pool.get(self.Bh, Tl, C)
        xn = pool.get(self.Bh, Tl, C) if pre_norm else None
        self.add(lambda: ops.ln_film(x, y, ss, self.ss_stride, y_stats, self.G, net.MOD_LN_EPS, y2=xn,
                                     eps2=net.ATT_LN_EPS))
        pool.put(x)
        return dict(x=x, y=y, ss=ss, xn=xn)

    def _inject(self, x: Tensor, jp: Dict, C: int, Tl: int, li: int, y_stats: Optional[Tensor]) -> Dict:
        """InjectChannelsItem: conv1x1(cat([x, ctx])) + x as two accumulating GEMMs
        (W = [W_x | W_c]): tmp = ctx W_c^T + b + x ; y = x W_x^T + tmp."""
        pool, ctxb = self.pool, self.io.ctx[li]
        tmp, y = pool.get(self.Bh, Tl, C), pool.get(self.Bh, Tl, C)
        self.add(lambda: ops.conv_gemm(ctxb, jp["w_c"], tmp, c_in=ctxb.shape[-1], n_valid=C, bias=jp["b"],
                                       residual=x))
        self.add(lambda: ops.conv_gemm(x, jp["w_x"], y, c_in=C, n_valid=C, residual=tmp, stats=y_stats,
                                       groups=self.G))
        pool.put(tmp)
        pool.put(x)
        return dict(x=x, y=y, ctx=ctxb)

    def _attention(self, x: Tensor, xn: Optional[Tensor], ap: Dict, cross: bool, C: int, Tl: int,
                   y_stats: Optional[Tensor]) -> Dict:
        """AttentionItem / CrossAttentionItem: y = x + to_out(softmax(q k^T / sqrt(D)) v) with
        q, k, v projected from xn = LayerNorm(x) (affine folded into the projections); xn None:
        the LayerNorm runs here."""
        net, pool, add, Bh, mid, D = self.net, self.pool, self.add, self.Bh, self.mid, self.D
        o, y = pool.get(Bh, Tl, mid), pool.get(Bh, Tl, C)
        if xn is None:
            xn = pool.get(Bh, Tl, C)
            add(lambda: ops.ln_film(x, xn, None, 0, None, self.G, net.ATT_LN_EPS))
        lse = torch.zeros(Bh, net.heads, Tl, device=x.device) if self.keep else None
        qkv = kv = None
        if not cross:
            qkv = pool.get(Bh, Tl, 3 * mid)
            q, k, v = qkv[..., :mid], qkv[..., mid:2 * mid], qkv[..., 2 * mid:]
            add(lambda: ops.conv_gemm(xn, ap["w_qkv"], qkv, c_in=C, n_valid=3 * mid, bias=ap["b_qkv"]))
        else:
            # context K/V do not depend on x or sigma: in sampling mode they are projected ONCE per
            # sample() call (plan.pre), not once per step
            E, M = net.embedding_features, self.io.embedding.shape[1]
            q = pool.get(Bh, Tl, mid)
            if self.en is None:
                self.en = torch.empty(Bh, M, E, dtype=pool.dtype, device=x.device)
                self.add_ctx(lambda en=self.en: ops.ln_film(self.io.embedding, en, None, 0, None, self.G,
                                                            net.ATT_LN_EPS))
            en = self.en
            kv = torch.empty(Bh, M, 2 * mid, dtype=pool.dtype, device=x.device)
            k, v = kv[..., :mid], kv[..., mid:]
            self.add_ctx(lambda: ops.conv_gemm(en, ap["w_kv"], kv, c_in=E, n_valid=2 * mid, bias=ap["b_kv"]))
            add(lambda: ops.conv_gemm(xn, ap["w_q"], q, c_in=C, n_valid=mid, bias=ap["b_q"]))
        add(lambda: ops.attention(q, k, v, o, net.heads, D ** -0.5, lse=lse, head_dim=D))
        pool.put(q if cross else qkv)
        add(lambda: ops.conv_gemm(o, ap["w_out"], y, c_in=mid, n_valid=C, residual=x, stats=y_stats,
                                  groups=self.G))
        pool.put(xn)
        pool.put(o)
        pool.put(x)
        return dict(x=x, xn=xn, q=q, k=k, v=v, kv=kv, qkv=qkv, o=o, lse=lse, y=y)

    def down(self, lv: "LevelParams", Lp: Dict, x_in: Tensor, Tl: int) -> Tuple[Tensor, Tensor]:
        """Down conv of a level >= 1 (k = stride = factor over the [Bh, Tl, f*ci] view)."""
        x, st, kdim = self.pool.get(self.Bh, Tl, lv.ch), self.new_stats(), lv.factor * lv.in_ch
        self.add(lambda: ops.conv_gemm(x_in.view(self.Bh, Tl, kdim), Lp["down_w"], x, c_in=kdim, n_valid=lv.ch,
                                       bias=Lp["down_b"], stats=st, groups=self.G))
        return x, st

    def up_merge(self, lv: "LevelParams", Lp: Dict, x: Tensor, x_in: Tensor, Tl: int, T_in: int,
                 gate: Optional[Tensor]):
        """Up conv of a level >= 1's chain output x and its merge with the level input x_in:
        MergeModulate's `gate`, SkipCat or SkipAdd (gate None).  Returns (output, its statistics,
        y_up = the up conv's own output, None when the merge runs in its epilogue)."""
        pool, add, G, Bh, f, C, Co = self.pool, self.add, self.G, self.Bh, lv.factor, lv.ch, lv.out_ch
        out, ost = pool.get(Bh, T_in, Co), self.new_stats()
        merge = self.net.merge
        geom = dict(up_factor=f) if f > 1 else dict(taps=(-1, 0, 1))

        def phases(t):          # [Bh, T_in, Co] as the [Bh, Tl, f*Co] output of the upsample GEMM
            return t.view(Bh, Tl, f * Co)
        # SkipAdd is the epilogue's residual without a gate; its backward needs no y_up either
        if merge == "add" or (merge == "modulate" and not self.keep):
            add(lambda: ops.conv_gemm(x, Lp["up_w"], phases(out), c_in=C, n_valid=Co, bias=Lp["up_b"],
                                      residual=phases(x_in), gate=gate, stats=ost, groups=G, **geom))
            pool.put(x)
            return out, ost, None
        y_up, tmp = pool.get(Bh, T_in, Co), None
        add(lambda: ops.conv_gemm(x, Lp["up_w"], phases(y_up), c_in=C, n_valid=Co, bias=Lp["up_b"], **geom))
        if merge == "modulate":
            add(lambda: ops.skip_gate(y_up, x_in, gate, out, ost, G))
        else:
            # SkipCat: tmp = Wc1 (skip * s) + bc; out = Wc2 y_up + tmp.  The tensor-core GEMM needs
            # K >= 16: an 8-channel level runs two positions per row against block-diagonal weights
            rp = max(1, 16 // Co)
            assert T_in % rp == 0, "SkipCat merge of an 8-channel level needs an even length"
            tmp = pool.get(Bh, T_in, Co)

            def rows(t):
                return t.view(Bh, T_in // rp, rp * Co)
            add(lambda: ops.conv_gemm(rows(x_in), Lp["cat_w1"], rows(tmp), c_in=rp * Co, n_valid=rp * Co,
                                      bias=Lp["cat_b"]))
            add(lambda: ops.conv_gemm(rows(y_up), Lp["cat_w2"], rows(out), c_in=rp * Co, n_valid=rp * Co,
                                      residual=rows(tmp), stats=ost if rp == 1 else None, groups=G))
            if rp > 1:           # the epilogue's group mapping does not see the paired layout
                add(lambda: ops.gn_stats(out, ost, G))
        for t in (y_up, tmp, x):
            pool.put(t)
        return out, ost, y_up


class B200UNet(nn.Module):
    """See module docstring.  Reference parity notes per block are in include/adp_b200.h."""

    GN_EPS = 1e-5      # nn.GroupNorm default (a_unet ConvBlock)
    ATT_LN_EPS = 1e-5  # nn.LayerNorm default (a_unet Attention norms)
    MOD_LN_EPS = 1e-6  # a_unet Modulation LayerNorm
    HEAD_DIMS = (32, 64, 128)   # attention_features the attention kernels are built for
    MAX_BOUNDARY = 64           # in_channels (x + appended) and out_channels of the stem kernels
    MAX_STEM_IN = 128           # in_channels * factors[0]: inputs of one stem_in output position
    MAX_C0 = 256                # channels[0]
    # channels[i] (8 or a multiple of 16), attention_heads * attention_features and
    # embedding_features: the LayerNorm, GroupNorm-backward and bias-gradient row kernels hold a
    # row of at most this many channels (csrc/rowwise.cu kMaxLnC, csrc/backward.cu kBwMaxC)
    MAX_WIDTH = 2048
    # widest level whose ConvBlocks fuse_groupnorm applies to: the conv GEMM's GroupNorm A transform
    # keeps the coefficients of at most this many input channels (csrc/conv_gemm.cu s_coef)
    MAX_FUSED_GN_C = 1024

    def __init__(self, dim: int, in_channels: int, channels: Sequence[int],
                 factors: Sequence[int], items: Sequence[int],
                 attentions: Optional[Sequence[int]] = None,
                 cross_attentions: Optional[Sequence[int]] = None,
                 context_channels: Optional[Sequence[int]] = None,
                 attention_features: Optional[int] = None,
                 attention_heads: Optional[int] = None,
                 embedding_features: Optional[int] = None, resnet_groups: int = 8,
                 use_modulation: bool = True, modulation_features: int = 1024,
                 embedding_max_length: Optional[int] = None,
                 use_time_conditioning: bool = True, use_embedding_cfg: bool = False,
                 use_text_conditioning: bool = False, out_channels: Optional[int] = None,
                 append_channels: int = 0):
        super().__init__()
        n = len(channels)
        attentions = default(attentions, [0] * n)
        cross_attentions = default(cross_attentions, [0] * n)
        context_channels = default(context_channels, [0] * n)
        xs = (channels, factors, items, attentions, cross_attentions, context_channels)
        assert all(len(x) == n for x in xs)                       # reference components.py:61
        # a_unet repeats each item as `[Item] * count`: True is one item, 0 / False / negative none
        attentions = [max(0, int(a)) for a in attentions]
        cross_attentions = [max(0, int(a)) for a in cross_attentions]
        assert dim == 1, "the CUDA path implements the 1-D (waveform) U-Net"
        if use_embedding_cfg:                                     # components.py:66-68
            assert exists(embedding_max_length), "use_embedding_cfg requires embedding_max_length"
        if use_time_conditioning:                                 # components.py:75
            assert use_modulation, "use_time_conditioning requires use_modulation=True"
        if use_text_conditioning:
            raise NotImplementedError(
                "use_text_conditioning builds a T5 encoder (a_unet TextConditioningPlugin); pass "
                "precomputed `embedding=` with use_text_conditioning=False (SURVEY.md 3.4)")
        self._setup(in_channels, out_channels, append_channels, channels, factors, items, attentions,
                    cross_attentions, context_channels, attention_features, attention_heads, embedding_features,
                    resnet_groups, use_modulation, "modulate" if use_modulation else "cat",   # SkipModulate / SkipCat
                    modulation_features, use_time_conditioning, use_embedding_cfg)

        # registration order mirrors a_unet: time plugin, cfg plugin, then the recursive blocks
        self.time = TimeParams(modulation_features) if use_time_conditioning else None
        self.fixed_embedding = (nn.Embedding(embedding_max_length, embedding_features)
                                if use_embedding_cfg else None)

        def build(i: int):
            if i == n:
                return None
            in_ch = in_channels if i == 0 else channels[i - 1]
            out_ch = self.out_channels if i == 0 else in_ch
            return LevelParams(in_ch, out_ch, channels[i], factors[i], items[i], build(i + 1),
                               groups=resnet_groups, features=modulation_features,
                               att=attentions[i], cross=cross_attentions[i],
                               head_features=attention_features, heads=attention_heads,
                               embedding_features=embedding_features, context=context_channels[i],
                               modulation=use_modulation)

        self.net = build(0)
        self._init_runtime()

    def _init_runtime(self) -> None:
        """Plans, packs and the program-building attributes of a freshly built net."""
        self._plans: Dict[Tuple, _Plan] = {}
        self._packed = None
        self._packed_version = None
        self._fingerprint = None
        self._storage_sig = None
        self._repack_graph = None
        self.use_cuda_graph = True
        # GroupNorm+SiLU applied to the A tile inside the conv GEMM (adp_conv_gemm gn_*).
        # Bit-compatible with the two-kernel path, but every N tile repeats the transform of
        # its A rows, so it only pays for N <= BN.  Off by default.  Levels wider than
        # MAX_FUSED_GN_C keep the two-kernel path under this flag.
        self.fuse_groupnorm = False
        # C = 32 / 64 ConvBlocks as ONE fused kernel (GroupNorm+SiLU -> conv3 -> +res -> LN/FiLM ->
        # statistics, csrc/mid_conv.cu) instead of three: those levels are HBM-bound
        self.fuse_thin_levels = True
        self.cond_table_rows = 4096    # sampler: rows (steps x batch) of conditioning per pass
        self.max_table_steps = 4096    # iterations per conditioning block (alpha/beta table rows)
        self.steps_per_graph = 10      # sampling steps captured back to back in one CUDA graph
        self._verify_fp32 = False

    def _setup(self, in_channels: int, out_channels: Optional[int], append_channels: int, channels: Sequence[int],
               factors: Sequence[int], items: Sequence[int], attentions: Sequence[int],
               cross_attentions: Sequence[int], context_channels: Sequence[int],
               attention_features: Optional[int], attention_heads: Optional[int],
               embedding_features: Optional[int], resnet_groups: int, use_modulation: bool, merge: str,
               modulation_features: int, use_time_conditioning: bool, use_embedding_cfg: bool) -> None:
        """The net's shape attributes and the size envelope of the kernels, shared by UNetV0 and XUNet
        (per level: `items` repetitions or items, `attentions` / `cross_attentions` counts).
        use_modulation: the net has a conditioning projection; merge: "modulate", "cat" or "add"."""
        for c, ctx in zip(channels, context_channels):
            assert ctx == 0 or c >= 16, "InjectChannelsItem is built for levels with >= 16 channels"
        if any(attentions) or any(cross_attentions):
            assert exists(attention_features) and exists(attention_heads), \
                "AttentionItem requires attention_features and attention_heads"
            assert attention_features in self.HEAD_DIMS, \
                f"attention_features={attention_features}: the attention kernels support head dims " \
                f"{', '.join(map(str, self.HEAD_DIMS))}"
        if any(cross_attentions):
            assert exists(embedding_features), "CrossAttentionItem requires embedding_features"

        self.x_channels = in_channels - append_channels   # channels of `x` (rest is appended)
        self.append_channels = append_channels
        self.in_channels, self.out_channels = in_channels, default(out_channels, in_channels)
        self.channels, self.factors, self.items = list(channels), list(factors), list(items)
        self.attentions, self.cross_attentions = list(attentions), list(cross_attentions)
        self.context_channels = list(context_channels)
        self.groups, self.features = resnet_groups, modulation_features
        self.heads, self.head_features = attention_heads, attention_features
        self.embedding_features = embedding_features
        self.use_time_conditioning, self.use_embedding_cfg = use_time_conditioning, use_embedding_cfg
        self.use_modulation = use_modulation
        self.merge = merge
        for c in self.channels:
            assert c % resnet_groups == 0 and c % 8 == 0, "channels must be multiples of 8 and groups"
        # every ResnetItem conv GEMM sums the GroupNorm statistics of its output in its epilogue,
        # which holds at most 8 groups (csrc/conv_gemm.cu kMaxGroups)
        assert 1 <= resnet_groups <= 8, \
            f"resnet_groups={resnet_groups}: the conv GEMM's fused GroupNorm statistics support at most 8 groups"
        # the level-0 stem kernels (csrc/stem.cu, stem_bwd.cu) hold the whole boundary of a position
        assert self.in_channels <= self.MAX_BOUNDARY, \
            f"in_channels={self.in_channels} (x plus appended channels): the stem kernels support at most " \
            f"{self.MAX_BOUNDARY} input channels"
        assert self.out_channels <= self.MAX_BOUNDARY, \
            f"out_channels={self.out_channels}: the stem kernels support at most {self.MAX_BOUNDARY} output channels"
        assert self.out_channels <= self.x_channels, \
            f"out_channels={self.out_channels} exceeds the {self.x_channels} channels of x (the identity skip " \
            f"and the sampler update need out_channels <= x channels)"
        assert self.in_channels * factors[0] <= self.MAX_STEM_IN, \
            f"in_channels * factors[0] = {self.in_channels * factors[0]}: the stem_in conv supports at most " \
            f"{self.MAX_STEM_IN} inputs per output position"
        assert channels[0] <= self.MAX_C0, \
            f"channels[0]={channels[0]}: the stem kernels support a level 0 at most {self.MAX_C0} wide"
        for i, c in enumerate(self.channels):
            # the conv GEMM's K step is 16 channels; an 8-wide level runs on its own kernels
            assert c == 8 or c % 16 == 0, \
                f"channels[{i}]={c}: levels are 8 channels wide or a multiple of 16"
            assert c <= self.MAX_WIDTH, \
                f"channels[{i}]={c}: the row kernels support levels at most {self.MAX_WIDTH} wide"
        if any(attentions) or any(cross_attentions):
            assert attention_heads * attention_features <= self.MAX_WIDTH, \
                f"attention_heads * attention_features = {attention_heads * attention_features}: the row " \
                f"kernels support an attention width of at most {self.MAX_WIDTH}"
        if exists(embedding_features) and (any(cross_attentions) or use_embedding_cfg):
            assert embedding_features % 8 == 0 and embedding_features <= self.MAX_WIDTH, \
                f"embedding_features={embedding_features}: the embedding LayerNorm supports a multiple of 8 " \
                f"up to {self.MAX_WIDTH}"


    @property
    def verify_fp32(self) -> bool:
        """fp32 VERIFICATION MODE (inference, sampling and training): the same launch programs,
        packed-weight layouts and folds -- under autograd the same training program, backward and
        gradient arena -- with fp32 storage and fp32 arithmetic on the simple kernels of
        csrc/verify_f32.cu and csrc/verify_f32_bwd.cu (the fused thin-level and C = 8 kernels are
        replaced by their unfused composition).  For checking the program against the reference at
        rtol 1e-3 / atol 1e-4; ~100x slower than the tensor-core path.  Not supported under
        OverlappedDataParallel.  Switching drops every plan and pack."""
        return self._verify_fp32

    @verify_fp32.setter
    def verify_fp32(self, on: bool) -> None:
        if bool(on) != self._verify_fp32:
            self._verify_fp32 = bool(on)
            self.invalidate()

    def _act_dtype(self):
        return torch.float32 if self._verify_fp32 else torch.bfloat16

    # ------------------------------------------------------------------ weights
    def levels(self) -> List[LevelParams]:
        out, lvl = [], self.net
        while lvl is not None:
            out.append(lvl)
            lvl = lvl.inner
        return out

    @torch.no_grad()
    def load_reference_parameters(self, reference_net: nn.Module) -> None:
        """Positional copy from a reference UNetV0 (same kwargs): both trees register
        parameters in a_unet order, so shapes must line up one to one."""
        src, dst = list(reference_net.parameters()), list(self.parameters())
        assert len(src) == len(dst), f"parameter count {len(src)} != {len(dst)}"
        for s, d in zip(src, dst):
            assert s.shape == d.shape, f"shape mismatch {tuple(s.shape)} vs {tuple(d.shape)}"
            d.copy_(s)

    @torch.no_grad()
    def load_reference_state_dict(self, state_dict, prefix: str = "") -> None:
        """Loads the U-Net part of a reference checkpoint (`torch.save(model.state_dict())` of a
        reference model built with the same kwargs) without depending on a_unet's module NAMES:
        the keys under `prefix` are taken in checkpoint order, which is a_unet's registration
        order = this tree's parameter order, except that the time MLP's Linear is listed twice
        (a_unet repeats one module object inside a Sequential; both entries hold the same tensor).
        Shapes are checked entry by entry."""
        entries = [(k, v) for k, v in state_dict.items() if k.startswith(prefix)]
        mine = []
        for name, p in self.named_parameters():
            mine.append((name, p))
            if name == "time.mlp.bias":
                mine += mine[-2:]
        assert len(entries) == len(mine), \
            f"checkpoint has {len(entries)} tensors under '{prefix}', this net expects {len(mine)}"
        seen = {}
        for (key, src), (name, dst) in zip(entries, mine):
            assert tuple(src.shape) == tuple(dst.shape), \
                f"{key}: shape {tuple(src.shape)} does not match {name} {tuple(dst.shape)}"
            if name in seen:
                assert torch.equal(src, seen[name]), f"{key}: repeated module entries differ"
                continue
            seen[name] = src
            dst.copy_(src)

    def _version(self) -> int:
        """Moves whenever a parameter may have changed in place: the tensors' version counters, plus
        the number of optimizer steps taken in the process.  Fused optimizers (`fused=True`) update
        the parameters through one multi-tensor kernel that bumps no version counter; without the
        second term the packs, and with them the whole forward and backward, stayed at the weights
        from before the step."""
        return sum(p._version for p in self.parameters()) + _OPTIMIZER_STEPS[0]

    def _storage_signature(self):
        return tuple((p.data_ptr(), p.dtype) for p in self.parameters())

    def invalidate(self) -> None:
        """Drops every packed weight, plan and captured graph.  Needed after a parameter was
        re-pointed (`p.data = ...`, `.to()`, `.half()`, `load_state_dict(assign=True)`); in-place
        updates through the Parameter (optimizers, `load_state_dict`, `copy_`) are tracked by the
        version counters and refresh the packs in place instead."""
        self._plans.clear()
        self._packed = None
        self._packed_version = None
        self._fingerprint = None
        self._repack_graph = None

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        if hasattr(self, "_plans"):
            self.invalidate()
        return out

    @torch.no_grad()
    def _check_untracked_updates(self) -> None:
        """`p.data.add_()` / `.data.copy_()` style updates (EMA wrappers, manual init, weight
        clipping) bump no version counter.  Inference entry points therefore compare a cheap device
        fingerprint of all parameters (one multi-tensor norm + one small device->host read per
        call, outside the step loop) and re-pack when it moved."""
        ps = [p for p in self.parameters()]
        if not ps or not ps[0].is_cuda:
            return
        fp = torch.stack(torch._foreach_norm(ps)).double().cpu()
        if self._fingerprint is not None and not torch.equal(fp, self._fingerprint):
            self._packed_version = None          # force an in-place re-pack
            for plan in self._plans.values():
                if hasattr(plan, "version"):
                    plan.version = None
        self._fingerprint = fp

    @torch.no_grad()
    def packed(self):
        """Kernel-layout copies of the weights (bf16 GEMM operands, folded LayerNorm affines,
        one concatenated conditioning projection).  Rebuilt when a parameter changes."""
        sig = self._storage_signature()
        if getattr(self, "_storage_sig", None) != sig:   # a parameter was re-pointed: addresses
            if getattr(self, "_storage_sig", None) is not None:   # baked into plans are stale
                self.invalidate()
            self._storage_sig = sig
        v = self._version()
        if self._packed is not None and self._packed_version == v:
            return self._packed
        if self._packed is not None:
            # weights changed (optimizer step): refresh the SAME tensors in place, so captured
            # CUDA graphs and plans that hold their addresses stay valid
            self._repack()
            self._packed_version = v
            return self._packed
        self._packed, self._packed_version = self._compute_packed(), v
        return self._packed

    @torch.no_grad()
    def _repack(self) -> None:
        """In-place refresh of every packed weight.  The re-layout is ~500 small permute / cast /
        fold launches whose HOST cost
        dwarfs their device time: sources (the parameters) and destinations (the packs) have
        fixed addresses, so the whole sequence is captured once into a CUDA graph and replayed."""
        self._repack_graph = _refreshed(self._repack_graph,
                                        lambda: _copy_tree(self._packed, self._compute_packed()),
                                        self.use_cuda_graph and self.net.down.weight.is_cuda)

    @torch.no_grad()
    def _compute_packed(self):
        with ops.pack_dtype(self._act_dtype()):
            return self._compute_packed_impl()

    def _compute_packed_impl(self):
        P: Dict = {}
        pd = self._act_dtype()
        f32 = lambda t: t.detach().float().contiguous()  # noqa: E731
        cond_w, cond_b, off = [], [], 0

        def add_cond(lin: nn.Linear) -> int:
            nonlocal off
            n_out = lin.weight.shape[0]
            pad = ops.round_up(n_out, 8)
            w = torch.zeros(pad, lin.weight.shape[1], device=lin.weight.device)
            b = torch.zeros(pad, device=lin.weight.device)
            w[:n_out], b[:n_out] = lin.weight.detach().float(), lin.bias.detach().float()
            cond_w.append(w)
            cond_b.append(b)
            start, off = off, off + pad
            return start

        def pack_att(a: AttentionParams, self_attn: bool) -> Dict:
            wq = a.to_q.weight.detach().float()
            wkv = a.to_kv.weight.detach().float()
            g1, b1 = a.norm.weight.detach().float(), a.norm.bias.detach().float()
            g2, b2 = a.norm_context.weight.detach().float(), a.norm_context.bias.detach().float()
            d: Dict = {"w_out": ops.pack_linear(a.to_out.weight.detach())}
            # LayerNorm affine folded into the projection: W (xhat*g + b) = (W*g) xhat + W b
            wq_f, bq = wq * g1[None, :], wq @ b1
            wkv_f, bkv = wkv * g2[None, :], wkv @ b2
            if self_attn:
                d["w_qkv"] = ops.pack_linear(torch.cat([wq_f, wkv_f], 0))
                d["b_qkv"] = torch.cat([bq, bkv]).contiguous()
            else:
                d["w_q"], d["b_q"] = ops.pack_linear(wq_f), bq.contiguous()
                d["w_kv"], d["b_kv"] = ops.pack_linear(wkv_f), bkv.contiguous()
            return d

        def pack_resnet(r: ResnetParams, narrow: bool) -> Dict:
            d: Dict = {"gn1": (f32(r.gn1.weight), f32(r.gn1.bias)),
                       "gn2": (f32(r.gn2.weight), f32(r.gn2.bias)),
                       "b1": f32(r.conv1.bias), "b2": f32(r.conv2.bias)}
            if narrow:
                d["w1"], d["w2"] = f32(r.conv1.weight), f32(r.conv2.weight)
            else:
                d["w1"], d["w2"] = ops.pack_conv(r.conv1.weight.detach()), ops.pack_conv(r.conv2.weight.detach())
                if r.conv1.weight.shape[0] in (32, 64):    # thin levels: fused ConvBlock kernel
                    d["w1_raw"], d["w2_raw"] = f32(r.conv1.weight), f32(r.conv2.weight)
                    d["w1_mid"], d["w2_mid"] = ops.pack_mid_conv(r.conv1.weight), ops.pack_mid_conv(r.conv2.weight)
            return d

        def pack_inject(conv: nn.Conv1d) -> Dict:
            C_ = conv.weight.shape[0]
            wi = conv.weight.detach().float()[:, :, 0]
            ctx = wi.shape[1] - C_
            wc = torch.zeros(C_, ops.round_up(ctx, 16), device=wi.device)
            wc[:, :ctx] = wi[:, C_:]
            return {"w_x": ops.pack_linear(wi[:, :C_]), "w_c": ops.pack_linear(wc), "b": f32(conv.bias)}

        def pack_chain(chain, narrow: bool) -> List[Tuple[str, Dict]]:
            """(kind, pack) per item; each cross-attention projects the context through its own K|V
            weights (its norm_context affine folded in)."""
            out = []
            for kind, m in chain:
                if kind == "resnet":
                    out.append((kind, pack_resnet(m, narrow)))
                elif kind == "mod":
                    out.append((kind, {"ss_off": add_cond(m.proj)}))
                elif kind == "inj":
                    out.append((kind, pack_inject(m)))
                else:
                    out.append((kind, pack_att(m, kind == "att")))
            return out

        P["levels"] = []
        for i, lvl in enumerate(self.levels()):
            narrow = lvl.ch == 8 and not self._verify_fp32
            L: Dict = {"down_b": f32(lvl.down.bias), "up_b": f32(lvl.up.bias)}
            if i == 0:
                L["down_w"], L["up_w"] = f32(lvl.down.weight), f32(lvl.up.weight)
                if lvl.adapter is not None:
                    L["adapt_w"] = f32(lvl.adapter.weight[:, :, 0])
                    L["adapt_b"] = f32(lvl.adapter.bias)
            else:
                L["down_w"] = ops.pack_conv(lvl.down.weight.detach())
                L["up_w"] = (ops.pack_upsample_conv(lvl.up.weight.detach(), lvl.factor)
                             if lvl.factor > 1 else ops.pack_conv(lvl.up.weight.detach()))
            L["items_down"] = pack_chain(lvl.chain(up=False), narrow)
            L["items_up"] = pack_chain(lvl.chain(up=True), narrow)
            if self.merge == "modulate":
                L["gate_off"] = add_cond(lvl.merge)
            elif self.merge == "cat":
                # SkipCat: out = Wc1 (skip * s) + Wc2 y + bc,  W = [Wc1 | Wc2]
                s_ = 2 ** -0.5
                wm = lvl.merge.weight.detach().float()[:, :, 0]
                co = wm.shape[0]
                wc1, wc2, bc = wm[:, :co] * s_, wm[:, co:], lvl.merge.bias.detach().float()
                if i > 0:
                    # the tensor-core GEMM needs K >= 16: an 8-channel level output is viewed as
                    # [B, T/2, 16] (two positions per row) against block-diagonal weights
                    rr = max(1, 16 // co)
                    L["cat_w1"] = ops.pack_linear(torch.block_diag(*[wc1] * rr))
                    L["cat_w2"] = ops.pack_linear(torch.block_diag(*[wc2] * rr))
                    L["cat_b"] = bc.repeat(rr).contiguous()
                else:
                    # level 0 runs in the stem kernel (skip adapter + upsample conv + merge): fold the
                    # 1x1 merge conv into both branches.  v = (Wc1 W_ad) x + Wc1 b_ad + conv'(h) + b',
                    # conv' = Wc2 o W_up, b' = Wc2 b_up + bc; the kernel's gate is 1.
                    w_up = lvl.up.weight.detach().float()
                    L["up_w"] = torch.einsum("om,mck->ock", wc2, w_up).contiguous()
                    L["up_b"] = (wc2 @ lvl.up.bias.detach().float() + bc).contiguous()
                    if lvl.adapter is not None:
                        L["adapt_w"] = (wc1 @ lvl.adapter.weight.detach().float()[:, :, 0]).contiguous()
                        L["adapt_b"] = (wc1 @ lvl.adapter.bias.detach().float()).contiguous()
                    else:
                        L["adapt_w"], L["adapt_b"] = wc1.contiguous(), torch.zeros_like(bc)
            P["levels"].append(L)
        n_tot = off
        if cond_w:
            w_all = torch.cat(cond_w, 0)
            n_pad = ops.round_up(n_tot, 256)
            w_pad = torch.zeros(n_pad, w_all.shape[1], dtype=pd, device=w_all.device)
            w_pad[:n_tot] = w_all.to(pd)
            P["cond_w"], P["cond_b"], P["cond_n"] = w_pad.contiguous(), torch.cat(cond_b).contiguous(), n_tot
        else:          # use_modulation=False: no conditioning linears at all
            P["cond_w"], P["cond_b"], P["cond_n"] = None, None, 0
        if self.time is not None:
            t = self.time
            kdim = t.to_out.weight.shape[1]
            kpad = ops.round_up(kdim, 8)
            w_emb = torch.zeros(self.features, kpad, dtype=pd, device=t.to_out.weight.device)
            w_emb[:, :kdim] = t.to_out.weight.detach().to(pd)
            P["time"] = {"freqs": f32(t.weights), "w_emb": w_emb.contiguous(), "b_emb": f32(t.to_out.bias),
                         # a copy also in fp32: an alias would have the in-place re-pack bump the
                         # version of a weight the time MLP's autograd saved
                         "w_mlp": t.mlp.weight.detach().to(pd, copy=True).contiguous(),
                         "b_mlp": f32(t.mlp.bias), "kpad": kpad}
        return P

    def _add_conditioning(self, plan: _Plan, P: Dict, Bh: int) -> Tensor:
        """Appends the conditioning launches for Bh rows of (plan.sigma, plan.features_in) to
        `plan`; returns ss_all [Bh, n] fp32 (every Modulation / MergeModulate scale, shift and
        gate of the network, concatenated)."""
        dev = plan.sigma.device
        Fm = self.features
        ss_all = self._ss_all(P, Bh)
        cond_bf = torch.zeros(1, Bh, Fm, dtype=self._act_dtype(), device=dev)
        fvec = torch.zeros(Bh, Fm, device=dev)
        plan.use_features_in = False
        if self.time is not None:
            tp = P["time"]
            feat = torch.zeros(Bh, tp["kpad"], device=dev)
            e0, e1 = torch.zeros(Bh, Fm, device=dev), torch.zeros(Bh, Fm, device=dev)
            plan.add(lambda: ops.time_features(plan.sigma, tp["freqs"], feat))
            plan.add(lambda: ops.skinny_linear(feat, tp["w_emb"], tp["b_emb"], e0, tp["kpad"], Fm,
                                               out_act=ops.ACT_GELU))
            plan.add(lambda: ops.skinny_linear(e0, tp["w_mlp"], tp["b_mlp"], e1, Fm, Fm,
                                               out_act=ops.ACT_GELU))
            plan.add(lambda: ops.skinny_linear(e1, tp["w_mlp"], tp["b_mlp"], fvec, Fm, Fm,
                                               out_act=ops.ACT_GELU))

            def add_features():
                if plan.use_features_in:
                    fvec.add_(plan.features_in)
            plan.add(add_features)
        else:
            plan.add(lambda: fvec.copy_(plan.features_in))
        plan.add(lambda: ops.silu_bf16(fvec, cond_bf))
        self._project_conditioning(plan.add, P, cond_bf, ss_all)
        return ss_all

    def _ss_all(self, P: Dict, rows: int) -> Tensor:
        """A zeroed ss_all [rows, n] fp32: the conditioning projection's output, n = its outputs padded
        to 8 (8 without a projection: the step selector and the walk keep one layout)."""
        return torch.zeros(rows, max(8, ops.round_up(P["cond_n"], 8)), device=self.net.down.weight.device)

    def _project_conditioning(self, add: Callable, P: Dict, cond_bf: Tensor, ss_all: Tensor) -> None:
        """Appends the conditioning projection ss_all = W_all cond_bf + b_all (cond_bf [1, rows,
        features] = SiLU(features), in the activation dtype) through `add`."""
        cond_bias = _pad_to(P["cond_b"], ss_all.shape[1])
        add(lambda: ops.conv_gemm(cond_bf, P["cond_w"], ss_all.view(1, ss_all.shape[0], -1), c_in=self.features,
                                  n_valid=ss_all.shape[1], bias=cond_bias))

    def _static_io(self, io, B: int, Bh: int, T: int, M: int) -> None:
        """The input buffers of a plan, set on `io`: x [B, x channels, T] and append (fp32, as the
        caller passes them), the embedding tokens [Bh, M, embedding_features] (M = 0: None) and the
        InjectChannelsItem context of each depth d, ctx[d] [Bh, T_d, channels padded to 16] (both in
        the activation dtype)."""
        dev, adt = self.net.down.weight.device, self._act_dtype()
        io.x = torch.zeros(B, self.x_channels, T, device=dev)
        io.append = torch.zeros(B, self.append_channels, T, device=dev) if self.append_channels else None
        io.embedding = torch.zeros(Bh, M, self.embedding_features, dtype=adt, device=dev) if M else None
        io.ctx = {i: torch.zeros(Bh, T // _prod(self.factors[:i + 1]), ops.round_up(c, 16), dtype=adt, device=dev)
                  for i, c in enumerate(self.context_channels) if c > 0}

    def _cond_table(self, sigmas: Tensor, features_in: Optional[Tensor]) -> Tensor:
        """ss_all for every row of `sigmas` [R] in one pass (the 97 MB of conditioning weights of
        the README network are read once per sample() call instead of once per step)."""
        R = sigmas.shape[0]
        key = ("cond", R)
        P = self.packed()
        if not self.use_modulation:       # nothing to evaluate: a dummy table keeps the step selector uniform
            plan = self._plans.get(key)
            if plan is None:
                plan = self._plans[key] = _Plan()
                plan.ss_all = self._ss_all(P, R)
            return plan.ss_all
        plan = self._plans.get(key)
        if plan is None:
            ops.device_check()
            plan = _Plan()
            plan.sigma = torch.zeros(R, device=sigmas.device)
            plan.features_in = torch.zeros(R, self.features, device=sigmas.device)
            plan.ss_all = self._add_conditioning(plan, P, R)
            self._plans[key] = plan
        plan.sigma.copy_(sigmas)
        plan.use_features_in = features_in is not None
        if features_in is not None:
            plan.features_in.copy_(features_in)
        plan.run_eager()
        return plan.ss_all

    # --------------------------------------------------------------------- plan
    def _build_plan(self, B: int, T: int, Bh: int, M: int, mode: str) -> _Plan:
        """B = batch of x; Bh = rows the trunk runs (2B under classifier-free guidance);
        M = embedding tokens (0 if none); mode in {'v', 'sample', 'sample_dpm'}.  'sample_dpm' is the
        'sample' plan with stem_out writing v and the DPM-Solver++(2M) update (adp_dpm_step, on
        x, a history buffer and a coefficient table picked by the step counter) before step_advance."""
        dev = self.net.down.weight.device
        P = self.packed()
        plan = _Plan()
        levels = self.levels()
        total_f = _prod(self.factors)
        assert T % total_f == 0, f"length {T} must be divisible by the product of factors {total_f}"

        # ---- static I/O
        self._static_io(plan, B, Bh, T, M)
        plan.sigma = torch.zeros(Bh, device=dev)
        plan.features_in = torch.zeros(Bh, self.features, device=dev)
        plan.v = torch.zeros(B, self.out_channels, T, device=dev)
        plan.ab = torch.zeros(4, device=dev)
        plan.cfg_scale = None
        plan.pre = []                        # step-invariant launches of a sampling plan

        # ---- statistics arena (zeroed once per forward)
        n_slots = 2 + sum(3 * (len(lv.items_down) + len(lv.items_up)) + 3 for lv in levels)
        arena = torch.zeros(n_slots, Bh, self.groups, 2, dtype=torch.float64, device=dev)
        sampling = mode in ("sample", "sample_dpm")
        if sampling:
            # the step's conditioning rows and alpha/beta are picked ON THE DEVICE from tables by a
            # step counter, so the captured graph is identical for every step (the host only
            # replays it, and several steps are captured back to back: _execute_steps)
            plan.step = torch.zeros(1, dtype=torch.int32, device=dev)
            plan.ctrl = torch.zeros(3, dtype=torch.int64, device=dev)
            plan.ab_table = torch.zeros(self.max_table_steps, 4, device=dev)
            plan.multi_graph, plan.multi_steps = None, 0
        if mode == "sample_dpm":
            from . import diffusion
            plan.dpm_table = torch.zeros(self.max_table_steps, 5, device=dev)
            plan.hist = torch.zeros_like(plan.x)          # x0 of the previous step
        plan.add(lambda: arena.zero_())

        # ---- conditioning: f = MLP(GELU(embed(sigma))) (+features); ss = W_all SiLU(f) + b.
        # The sampler knows every sigma_i up front and evaluates this ONCE for all steps
        # (_cond_table): its plan only receives the step's rows of the table.
        if sampling:
            ss_all = plan.ss_all = self._ss_all(P, Bh)
            plan.use_features_in = False
            plan.add(lambda: ops.step_select(plan.step, plan.ctrl, plan.ab_table, plan.ab, ss_all))
        elif self.use_modulation:
            ss_all = self._add_conditioning(plan, P, Bh)
        else:
            ss_all = self._ss_all(P, Bh)
            plan.use_features_in = False
        walk = _ForwardWalk(self, P, plan, plan.add, Bh, arena, ss_all, keep=False,
                            add_ctx=plan.pre.append if sampling else plan.add)
        if mode == "sample":       # v and the VSampler update in one pass; x advanced in place
            walk.trunk(lambda: dict(x_next=plan.x, ab=plan.ab, cfg_scale=plan.cfg_scale))
            plan.add(lambda: ops.step_advance(plan.step))
        elif mode == "sample_dpm":
            walk.trunk(lambda: dict(v_out=plan.v, cfg_scale=plan.cfg_scale))
            plan.add(lambda: diffusion._dpm_step(plan.x, plan.v, plan.hist, plan.dpm_table, plan.step,
                                                 plan.dpm_table.shape[0]))
            plan.add(lambda: ops.step_advance(plan.step))
        else:
            walk.trunk(lambda: dict(v_out=plan.v, cfg_scale=plan.cfg_scale))
        plan.workspace_bytes = walk.pool.total_bytes
        return plan

    def _plan(self, B: int, T: int, Bh: int, M: int, mode: str, baked: Tuple = ()) -> _Plan:
        """`baked` = host-side values frozen into the captured graph (cfg scale, features flag)."""
        key = (B, T, Bh, M, mode, baked)
        self.packed()                      # refreshes the packed weights in place if needed
        plan = self._plans.get(key)
        if plan is None:
            ops.device_check()
            plan = self._plans[key] = self._build_plan(B, T, Bh, M, mode)
        return plan

    def profile_plan(self, plan: _Plan, iters: int = 5):
        """Instrumented eager passes of a plan: CUDA events around every launch, aggregated
        per kernel/shape -> {label: count per pass, avg/total ms per pass, flops, bytes}."""
        with ops.trace(timing=True) as tr:
            for _ in range(iters):
                if hasattr(plan, "step"):
                    plan.step.zero_()
                plan.run_eager()
        table = tr.table()
        for row in table.values():
            row["count"] //= iters
            row["ms_total"] /= iters
        return table

    def _execute(self, plan: _Plan) -> None:
        """One evaluation of the plan (_Graphed); the first eager run under graphs also counts the
        kernels of one net evaluation."""
        if self.use_cuda_graph and plan.runs == 0:
            with ops.trace() as tr:
                plan(True)
            plan.n_kernels = len(tr.records)
        else:
            plan(self.use_cuda_graph)

    def _execute_steps(self, plan: _Plan, n: int) -> None:
        """n consecutive sampling steps of a 'sample' plan.  Once the single-step graph exists, a
        second graph holding `steps_per_graph` steps back to back is captured and used for full
        groups: 5 graph launches instead of 50 per 50-step sample (host-side launch cost and its
        variance between boxes stay off the critical path)."""
        S = self.steps_per_graph
        while n > 0:
            if (self.use_cuda_graph and S > 1 and n >= S and plan.graph is not None):
                if plan.multi_graph is None or plan.multi_steps != S:
                    def steps():
                        for _ in range(S):
                            plan.run_eager()
                    plan.multi_graph, plan.multi_steps = _capture(steps, early_weights=True), S
                plan.multi_graph.replay()
                plan.runs += S
                n -= S
            else:
                self._execute(plan)
                n -= 1

    def _set_step_tables(self, plan: _Plan, table: Tensor, ab_rows: Tensor, share: int = 1,
                         dpm_rows: Optional[Tensor] = None) -> None:
        """Points the plan's step selector at a block of conditioning rows [n, Bh, stride] and its
        alpha/beta rows [n_iterations, 4] (and a 'sample_dpm' plan's update at its coefficient rows
        [n_iterations, 5]); resets the device step counter."""
        assert ab_rows.shape[0] <= plan.ab_table.shape[0], "too many iterations per conditioning block"
        plan.ab_table[: ab_rows.shape[0]].copy_(ab_rows, non_blocking=True)
        if dpm_rows is not None:
            plan.dpm_table[: dpm_rows.shape[0]].copy_(dpm_rows, non_blocking=True)
        plan.ctrl.copy_(torch.tensor([table.data_ptr(), share, table.shape[0]], dtype=torch.int64),
                        non_blocking=True)
        plan.step.zero_()

    def _stage_inputs(self, plan: _Plan, x: Tensor, time: Optional[Tensor], features, embedding,
                      embedding_scale: float, embedding_mask_proba: float, append_channels,
                      channels=None):
        B = x.shape[0]
        Bh = plan.sigma.shape[0]
        cfg = Bh == 2 * B
        for d, buf in plan.ctx.items():       # InjectChannelsItem context: [B, ctx, T_d] -> channels-last bf16
            assert channels is not None and channels[d] is not None, \
                f"context `channels[{d}]` is required (context_channels[{d}] > 0)"
            c = channels[d]
            assert c.shape[1] == self.context_channels[d] and c.shape[2] == buf.shape[1], \
                "context `channels` at depth must match resolution and context_channels"
            buf[:B, :, : c.shape[1]].copy_(c.transpose(1, 2))
            if cfg:
                buf[B:, :, : c.shape[1]].copy_(c.transpose(1, 2))
        if plan.x.data_ptr() != x.data_ptr():
            plan.x.copy_(x)
        if self.append_channels:
            assert exists(append_channels), "append_channels is required (AppendChannelsPlugin)"
            plan.append.copy_(append_channels)
        if self.time is not None:
            assert exists(time), "time conditioning requires the time argument"
            plan.sigma[:B].copy_(time.reshape(-1))
            if cfg:
                plan.sigma[B:].copy_(time.reshape(-1))
            plan.use_features_in = exists(features)
        elif self.use_modulation:
            assert exists(features), "use_time_conditioning=False needs features="
        if exists(features):
            plan.features_in[:B].copy_(features)
            if cfg:
                plan.features_in[B:].copy_(features)
        if plan.embedding is not None:
            assert exists(embedding), "ClassiferFreeGuidancePlugin requires embedding"
            emb = embedding
            if self.fixed_embedding is not None:
                fixed = self.fixed_embedding.weight[: emb.shape[1]].unsqueeze(0).expand_as(emb)
                if embedding_mask_proba > 0.0:          # a_unet CFG plugin, training-time masking
                    mask = torch.bernoulli(torch.full((B, 1, 1), embedding_mask_proba,
                                                      device=emb.device)).to(torch.bool)
                    emb = torch.where(mask, fixed, emb)
                if cfg:
                    plan.embedding[B:].copy_(fixed)
            plan.embedding[:B].copy_(emb)
        plan.cfg_scale = float(embedding_scale) if cfg else None

    def _shape_key(self, x: Tensor, embedding, embedding_scale: float):
        B, _, T = x.shape
        cfg = self.use_embedding_cfg and exists(embedding) and embedding_scale != 1.0
        M = embedding.shape[1] if (exists(embedding) and any(self.cross_attentions)) else 0
        return B, T, (2 * B if cfg else B), M

    def forward(self, x: Tensor, time: Optional[Tensor] = None, *, features: Optional[Tensor] = None,
                embedding: Optional[Tensor] = None, embedding_scale: float = 1.0,
                embedding_mask_proba: float = 0.0, channels=None,
                append_channels: Optional[Tensor] = None) -> Tensor:
        if self.use_embedding_cfg:
            assert exists(embedding), "ClassiferFreeGuidancePlugin requires embedding"
        ctx_list = [c for c in (channels or []) if exists(c)]
        if torch.is_grad_enabled() and (
                any(p.requires_grad for p in self.parameters()) or
                any(exists(t) and t.requires_grad for t in (x, features, embedding, append_channels, *ctx_list))):
            # differentiable: custom loss_fn / diffusion_t (reference models.py:28,37)
            from .training import differentiable_forward
            return differentiable_forward(self, x, time, features=features, embedding=embedding,
                                          embedding_scale=embedding_scale,
                                          embedding_mask_proba=embedding_mask_proba,
                                          append_channels=append_channels, channels=channels)
        with torch.no_grad():
            plan = self._prelude(x, "v", time, features=features, embedding=embedding,
                                 embedding_scale=embedding_scale, embedding_mask_proba=embedding_mask_proba,
                                 append_channels=append_channels, channels=channels)
            self._execute(plan)
            return plan.v.clone().to(x.dtype)

    def _prelude(self, x: Tensor, mode: str, time: Optional[Tensor], **kwargs) -> _Plan:
        """What every inference entry point does before its first evaluation: checks the input device
        and the weights, picks the plan of x's shape, stages the inputs and runs the plan's
        step-invariant launches (plan.pre: the cross-attention context K/V of a sampling plan, once
        per call).  kwargs: forward's keyword arguments."""
        ops.require_cuda(x)
        self._check_untracked_updates()
        embedding, scale, features = kwargs.get("embedding"), kwargs.get("embedding_scale", 1.0), kwargs.get("features")
        B, T, Bh, M = self._shape_key(x, embedding, scale)
        plan = self._plan(B, T, Bh, M, mode, (float(scale) if Bh != B else None, exists(features)))
        self._stage_inputs(plan, x.float(), time, features, embedding, scale,
                           kwargs.get("embedding_mask_proba", 0.0), kwargs.get("append_channels"),
                           kwargs.get("channels"))
        for fn in plan.pre:
            fn()
        return plan

    def _table_steps(self, plan: _Plan, sigmas: Tensor, ab_rows: Tensor, share: int, progress,
                     each: Optional[Callable[[], None]] = None, dpm_rows: Optional[Tensor] = None) -> None:
        """The steps of a 'sample' plan from sigmas [N+1, B]: `share` evaluations per step, each
        followed by each(); ab_rows [N * share, 4] holds every evaluation's alpha/beta (dpm_rows
        [N, 5] a 'sample_dpm' plan's update coefficients, re-based per block like ab_rows).  The
        conditioning table is evaluated in blocks of <= ~4096 rows (190 KB of fp32 per row for the
        README net); inside a block the device picks each step's rows: graph launches only, no host
        sync.  Without a progress iterator and each(), _execute_steps runs a block's steps."""
        B, Bh = plan.x.shape[0], plan.sigma.shape[0]
        num_steps = sigmas.shape[0] - 1
        sig = sigmas.float().repeat(1, Bh // B).contiguous()      # [N+1, Bh]
        block = max(1, min(self.cond_table_rows // Bh, self.max_table_steps // share))
        ticks = _ticks(progress, num_steps)
        for first in range(0, num_steps, block):
            n = min(block, num_steps - first)
            feats = plan.features_in.repeat(n, 1) if plan.use_features_in else None
            table = self._cond_table(sig[first:first + n].reshape(-1), feats).view(n, Bh, -1)
            self._set_step_tables(plan, table, ab_rows[first * share:(first + n) * share], share,
                                  None if dpm_rows is None else dpm_rows[first:first + n])
            if progress is None and each is None:
                self._execute_steps(plan, n)
                continue
            for _ in range(n):         # progress bar: one graph launch per evaluation
                next(ticks)
                for _ in range(share):
                    self._execute(plan)
                    if each is not None:
                        each()
        for _ in ticks:
            pass

    @torch.no_grad()
    def sample_loop(self, x_noisy: Tensor, sigmas: Tensor, alphas: Tensor, betas: Tensor,
                    progress=None, **kwargs) -> Tensor:
        """VSampler's loop (reference diffusion.py:183-188) with the per-step update fused into
        the net's last kernel: one graph launch per step, no host sync inside the loop."""
        plan = self._prelude(x_noisy, "sample", sigmas[0], **kwargs)
        ab = torch.stack([alphas[:-1], betas[:-1], alphas[1:], betas[1:]], dim=1).float().contiguous()
        self._table_steps(plan, sigmas, ab, 1, progress)
        return plan.x.clone().to(x_noisy.dtype)

    @torch.no_grad()
    def dpm_loop(self, x_noisy: Tensor, sigmas: Tensor, coefficients: Tensor, progress=None, **kwargs) -> Tensor:
        """DPMSolverSampler's loop: per step one graph launch of the 'sample_dpm' plan (the net's v,
        then adp_dpm_step on x and the history with row i of `coefficients` [N, 5], from
        diffusion.dpm_coefficients), no host sync inside the loop."""
        assert self.out_channels == self.x_channels, \
            f"out_channels={self.out_channels} differs from the {self.x_channels} channels of x"
        plan = self._prelude(x_noisy, "sample_dpm", sigmas[0], **kwargs)
        unused_ab = torch.zeros(coefficients.shape[0], 4, device=plan.x.device)   # stem_out writes v: plan.ab is not read
        self._table_steps(plan, sigmas, unused_ab, 1, progress, dpm_rows=coefficients)
        return plan.x.clone().to(x_noisy.dtype)

    @torch.no_grad()
    def inpaint_loop(self, x_noisy: Tensor, source: Tensor, mask: Tensor, sigmas: Tensor, alphas: Tensor,
                     betas: Tensor, num_resamples: int, progress=None, **kwargs) -> Tensor:
        """VInpainter's loop (reference diffusion.py:338-352): per step `num_resamples` net
        evaluations; each one advances x to the level of the NEXT step only on the last resample
        (otherwise it is re-noised back to the current level), then the known region (mask) is
        replaced by the source noised to that level.  One graph launch + one blend kernel per
        evaluation; the noise is drawn with torch.randn_like(source) in the reference's order."""
        plan = self._prelude(x_noisy, "sample", sigmas[0], **kwargs)
        a, b = alphas.float(), betas.float()
        # ab[i][j]: coefficients of a step from level i to level i + j (j = 0: stay, re-noise)
        ab = torch.stack([torch.stack([a[:-1], b[:-1], a[:-1], b[:-1]], 1),
                          torch.stack([a[:-1], b[:-1], a[1:], b[1:]], 1)], 1).contiguous()
        # per iteration (step i, resample r): alpha/beta row = ab[i][r is the last]
        last = torch.zeros(num_resamples, dtype=torch.long, device=ab.device)
        last[-1] = 1
        src = source.float().expand_as(plan.x).contiguous()
        mask_u8 = mask.expand_as(plan.x).to(torch.uint8).contiguous()

        def blend():
            ops.inpaint_blend(plan.x, src, torch.randn_like(source).float().expand_as(plan.x).contiguous(),
                              mask_u8, plan.ab)
        self._table_steps(plan, sigmas, ab[:, last].reshape(-1, 4), num_resamples, progress, blend)
        return plan.x.clone().to(x_noisy.dtype)

    @torch.no_grad()
    def arv_loop(self, current: Tensor, sigmas: Tensor, progress=None, **kwargs) -> Tensor:
        """ARVSampler.sample_loop (reference diffusion.py:223-238): the net input is cat([current,
        sigma_i]) with a noise level PER POSITION (sigmas [N+1, B, 1, T]) and no time conditioning.
        The plan's input buffer holds that concatenation for the whole loop: one graph launch (the
        net) + one adp_arv_step (the update, which also writes sigma_{i+1} into the last channel)."""
        B, C, T = current.shape
        assert C + 1 == self.x_channels and sigmas.shape[1:] == (B, 1, T)
        plan = self._prelude(torch.cat([current.float(), sigmas[0].float()], dim=1), "v", None, **kwargs)
        sig = sigmas.float().reshape(sigmas.shape[0], B, T).contiguous()
        for i in _ticks(progress, sigmas.shape[0] - 1):
            self._execute(plan)
            ops.arv_step(plan.x, plan.v, sig[i + 1])
        return plan.x[:, :C].clone().to(current.dtype)


def _ticks(progress, n: int):
    """n steps: advances `progress` (any iterable) before each, then lets it finish (a progress
    generator's last description update runs after the last step)."""
    it = iter(progress if progress is not None else range(n))
    for i in range(n):
        next(it)
        yield i
    for _ in it:
        pass


_OPTIMIZER_STEPS = [0]


def _count_optimizer_step(optimizer, args, kwargs) -> None:
    _OPTIMIZER_STEPS[0] += 1


# every torch.optim step in the process: a step of an unrelated optimizer costs one in-place re-pack
register_optimizer_step_post_hook(_count_optimizer_step)


def _copy_tree(dst, src) -> None:
    """In-place refresh of a nested dict/list/tuple of tensors (same structure)."""
    if isinstance(dst, Tensor):
        dst.copy_(src)
    elif isinstance(dst, dict):
        for k in dst:
            _copy_tree(dst[k], src[k])
    elif isinstance(dst, (list, tuple)):
        for d, s_ in zip(dst, src):
            _copy_tree(d, s_)


def _prod(vals) -> int:
    out = 1
    for v in vals:
        out *= v
    return out


def _pad_to(t: Tensor, n: int) -> Tensor:
    if t.shape[0] == n:
        return t
    out = torch.zeros(n, dtype=t.dtype, device=t.device)
    out[: t.shape[0]] = t
    return out


def UNetV0(dim: int, in_channels: int, channels: Sequence[int], factors: Sequence[int],
           items: Sequence[int], **kwargs) -> nn.Module:
    """Drop-in for reference components.py:34 `UNetV0` (same kwargs, asserts and call
    signature); returns the CUDA-native module."""
    return B200UNet(dim=dim, in_channels=in_channels, channels=channels, factors=factors,
                    items=items, **kwargs)
