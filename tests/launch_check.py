"""Checks every kernel launch of a real program against an fp64 restatement of what it computes.

`Shadow` replaces the launch functions of `ops` (as tests/test_launch_programs_cpu.py's Recorder
does) by wrappers that, around each launch, synchronise, snapshot every storage the arguments
touch, run the real kernel (or, with `fake=True`, write the restatement itself, so whole programs
run on the CPU), and then compare everything the launch wrote with an fp64 reference computed from
the snapshot -- the exact inputs the kernel saw, with the real buffer aliasing (`residual is out`,
`stem_out(x_next=plan.x)`).  Errors do not carry from launch to launch, so every kernel is held to
its own bound at the shape and on the activations the program gives it.

Bounds (err = |got - ref| element-wise, `absref` = the same operation applied to absolute
values: conv of |a| with |w|, P |V|, ...):
    bf16 outputs   err <= 2^-7 |ref| + tau absref
                   tau = 2^-8 where the kernel rounds an internal operand to bf16 (the GroupNorm +
                   SiLU A operand of the fused conv GEMM and of narrow_conv, attention's P),
                   tau = 2^-12 elsewhere
    fp32 outputs   err <= 1e-5 |ref| + 2^-14 absref
    statistics     the launch's contribution (after - before) against stats_of() of the kernel's
                   own rounded output, within 1e-4 of sum|x| and sum x^2; the variance the
                   consumers derive, E[x^2] - mean^2, within 1e-3 (var + 1e-5) of a two-pass fp64
                   variance (GroupNorm normalises by sqrt(var + 1e-5); the plain relative error
                   of the variance is recorded as `.var_rel`, unbounded: a single-pass variance
                   of a near-constant group, var << mean^2, keeps only a few digits)
    accumulators   (Acc: fp32 parameter / conditioning gradients, fp64 sums) the launch's own
                   contribution, after - before, against the fp64 sum of its terms:
                   fp32  err <= 1e-5 |ref| + 2^-14 absref + 2^-23 (|before| + |after|)
                   fp64  err <= 1e-4 absref      (GroupNorm backward sums, the loss sum)
                   absref = the same sum over absolute terms; the GroupNorm backward sums are taken
                   over dxh as stored, as statistics are over the stored output
    attention lse  the fp32 bound + 2^-9 (LSE_FLOOR: the row sum is taken over P rounded to bf16)
    log mel        the fp32 bound b of the linear value carried through log(max(., 1e-5)): b divided
                   by max(ref - b, 1e-5), + 1e-5 |ref| of the log
    copies         bitwise (the step selector's rows, arv_step's sigma channel, and inpaint_blend's
                   positions outside the mask, which hold the sampler's value)
The fp32 verification mode (B200UNet.verify_fp32: the f32_* kernels of verify_f32.cu and
verify_f32_bwd.cu, one thread per output, fixed sequential fp32 sums) is held to fp32 round-off, none
of the bf16 allowances above (no tau = 2^-8, no LSE_FLOOR, no bf16 rounding of operands or P):
    f32 outputs    err <= 2^-23 |ref| + lambda sqrt(n) 2^-24 absref,   lambda = 10
                   accumulators: + 2^-23 (|before| + |after|) (fp32), 2^-52 (...) (fp64: loss_sum, S)
the probabilistic bound of Higham and Mary (SIAM J. Sci. Comput. 41(5), 2019): with independent
roundings an element exceeds it with probability at most 2n exp(-lambda^2 / 2), negligible at
lambda = 10.  n is the longest fp32 chain forming the element in that kernel:
    kind            n                                  kind            n
    conv_gemm       c_in * slots + 3                   wgrad           B T
    skinny_linear   K + 2                              colsum          B T + 2
    ln_film (y, y2) C + 4                              gn_silu_bwd     8 (dxh), B T (dgamma, dbeta), T + 8 (S)
    attention       2 Tk + 4 (o, lse)                  gn_bwd_apply    8 (dx), B T + 8 (colsum)
    stem_in         cin f + 3                          ln_film_bwd     C + 8 (dx), T + C (dss), B T + C (colsum)
    stem_out        3 c0 + cin + 8                     skip_gate_bwd   8 (dys), T + 2 (dgate)
    gn_silu, silu,  8 (F32_SHORT: a few roundings,     cond_bwd        B + 2 (dw, dbias), N + 2 (dcond)
    skip_gate         transcendentals included)        stem_in_bwd     B T/f + 3 (dw), c0 + 1 (dxin)
    attention_bwd   D + 2 (delta), Tk + D + 4 (dq),    stem_out_bwd    3 f co + 2 (dh), B T + 2 (dw, dbias,
                    Tq + D + 4 (dk, dv)                                dw_adapt), co + 2 (dxin), 2 (T + 3 c0 + 2) (dgate)
Where the arithmetic leaves that model, absref carries the magnitude the rounding is relative to,
as the bf16 checkers do: x - mean in fp32 (gn_silu, the GroupNorm backward: |x| + |mean|), xhat
formed in fp32 (ln_film_bwd: (|x| + mean|x|) / std), SiLU' near its zero (DSILU_MAX |da| + the
rounding of z through |SiLU''| <= 1/2), exp(s - max) (an absolute error of the score, a D-chain over
|q| |k| scale, is a relative one of p: attention's o and lse, attention_bwd's P and dS), and the
stems' noising alpha x + beta noise (|alpha x| + |beta noise|).  GroupNorm statistics keep their
check above (fp64 sums of the stored fp32 output).  attention's online softmax rounds twice per key
(acc corr + p v, and l the same way): its n counts both.  A 2^-12 relative change of an element is
outside the bound wherever sqrt(n) absref / |ref| < (2^-12 - 2^-23) / (lambda 2^-24) = (2^12 - 2) /
lambda, about 409: a chain of 256 catches it while absref / |ref| < 25.
In the fp32 mode conv_gemm, ln_film, stem_in and skip_gate make their GroupNorm statistics with a
gn_stats launch of their own inside the ops call: it is checked once, as the caller's `stats`
output, runs on the caller's (relocated) storages, and the caller's label names the caller.

Every launch also checks that read-only arguments are bitwise unchanged and that no byte of a
written tensor's storage outside the written view changed -- the rest of the gradient arena
included, every accumulator being a view of that one storage.

Checked kinds are every launching function of `ops`, in both modes (UNCHECKED is empty: the
launching functions without a checker; the f32 routes of a function share its checker): the launches of the
inference, sampling and training programs (forward, fused loss and backward; tau = 2^-8 also for
attention_bwd, which rounds P and dS to bf16); the tensors fir_resample, mel_spectrogram, to_flat
and to_flat_bwd allocate and return (RESULT); and the in-place sampler steps of VSampler's generic
loop (sampler_step), VInpainter (inpaint_blend) and ARVSampler (arv_step).

Guard mode (`Shadow(guard=True)`) also holds every launch to the bytes it is given.  After the
snapshot, each distinct storage among the tensor arguments (nested tuples such as `gn` included) is
copied into a fresh buffer laid out as [front guard | copy | back guard], each guard GUARD_BYTES,
the copy at its storage's address modulo GUARD_ALIGN (every TMA and vector alignment holds) and the
back guard starting at the storage's last byte + 1.  The guards and every byte of the copy outside
all of the launch's argument views are poisoned: POISON_FLOAT (0x7F bytes: bf16 / fp32 3.39e38, fp64
~1.4e306, finite, so a read survives fmaxf / fminf and comparisons where a NaN would not) for
storages only floating tensors view, POISON_INT (zero) for any storage an integer tensor views
(`step`, `ctrl`, `mask_u8`, the mel `band`), so no poisoned value becomes an index, an address or a
loop bound.  The launch runs on views of the copies with the original offsets, shapes and strides
(memoised by id(): `residual is out` and `x_next=plan.x` stay aliases); the tensors the RESULT
kinds allocate inside `ops` come from a `torch` proxy (`_TorchProxy`) that puts them between guards
too.  Afterwards every poisoned byte must be unchanged -- a failure names the launch, the argument
view nearest the byte, whether it lies before the start, in an unviewed gap or past the end of the
storage, and its distance in bytes and in rows of that view -- and the viewed bytes go back to the
original storages, where the value and side-effect checks above run unchanged: a kernel that read
poison shows there as a huge error.  `n_guarded` counts the guarded launches.

Guard mode does not cover storages a kernel reaches only through a device-side address (the
conditioning table whose address `ctrl[0]` holds: step_select reads it in place), arguments of
kinds listed in READS_OUTSIDE_VIEW (none), nor workspaces the C library allocates itself.
"""
import inspect
import math
from typing import Callable, Dict, FrozenSet, List, Optional, Tuple

import torch

from audio_diffusion_pytorch_b200 import ops

F64 = torch.float64
TAU_BF16_OPERAND = 2.0 ** -8
TAU_FP32_ACC = 2.0 ** -12
BF16_REL = 2.0 ** -7
FP32_REL, FP32_TAU = 1e-5, 2.0 ** -14
STATS_TOL = 1e-4
VAR_TOL = 1e-3
GN_EPS = 1e-5                    # every statistics slot feeds a GroupNorm: it divides by sqrt(var + eps)
# attention's lse is log of the fp32 row sum of P, taken before P is rounded to bf16 for the P V GEMM
# (the rounded sum normalises o only: when a row's terms all round the same way, near-equal scores,
# the two sums differ by up to 2^-8).  LSE_FLOOR is the absolute allowance of 2^-9 kept for the log;
# attention_bwd rounds the P it recomputes from lse to bf16.
LSE_FLOOR = 2.0 ** -9
ACC_EPS = 2.0 ** -23              # an fp32 accumulator's own rounding, per unit of |before| + |after|
# the fp32 verification kernels (chain = n): err <= F32_REL |ref| + F32_LAMBDA sqrt(n) F32_U absref
F32_REL, F32_U, F32_LAMBDA = 2.0 ** -23, 2.0 ** -24, 10.0
F32_SHORT = 8                     # chain of an element-wise f32 kernel: a few roundings, transcendentals included
F64_ACC_EPS = 2.0 ** -52          # an fp64 accumulator's own rounding (loss_sum, S in the fp32 mode)
SIDE_CHUNK = 1 << 28              # bytes compared at a time by the side-effect check
ROW_TILE = 64                    # rows left stale by the mutation: half the conv GEMM's 128-row M tile

UNCHECKED: Dict[str, str] = {}          # launching functions of `ops` without a checker: none
# In the fp32 mode these kinds make their GroupNorm statistics with an adp_f32_gn_stats launch inside
# the ops call (kind -> its statistics argument); no other launch may nest in a checked one.
NESTED_STATS: Dict[str, str] = {"conv_gemm": "stats", "ln_film": "stats_out", "stem_in": "stats",
                                "skip_gate": "stats"}


class CheckError(AssertionError):
    pass


def launching_functions() -> List[str]:
    """Every function of `ops` that launches a kernel (calls ops._launch)."""
    out = []
    for name, fn in inspect.getmembers(ops, inspect.isfunction):
        if fn.__module__ == ops.__name__ and not name.startswith("_") and "_launch(" in inspect.getsource(fn):
            out.append(name)
    return sorted(out)


# ------------------------------------------------------------------------------ outputs
class Val:
    """A stored output: `view(args)` is the written view; ref / absref fp64 of its shape (or a
    callable(post args) -> (ref, absref) when the reference reads another output of the launch).
    keep: a bool mask of the view's positions the launch must leave bitwise unchanged (an in-place
    update of part of a tensor).  of: the argument the view belongs to (default: name), when one
    argument has several outputs."""

    def __init__(self, name, view, ref, absref=None, tau=TAU_FP32_ACC, exact=False, floor=0.0, keep=None,
                 of=None, chain: Optional[float] = None):
        self.name, self.view, self.ref, self.absref, self.tau, self.exact = name, view, ref, absref, tau, exact
        self.acc, self.floor = False, floor      # floor: an absolute term of the bound (see LSE_FLOOR)
        self.keep, self.of = keep, of or name
        self.chain = chain                       # an fp32 verification kernel's chain length n, or None


class Stat:
    """fp64 GroupNorm statistics [B, G, 2] accumulated (+=) by the launch over src(post args)."""

    def __init__(self, name, view, src, groups):
        self.name, self.view, self.src, self.groups = name, view, src, groups
        self.acc, self.of = True, name


class Acc:
    """An accumulator the launch adds to (+=): fp32 parameter / conditioning gradients, or fp64 sums.
    Checked as after - before against ref, the launch's own contribution (fp64; absref = the same sum
    over absolute terms), or a callable(post args) -> (ref, absref) when the contribution is defined
    on another output of the launch as stored (the GroupNorm backward sums of the rounded dxh)."""

    def __init__(self, name, view, ref, absref=None, chain: Optional[float] = None):
        self.name, self.view, self.ref, self.absref = name, view, ref, absref
        self.acc, self.exact, self.of, self.keep = True, False, name, None
        self.chain = chain


def arg(name):
    return lambda a: a[name]


def cols(name, n):
    return lambda a: a[name][..., :n]


def stats_of(y: torch.Tensor, groups: int) -> torch.Tensor:
    """(sum, sumsq) per (batch, group) of a channels-last tensor [B, T, C], fp64."""
    B, T, Cc = y.shape
    yg = y.to(F64).reshape(B, T, groups, Cc // groups)
    return torch.stack([yg.sum(dim=(1, 3)), (yg * yg).sum(dim=(1, 3))], dim=-1)


def _silu(x):
    return x * torch.sigmoid(x)


def _gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def _gn_coef(stats, gamma, beta, groups, eps, T, C):
    """(scale, shift) [B, 1, C] of GroupNorm from the statistics slots the kernel reads."""
    st = stats.to(F64)
    n = float(T * (C // groups))
    mean = st[..., 0] / n
    var = (st[..., 1] / n - mean * mean).clamp_min(0.0)
    rep = C // groups
    mean, var = mean.repeat_interleave(rep, dim=1), var.repeat_interleave(rep, dim=1)
    ga = gamma.to(F64)[None] / torch.sqrt(var + eps)
    return ga[:, None, :], (beta.to(F64)[None] - mean * ga)[:, None, :]


def _conv3(a, w3, bias=None):
    """a [T, Ci] fp64, w3 [3, Co, Ci] (tap -1, 0, +1), zero padding -> [T, Co]."""
    T = a.shape[0]
    z = a.new_zeros(1, a.shape[1])
    ap = torch.cat([z, a, z])
    out = ap[0:T] @ w3[0].t() + ap[1:T + 1] @ w3[1].t() + ap[2:T + 2] @ w3[2].t()
    return out if bias is None else out + bias


def _layer_norm(x, eps):
    """(LayerNorm(x), its std, its absref (|x| + mean|x|) / std): the centring cancels, so an
    output's rounding error scales with the row's magnitude, not with the output itself."""
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    std = torch.sqrt(var + eps)
    return (x - mean) / std, std, (x.abs() + x.abs().mean(-1, keepdim=True)) / std


# ----------------------------------------------------------------------------- checkers
def c_conv_gemm(a, ctx):
    x, w, out = a["a"], a["w"], a["out"]
    f32 = x.dtype == torch.float32         # f32_conv_gemm: fp32 operands, residual read, statistics a gn_stats pass
    B, T, _ = x.shape
    c_in, n_valid, taps, up = a["c_in"], a["n_valid"], tuple(a["taps"]), a["up_factor"]
    phases = up if up > 1 else 1
    n_pad = w.shape[0] // phases
    W = w.to(F64).reshape(phases, n_pad, w.shape[1])[:, :n_valid]
    xa = x[..., :c_in].to(F64)
    tau = TAU_FP32_ACC
    if a["gn"] is not None:
        gst, gg, gb, gG, geps = a["gn"]
        sc, sh = _gn_coef(gst, gg, gb, gG, geps, T, c_in)
        xa = _silu(xa * sc + sh)
        tau = TAU_BF16_OPERAND
    bias = a["bias"].to(F64)[:n_valid] if a["bias"] is not None else None
    gate = a["gate"].to(F64)[:, :n_valid][:, None, None, :] if a["gate"] is not None else None

    def shifted(t, off):
        if off == 0:
            return t
        z = t.new_zeros(t.shape[0], abs(off), t.shape[2])
        return torch.cat([t[:, off:], z], 1) if off > 0 else torch.cat([z, t[:, :off]], 1)

    ref = xa.new_zeros(B, T, phases, n_valid)
    absr = torch.zeros_like(ref)
    xabs = xa.abs()
    Wabs = W.abs()
    for p in range(phases):
        if up > 1:
            offs = (-1, 0) if p == 0 else ((0, 1) if p == up - 1 else (0,))
        else:
            offs = taps
        for j, off in enumerate(offs):
            Wt, Wa = W[p, :, j * c_in:(j + 1) * c_in], Wabs[p, :, j * c_in:(j + 1) * c_in]
            ref[:, :, p] += shifted(xa, off) @ Wt.t()
            absr[:, :, p] += shifted(xabs, off) @ Wa.t()
    if bias is not None:
        ref += bias
        absr += bias.abs()
    if gate is not None:
        ref *= gate
        absr *= gate.abs()
    if a["residual"] is not None and (f32 or out.dtype != torch.float32):
        r = a["residual"][..., :phases * n_valid].to(F64).reshape(B, T, phases, n_valid)
        ref += r
        absr += r.abs()
    ncols = phases * n_valid

    def view(args):
        return args["out"][..., :ncols]
    # f32: one fmaf chain of c_in per tap slot, the slots added in turn (+ bias, gate, residual)
    chain = c_in * (2 if up > 1 else len(taps)) + 3 if f32 else None
    outs = [Val("out", view, ref.reshape(B, T, ncols), absr.reshape(B, T, ncols), tau, chain=chain)]
    if a["stats"] is not None:
        outs.append(Stat("stats", arg("stats"),
                         lambda p: p["out"][..., :ncols].reshape(B, T * phases, n_valid), a["groups"]))
    return outs


def c_gn_silu(a, ctx):
    x = a["x"]
    B, T, C = x.shape
    sc, sh = _gn_coef(a["stats"], a["gamma"], a["beta"], a["groups"], a["eps"], T, C)
    z = x.to(F64) * sc + sh
    if x.dtype == torch.float32:         # f32_gn_silu forms x - mean in fp32: relative to |x| + |mean|
        be = a["beta"].to(F64)[None, None]
        return [Val("y", arg("y"), _silu(z), 1.2 * ((x.to(F64) * sc).abs() + (be - sh).abs() + be.abs()),
                    chain=F32_SHORT)]
    return [Val("y", arg("y"), _silu(z), 1.2 * ((x.to(F64) * sc).abs() + sh.abs()))]


def c_gn_stats(a, ctx):
    return [Stat("stats", arg("stats"), arg("x"), a["groups"])]


def c_ln_film(a, ctx):
    x = a["x"]
    B, T, C = x.shape
    chain = C + 4 if x.dtype == torch.float32 else None      # f32_ln_film: the row sums over C
    xn, _, lnabs = _layer_norm(x.to(F64), a["eps"])
    ref, absr = xn, lnabs
    if a["scale_shift"] is not None:
        ss = a["scale_shift"].to(F64)
        s, t = ss[:, None, :C], ss[:, None, C:2 * C]
        ref, absr = xn * (1 + s) + t, lnabs * (1 + s).abs() + t.abs()
    outs = [Val("y", arg("y"), ref, absr, chain=chain)]
    if a["y2"] is not None:
        def ref2(p, eps2=a["eps2"]):
            y2, _, y2abs = _layer_norm(p["y"].to(F64), eps2)
            return y2, y2abs
        outs.append(Val("y2", arg("y2"), ref2, chain=chain))
    if a["stats_out"] is not None:
        outs.append(Stat("stats_out", arg("stats_out"), arg("y"), a["groups"]))
    return outs


def c_attention(a, ctx):
    q, k, v = a["q"], a["k"], a["v"]
    H, D, scale = a["heads"], a["head_dim"], a["scale"]
    B, Tq, Tk, mid = q.shape[0], q.shape[1], k.shape[1], a["heads"] * a["head_dim"]
    f32 = q.dtype == torch.float32
    ref = torch.empty(B, Tq, mid, dtype=F64, device=q.device)
    absr = torch.empty_like(ref)
    lse = torch.empty(B, H, Tq, dtype=F64, device=q.device) if a["lse"] is not None else None
    lse_abs = torch.empty_like(lse) if lse is not None else None
    for b in range(B):                 # one batch element at a time: S is [H, Tq, Tk] in fp64
        Q = q[b, :, :mid].to(F64).reshape(Tq, H, D).transpose(0, 1)
        K = k[b, :, :mid].to(F64).reshape(Tk, H, D).transpose(0, 1)
        V = v[b, :, :mid].to(F64).reshape(Tk, H, D).transpose(0, 1)
        S = (Q @ K.transpose(1, 2)) * scale
        P = torch.softmax(S, dim=-1)
        ref[b] = (P @ V).transpose(0, 1).reshape(Tq, mid)
        absr[b] = (P @ V.abs()).transpose(0, 1).reshape(Tq, mid)
        if f32:
            # exp(s - max) turns an absolute error e_j of the score (a D-chain over |q| |k| scale)
            # into a relative one of p_j: o moves by sum_j p_j e_j (v_j - o), at most 2 max_j e_j P|V|
            smax = ((Q.abs() @ K.abs().transpose(1, 2)) * scale).amax(-1)                   # [H, Tq]
            absr[b] *= (1 + 2 * math.sqrt(D / (2 * Tk)) * smax).transpose(0, 1).repeat_interleave(D, dim=1)
        if lse is not None:
            lse[b] = torch.logsumexp(S, dim=-1)
            # f32: max + logf(l): the score error, l's relative error (a Tk-chain) and the log's rounding
            lse_abs[b] = S.abs().amax(-1) if not f32 else \
                math.sqrt(D / (2 * Tk)) * smax + 1 + lse[b].abs()
    if f32:
        # each key rounds twice (acc * corr + p v; l * corr + p): n = 2 Tk
        outs = [Val("o", lambda p: p["o"][..., :mid], ref, absr, chain=2 * Tk + 4)]
        if lse is not None:
            outs.append(Val("lse", arg("lse"), lse, lse_abs, chain=2 * Tk + 4))
        return outs
    outs = [Val("o", lambda p: p["o"][..., :mid], ref, absr, TAU_BF16_OPERAND)]
    if lse is not None:
        outs.append(Val("lse", arg("lse"), lse, lse_abs, floor=LSE_FLOOR))
    return outs


def c_skinny_linear(a, ctx):
    x, w, K, N = a["x"], a["w"], a["K"], a["N"]
    acts = {ops.ACT_NONE: (lambda t: t, 1.0), ops.ACT_GELU: (_gelu, 1.2), ops.ACT_SILU: (_silu, 1.2)}
    fin, gin = acts[a["in_act"]]
    fout, gout = acts[a["out_act"]]
    xi = fin(x[:, :K].to(F64))
    W = w[:N, :K].to(F64)
    pre = xi @ W.t()
    absr = xi.abs() @ W.abs().t()
    if a["bias"] is not None:
        pre = pre + a["bias"].to(F64)[:N]
        absr = absr + a["bias"].to(F64)[:N].abs()
    chain = K + 2 if w.dtype == torch.float32 else None          # f32_linear: one fmaf chain over K
    return [Val("y", lambda p: p["y"][:, :N], fout(pre), gout * absr, chain=chain)]


def c_time_features(a, ctx):
    s, fr, out = a["sigma"].to(F64), a["freqs"].to(F64), a["out"]
    B, nf = s.shape[0], fr.shape[0]
    arg_ = s[:, None] * fr[None] * (2 * math.pi)
    ref = torch.zeros(B, out.shape[1], dtype=F64, device=out.device)
    absr = torch.zeros_like(ref)
    ref[:, 0], absr[:, 0] = s, s.abs()
    ref[:, 1:1 + nf], ref[:, 1 + nf:1 + 2 * nf] = arg_.sin(), arg_.cos()
    absr[:, 1:1 + nf] = absr[:, 1 + nf:1 + 2 * nf] = arg_.abs()
    return [Val("out", lambda p: p["out"][:B], ref, absr)]


def c_silu_bf16(a, ctx):
    x = a["x"].to(F64)
    chain = F32_SHORT if a["y"].dtype == torch.float32 else None
    return [Val("y", arg("y"), _silu(x).reshape(a["y"].shape), 1.2 * x.abs().reshape(a["y"].shape), chain=chain)]


def _stem_input(a, absolute=False):
    """cat([alpha x + beta noise, append]) fp64 [B, cin, T] (VDiffusion noising in the stems);
    absolute=True: its magnitude |alpha x| + |beta noise| (the fp32 kernels round the noising)."""
    x = a["x"].to(F64)
    if absolute:
        x = x.abs()
    if a["noise"] is not None:
        al, be, nz = a["alpha"].to(F64), a["beta"].to(F64), a["noise"].to(F64)
        if absolute:
            al, be, nz = al.abs(), be.abs(), nz.abs()
        x = al[:, None, None] * x + be[:, None, None] * nz
    if a["append"] is not None:
        x = torch.cat([x, a["append"].to(F64).abs() if absolute else a["append"].to(F64)], dim=1)
    return x


def c_stem_in(a, ctx):
    xin, w, f = _stem_input(a), a["w"].to(F64), a["f"]
    f32 = a["out"].dtype == torch.float32
    B, cin, T = xin.shape
    c0 = w.shape[0]

    def rows(t):
        return t.reshape(B, cin, T // f, f).permute(0, 2, 1, 3).reshape(B, T // f, cin * f)
    xr = rows(xin)
    xa = rows(_stem_input(a, absolute=True)) if f32 else xr.abs()
    Wm = w.reshape(c0, cin * f)
    ref, absr = xr @ Wm.t(), xa @ Wm.abs().t()
    if a["bias"] is not None:
        ref, absr = ref + a["bias"].to(F64), absr + a["bias"].to(F64).abs()
    outs = [Val("out", arg("out"), ref, absr, chain=cin * f + 3 if f32 else None)]
    if a["stats"] is not None:
        outs.append(Stat("stats", arg("stats"), arg("out"), a["groups"]))
    return outs


def c_stem_out(a, ctx):
    h, f = a["h"], a["f"]
    xin = _stem_input(a)
    f32 = h.dtype == torch.float32
    xin_abs = _stem_input(a, absolute=True) if f32 else xin.abs()
    B, cin, T = xin.shape
    w = a["w"].to(F64)
    co = w.shape[0]
    # f32_stem_out: the branch is one fmaf chain over 3 c0, the adapter one over cin; then the
    # merge, the guidance combine, the sampler update or the loss term
    chain = 3 * h.shape[-1] + cin + 8 if f32 else None
    w3 = w.permute(2, 0, 1)                                    # [3, co, c0]
    bias = a["bias"].to(F64) if a["bias"] is not None else None
    if a["w_adapt"] is not None:
        wa = a["w_adapt"].to(F64)
        skip = torch.einsum("oc,bct->bot", wa, xin) + a["b_adapt"].to(F64)[None, :, None]
        skip_abs = torch.einsum("oc,bct->bot", wa.abs(), xin_abs) + a["b_adapt"].to(F64).abs()[None, :, None]
    else:
        skip, skip_abs = xin[:, :co], xin_abs[:, :co]
    gate = a["gate"].to(F64)[:, :co]

    def branch(b):               # gate * conv3(nearest_up(h)) of trunk row b -> [co, T]
        up = h[b].to(F64).repeat_interleave(f, dim=0)
        y = _conv3(up, w3, bias).t()
        ya = _conv3(up.abs(), w3.abs(), None if bias is None else bias.abs()).t()
        return gate[b][:, None] * y, gate[b].abs()[:, None] * ya
    v = torch.empty(B, co, T, dtype=F64, device=h.device)
    vabs = torch.empty_like(v)
    s = a["cfg_scale"]
    for b in range(B):
        yc, yca = branch(b)
        if s is None:
            v[b], vabs[b] = skip[b] + yc, skip_abs[b] + yca
        else:
            ym, yma = branch(b + B)
            vc, vm = skip[b] + yc, skip[b] + ym
            v[b] = vm + (vc - vm) * s
            vabs[b] = (abs(s) + abs(1 - s)) * skip_abs[b] + abs(s) * yca + abs(1 - s) * yma
    outs = []
    if a["v_out"] is not None:
        outs.append(Val("v_out", arg("v_out"), v, vabs, chain=chain))
    if a["x_next"] is not None:
        a0, b0, a1, b1 = a["ab"].to(F64).tolist()
        xs = xin[:, :co]
        xn = a1 * (a0 * xs - b0 * v) + b1 * (b0 * xs + a0 * v)
        xna = (abs(a1 * a0) + abs(b1 * b0)) * xs.abs() + (abs(a1 * b0) + abs(b1 * a0)) * vabs
        outs.append(Val("x_next", arg("x_next"), xn, xna, chain=chain))
    if a["loss_sum"] is not None:      # VDiffusion: sum (v - (alpha noise - beta x))^2, dv = 2 (v - target) / numel
        al, be = a["alpha"].to(F64)[:, None, None], a["beta"].to(F64)[:, None, None]
        nz, x0 = a["noise"].to(F64), a["x"].to(F64)
        d = v - (al * nz - be * x0)
        dabs = vabs + (al * nz).abs() + (be * x0).abs()
        if f32:        # d^2 summed in fp64: an error e of d (its chain bound) moves a term by 2 |d| e
            outs.append(Acc("loss_sum", arg("loss_sum"), (d * d).sum().reshape(1),
                            (2 * d.abs() * dabs).sum().reshape(1), chain=chain))
        else:
            # an error e of v within its fp32 bound moves d^2 by 2 |d| e: carried at the same weight
            outs.append(Acc("loss_sum", arg("loss_sum"), (d * d).sum().reshape(1),
                            ((d * d).sum() + (FP32_TAU / STATS_TOL) * (2 * d.abs() * dabs).sum()).reshape(1)))
        if a["dv"] is not None:
            outs.append(Val("dv", arg("dv"), 2 * d / d.numel(), 2 * dabs / d.numel(), chain=chain))
    return outs


def c_narrow_conv(a, ctx):
    x = a["x"]
    B, T, C = x.shape
    G = a["groups"]
    sc, sh = _gn_coef(a["stats_in"], a["gamma"], a["beta"], G, a["gn_eps"], T, C)
    act = _silu(x.to(F64) * sc + sh)
    if a["w_packed"] is not None:          # bf16 [C][3C], k = tap * C + ci
        w3 = a["w_packed"].to(F64).reshape(C, 3, C).permute(1, 0, 2)
    else:                                  # fp32 [C][C][3], rounded to bf16 for the tensor cores
        w3 = a["w"].to(torch.bfloat16).to(F64).permute(2, 0, 1)
    bias = a["bias"].to(F64) if a["bias"] is not None else None
    r = torch.stack([_conv3(act[b], w3, bias) for b in range(B)])
    ra = torch.stack([_conv3(act[b].abs(), w3.abs(), None if bias is None else bias.abs()) for b in range(B)])
    if a["residual"] is not None:
        r, ra = r + a["residual"].to(F64), ra + a["residual"].to(F64).abs()
    ref, absr = r, ra
    if a["scale_shift"] is not None:
        ss = a["scale_shift"].to(F64)
        s, t = ss[:, None, :C], ss[:, None, C:2 * C]
        xn, std, lnabs = _layer_norm(r, a["ln_eps"])
        ref = xn * (1 + s) + t
        # an error e in r moves LN(r) by up to ~2 max|e| / std (the row's own entry, its mean, its variance)
        absr = (2 * ra.amax(-1, keepdim=True) / std + lnabs) * (1 + s).abs() + t.abs()
    outs = [Val("y", arg("y"), ref, absr, TAU_BF16_OPERAND)]
    if a["stats_out"] is not None:
        outs.append(Stat("stats_out", arg("stats_out"), arg("y"), G))
    return outs


def c_sampler_step(a, ctx):
    x, v = a["x"].to(F64), a["v"].to(F64)
    a0, b0, a1, b1 = a["ab"].to(F64).tolist()
    ref = a1 * (a0 * x - b0 * v) + b1 * (b0 * x + a0 * v)
    absr = (abs(a1 * a0) + abs(b1 * b0)) * x.abs() + (abs(a1 * b0) + abs(b1 * a0)) * v.abs()
    return [Val("x_next", arg("x_next"), ref, absr)]


def c_step_select(a, ctx):
    ctrl = a["ctrl"].tolist()
    div = ctrl[1] if ctrl[1] > 0 else 1
    n_it = (ctrl[2] if ctrl[2] > 0 else 1) * div
    it = min(int(a["step"].item()), n_it - 1)
    n = a["ss_out"].numel()
    table = ctx.lookup(ctrl[0], (it // div + 1) * n, torch.float32)
    return [Val("ss_out", arg("ss_out"), table[(it // div) * n:(it // div + 1) * n].reshape(a["ss_out"].shape),
                exact=True),
            Val("ab_out", arg("ab_out"), a["ab_table"][it].clone(), exact=True)]


def c_step_advance(a, ctx):
    return [Val("step", arg("step"), a["step"] + 1, exact=True)]


# ------------------------------------------------------------- training launch kinds
def _shift(t, off):
    """t[:, i] <- t[:, i + off] along dim 1, zeros outside."""
    if off == 0:
        return t
    z = t.new_zeros(t.shape[0], abs(off), *t.shape[2:])
    return torch.cat([t[:, off:], z], 1) if off > 0 else torch.cat([z, t[:, :off]], 1)


def _gn_xhat(x, stats, groups, eps):
    """(xhat, rstd [B, 1, C], |xhat|'s magnitude) of GroupNorm from the statistics slots (arithmetic
    of _gn_coef).  The kernels form xhat = (x - mean) rstd in fp32: its rounding is relative to
    (|x| + |mean|) rstd, which is far above |xhat| where x lies close to its group's mean.  A sum over
    many rows hides that; a group of one row (an innermost level of length 1 at B = 1) does not."""
    B, T, C = x.shape
    one = torch.ones(C, dtype=F64, device=x.device)
    sc, sh = _gn_coef(stats, one, torch.zeros_like(one), groups, eps, T, C)     # rstd, -mean rstd
    xf = x.to(F64)
    return xf * sc + sh, sc, xf.abs() * sc + sh.abs()


def _dsilu(z):
    sg = torch.sigmoid(z)
    return sg * (1 + z * (1 - sg))


DSILU_MAX = 1.1                  # max |SiLU'|


def _group_sums(t, groups):
    B, T, C = t.shape
    return t.reshape(B, T, groups, C // groups).sum(dim=(1, 3))


def _gn_S(xh, xha, groups):
    """The GroupNorm backward sums S[b, g] = (sum dxh, sum dxh xhat) of dxh AS STORED (xha: the
    magnitude of xhat, _gn_xhat)."""
    def ref(p):
        d = p["dxh"].to(F64)
        return (torch.stack([_group_sums(d, groups), _group_sums(d * xh, groups)], -1),
                torch.stack([_group_sums(d.abs(), groups), _group_sums(d.abs() * xha, groups)], -1))
    return ref


def c_wgrad(a, ctx):
    g, x, n, k = a["g"], a["x"], a["n"], a["k"]
    chain = g.shape[0] * g.shape[1] if g.dtype == torch.float32 else None     # f32_wgrad: one chain over B T
    G = g[..., a["g_col0"]:a["g_col0"] + n].to(F64).reshape(-1, n)
    X = x[..., a["x_col0"]:a["x_col0"] + k].to(F64)
    taps = 3 if a["ntaps"] == 3 else 1
    ref = [G.t() @ _shift(X, a["off"] + j).reshape(-1, k) for j in range(taps)]
    absr = [G.abs().t() @ _shift(X.abs(), a["off"] + j).reshape(-1, k) for j in range(taps)]
    if taps == 3:
        return [Acc("dw", lambda p: p["dw"][:, :n, :k], torch.stack(ref), torch.stack(absr), chain=chain)]
    return [Acc("dw", lambda p: p["dw"][:n, :k], ref[0], absr[0], chain=chain)]


def c_gn_silu_bwd(a, ctx):
    x, G = a["x"], a["groups"]
    B, T, _ = x.shape
    xh, _, xha = _gn_xhat(x, a["stats"], G, a["eps"])
    ga, da, be = a["gamma"].to(F64), a["da"].to(F64), a["beta"].to(F64)
    dz = da * _dsilu(xh * ga + be)
    # SiLU' crosses zero (z = -1.28) by cancellation: dz's rounding is relative to DSILU_MAX |da|, as for
    # dxh and narrow_conv_bwd; a sum over one row (M = 1) shows it
    dza = DSILU_MAX * da.abs()
    f32 = x.dtype == torch.float32
    if f32:            # + z's own rounding (relative to |xhat gamma| + |beta|) through |SiLU''| <= 1/2
        dza = dza + 0.5 * da.abs() * (xha * ga.abs() + be.abs())
    c = (lambda n: n) if f32 else (lambda n: None)
    return [Val("dxh", arg("dxh"), dz * ga, dza * ga.abs(), chain=c(F32_SHORT)),
            Acc("dgamma", arg("dgamma"), (dz * xh).sum((0, 1)), (dza * xha).sum((0, 1)), chain=c(B * T)),
            Acc("dbeta", arg("dbeta"), dz.sum((0, 1)), dza.sum((0, 1)), chain=c(B * T)),
            Acc("S", arg("S"), _gn_S(xh, xha, G), chain=c(T + F32_SHORT))]


def c_gn_bwd_apply(a, ctx):
    x, G = a["x"], a["groups"]
    B, T, C = x.shape
    xh, rstd, xha = _gn_xhat(x, a["stats"], G, a["eps"])
    c = (a["S"].to(F64) / float(T * (C // G))).repeat_interleave(C // G, dim=1)[:, None]     # [B, 1, C, 2]
    d = a["dxh"].to(F64)
    ref = rstd * (d - c[..., 0] - xh * c[..., 1])
    absr = rstd.abs() * (d.abs() + c[..., 0].abs() + xha * c[..., 1].abs())
    if a["dres"] is not None:
        ref, absr = ref + a["dres"].to(F64), absr + a["dres"].to(F64).abs()
    f32 = x.dtype == torch.float32
    outs = [Val("dx", arg("dx"), ref, absr, chain=F32_SHORT if f32 else None)]
    if a["colsum"] is not None:        # the kernel sums the values before they are rounded to bf16
        outs.append(Acc("colsum", cols("colsum", C), ref.sum((0, 1)), absr.sum((0, 1)),
                        chain=B * T + F32_SHORT if f32 else None))
    return outs


def c_ln_film_bwd(a, ctx):
    x = a["x"]
    B, T, C = x.shape
    xh, std, lnabs = _layer_norm(x.to(F64), a["eps"])
    dy = a["dy"].to(F64)
    f = 1 + a["scale_shift"].to(F64)[:, None, :C] if a["scale_shift"] is not None else 1.0
    g = dy * f
    m1, m2 = g.mean(-1, keepdim=True), (g * xh).mean(-1, keepdim=True)
    ref = (g - m1 - xh * m2) / std
    f32 = x.dtype == torch.float32
    # f32_ln_film_bwd forms xhat in fp32: its rounding is relative to lnabs ((|x| + mean|x|) / std)
    xa = lnabs if f32 else xh.abs()
    absr = (g.abs() + g.abs().mean(-1, keepdim=True) + xa * (g.abs() * xa).mean(-1, keepdim=True)) / std
    if a["dres"] is not None:
        ref, absr = ref + a["dres"].to(F64), absr + a["dres"].to(F64).abs()
    c = (lambda n: n) if f32 else (lambda n: None)
    outs = [Val("dx", arg("dx"), ref, absr, chain=c(C + F32_SHORT))]
    if a["dss"] is not None:
        outs.append(Acc("dss", cols("dss", 2 * C), torch.cat([(dy * xh).sum(1), dy.sum(1)], -1),
                        torch.cat([(dy.abs() * xa).sum(1), dy.abs().sum(1)], -1), chain=c(T + C)))
    if a["colsum"] is not None:
        outs.append(Acc("colsum", cols("colsum", C), ref.sum((0, 1)), absr.sum((0, 1)), chain=c(B * T + C)))
    return outs


def c_colsum(a, ctx):
    x = a["x"].to(F64)
    B, T, C = x.shape
    chain = B * T + 2 if a["x"].dtype == torch.float32 else None      # f32_colsum: B T-sums, gated, summed
    if a["gate"] is not None:
        x = x * a["gate"].to(F64)[:, None, :C]
    return [Acc("out", cols("out", C), x.sum((0, 1)), x.abs().sum((0, 1)), chain=chain)]


def c_skip_gate(a, ctx):
    y, skip = a["y"].to(F64), a["skip"].to(F64)
    gy = a["gate"].to(F64)[:, None, :y.shape[-1]] * y
    chain = F32_SHORT if a["y"].dtype == torch.float32 else None
    outs = [Val("out", arg("out"), skip + gy, skip.abs() + gy.abs(), chain=chain)]
    if a["stats"] is not None:
        outs.append(Stat("stats", arg("stats"), arg("out"), a["groups"]))
    return outs


def c_skip_gate_bwd(a, ctx):
    d, y = a["dout"].to(F64), a["y"].to(F64)
    T, C = y.shape[1], y.shape[-1]
    ref = a["gate"].to(F64)[:, None, :C] * d
    c = (lambda n: n) if a["y"].dtype == torch.float32 else (lambda n: None)
    return [Val("dys", arg("dys"), ref, ref.abs(), chain=c(F32_SHORT)),
            Acc("dgate", cols("dgate", C), (d * y).sum(1), (d * y).abs().sum(1), chain=c(T + 2))]


def c_cond_bwd(a, ctx):
    N = a["N"]
    d, c, W = a["dss"][:, :N].to(F64), a["cond"].to(F64), a["w"][:N].to(F64)
    B = d.shape[0]
    f = (lambda n: n) if a["w"].dtype == torch.float32 else (lambda n: None)
    outs = [Val("dw", lambda p: p["dw"][:N], d.t() @ c, d.abs().t() @ c.abs(), chain=f(B + 2)),
            Val("dbias", lambda p: p["dbias"][:N], d.sum(0), d.abs().sum(0), chain=f(B + 2))]
    if a["dcond"] is not None:
        outs.append(Acc("dcond", arg("dcond"), d @ W, d.abs() @ W.abs(), chain=f(N + 2)))
    return outs


def _conv3_t(dy, w3):
    """Transpose of _conv3 over [B, T, Co]: da[t] = sum_k dy[t - (k - 1)] @ w3[k]  (w3 [3, Co, Ci])."""
    return sum(_shift(dy, 1 - k) @ w3[k] for k in range(3))


def c_narrow_conv_bwd(a, ctx):
    x, G = a["x"], a["groups"]
    xh, _, xha = _gn_xhat(x, a["stats_in"], G, a["gn_eps"])
    ga = a["gamma"].to(F64)
    z = xh * ga + a["beta"].to(F64)
    act, dy = _silu(z), a["dy"].to(F64)
    w3 = a["w"].to(F64).permute(2, 0, 1)                        # [3, co, ci]
    da, da_abs = _conv3_t(dy, w3), _conv3_t(dy.abs(), w3.abs())
    dz = da * _dsilu(z)
    C = x.shape[-1]
    dw = torch.stack([dy.reshape(-1, C).t() @ _shift(act, k - 1).reshape(-1, C) for k in range(3)], -1)
    dwa = torch.stack([dy.abs().reshape(-1, C).t() @ _shift(act.abs(), k - 1).reshape(-1, C) for k in range(3)], -1)
    # the sums of dz inherit the error of da (fp32 dot products of 3 C terms): its absref, not |dz|
    dza = DSILU_MAX * da_abs
    return [Val("dxh", arg("dxh"), dz * ga, dza * ga.abs()),
            Acc("dgamma", arg("dgamma"), (dz * xh).sum((0, 1)), (dza * xha).sum((0, 1))),
            Acc("dbeta", arg("dbeta"), dz.sum((0, 1)), dza.sum((0, 1))),
            Acc("S", arg("S"), _gn_S(xh, xha, G)),
            Acc("dw", arg("dw"), dw, dwa),
            Acc("dbias", arg("dbias"), dy.sum((0, 1)), dy.abs().sum((0, 1)))]


def c_stem_out_bwd(a, ctx):
    h, f = a["h"], a["f"]
    B, Tl, c0 = h.shape
    w = a["w"].to(F64)
    co = w.shape[0]
    w3 = w.permute(2, 0, 1)                                     # [3, co, c0]
    gs = a["gscale"].to(F64)[0] if a["gscale"] is not None else 1.0
    dvs = (a["dv"].to(F64) * gs).transpose(1, 2)                # [B, T, co]
    gate = a["gate"].to(F64)[:, None, :co]
    dy = dvs * gate
    up = h.to(F64).repeat_interleave(f, dim=1)                  # nearest upsampling [B, T, c0]
    dup, dupa = _conv3_t(dy, w3), _conv3_t(dy.abs(), w3.abs())
    bias = a["bias"].to(F64) if a["bias"] is not None else None
    y = torch.stack([_conv3(up[b], w3, bias) for b in range(B)])
    ya = torch.stack([_conv3(up[b].abs(), w3.abs(), None if bias is None else bias.abs()) for b in range(B)])
    T = up.shape[1]
    dw = torch.stack([dy.reshape(-1, co).t() @ _shift(up, k - 1).reshape(-1, c0) for k in range(3)], -1)
    dwa = torch.stack([dy.abs().reshape(-1, co).t() @ _shift(up.abs(), k - 1).reshape(-1, c0) for k in range(3)], -1)
    # f32_stem_out_bwd: dh sums f 3 co terms, the parameter gradients B T terms; dgate's terms carry
    # the branch y, itself a chain over 3 c0: (sqrt(T) + sqrt(3 c0))^2 <= 2 (T + 3 c0)
    f32 = h.dtype == torch.float32
    c = (lambda n: n) if f32 else (lambda n: None)
    outs = [Val("dh", arg("dh"), dup.reshape(B, Tl, f, c0).sum(2), dupa.reshape(B, Tl, f, c0).sum(2),
                chain=c(3 * f * co + 2)),
            Acc("dw", arg("dw"), dw, dwa, chain=c(B * T + 2)),
            Acc("dbias", cols("dbias", co), dy.sum((0, 1)), dy.abs().sum((0, 1)), chain=c(B * T + 2)),
            Acc("dgate", cols("dgate", co), (dvs * y).sum(1), (dvs.abs() * ya).sum(1), chain=c(2 * (T + 3 * c0 + 2)))]
    xin = None
    if a["w_adapt"] is not None:
        xin = _stem_input(a).transpose(1, 2)                    # [B, T, cin]
        xin_abs = _stem_input(a, absolute=True).transpose(1, 2) if f32 else xin.abs()
        cin = xin.shape[-1]
        outs += [Acc("dw_adapt", arg("dw_adapt"), dvs.reshape(-1, co).t() @ xin.reshape(-1, cin),
                     dvs.abs().reshape(-1, co).t() @ xin_abs.reshape(-1, cin), chain=c(B * T + 3)),
                 Acc("db_adapt", arg("db_adapt"), dvs.sum((0, 1)), dvs.abs().sum((0, 1)), chain=c(B * T + 1))]
    if a["dxin"] is not None:          # through the skip path only, stored
        cin = a["dxin"].shape[1]
        if a["w_adapt"] is not None:
            wa = a["w_adapt"].to(F64)
            ref, absr = dvs @ wa, dvs.abs() @ wa.abs()
        else:
            ref = torch.cat([dvs, dvs.new_zeros(B, T, cin - co)], -1)
            absr = ref.abs()
        outs.append(Val("dxin", arg("dxin"), ref.transpose(1, 2), absr.transpose(1, 2), chain=c(co + 2)))
    return outs


def c_stem_in_bwd(a, ctx):
    f = a["f"]
    xin, d = _stem_input(a), a["dout"].to(F64)
    f32 = a["dout"].dtype == torch.float32
    B, cin, T = xin.shape
    c0 = d.shape[-1]

    def rows(t):
        return t.reshape(B, cin, T // f, f).permute(0, 2, 1, 3).reshape(-1, cin * f)
    xr = rows(xin)
    xa = rows(_stem_input(a, absolute=True)) if f32 else xr.abs()
    d2 = d.reshape(-1, c0)
    c = (lambda n: n) if f32 else (lambda n: None)
    outs = [Acc("dw", arg("dw"), (d2.t() @ xr).reshape(c0, cin, f), (d2.abs().t() @ xa).reshape(c0, cin, f),
                chain=c(d2.shape[0] + 3)),
            Acc("dbias", arg("dbias"), d2.sum(0), d2.abs().sum(0), chain=c(d2.shape[0] + 1))]
    if a["dxin"] is not None:
        Wm = a["w"].to(F64).reshape(c0, cin * f)

        def back(t):
            return t.reshape(B, T // f, cin, f).permute(0, 2, 1, 3).reshape(B, cin, T)
        outs.append(Acc("dxin", arg("dxin"), back(d2 @ Wm), back(d2.abs() @ Wm.abs()), chain=c(c0 + 1)))
    return outs


def c_attention_bwd(a, ctx):
    q, k, v = a["q"], a["k"], a["v"]
    H, D, scale = a["heads"], a["head_dim"], a["scale"]
    B, Tq, Tk, mid = q.shape[0], q.shape[1], k.shape[1], H * D
    dev = q.device
    f32 = q.dtype == torch.float32
    r = {n: torch.empty(B, t, mid, dtype=F64, device=dev) for n, t in
         (("dq", Tq), ("dk", Tk), ("dv", Tk), ("dqa", Tq), ("dka", Tk), ("dva", Tk))}
    delta = torch.empty(B, H, Tq, dtype=F64, device=dev)
    delta_abs = torch.empty_like(delta)

    def heads(t, b, n):
        return t[b, :, :mid].to(F64).reshape(n, H, D).transpose(0, 1)

    def rows(t, n):
        return t.transpose(0, 1).reshape(n, mid)
    for b in range(B):
        Q, K, V = heads(q, b, Tq), heads(k, b, Tk), heads(v, b, Tk)
        O, dO = heads(a["o"], b, Tq), heads(a["d_o"], b, Tq)
        P = torch.exp((Q @ K.transpose(1, 2)) * scale - a["lse"][b].to(F64)[..., None])
        dl, dla = (dO * O).sum(-1), (dO * O).abs().sum(-1)
        dS = P * (dO @ V.transpose(1, 2) - dl[..., None])
        dSa = P * (dO.abs() @ V.abs().transpose(1, 2) + dla[..., None])
        Pa = P
        if f32:
            # the f32 kernels recompute s (a D-chain over |q| |k| scale): its absolute error is a
            # relative one of P = exp(s - lse), carried into P and dS at the weight of one chain
            sa = 1 + (Q.abs() @ K.abs().transpose(1, 2)) * scale
            Pa, dSa = P * sa, dSa * sa
        delta[b], delta_abs[b] = dl, dla
        r["dv"][b], r["dva"][b] = rows(P.transpose(1, 2) @ dO, Tk), rows(Pa.transpose(1, 2) @ dO.abs(), Tk)
        r["dq"][b], r["dqa"][b] = rows(dS @ K * scale, Tq), rows(dSa @ K.abs() * scale, Tq)
        r["dk"][b], r["dka"][b] = rows(dS.transpose(1, 2) @ Q * scale, Tk), rows(dSa.transpose(1, 2) @ Q.abs() * scale, Tk)
    # P and dS are rounded to bf16 for the second GEMMs
    def delta_view(p):       # a flat workspace sized for the largest item: this launch's rows come first
        return p["delta"].reshape(-1)[:B * H * Tq].view(B, H, Tq)
    if f32:                  # dq sums Tk terms, dk and dv Tq terms, each over a D-chain of s and dO.v
        return [Val("delta", delta_view, delta, delta_abs, chain=D + 2),
                Val("dq", cols("dq", mid), r["dq"], r["dqa"], chain=Tk + D + 4),
                Val("dk", cols("dk", mid), r["dk"], r["dka"], chain=Tq + D + 4),
                Val("dv", cols("dv", mid), r["dv"], r["dva"], chain=Tq + D + 4)]
    return [Val("delta", delta_view, delta, delta_abs),
            Val("dq", cols("dq", mid), r["dq"], r["dqa"], TAU_BF16_OPERAND),
            Val("dk", cols("dk", mid), r["dk"], r["dka"], TAU_BF16_OPERAND),
            Val("dv", cols("dv", mid), r["dv"], r["dva"], TAU_BF16_OPERAND)]


def c_ln_fold_bwd(a, ctx):
    W, g, b = a["w"].to(F64), a["g"].to(F64), a["b"].to(F64)
    N, C = W.shape
    dwf, dbf = a["dwf"][:N, :C].to(F64), a["dbf"][:N].to(F64)
    return [Val("dw", arg("dw"), dwf * g + dbf[:, None] * b, (dwf * g).abs() + (dbf[:, None] * b).abs()),
            Acc("dg", arg("dg"), (dwf * W).sum(0), (dwf * W).abs().sum(0)),
            Acc("db", arg("db"), W.t() @ dbf, W.abs().t() @ dbf.abs())]


def _fir_result(a):
    n = a["t_out"] if a["adjoint_of"] is None else a["adjoint_of"]
    return {"_result": (a["x"].shape[0], n)}


def c_fir_resample(a, ctx):
    """y[r, i fo + p] = sum_k xpad[r, i fi + k] bank[p, k], xpad[j] = x[j - half]; or its transpose."""
    x, bank = a["x"].to(F64), a["bank"].to(F64)
    fi, fo, half, t_out = a["factor_in"], a["factor_out"], a["half"], a["t_out"]
    taps = bank.shape[1]
    rows = x.shape[0]
    frames = -(-t_out // fo)
    span = (frames - 1) * fi + taps

    def forward(xs, bk):
        t = xs.shape[1]
        xp = torch.cat([xs.new_zeros(rows, half), xs, xs.new_zeros(rows, max(0, span - half - t))], 1)[:, :span]
        return (xp.unfold(1, taps, fi) @ bk.t()).reshape(rows, frames * fo)[:, :t_out]

    def adjoint(dy, bk):
        t = a["adjoint_of"]
        d = torch.cat([dy, dy.new_zeros(rows, frames * fo - t_out)], 1).reshape(rows, frames, fo) @ bk
        idx = (torch.arange(frames, device=x.device)[:, None] * fi + torch.arange(taps, device=x.device)).reshape(-1)
        xp = dy.new_zeros(rows, max(span, half + t)).index_add_(1, idx, d.reshape(rows, -1))
        return xp[:, half:half + t]
    op = forward if a["adjoint_of"] is None else adjoint
    return [Val("_result", arg("_result"), op(x, bank), op(x.abs(), bank.abs()))]


# ---------------------------------------------------- vocoder front-end and sampler steps
# Keyword options of these restatements state an alternative operation (a padding, a frame order, a
# batch stride): the kind-specific mutations below write it over the output, so the checker must
# tell the two apart.
def _mel_result(a):
    rows, t = a["wave"].shape
    frames = 1 + (t + 2 * a["pad"] - a["n_fft"]) // a["hop"]
    return {"mel": (rows, a["fb"].shape[1], frames)}


def _frames(wave, n_fft, hop, pad, frames, symmetric=False):
    """[rows, frames, n_fft]: frame f is padded[f hop : f hop + n_fft] of the row padded by `pad` on
    both sides, by reflection (F.pad mode="reflect": the edge sample is not repeated) or, with
    symmetric=True, by mirroring (the edge sample repeated)."""
    t = wave.shape[1]
    j = torch.arange(frames, device=wave.device)[:, None] * hop + torch.arange(n_fft, device=wave.device) - pad
    if symmetric:
        j = torch.where(j < 0, -j - 1, torch.where(j >= t, 2 * t - 1 - j, j))
    else:
        j = torch.where(j < 0, -j, torch.where(j >= t, 2 * (t - 1) - j, j))
    return wave[:, j]


def c_mel_spectrogram(a, ctx, symmetric=False, swap_pairs=False):
    """mel[r, m, f] = sum_k fb[k, m] |rfft(window frame_f)[k]|, then log(max(., 1e-5)) if apply_log.
    absref = sum_k |fb[k, m]| sum_n |window_n frame_f[n]|, which bounds every |X_k| (triangle
    inequality); a float FFT's error is ~log2(N) 2^-24 of it."""
    wave, window, fb = a["wave"].to(F64), a["window"].to(F64), a["fb"].to(F64)
    n_fft, hop, pad = a["n_fft"], a["hop"], a["pad"]
    rows, n_mels, frames = _mel_result(a)["mel"]
    fr = _frames(wave, n_fft, hop, pad, frames, symmetric) * window
    mel = (torch.fft.rfft(fr, dim=-1).abs() @ fb).transpose(1, 2)              # [rows, n_mels, frames]
    absr = (fr.abs().sum(-1)[:, None, :] * fb.abs().sum(0)[None, :, None])
    if swap_pairs:                     # the two frames of each FFT pair exchanged (2p <-> 2p + 1)
        f = torch.arange(frames, device=wave.device)
        f = torch.where((f ^ 1) < frames, f ^ 1, f)
        mel, absr = mel[..., f], absr[..., f]
    if not a["apply_log"]:
        return [Val("mel", arg("mel"), mel, absr)]
    # an error within b of the linear value moves log(max(., 1e-5)) by at most b / max(ref - b, 1e-5)
    # (the clamped log's Lipschitz constant on [ref - b, ref + b]); 1e-5 |log| is the log's own rounding
    b = FP32_REL * mel.abs() + FP32_TAU * absr
    return [Val("mel", arg("mel"), torch.log(mel.clamp_min(1e-5)), b / (mel - b).clamp_min(1e-5) / FP32_TAU)]


def _to_flat_result(a):
    B, _, frames = a["spec"].shape
    return {"out": (B, (frames - 1) * a["hop"] - 2 * a["pad"] + a["w"].shape[1])}


def _overlap_add(spec, w, hop, start, t_out):
    """out[b, t] = sum_c sum_j spec[b, c, j] w[c, t + start - j hop] (0 <= t + start - j hop < win)."""
    B, _, frames = spec.shape
    win = w.shape[1]
    cols = torch.einsum("bcj,ck->bjk", spec, w)                                 # frame j's window
    at = (torch.arange(frames, device=spec.device)[:, None] * hop + torch.arange(win, device=spec.device)).reshape(-1)
    full = cols.new_zeros(B, (frames - 1) * hop + win).index_add_(1, at, cols.reshape(B, -1))
    return full[:, start:start + t_out]


def c_to_flat(a, ctx, shift=0):
    """The bias-free ConvTranspose1d(C -> 1, kernel win, stride hop, padding pad); shift=1: the output
    one sample late."""
    spec, w, hop, pad = a["spec"].to(F64), a["w"].to(F64), a["hop"], a["pad"]
    t_out = _to_flat_result(a)["out"][1]
    return [Val("out", arg("out"), _overlap_add(spec, w, hop, pad - shift, t_out),
                _overlap_add(spec.abs(), w.abs(), hop, pad - shift, t_out))]


def _to_flat_bwd_result(a):
    return {"dspec": tuple(a["spec"].shape) if a["need_dspec"] else None,
            "dw": tuple(a["w"].shape) if a["need_dw"] else None}


def c_to_flat_bwd(a, ctx, dw_rows=None):
    """dspec[b, c, j] = sum_k w[c, k] dout[b, j hop + k - pad] and dw[c, k] = sum_b sum_j spec[b, c, j]
    dout[b, j hop + k - pad] (dout zero outside [0, t_out)); both are tensors the launch allocates and
    returns (dw zeroed inside ops.to_flat_bwd: stored, not accumulated).  dw_rows: dw over the first
    rows only (a lost batch row)."""
    spec, w, dout, hop, pad = a["spec"].to(F64), a["w"].to(F64), a["dout"].to(F64), a["hop"], a["pad"]
    B, win = dout.shape[0], w.shape[1]
    z = dout.new_zeros(B, pad)
    d = torch.cat([z, dout, z], 1).unfold(1, win, hop)                        # [B, frames, win]
    outs = []
    if a["need_dspec"]:
        outs.append(Val("dspec", arg("dspec"), torch.einsum("bjk,ck->bcj", d, w),
                        torch.einsum("bjk,ck->bcj", d.abs(), w.abs())))
    if a["need_dw"]:
        n = B if dw_rows is None else dw_rows
        outs.append(Val("dw", arg("dw"), torch.einsum("bcj,bjk->ck", spec[:n], d[:n]),
                        torch.einsum("bcj,bjk->ck", spec[:n].abs(), d[:n].abs())))
    return outs


def c_inpaint_blend(a, ctx, level=2):
    """x <- ab[2] source + ab[3] noise where mask, in place; elsewhere x keeps the sampler's value, bit
    for bit.  level=0: blended to the level the step started from (ab[0], ab[1])."""
    x, keep = a["x"], a["mask_u8"] == 0
    al, be = (float(c) for c in a["ab"].to(F64)[level:level + 2])
    src, nz = a["source"].to(F64), a["noise"].to(F64)
    ref = torch.where(keep, x.to(F64), al * src + be * nz)
    absr = torch.where(keep, 0.0, abs(al) * src.abs() + abs(be) * nz.abs())
    return [Val("x", arg("x"), ref, absr, keep=keep)]


def c_arv_step(a, ctx, advance_sigma=True, v_batch_stride=None):
    """In place on chan [B, C+1, T] = (x | sigma_0), with a = cos(sigma pi / 2), b = sin(sigma pi / 2):
    x <- a_1 (a_0 x - b_0 v) + b_1 (b_0 x + a_0 v), sigma_1 = sig_next [B, T] (bitwise) into channel C.
    v_batch_stride: v [B, C, T] read with another batch stride (zero past its end)."""
    chan, sig1 = a["chan"].to(F64), a["sig_next"].to(F64)
    B, C1, T = chan.shape
    C = C1 - 1
    v = a["v"].to(F64)
    if v_batch_stride is not None:
        flat = torch.cat([v.reshape(-1), v.new_zeros(B * v_batch_stride)])
        at = (torch.arange(B, device=v.device)[:, None, None] * v_batch_stride +
              torch.arange(C, device=v.device)[:, None] * T + torch.arange(T, device=v.device))
        v = flat[at]
    x, s0, s1 = chan[:, :C], chan[:, C:], sig1.reshape(B, 1, T)
    a0, b0, a1, b1 = torch.cos(s0 * math.pi / 2), torch.sin(s0 * math.pi / 2), \
        torch.cos(s1 * math.pi / 2), torch.sin(s1 * math.pi / 2)
    ref = a1 * (a0 * x - b0 * v) + b1 * (b0 * x + a0 * v)
    absr = ((a1 * a0).abs() + (b1 * b0).abs()) * x.abs() + ((a1 * b0).abs() + (b1 * a0).abs()) * v.abs()
    return [Val("chan", lambda p: p["chan"][:, :C], ref, absr),
            Val("chan.sigma", lambda p: p["chan"][:, C], (s1 if advance_sigma else s0)[:, 0], exact=True, of="chan")]


# Role of every tensor argument of each checked kind: read, stored (the launch writes it), or
# accumulated (+=, checked as after - before).  Shadow refuses a launch whose checker returns
# outputs other than these, or leaves a passed output argument unchecked; `probe=True` also
# perturbs each read argument and requires some reference to move (an input the restatement
# ignores is a gap).
ARGS: Dict[str, Tuple[FrozenSet[str], FrozenSet[str], FrozenSet[str]]] = {k: (frozenset(r), frozenset(st), frozenset(ac)) for k, (r, st, ac) in {
    "conv_gemm": ({"a", "w", "bias", "residual", "gate", "gn"}, {"out"}, {"stats"}),
    "gn_silu": ({"x", "stats", "gamma", "beta"}, {"y"}, ()),
    "gn_stats": ({"x"}, (), {"stats"}),
    "ln_film": ({"x", "scale_shift"}, {"y", "y2"}, {"stats_out"}),
    "attention": ({"q", "k", "v"}, {"o", "lse"}, ()),
    "skinny_linear": ({"x", "w", "bias"}, {"y"}, ()),
    "time_features": ({"sigma", "freqs"}, {"out"}, ()),
    "silu_bf16": ({"x"}, {"y"}, ()),
    "stem_in": ({"x", "w", "bias", "append", "noise", "alpha", "beta"}, {"out"}, {"stats"}),
    "stem_out": ({"h", "x", "w", "bias", "gate", "append", "w_adapt", "b_adapt", "ab", "noise", "alpha", "beta"},
                 {"v_out", "x_next", "dv"}, {"loss_sum"}),
    "narrow_conv": ({"x", "stats_in", "gamma", "beta", "w", "bias", "residual", "scale_shift", "w_packed"},
                    {"y"}, {"stats_out"}),
    "sampler_step": ({"x", "v", "ab"}, {"x_next"}, ()),
    "step_select": ({"step", "ctrl", "ab_table"}, {"ab_out", "ss_out"}, ()),
    "step_advance": ((), {"step"}, ()),       # step += 1, checked against the snapshot + 1
    # training (training.py's plans): the third set holds fp32 / fp64 accumulators (Acc) and statistics
    "wgrad": ({"g", "x"}, (), {"dw"}),
    "gn_silu_bwd": ({"da", "x", "stats", "gamma", "beta"}, {"dxh"}, {"dgamma", "dbeta", "S"}),
    "gn_bwd_apply": ({"dxh", "x", "stats", "S", "dres"}, {"dx"}, {"colsum"}),
    "ln_film_bwd": ({"dy", "x", "scale_shift", "dres"}, {"dx"}, {"dss", "colsum"}),
    "colsum": ({"x", "gate"}, (), {"out"}),
    "skip_gate": ({"y", "skip", "gate"}, {"out"}, {"stats"}),
    "skip_gate_bwd": ({"dout", "y", "gate"}, {"dys"}, {"dgate"}),
    "cond_bwd": ({"dss", "cond", "w"}, {"dw", "dbias"}, {"dcond"}),
    "narrow_conv_bwd": ({"dy", "x", "stats_in", "gamma", "beta", "w"}, {"dxh"},
                        {"dgamma", "dbeta", "S", "dw", "dbias"}),
    "stem_out_bwd": ({"dv", "h", "x", "w", "bias", "gate", "gscale", "append", "noise", "alpha", "beta", "w_adapt"},
                     {"dh", "dxin"}, {"dw", "dbias", "dgate", "dw_adapt", "db_adapt"}),
    "stem_in_bwd": ({"dout", "x", "append", "noise", "alpha", "beta", "w"}, (), {"dw", "dbias", "dxin"}),
    "attention_bwd": ({"q", "k", "v", "o", "d_o", "lse"}, {"delta", "dq", "dk", "dv"}, ()),
    "ln_fold_bwd": ({"w", "g", "b", "dwf", "dbf"}, {"dw"}, {"dg", "db"}),
    "fir_resample": ({"x", "bank"}, {"_result"}, ()),      # the output is the tensor the launch returns
    # the vocoder front-end: outputs are tensors the launch returns (RESULT)
    "mel_spectrogram": ({"wave", "window", "fb", "band"}, {"mel"}, ()),
    "to_flat": ({"spec", "w"}, {"out"}, ()),
    "to_flat_bwd": ({"spec", "w", "dout"}, {"dspec", "dw"}, ()),
    # the sampler steps of VInpainter and ARVSampler, in place (x / chan are read too)
    "inpaint_blend": ({"source", "noise", "mask_u8", "ab"}, {"x"}, ()),
    "arv_step": ({"v", "sig_next"}, {"chan"}, ()),
}.items()}

# Kinds whose outputs are tensors the launch allocates and returns: RESULT[kind](args) gives
# {name: fp32 shape, or None for an output the launch does not make}, in the order of the returned
# tuple (one name: the returned tensor itself).  The names are the stored roles above.
RESULT: Dict[str, Callable] = {"fir_resample": _fir_result, "mel_spectrogram": _mel_result,
                               "to_flat": _to_flat_result, "to_flat_bwd": _to_flat_bwd_result}

# Read arguments the kernel does not read for some argument combinations (the probe skips them):
# narrow_conv copies the host-packed bf16 image instead of converting `w`, and the tensor-core conv
# GEMM's fp32-output epilogue has no residual (adp_conv_gemm refuses one); f32_conv_gemm, whose
# operands are fp32 too, adds it.
# stem_out_bwd reads the block input only for the SkipAdapter's weight gradient, and stem_in_bwd
# the weight only for dxin; stem_out reads x un-noised only for the loss target.
# attention over a single key (the innermost level of length 1) has softmax identically 1: its
# output is v whatever q and k are, and only the lse rows, when the launch writes them, read q and
# k.  attention_bwd needs no entry: its P = exp(q k * scale - lse) takes lse as an input.
NOT_READ: Dict[str, Callable] = {
    "attention": lambda a: {"q", "k"} if a["k"].shape[1] == 1 and a["lse"] is None else set(),
    "narrow_conv": lambda a: {"w"} if a["w_packed"] is not None else set(),
    "conv_gemm": lambda a: {"residual"} if a["out"].dtype == torch.float32 and a["a"].dtype != torch.float32
    else set(),
    "stem_out_bwd": lambda a: {"x", "append", "noise", "alpha", "beta"} if a["w_adapt"] is None else set(),
    "stem_in_bwd": lambda a: {"w"} if a["dxin"] is None else set(),
    "cond_bwd": lambda a: {"w"} if a["dcond"] is None else set(),     # the weights serve dcond only
    # to_flat_bwd: the spectrogram serves dw only, the weights dspec only
    "to_flat_bwd": lambda a: ({"spec"} if not a["need_dw"] else set()) | ({"w"} if not a["need_dspec"] else set()),
}

CHECKERS: Dict[str, Callable] = {
    "conv_gemm": c_conv_gemm, "gn_silu": c_gn_silu, "gn_stats": c_gn_stats, "ln_film": c_ln_film,
    "attention": c_attention, "skinny_linear": c_skinny_linear, "time_features": c_time_features,
    "silu_bf16": c_silu_bf16, "stem_in": c_stem_in, "stem_out": c_stem_out, "narrow_conv": c_narrow_conv,
    "sampler_step": c_sampler_step, "step_select": c_step_select, "step_advance": c_step_advance,
    "wgrad": c_wgrad, "gn_silu_bwd": c_gn_silu_bwd, "gn_bwd_apply": c_gn_bwd_apply, "ln_film_bwd": c_ln_film_bwd,
    "colsum": c_colsum, "skip_gate": c_skip_gate, "skip_gate_bwd": c_skip_gate_bwd, "cond_bwd": c_cond_bwd,
    "narrow_conv_bwd": c_narrow_conv_bwd, "stem_out_bwd": c_stem_out_bwd, "stem_in_bwd": c_stem_in_bwd,
    "attention_bwd": c_attention_bwd, "ln_fold_bwd": c_ln_fold_bwd, "fir_resample": c_fir_resample,
    "mel_spectrogram": c_mel_spectrogram, "to_flat": c_to_flat, "to_flat_bwd": c_to_flat_bwd,
    "inpaint_blend": c_inpaint_blend, "arv_step": c_arv_step,
}


# ------------------------------------------------------------------------------ harness
def _tensors(v):
    if isinstance(v, torch.Tensor):
        yield v
    elif isinstance(v, (tuple, list)):
        for x in v:
            yield from _tensors(x)


def _key(t):
    return t.untyped_storage().data_ptr()


def _on(storage, t):
    """t's view over another storage of the same layout (its snapshot)."""
    return torch.empty(0, dtype=t.dtype, device=t.device).set_(storage, t.storage_offset(), t.shape, t.stride())


def _bits(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _flat(storage, dtype, device):
    n = storage.nbytes() // torch.empty(0, dtype=dtype).element_size()
    return torch.empty(0, dtype=dtype, device=device).set_(storage, 0, (n,), (1,))


def _where(idx, shape):
    out = []
    for s in reversed(shape):
        out.append(idx % s)
        idx //= s
    return tuple(reversed(out))


class Record:
    def __init__(self):
        self.count, self.worst, self.label, self.where = 0, 0.0, "", ""


# ---------------------------------------------------------------------------- guard bands
GUARD_BYTES = 2 << 20          # each guard: twice the largest tile store (256 rows x 2048 bf16 columns)
GUARD_ALIGN = 4096             # a copy keeps its storage's address modulo this (TMA and vector alignment)
POISON_FLOAT = 0x7F            # bf16 / fp32 3.39e38, fp64 ~1.4e306: finite, so fmaxf and compares keep it
POISON_INT = 0x00              # an index, address or loop bound read from a guard stays in range
_INT_OF_SIZE = {1: torch.int8, 2: torch.int16, 4: torch.int32, 8: torch.int64}

# Kinds whose contract is to read bytes outside the views they are passed: the guard check would
# poison those bytes.  READS_OUTSIDE_VIEW[kind](args) -> names of such arguments, left in place.
READS_OUTSIDE_VIEW: Dict[str, Callable] = {}


def _extent(t):
    """[first, last + 1) byte of t's view within its storage."""
    es = t.element_size()
    lo = t.storage_offset() * es
    if t.numel() == 0:
        return lo, lo
    return lo, lo + (sum((s - 1) * st for s, st in zip(t.shape, t.stride())) + 1) * es


def _row_bytes(t):
    return (t.stride(-2) if t.dim() >= 2 else max(t.numel(), 1)) * t.element_size()


class _Guarded:
    """One storage's copy placed as [front guard | copy | back guard] in a fresh buffer, at the
    storage's address modulo GUARD_ALIGN; the guards and every byte of the copy outside the viewed
    bytes (`mask`) hold the poison byte."""

    def __init__(self, nbytes, device, residue, poison):
        self.n, self.poison = nbytes, poison
        self.buf = torch.full((2 * GUARD_BYTES + GUARD_ALIGN + nbytes,), poison, dtype=torch.uint8, device=device)
        self.off = GUARD_BYTES + (residue - (self.buf.data_ptr() + GUARD_BYTES)) % GUARD_ALIGN
        self.copy = self.buf[self.off:self.off + nbytes]
        self.mask = torch.zeros(nbytes, dtype=torch.uint8, device=device)
        self.views: List[Tuple[str, torch.Tensor]] = []          # (argument, relocated view)

    def view_of(self, name, t):
        """t's view (same storage offset, shape and strides) over the copy; its bytes marked viewed."""
        es = t.element_size()
        assert self.off % es == 0
        if t.numel():
            _flat(self.mask.untyped_storage(), _INT_OF_SIZE[es], t.device).as_strided(
                t.shape, t.stride(), t.storage_offset()).fill_(-1)
        r = torch.empty(0, dtype=t.dtype, device=t.device).set_(
            self.buf.untyped_storage(), self.off // es + t.storage_offset(), t.shape, t.stride())
        self.views.append((name, r))
        return r

    def fill_from(self, storage):
        """The viewed bytes from `storage`, poison elsewhere."""
        src = _flat(storage, torch.uint8, self.buf.device)
        for lo in range(0, self.n, SIDE_CHUNK):
            c, m = self.copy[lo:lo + SIDE_CHUNK], self.mask[lo:lo + SIDE_CHUNK]
            c.copy_(torch.where(m.bool(), src[lo:lo + SIDE_CHUNK], self.poison))

    def copy_back(self, storage):
        """The viewed bytes of the copy into `storage`; its other bytes stay as they are."""
        dst = _flat(storage, torch.uint8, self.buf.device)
        for lo in range(0, self.n, SIDE_CHUNK):
            d, m = dst[lo:lo + SIDE_CHUNK], self.mask[lo:lo + SIDE_CHUNK]
            d.copy_(torch.where(m.bool(), self.copy[lo:lo + SIDE_CHUNK], d))

    def first_damage(self):
        """(region, buffer index) of the poisoned byte nearest the copy that changed, or None."""
        front = (self.buf[:self.off] != self.poison).nonzero()
        if front.numel():
            return "before the start", int(front[-1, 0])
        for lo in range(0, self.n, SIDE_CHUNK):
            bad = ((self.copy[lo:lo + SIDE_CHUNK] != self.poison) & (self.mask[lo:lo + SIDE_CHUNK] == 0)).nonzero()
            if bad.numel():
                return "in an unviewed gap", self.off + lo + int(bad[0, 0])
        back = (self.buf[self.off + self.n:] != self.poison).nonzero()
        if back.numel():
            return "past the end", self.off + self.n + int(back[0, 0])
        return None

    def describe(self, region, i):
        """Which argument view the damaged byte i lies nearest, and how far from it."""
        rel = i - self.off
        best = None
        for name, v in self.views:
            lo, hi = (e - self.off for e in _extent(v))
            d = lo - rel if rel < lo else (rel - hi + 1 if rel >= hi else 0)
            if best is None or d < best[0]:
                best = (d, name, v, "before" if rel < lo else "past the end of")
        d, name, v, side = best
        row = _row_bytes(v)
        where = (f"{self.off - i} bytes before the start of the storage" if region == "before the start" else
                 f"{rel - self.n + 1} bytes past the end of the storage" if region == "past the end" else
                 f"storage byte {rel}")
        return (f"`{name}` damaged {region}: {where}, {d} bytes ({d / row:.3g} rows of {row} bytes) {side} "
                f"its view {tuple(v.shape)}, byte {int(self.buf[i]):#04x} where poison {self.poison:#04x}")


class Guards:
    """The storages of one launch (or one direct call) relocated between poisoned guard bands.

    relocate(args) gives the arguments as views of the copies (memoised by id(): one object stays
    one object, views of one storage stay views of one copy); alloc() makes a tensor between guards
    for a kernel to write (`torch_proxy()` hands these out as torch.empty / empty_like /
    zeros_like); check() reports the first poisoned byte that changed; copy_back() returns the
    viewed bytes to the original storages."""

    def __init__(self):
        self.items: Dict[int, Tuple[_Guarded, object]] = {}     # storage key -> (copy, original storage)
        self.made: List[_Guarded] = []

    def relocate(self, args: Dict[str, object], keep=frozenset()) -> Dict[str, object]:
        """args with every tensor (nested tuples included) but those of the arguments in `keep`
        replaced by its view of the relocated copy of its storage."""
        owners: Dict[int, List[Tuple[str, torch.Tensor]]] = {}
        for n, v in args.items():
            for t in _tensors([v] if n not in keep else []):
                owners.setdefault(_key(t), []).append((n, t))
        for k, ts in owners.items():
            st = ts[0][1].untyped_storage()
            poison = POISON_FLOAT if all(t.is_floating_point() for _, t in ts) else POISON_INT
            self.items[k] = (_Guarded(st.nbytes(), ts[0][1].device, st.data_ptr() % GUARD_ALIGN, poison), st)
        memo: Dict[int, torch.Tensor] = {}

        def sub(n, v):
            if n in keep:
                return v
            if isinstance(v, torch.Tensor):
                if id(v) not in memo:
                    memo[id(v)] = self.items[_key(v)][0].view_of(n, v)
                return memo[id(v)]
            if isinstance(v, (tuple, list)):
                return type(v)(sub(n, x) for x in v)
            return v
        out = {n: sub(n, v) for n, v in args.items()}
        for g, st in self.items.values():
            g.fill_from(st)
        return out

    def alloc(self, shape, dtype, device, name="result", zero=False):
        shape = tuple(shape)
        t = torch.empty(shape, dtype=dtype, device="meta")
        g = _Guarded(t.numel() * t.element_size(), device, 0,
                     POISON_FLOAT if t.is_floating_point() else POISON_INT)
        r = g.view_of(name, torch.empty(shape, dtype=dtype, device=device))
        if zero:
            r.zero_()
        self.made.append(g)
        return r

    def torch_proxy(self):
        return _TorchProxy(self)

    def name(self, t, name):
        """Names the allocated tensor t (as its launch's output) in the check's messages."""
        for g in self.made:
            g.views = [(name if v.data_ptr() == t.data_ptr() else n, v) for n, v in g.views]

    def check(self, fail):
        for g in [g for g, _ in self.items.values()] + self.made:
            bad = g.first_damage()
            if bad is not None:
                fail(g.describe(*bad))

    def copy_back(self):
        for g, st in self.items.values():
            g.copy_back(st)


class _TorchProxy:
    """`torch` for a module whose calls allocate the outputs of a guarded launch: empty, empty_like
    and zeros_like give tensors between guard bands, every other name is torch's."""

    def __init__(self, guards):
        self._guards = guards

    def empty(self, *size, dtype=None, device=None):
        if len(size) == 1 and isinstance(size[0], (tuple, list, torch.Size)):
            size = size[0]
        return self._guards.alloc(size, dtype or torch.get_default_dtype(), device or "cpu")

    def empty_like(self, t):
        return self._guards.alloc(t.shape, t.dtype, t.device)

    def zeros_like(self, t):
        return self._guards.alloc(t.shape, t.dtype, t.device, zero=True)

    def __getattr__(self, name):
        return getattr(torch, name)


class Shadow:
    """Context manager: every ops launch of a CHECKERS kind is checked (see the module docstring).

    fake=True: no kernel runs; each launch writes its restatement rounded to the output dtype
    (statistics: those of the written output).  probe=True: the first launch of each kind and set
    of passed tensors also runs _probe.  mutate=(kind, fn): after the first launch of that
    kind where fn(args, outs, snapshot) applies (does not return False), fn damages what it
    wrote (the checker's self-test).  guard=True: each launch runs on copies of its storages
    between poisoned guard bands (Guards; see the module docstring), and mutate's fn sees those."""

    def __init__(self, fake: bool = False, mutate=None, probe: bool = False, guard: bool = False):
        self.fake, self.mutate, self.probe, self.guard = fake, mutate, probe, guard
        self.probed = set()
        self.records: Dict[str, Record] = {}
        self.n_launch, self.n_checked, self.n_guarded = 0, 0, 0
        self.labels = set()                      # trace labels of the launches seen (shapes included)
        self.symbols = set()                     # C entry points the checked launches called (ops._launch)
        self.known: Dict[int, torch.Tensor] = {}
        self._depth = 0                          # > 0 inside a checked launch (a nested launch: see _wrap)

    # ---- install
    def __enter__(self):
        self._saved = {}
        for name in launching_functions():
            self._saved[name] = getattr(ops, name)
            setattr(ops, name, self._wrap(name, self._saved[name]))
        return self

    def __exit__(self, *exc):
        for name, fn in self._saved.items():
            setattr(ops, name, fn)
        self.known.clear()

    def lookup(self, ptr, n, dtype):
        """n elements of `dtype` at device address ptr, from a storage seen in an earlier launch."""
        for t in self.known.values():
            st = t.untyped_storage()
            base = st.data_ptr()
            if base <= ptr and ptr + n * 4 <= base + st.nbytes():
                return _flat(st, dtype, t.device)[(ptr - base) // 4:][:n]
        raise CheckError(f"step_select: no known tensor holds address {ptr:#x}")

    # ---- one launch
    def _wrap(self, name, real):
        sig = inspect.signature(real)

        def launch(*args, **kwargs):
            if self._depth:           # a launch made by a checked launch's own ops call: part of it
                return real(*args, **kwargs)
            if name not in CHECKERS:
                raise CheckError(f"launch {self.n_launch}: {name} has no checker ({UNCHECKED.get(name, '?')})")
            b = sig.bind(*args, **kwargs)
            b.apply_defaults()
            post = dict(b.arguments)
            idx = self.n_launch
            self.n_launch += 1
            label0 = self._label(name, post)
            for t in _tensors(list(post.values())):
                self.known[_key(t)] = t
            if post[next(iter(post))].is_cuda:
                torch.cuda.synchronize()
            snaps = {}
            for t in _tensors(list(post.values())):
                k = _key(t)
                if k not in snaps:
                    snaps[k] = t.untyped_storage().clone()

            def snap(v):
                if isinstance(v, torch.Tensor):
                    return _on(snaps[_key(v)], v)
                if isinstance(v, tuple):
                    return tuple(snap(x) for x in v)
                return v
            pre = {k: snap(v) for k, v in post.items()}
            outs = CHECKERS[name](pre, self)
            made = RESULT[name](pre) if name in RESULT else {}
            self._check_roles(idx, name, outs, post, made)
            variant = (name, frozenset(n for n, v in post.items() if list(_tensors([v]))) |
                       frozenset(n for n, s in made.items() if s is not None))
            if self.probe and variant not in self.probed:      # once per set of passed / returned tensors
                self._probe(idx, name, outs, pre)
                self.probed.add(variant)
            guards = Guards() if self.guard else None
            run = post                           # the arguments the launch runs on
            if guards is not None:
                run = guards.relocate(post, READS_OUTSIDE_VIEW[name](pre) if name in READS_OUTSIDE_VIEW else ())
            if self.fake:
                dev = next(_tensors(list(post.values()))).device
                for n, shape in made.items():
                    run[n] = None if shape is None else \
                        guards.alloc(shape, torch.float32, dev, n) if guards is not None else \
                        torch.empty(shape, dtype=torch.float32, device=dev)
                result = tuple(run[n] for n in made) if len(made) > 1 else \
                    (run[next(iter(made))] if made else None)
                self._fake_write(outs, pre, run)
                label = label0
            else:
                self._depth += 1
                try:
                    if guards is None:
                        with ops.trace() as tr:
                            result = real(*args, **kwargs)
                    else:
                        call = inspect.BoundArguments(sig, {n: run[n] for n in b.arguments})
                        saved = ops.torch
                        if name in RESULT:           # the outputs ops allocates go between guards too
                            ops.torch = guards.torch_proxy()
                        try:
                            with ops.trace() as tr:
                                result = real(*call.args, **call.kwargs)
                        finally:
                            ops.torch = saved
                finally:
                    self._depth -= 1
                # the first record is the launch itself; a nested one (gn_stats) follows it
                label = tr.records[0]["name"] if tr.records else label0
                nested = [r["symbol"] for r in tr.records[1:]]
                if nested and (nested != ["adp_f32_gn_stats"] or name not in NESTED_STATS
                               or post[NESTED_STATS[name]] is None):
                    self._fail(idx, name, label, f"launches {nested} inside the ops call: only the fp32 "
                                                 f"statistics pass of {sorted(NESTED_STATS)} is checked as part of "
                                                 f"its caller")
                self.symbols.update(r["symbol"] for r in tr.records)
                if post[next(iter(post))].is_cuda:
                    torch.cuda.synchronize()
                run.update(zip(made, result if len(made) > 1 else (result,)))
            if self.mutate is not None and self.mutate[0] == name:
                if self.mutate[1](run, outs, pre) is not False:       # False: not applicable here
                    self.mutate = None
            self.labels.add(label)
            if guards is not None:
                result = self._unguard(idx, name, label, guards, post, run, made, result)
            self._check(idx, name, label, outs, pre, post, snaps)
            snaps.clear()            # `snap` refers to itself: without this the snapshots wait for the cycle collector
            self.n_checked += 1
            return result
        return launch

    def _unguard(self, idx, name, label, guards, post, run, made, result):
        """Guard check of a relocated launch; then its viewed bytes go back to the original
        storages, the tensors it allocated are handed back as plain copies, and `result` (the
        launch's return value) refers to those and to the original arguments."""
        for n in made:
            if run[n] is not None:
                guards.name(run[n], n)
        guards.check(lambda msg: self._fail(idx, name, label, f"guard: {msg}"))
        guards.copy_back()
        back = {}
        for n, v in post.items():
            for o, r in zip(_tensors([v]), _tensors([run[n]])):
                back[id(r)] = o
        for n in made:
            post[n] = None if run[n] is None else run[n].clone()
            if run[n] is not None:
                back[id(run[n])] = post[n]
        self.n_guarded += 1
        if isinstance(result, tuple):
            return tuple(back.get(id(r), r) if r is not None else None for r in result)
        return back.get(id(result), result) if result is not None else None

    def _check_roles(self, idx, name, outs, post, made):
        """The checker's outputs are exactly the output arguments the launch was given and the
        tensors it returns (`made`: RESULT)."""
        _, stored, accumulated = ARGS[name]
        got = {(o.of, o.acc) for o in outs}
        want = {(n, False) for n in stored if post.get(n) is not None or made.get(n) is not None} | \
            {(n, True) for n in accumulated if post.get(n) is not None}
        if got != want:
            raise CheckError(f"launch {idx}: {name}: checker outputs {sorted(got)}, declared {sorted(want)}")

    def _probe(self, idx, name, outs, pre):
        """Every tensor the launch reads must move the reference when it changes."""
        def values(args, os_):
            return [stats_of(o.src(args), o.groups) if isinstance(o, Stat)
                    else (o.ref(args)[0] if callable(o.ref) else o.ref) for o in os_]
        base = values(pre, outs)
        skip = NOT_READ[name](pre) if name in NOT_READ else set()
        for n in sorted(ARGS[name][0] - skip):
            v = pre.get(n)
            ts = list(_tensors([v]))
            if not ts or not all(t.is_floating_point() for t in ts):
                continue                          # absent, or integer control words (step_select)

            def moved(t):
                return t.clone().mul_(1.25).add_(0.125)
            args = dict(pre)
            args[n] = moved(v) if isinstance(v, torch.Tensor) else \
                tuple(moved(x) if isinstance(x, torch.Tensor) else x for x in v)
            after = values(args, CHECKERS[name](args, self))
            if all(torch.equal(a, b) for a, b in zip(base, after)):
                raise CheckError(f"launch {idx}: {name}: the reference does not depend on `{n}`")

    @staticmethod
    def _label(name, post):
        shapes = [tuple(t.shape) for t, _ in zip(_tensors(list(post.values())), range(2))]
        return f"{name}{shapes}"

    def _fake_write(self, outs, pre, post):
        for o in outs:
            if isinstance(o, Val) or (isinstance(o, Acc) and not callable(o.ref)):
                got = o.view(post)
                ref = o.ref(post)[0] if callable(o.ref) else o.ref
                got.add_(ref.to(got.dtype)) if o.acc else got.copy_(ref.to(got.dtype))
        for o in outs:                       # statistics / sums of the values just written
            if isinstance(o, Stat):
                o.view(post).add_(stats_of(o.src(post), o.groups))
            elif isinstance(o, Acc) and callable(o.ref):
                o.view(post).add_(o.ref(post)[0].to(o.view(post).dtype))

    # ---- comparisons
    def _fail(self, idx, name, label, msg):
        raise CheckError(f"launch {idx} ({label}): {name}: {msg}")

    def _note(self, key, ratio, label, where):
        r = self.records.setdefault(key, Record())
        r.count += 1
        if ratio >= r.worst:
            r.worst, r.label, r.where = ratio, label, where

    def _check(self, idx, name, label, outs, pre, post, snaps):
        for o in outs:
            got = o.view(post)
            key = f"{name}.{o.name}"
            if isinstance(o, Stat):
                self._check_stats(idx, name, label, key, o, got.to(F64) - o.view(pre).to(F64), o.src(post))
                continue
            ref, absr = o.ref(post) if callable(o.ref) else (o.ref, o.absref)
            if o.exact:
                if not torch.equal(_bits(got.contiguous()), _bits(ref.to(got.dtype).contiguous())):
                    self._fail(idx, name, label, f"{o.name} differs from the copy it must make")
                self._note(key, 0.0, label, "")
                continue
            g = got.to(F64)
            if o.chain is not None:                   # an fp32 verification kernel (f32_*)
                bound = F32_REL * ref.abs() + (F32_LAMBDA * math.sqrt(o.chain) * F32_U) * absr
                val = g
                if isinstance(o, Acc):
                    before = o.view(pre).to(F64)
                    val = g - before
                    eps = F64_ACC_EPS if got.dtype == torch.float64 else ACC_EPS
                    bound = bound + eps * (before.abs() + g.abs())
            elif isinstance(o, Acc):                  # the launch's own contribution
                before = o.view(pre).to(F64)
                val = g - before
                if got.dtype == torch.float64:
                    bound = STATS_TOL * absr
                else:                                 # + the rounding of the two fp32 values subtracted
                    bound = FP32_REL * ref.abs() + FP32_TAU * absr + ACC_EPS * (before.abs() + g.abs())
            else:
                val = g
                if got.dtype == torch.bfloat16:
                    bound = BF16_REL * ref.abs() + o.tau * absr
                else:
                    bound = FP32_REL * ref.abs() + FP32_TAU * absr + o.floor
            err = (val - ref).abs()
            ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
            ratio = torch.where(torch.isnan(g), math.inf, ratio)
            if o.keep is not None:                    # positions the launch must not touch: bitwise
                changed = o.keep & (_bits(got) != _bits(o.view(pre)))
                if bool(changed.any()):
                    j = tuple(int(c) for c in changed.nonzero()[0])
                    self._fail(idx, name, label, f"{o.name}{list(j)}: changed outside the written positions, "
                                                 f"got {float(got[j]):.6g}, before {float(o.view(pre)[j]):.6g}")
                ratio = ratio.masked_fill(o.keep, 0.0)
            i = int(ratio.reshape(-1).argmax())
            worst = float(ratio.reshape(-1)[i])
            where = _where(i, tuple(ratio.shape))
            desc = (f"{o.name}{list(where)}: {'added' if o.acc else 'got'} {float(val.reshape(-1)[i]):.6g}, "
                    f"ref {float(ref.reshape(-1)[i]):.6g}, "
                    f"bound {float(bound.reshape(-1)[i]):.3g} (err/bound {worst:.3g})")
            if worst > 1.0:
                self._fail(idx, name, label, desc)
            self._note(key, worst, label, f"{list(where)}")
        self._check_side_effects(idx, name, label, outs, post, snaps)

    def _check_side_effects(self, idx, name, label, outs, post, snaps):
        """Read-only storages are bitwise unchanged, written ones outside their written views: the
        written views are copied into the snapshot, which must then equal the live storage byte for
        byte (in chunks: the gradient arena and the activation arena are one storage each)."""
        written = {}
        for o in outs:
            v = o.view(post)
            written.setdefault(_key(v), []).append(v)
        for k, st in snaps.items():
            t = next(t for t in _tensors(list(post.values())) if _key(t) == k)
            for v in written.get(k, ()):
                _on(st, v).copy_(v)
            before, after = _flat(st, torch.uint8, t.device), _flat(t.untyped_storage(), torch.uint8, t.device)
            for lo in range(0, before.numel(), SIDE_CHUNK):
                bb, aa = before[lo:lo + SIDE_CHUNK], after[lo:lo + SIDE_CHUNK]
                if torch.equal(bb, aa):
                    continue
                if k not in written:
                    argn = next(n for n, v in post.items() if any(_key(x) == k for x in _tensors([v])))
                    self._fail(idx, name, label, f"read-only argument `{argn}` was modified")
                i = lo + int((bb != aa).nonzero()[0, 0])
                self._fail(idx, name, label, f"wrote byte {i} of a storage outside its output view")

    def _check_stats(self, idx, name, label, key, o, got, src):
        B, T, C = src.shape
        G = o.groups
        ref = stats_of(src, G)
        yg = src.to(F64).reshape(B, T, G, C // G)
        scale = torch.stack([yg.abs().sum(dim=(1, 3)), (yg * yg).sum(dim=(1, 3))], dim=-1)
        err = (got - ref).abs()
        bound = STATS_TOL * scale
        ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
        i = int(ratio.reshape(-1).argmax())
        worst = float(ratio.reshape(-1)[i])
        where = list(_where(i, tuple(ratio.shape)))
        if worst > 1.0:
            self._fail(idx, name, label, f"{o.name}{where}: got {float(got.reshape(-1)[i]):.10g}, "
                                         f"ref {float(ref.reshape(-1)[i]):.10g} (err/bound {worst:.3g})")
        self._note(key, worst, label, f"{where}")
        # the variance GroupNorm derives from the slots, against a two-pass fp64 variance
        n = float(T * (C // G))
        mean = got[..., 0] / n
        var = got[..., 1] / n - mean * mean
        mu = yg.mean(dim=(1, 3), keepdim=True)
        var2 = ((yg - mu) ** 2).mean(dim=(1, 3))
        vr = (var - var2).abs() / (VAR_TOL * (var2 + GN_EPS))
        j = int(vr.reshape(-1).argmax())
        vworst = float(vr.reshape(-1)[j])
        vwhere = list(_where(j, tuple(vr.shape)))
        if vworst > 1.0:
            self._fail(idx, name, label, f"{o.name} variance {vwhere}: E[x^2]-mean^2 = {float(var.reshape(-1)[j]):.8g}, "
                                         f"two-pass {float(var2.reshape(-1)[j]):.8g} (err/bound {vworst:.3g})")
        self._note(key + ".var", vworst, label, f"{vwhere}")
        # not bounded: the relative error of the variance itself, large only for near-constant groups
        rel = ((var - var2).abs() / var2.clamp_min(1e-300)).reshape(-1)
        j = int(rel.argmax())
        self._note(key + ".var_rel", float(rel[j]), label, f"{list(_where(j, tuple(var2.shape)))} "
                                                           f"var {float(var2.reshape(-1)[j]):.3g}")

    def table(self) -> str:
        lines = [f"{'kind.output':28s} {'count':>6s} {'worst err/bound':>16s}  label (where)"]
        for k in sorted(self.records):
            r = self.records[k]
            lines.append(f"{k:28s} {r.count:6d} {r.worst:16.4f}  {r.label} {r.where}")
        lines.append(f"launches {self.n_launch}, checked {self.n_checked}" +
                     (f", guarded {self.n_guarded}" if self.guard else ""))
        return "\n".join(lines)


# ---------------------------------------------------------------------------- mutations
def m_scale_largest(post, outs, pre):
    """The largest-|ref| element of the first stored output scaled by 1 + 2^-5."""
    o = next((o for o in outs if isinstance(o, Val)), None)
    if o is None:
        return False
    ref = o.ref(post)[0] if callable(o.ref) else o.ref
    g = o.view(post)
    i = int(ref.abs().to(F64).reshape(-1).argmax())
    idx = _where(i, tuple(g.shape))
    if g.is_floating_point():
        g[idx] = (g[idx].to(F64) * (1 + 2 ** -5)).to(g.dtype)
    else:                                      # the step counter
        g[idx] += 1


def m_stale_tile(post, outs, pre):
    """The last row tile of the last batch element of the first [B, T, C] output left unwritten."""
    o = next((o for o in outs if isinstance(o, Val) and not o.exact and o.view(post).dim() == 3), None)
    if o is None:
        return False
    g, old = o.view(post), o.view(pre)
    g[-1, -ROW_TILE:] = old[-1, -ROW_TILE:]


def m_stats_slot(post, outs, pre):
    """One statistics slot scaled by 1 + 1e-3."""
    o = next((o for o in outs if isinstance(o, Stat)), None)
    if o is None:
        return False
    g = o.view(post)
    g[-1, -1, 1] *= 1 + 1e-3


def _first_acc(outs, post, pre):
    for o in outs:
        if isinstance(o, Acc) and bool((o.view(pre) != 0).any()):
            return o
    return None


def m_acc_stored(post, outs, pre):
    """An accumulator with a non-zero value before the launch stored to instead of added to
    (what wgrad's single-split configuration once did)."""
    o = _first_acc(outs, post, pre)
    if o is None:
        return False
    o.view(post).sub_(o.view(pre))


def m_acc_lost_split(post, outs, pre):
    """The largest element of an accumulator's contribution short of 2^-5 of itself (a lost split)."""
    o = next((o for o in outs if isinstance(o, Acc)), None)
    if o is None:
        return False
    g, old = o.view(post), o.view(pre)
    ref = o.ref(post)[0] if callable(o.ref) else o.ref
    idx = _where(int(ref.abs().reshape(-1).argmax()), tuple(g.shape))
    g[idx] = (old[idx].to(F64) + (g[idx].to(F64) - old[idx].to(F64)) * (1 - 2 ** -5)).to(g.dtype)


def m_outside_view(post, outs, pre):
    """One element of a written tensor's storage outside the written views changed."""
    for o in outs:
        v = o.view(post)
        flat = _flat(v.untyped_storage(), v.dtype, v.device)
        mask = torch.zeros(flat.shape, dtype=torch.bool, device=v.device)
        for w in (o2.view(post) for o2 in outs):       # every output the launch writes into this storage
            if _key(w) == _key(v) and w.dtype == v.dtype:
                mask.as_strided(w.shape, w.stride(), w.storage_offset()).fill_(True)
        free = (~mask).nonzero()
        if free.numel():
            i = int(free[-1, 0])
            flat[i] += 1
            return None
    return False


def m_readonly(post, outs, pre):
    """One element of a read-only input changed."""
    written = {_key(o.view(post)) for o in outs}
    for v in post.values():
        for t in _tensors([v]):
            if _key(t) not in written and t.numel():
                t[(0,) * t.dim()] += 1
                return None
    return False


def m_scale_largest_f32(post, outs, pre):
    """The largest-|ref| element of the first stored output scaled by 1 + 2^-12 (an fp32 output
    one bf16-class rounding off, which the fp32 bound must see)."""
    o = next((o for o in outs if isinstance(o, (Val, Acc)) and not o.exact), None)
    if o is None:
        return False
    ref = o.ref(post)[0] if callable(o.ref) else o.ref
    g = o.view(post)
    idx = _where(int(ref.abs().to(F64).reshape(-1).argmax()), tuple(g.shape))
    if isinstance(o, Acc):                     # the launch's contribution, not the value before it
        old = o.view(pre)[idx].to(F64)
        g[idx] = (old + (g[idx].to(F64) - old) * (1 + 2 ** -12)).to(g.dtype)
    else:
        g[idx] = (g[idx].to(F64) * (1 + 2 ** -12)).to(g.dtype)


def _alternative(kind, doc, **option):
    """A mutation that writes an alternative fp64 restatement of `kind` (CHECKERS[kind] with
    `option`) over the outputs, rounded to their dtype."""
    def mutate(post, outs, pre):
        for o in CHECKERS[kind](pre, None, **option):
            got = o.view(post)
            got.copy_((o.ref(post)[0] if callable(o.ref) else o.ref).to(got.dtype))
    mutate.__doc__ = doc
    return mutate


def m_unmasked_write(post, outs, pre):
    """inpaint_blend: the blend also written at one position outside the mask."""
    keep = next((o.keep for o in outs if getattr(o, "keep", None) is not None), None)
    if keep is None or not bool(keep.any()):
        return False
    j = tuple(int(c) for c in keep.nonzero()[0])
    a = pre["ab"].to(F64)
    post["x"][j] = float(a[2] * pre["source"][j].double() + a[3] * pre["noise"][j].double())


def m_v_chan_stride(post, outs, pre):
    """arv_step: v read with chan's batch stride (C+1) T instead of its own C T."""
    B, C1, T = pre["chan"].shape
    if B < 2 or C1 < 3:
        return False                  # one batch row, or one channel: the two strides read the same
    _alternative("arv_step", "", v_batch_stride=C1 * T)(post, outs, pre)


MUTATIONS = {"scale_largest": m_scale_largest, "stale_tile": m_stale_tile, "stats_slot": m_stats_slot,
             "outside_view": m_outside_view, "readonly": m_readonly, "acc_stored": m_acc_stored,
             "acc_lost_split": m_acc_lost_split, "scale_largest_f32": m_scale_largest_f32,
             # kind-specific: an alternative operation written over the output
             "mel_symmetric_pad": _alternative(
                 "mel_spectrogram", "The edge frames cut from a symmetric pad (edge sample repeated).",
                 symmetric=True),
             "mel_pairs_swapped": _alternative(
                 "mel_spectrogram", "The two frames of each FFT pair exchanged.", swap_pairs=True),
             "to_flat_shifted": _alternative("to_flat", "The output one sample late.", shift=1),
             "to_flat_dw_lost_row": _alternative(
                 "to_flat_bwd", "dw without the last batch row's contribution (a lost atomic).", dw_rows=-1),
             "blend_start_level": _alternative(
                 "inpaint_blend", "The known region noised to the step's starting level (ab[0:2]).", level=0),
             "blend_unmasked_write": m_unmasked_write,
             "arv_sigma_kept": _alternative("arv_step", "The sigma channel not advanced.", advance_sigma=False),
             "arv_v_chan_stride": m_v_chan_stride}
