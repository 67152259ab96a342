"""The training half of the per-launch checker (tests/launch_check.py), without a GPU.

  * every training launch kind, the vocoder front-end and the VInpainter / ARVSampler steps, with and
    without their optional arguments, as one small direct launch on fake kernels with probes: each
    read argument must move the restatement, and the declared roles must be exactly the outputs the
    checker returns;
  * the restatements against float64 autograd of the forward operation they are the backward of
    (written here from the operation's definition with plain tensor operations), the front-end's
    against its float64 modules and the sampler steps' against the reference's formulas;
  * mutations: the accumulator stored instead of added, a lost share of the largest contribution, a
    scaled element, a stale tile, a write outside the view, a modified input -- each must be caught
    on every kind it applies to, into accumulators that are non-zero before the launch -- and, for
    the front-end and sampler steps, alternative operations written over the output.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import launch_check as lc
from audio_diffusion_pytorch_b200 import _lib, ops

BF, F64 = torch.bfloat16, torch.float64
B, T, C, G = 2, 320, 32, 4


@pytest.fixture
def cpu_launches(monkeypatch):
    monkeypatch.setattr(ops, "device_check", lambda: None)

    def no_library():
        raise AssertionError("a launch reached the CUDA library")
    monkeypatch.setattr(_lib, "lib", no_library)


class Rand:
    def __init__(self, seed):
        self.g = torch.Generator().manual_seed(seed)

    def bf(self, *shape):
        return torch.randn(*shape, generator=self.g).to(BF)

    def f32(self, *shape, scale=1.0):
        return torch.randn(*shape, generator=self.g) * scale

    def acc(self, *shape, dtype=torch.float32):
        """An accumulator that already holds something."""
        return torch.randn(*shape, generator=self.g).to(dtype)


def _stats(x, groups):
    return lc.stats_of(x, groups)


# ------------------------------------------------------------------------ direct launches
def _wgrad(r, variant):
    g, x = r.bf(B, T, 48), r.bf(B, T, 40)
    if variant == "taps3":
        return lambda: ops.wgrad(g, x, r.acc(3, 48, 40), n=48, k=40, off=-1, ntaps=3)
    if variant == "views":      # column windows of wider rows, into a column window of a wider dw
        dw = r.acc(16, 64)
        return lambda: ops.wgrad(g, x, dw[:, 24:], n=16, k=24, off=1, g_col0=32, x_col0=8)
    return lambda: ops.wgrad(g, x, r.acc(48, 40), n=48, k=40)


def _gn_silu_bwd(r, variant):
    x = r.bf(B, T, C) + 0.5
    return lambda: ops.gn_silu_bwd(r.bf(B, T, C), x, _stats(x, G), r.f32(C), r.f32(C), torch.empty(B, T, C, dtype=BF),
                                   r.acc(C), r.acc(C), r.acc(B, G, 2, dtype=F64), G)


def _gn_bwd_apply(r, variant):
    x = r.bf(B, T, C) + 0.5
    full = variant == "dres_colsum"
    return lambda: ops.gn_bwd_apply(r.bf(B, T, C), x, _stats(x, G), r.acc(B, G, 2, dtype=F64) * 30,
                                    torch.empty(B, T, C, dtype=BF), G, dres=r.bf(B, T, C) if full else None,
                                    colsum=r.acc(C) if full else None)


def _ln_film_bwd(r, variant):
    x = r.bf(B, T, C) + 0.5
    if variant == "plain":      # the affine-free attention pre-norm with the residual's gradient
        return lambda: ops.ln_film_bwd(r.bf(B, T, C), x, None, 0, torch.empty(B, T, C, dtype=BF), dres=r.bf(B, T, C))
    ss, dss = r.f32(B, 96, scale=0.3), r.acc(B, 96)
    return lambda: ops.ln_film_bwd(r.bf(B, T, C), x, ss[:, 16:], 96, torch.empty(B, T, C, dtype=BF),
                                   dss=dss[:, 16:], dss_stride=96, colsum=r.acc(C))


def _colsum(r, variant):
    gate = r.f32(B, 2 * C) if variant == "gate" else None
    return lambda: ops.colsum(r.bf(B, T, C), r.acc(C), gate)


def _skip_gate(r, variant):
    st = r.acc(B, G, 2, dtype=F64) if variant == "stats" else None
    return lambda: ops.skip_gate(r.bf(B, T, C), r.bf(B, T, C), r.f32(B, 2 * C), torch.empty(B, T, C, dtype=BF), st, G)


def _skip_gate_bwd(r, variant):
    return lambda: ops.skip_gate_bwd(r.bf(B, T, C), r.bf(B, T, C), r.f32(B, 2 * C), torch.empty(B, T, C, dtype=BF),
                                     r.acc(B, 2 * C))


def _cond_bwd(r, variant):
    N, K = 70, 24
    dcond = r.acc(B, K) if variant == "dcond" else None
    return lambda: ops.cond_bwd(r.f32(B, 72), r.f32(B, K), r.bf(80, K), torch.zeros(80, K), torch.zeros(80), dcond, N)


def _narrow_conv_bwd(r, variant):
    x = r.bf(B, T, 8) + 0.5
    return lambda: ops.narrow_conv_bwd(r.bf(B, T, 8), x, _stats(x, 2), r.f32(8), r.f32(8), r.f32(8, 8, 3, scale=0.3),
                                       torch.empty(B, T, 8, dtype=BF), r.acc(8), r.acc(8),
                                       r.acc(B, 2, 2, dtype=F64), r.acc(8, 8, 3), r.acc(8), 2)


def _stem_out_bwd(r, variant):
    f, Tf, co, cx, ca = 4, 256, 2, 2, 1
    kw = {}
    if variant == "adapter":    # loss-mode noising, appended channels, SkipAdapter, dxin
        kw = dict(gscale=torch.tensor([0.7]), append=r.f32(B, ca, Tf), noise=r.f32(B, cx, Tf),
                  alpha=torch.tensor([0.8, 0.6]), beta=torch.tensor([0.6, 0.8]), w_adapt=r.f32(co, cx + ca),
                  dw_adapt=r.acc(co, cx + ca), db_adapt=r.acc(co), dxin=torch.empty(B, cx + ca, Tf))
    elif variant == "dxin":     # identity skip into a wider block input
        kw = dict(append=r.f32(B, ca, Tf), dxin=torch.empty(B, cx + ca, Tf))
    return lambda: ops.stem_out_bwd(r.f32(B, co, Tf), r.bf(B, Tf // f, 8), r.f32(B, cx, Tf), r.f32(co, 8, 3), r.f32(co),
                                    r.f32(B, 4), f, torch.empty(B, Tf // f, 8, dtype=BF), r.acc(co, 8, 3), r.acc(co),
                                    r.acc(B, 4), **kw)


def _stem_in_bwd(r, variant):
    f, Tf, cx, ca, c0 = 4, 256, 2, 1, 8
    kw = {}
    if variant == "dxin":
        kw = dict(append=r.f32(B, ca, Tf), noise=r.f32(B, cx, Tf), alpha=torch.tensor([0.8, 0.6]),
                  beta=torch.tensor([0.6, 0.8]), w=r.f32(c0, cx + ca, f), dxin=r.acc(B, cx + ca, Tf))
    cin = cx + (ca if kw else 0)
    return lambda: ops.stem_in_bwd(r.bf(B, Tf // f, c0), r.f32(B, cx, Tf), r.acc(c0, cin, f), r.acc(c0), f, **kw)


def _attention_bwd(r, variant):
    H, D = 2, 32
    Tq, Tk = (96, 40) if variant == "cross" else (96, 96)
    mid = H * D
    q, kv = r.bf(B, Tq, mid + 16), r.bf(B, Tk, 2 * mid)
    k, v = kv[..., :mid], kv[..., mid:]
    S = torch.einsum("bqhd,bkhd->bhqk", q[..., :mid].double().reshape(B, Tq, H, D),
                     k.double().reshape(B, Tk, H, D)) * D ** -0.5
    lse = torch.logsumexp(S, -1).float()
    dqkv = torch.empty(B, Tq, 3 * mid, dtype=BF) if variant == "self" else None
    dq = dqkv[..., :mid] if dqkv is not None else torch.empty(B, Tq, mid, dtype=BF)
    dkv = torch.empty(B, Tk, 2 * mid, dtype=BF)
    dk, dv = (dqkv[..., mid:2 * mid], dqkv[..., 2 * mid:]) if dqkv is not None else (dkv[..., :mid], dkv[..., mid:])
    return lambda: ops.attention_bwd(q[..., :mid], k, v, r.bf(B, Tq, mid), r.bf(B, Tq, mid), lse,
                                     torch.zeros(2 * B * H * Tq), dq, dk, dv, H, D ** -0.5, head_dim=D)


def _ln_fold_bwd(r, variant):
    N, Cc = 48, 24
    gwf = r.f32(2 * N, Cc)
    return lambda: ops.ln_fold_bwd(r.f32(N, Cc), r.f32(Cc), r.f32(Cc), gwf[N:], r.f32(N), torch.empty(N, Cc),
                                   r.acc(Cc), r.acc(Cc))


def _fir_resample(r, variant):
    from audio_diffusion_pytorch_b200.utils import _polyphase_bank
    fi, fo = (4, 1) if variant in ("down", "adjoint") else (1, 4)
    bank, half = _polyphase_bank(fi, fo, 0.99, 6, torch.float32, "cpu")
    t = 500
    t_out = fo * t // fi
    if variant == "adjoint":
        return lambda: ops.fir_resample(r.f32(3, t_out), bank[:, 0].contiguous(), fi, fo, half, t_out, adjoint_of=t)
    return lambda: ops.fir_resample(r.f32(3, t), bank[:, 0].contiguous(), fi, fo, half, t_out)


def _stem_out_loss(r, variant):
    f, Tf, co = 4, 256, 2
    return lambda: ops.stem_out(r.bf(B, Tf // f, 8), r.f32(B, co, Tf), r.f32(co, 8, 3, scale=0.3), r.f32(co),
                                r.f32(B, 4), f, noise=r.f32(B, co, Tf), alpha=torch.tensor([0.8, 0.6]),
                                beta=torch.tensor([0.6, 0.8]), loss_sum=r.acc(1, dtype=F64).abs() * 100,
                                dv=torch.empty(B, co, Tf))


MEL = dict(n_fft=256, hop_length=64, win_length=200, sample_rate=16000, n_mel_channels=24)


def _mel_front(normalize_log):
    from audio_diffusion_pytorch_b200.components import MelSpectrogram
    return MelSpectrogram(normalize_log=normalize_log, **MEL)


def _mel_spectrogram(r, variant):
    """15 frames (an odd count: the last FFT pair has one frame), a window shorter than n_fft."""
    front = _mel_front(variant == "log")
    window, fb, band = front._kernel_tables("cpu")
    return lambda: ops.mel_spectrogram(r.f32(3, 1000), window, fb, band, MEL["n_fft"], MEL["hop_length"],
                                       front.padding, apply_log=variant == "log")


FLAT = dict(C=16, frames=9, win=64, hop=16, pad=24)          # t_out = 8 * 16 - 48 + 64 = 144


def _to_flat(r, variant):
    return lambda: ops.to_flat(r.f32(3, FLAT["C"], FLAT["frames"]), r.f32(FLAT["C"], FLAT["win"], scale=0.1),
                               FLAT["hop"], FLAT["pad"])


def _to_flat_bwd(r, variant):
    return lambda: ops.to_flat_bwd(r.f32(3, FLAT["C"], FLAT["frames"]), r.f32(FLAT["C"], FLAT["win"], scale=0.1),
                                   r.f32(3, 144), FLAT["hop"], FLAT["pad"], need_dspec=variant != "dw",
                                   need_dw=variant != "dspec")


def _inpaint_blend(r, variant):
    """x is rows 1.. of a wider buffer (room outside the written view); the two alpha / beta rows differ."""
    x = r.f32(3, 2, 500)[1:]
    mask = (torch.rand(2, 2, 500, generator=r.g) < 0.4).to(torch.uint8)
    return lambda: ops.inpaint_blend(x, r.f32(2, 2, 500), r.f32(2, 2, 500), mask,
                                     torch.tensor([0.8, 0.6, 0.9, 0.43589]))


def _arv_step(r, variant):
    """B = 3, C = 2, T = 300; chan is rows 1.. of a wider buffer, sigma_1 <= sigma_0 per position."""
    chan = r.f32(4, 3, 300)[1:]
    chan[:, 2] = torch.rand(3, 300, generator=r.g)
    sig_next = chan[:, 2] * torch.rand(3, 300, generator=r.g)
    return lambda: ops.arv_step(chan, r.f32(3, 2, 300), sig_next)


DIRECT = {
    "wgrad": (_wgrad, ("tap1", "taps3", "views")),
    "gn_silu_bwd": (_gn_silu_bwd, ("all",)),
    "gn_bwd_apply": (_gn_bwd_apply, ("bare", "dres_colsum")),
    "ln_film_bwd": (_ln_film_bwd, ("film", "plain")),
    "colsum": (_colsum, ("bare", "gate")),
    "skip_gate": (_skip_gate, ("stats", "bare")),
    "skip_gate_bwd": (_skip_gate_bwd, ("all",)),
    "cond_bwd": (_cond_bwd, ("dcond", "bare")),
    "narrow_conv_bwd": (_narrow_conv_bwd, ("all",)),
    "stem_out_bwd": (_stem_out_bwd, ("adapter", "bare", "dxin")),
    "stem_in_bwd": (_stem_in_bwd, ("dxin", "bare")),
    "attention_bwd": (_attention_bwd, ("self", "cross")),
    "ln_fold_bwd": (_ln_fold_bwd, ("all",)),
    "fir_resample": (_fir_resample, ("up", "down", "adjoint")),
    "stem_out": (_stem_out_loss, ("loss",)),
    "mel_spectrogram": (_mel_spectrogram, ("log", "linear")),
    "to_flat": (_to_flat, ("plain",)),
    "to_flat_bwd": (_to_flat_bwd, ("both", "dspec", "dw")),
    "inpaint_blend": (_inpaint_blend, ("all",)),
    "arv_step": (_arv_step, ("all",)),
}
CASES = [(k, v) for k, (_, vs) in DIRECT.items() for v in vs]


def _launch(kind, variant, seed=11):
    make, _ = DIRECT[kind]
    return make(Rand(seed), variant)


def test_every_training_kind_has_a_direct_launch():
    """The direct launches above cover every checked kind the recorded inference programs do not
    reach: the training kinds, the resampler, the vocoder front-end and the two sampler steps."""
    from test_launch_check_cpu import _fixture_launches
    inference = {launch[0] for launch in _fixture_launches()} | {"sampler_step"}
    assert set(DIRECT) - {"stem_out"} == set(lc.CHECKERS) - inference


@pytest.mark.parametrize("kind,variant", CASES, ids=[f"{k}-{v}" for k, v in CASES])
def test_direct_launch_probe(cpu_launches, kind, variant):
    """The fake launch passes its own check, and every read argument moves the restatement."""
    with lc.Shadow(fake=True, probe=True) as sh:
        _launch(kind, variant)()
    assert sh.n_checked == sh.n_launch == 1
    assert {k for k, _ in sh.probed} == {kind}


# ------------------------------------------------- the restatements against float64 autograd
def _grad_check(got, want, what):
    e = float((got.double() - want.double()).norm() / want.double().norm().clamp_min(1e-300))
    assert e <= 1e-9, f"{what}: rel-L2 {e:.3e} against float64 autograd"


def _ref(o, args=None):
    return o.ref(args)[0] if callable(o.ref) else o.ref


def _outs(kind, args):
    return {o.name: o for o in lc.CHECKERS[kind](args, None)}


def _gn_silu_forward(x, stats_n, gamma, beta, groups, eps=1e-5):
    """SiLU(GroupNorm(x)) with the statistics held constant is NOT the operation: autograd goes
    through mean and variance, which is what the two backward passes together compute."""
    Bb, Tt, Cc = x.shape
    return F.silu(F.group_norm(x.transpose(1, 2), groups, gamma, beta, eps)).transpose(1, 2)


def test_groupnorm_backward_pair_vs_autograd():
    """gn_silu_bwd followed by gn_bwd_apply (fed the fp64 dxh and S of the first) is the gradient of
    SiLU(GroupNorm(x)); dgamma / dbeta are its parameter gradients."""
    r = Rand(3)
    x = (r.bf(B, T, C) + 0.5).double().requires_grad_()
    gamma, beta = r.f32(C).double().requires_grad_(), r.f32(C).double().requires_grad_()
    da = r.bf(B, T, C).double()
    _gn_silu_forward(x, None, gamma, beta, G).backward(da)
    st = _stats(x.detach(), G)
    o1 = _outs("gn_silu_bwd", dict(da=da, x=x.detach(), stats=st, gamma=gamma.detach(), beta=beta.detach(),
                                   dxh=None, dgamma=None, dbeta=None, S=None, groups=G, eps=1e-5))
    dxh = o1["dxh"].ref
    S = _ref(o1["S"], {"dxh": dxh})
    o2 = _outs("gn_bwd_apply", dict(dxh=dxh, x=x.detach(), stats=st, S=S, dx=None, groups=G, dres=None,
                                    colsum=torch.zeros(C), eps=1e-5))
    _grad_check(o2["dx"].ref, x.grad, "gn dx")
    _grad_check(o1["dgamma"].ref, gamma.grad, "dgamma")
    _grad_check(o1["dbeta"].ref, beta.grad, "dbeta")
    _grad_check(o2["colsum"].ref, x.grad.sum((0, 1)), "colsum")


def test_ln_film_bwd_vs_autograd():
    r = Rand(4)
    x = (r.bf(B, T, C) + 0.5).double().requires_grad_()
    ss = r.f32(B, 2 * C, scale=0.3).double().requires_grad_()
    dy, dres = r.bf(B, T, C).double(), r.bf(B, T, C).double()
    y = F.layer_norm(x, (C,), eps=1e-6) * (1 + ss[:, None, :C]) + ss[:, None, C:]
    (y * dy).sum().add((x * dres).sum()).backward()
    o = _outs("ln_film_bwd", dict(dy=dy, x=x.detach(), scale_shift=ss.detach(), ss_stride=2 * C, dx=None,
                                  dss=torch.zeros(B, 2 * C), dss_stride=2 * C, colsum=None, dres=dres, eps=1e-6))
    _grad_check(o["dx"].ref, x.grad, "ln dx")
    _grad_check(o["dss"].ref, ss.grad, "dss")


def test_conv_weight_gradients_vs_autograd():
    """wgrad with three taps, and narrow_conv_bwd (conv3 of SiLU(GroupNorm)) with gn_bwd_apply."""
    r = Rand(5)
    a, dy = r.bf(B, T, 40).double(), r.bf(B, T, 48).double()
    w = r.f32(48, 40, 3).double().requires_grad_()
    F.conv1d(a.transpose(1, 2), w, padding=1).backward(dy.transpose(1, 2))
    o = _outs("wgrad", dict(g=dy.to(BF), x=a.to(BF), dw=None, n=48, k=40, off=-1, g_col0=0, x_col0=0, ntaps=3))
    _grad_check(o["dw"].ref.permute(1, 2, 0), w.grad, "wgrad x3")

    x = (r.bf(B, T, 8) + 0.5).double().requires_grad_()
    gamma, beta = r.f32(8).double().requires_grad_(), r.f32(8).double().requires_grad_()
    w = r.f32(8, 8, 3, scale=0.3).double().requires_grad_()
    bias = r.f32(8).double().requires_grad_()
    dy = r.bf(B, T, 8).double()
    act = _gn_silu_forward(x, None, gamma, beta, 2)
    F.conv1d(act.transpose(1, 2), w, bias, padding=1).backward(dy.transpose(1, 2))
    st = _stats(x.detach(), 2)
    o = _outs("narrow_conv_bwd", dict(dy=dy, x=x.detach(), stats_in=st, gamma=gamma.detach(), beta=beta.detach(),
                                      w=w.detach(), dxh=None, dgamma=None, dbeta=None, S=None, dw=None, dbias=None,
                                      groups=2, gn_eps=1e-5))
    dxh = o["dxh"].ref
    o2 = _outs("gn_bwd_apply", dict(dxh=dxh, x=x.detach(), stats=st, S=_ref(o["S"], {"dxh": dxh}), dx=None, groups=2,
                                    dres=None, colsum=None, eps=1e-5))
    for name, p in (("dw", w), ("dbias", bias), ("dgamma", gamma), ("dbeta", beta)):
        _grad_check(o[name].ref, p.grad, f"narrow_conv_bwd {name}")
    _grad_check(o2["dx"].ref, x.grad, "narrow_conv_bwd dx")


def test_attention_bwd_vs_autograd():
    r = Rand(6)
    H, D, Tq, Tk = 2, 32, 96, 40
    mid = H * D
    q, k, v = (t.double().requires_grad_() for t in (r.bf(B, Tq, mid), r.bf(B, Tk, mid), r.bf(B, Tk, mid)))
    d_o = r.bf(B, Tq, mid).double()

    def heads(t, n):
        return t.reshape(B, n, H, D).transpose(1, 2)
    S = heads(q, Tq) @ heads(k, Tk).transpose(2, 3) * D ** -0.5
    o = (torch.softmax(S, -1) @ heads(v, Tk)).transpose(1, 2).reshape(B, Tq, mid)
    o.backward(d_o)
    outs = _outs("attention_bwd", dict(q=q.detach(), k=k.detach(), v=v.detach(), o=o.detach(), d_o=d_o,
                                       lse=torch.logsumexp(S.detach(), -1), delta=None, dq=None, dk=None, dv=None,
                                       heads=H, scale=D ** -0.5, head_dim=D))
    for name, p in (("dq", q), ("dk", k), ("dv", v)):
        _grad_check(outs[name].ref, p.grad, f"attention_bwd {name}")


def test_stems_vs_autograd():
    """stem_out in loss mode (loss, dv), stem_out_bwd and stem_in_bwd against autograd of
    the VDiffusion loss through the two boundary convolutions, SkipAdapter and appended channels."""
    r = Rand(7)
    f, Tf, co, cx, ca, c0 = 4, 256, 2, 2, 1, 8
    x, noise, app = r.f32(B, cx, Tf).double(), r.f32(B, cx, Tf).double(), r.f32(B, ca, Tf).double()
    al, be = torch.tensor([0.8, 0.6], dtype=F64), torch.tensor([0.6, 0.8], dtype=F64)
    leaf = lambda *s, scale=1.0: r.f32(*s, scale=scale).double().requires_grad_()     # noqa: E731
    w_in, b_in, w_out, b_out = leaf(c0, cx + ca, f), leaf(c0), leaf(co, c0, 3, scale=0.3), leaf(co)
    w_ad, b_ad, gate = leaf(co, cx + ca), leaf(co), leaf(B, 4)
    xin = torch.cat([al[:, None, None] * x + be[:, None, None] * noise, app], 1).requires_grad_()
    h_exact = F.conv1d(xin, w_in, b_in, stride=f)                         # [B, c0, Tf / f]
    h = h_exact.detach().transpose(1, 2).to(BF)                           # what the trunk would hand on
    hl = h.double().requires_grad_()
    y = F.conv1d(hl.transpose(1, 2).repeat_interleave(f, dim=2), w_out, b_out, padding=1)
    skip = torch.einsum("oc,bct->bot", w_ad, xin) + b_ad[None, :, None]
    v = skip + gate[:, :co, None] * y
    loss = ((v - (al[:, None, None] * noise - be[:, None, None] * x)) ** 2).mean()
    d_h = r.bf(B, Tf // f, c0).double()                                   # gradient reaching stem_in's output
    (0.7 * loss + (h_exact.transpose(1, 2) * d_h).sum()).backward()

    fwd = _outs("stem_out", dict(h=h, x=x, w=w_out.detach(), bias=b_out.detach(), gate=gate.detach(), f=f, append=app,
                                 w_adapt=w_ad.detach(), b_adapt=b_ad.detach(), v_out=None, x_next=None, ab=None,
                                 noise=noise, alpha=al, beta=be, loss_sum=torch.zeros(1, dtype=F64),
                                 dv=torch.zeros(B, co, Tf), cfg_scale=None))
    assert abs(float(fwd["loss_sum"].ref) / v.numel() - float(loss.detach())) <= 1e-12 * float(loss.detach())
    common = dict(x=x, append=app, noise=noise, alpha=al, beta=be, f=f)
    o = _outs("stem_out_bwd", dict(common, dv=fwd["dv"].ref, h=h, w=w_out.detach(), bias=b_out.detach(),
                                   gate=gate.detach(), dh=None, dw=None, dbias=None, dgate=None,
                                   gscale=torch.tensor([0.7], dtype=F64), w_adapt=w_ad.detach(), dw_adapt=None,
                                   db_adapt=None, dxin=torch.zeros(B, cx + ca, Tf)))
    for name, p in (("dw", w_out), ("dbias", b_out), ("dw_adapt", w_ad), ("db_adapt", b_ad)):
        _grad_check(o[name].ref, p.grad, f"stem_out_bwd {name}")
    _grad_check(o["dgate"].ref, gate.grad[:, :co], "stem_out_bwd dgate")
    _grad_check(o["dh"].ref, hl.grad, "stem_out_bwd dh")
    i = _outs("stem_in_bwd", dict(common, dout=d_h, dw=None, dbias=None, w=w_in.detach(),
                                  dxin=torch.zeros(B, cx + ca, Tf)))
    _grad_check(i["dw"].ref, w_in.grad, "stem_in_bwd dw")
    _grad_check(i["dbias"].ref, b_in.grad, "stem_in_bwd dbias")
    _grad_check(o["dxin"].ref + i["dxin"].ref, xin.grad, "dxin (skip path + down path)")


def test_small_backward_kinds_vs_autograd():
    """skip_gate / skip_gate_bwd, colsum with a gate, cond_bwd, ln_fold_bwd, fir_resample's adjoint."""
    r = Rand(8)
    y, skip, d = r.bf(B, T, C).double().requires_grad_(), r.bf(B, T, C).double(), r.bf(B, T, C).double()
    gate = r.f32(B, 2 * C).double().requires_grad_()
    (skip + gate[:, None, :C] * y).backward(d)
    o = _outs("skip_gate_bwd", dict(dout=d, y=y.detach(), gate=gate.detach(), dys=None, dgate=None))
    _grad_check(o["dys"].ref, y.grad, "dys")
    _grad_check(o["dgate"].ref, gate.grad[:, :C], "dgate")
    o = _outs("colsum", dict(x=d, out=torch.zeros(C), gate=gate.detach()))
    _grad_check(o["out"].ref, (d * gate.detach()[:, None, :C]).sum((0, 1)), "gated colsum")

    N, K = 70, 24
    cond, W, bias = r.f32(B, K).double().requires_grad_(), r.bf(80, K).double().requires_grad_(), \
        r.f32(N).double().requires_grad_()
    dss = r.f32(B, 72).double()
    (cond @ W[:N].t() + bias).backward(dss[:, :N])
    o = _outs("cond_bwd", dict(dss=dss, cond=cond.detach(), w=W.detach(), dw=None, dbias=None,
                               dcond=torch.zeros(B, K), N=N))
    _grad_check(o["dw"].ref, W.grad[:N], "cond dw")
    _grad_check(o["dbias"].ref, bias.grad, "cond dbias")
    _grad_check(o["dcond"].ref, cond.grad, "dcond")

    Wp, g, b = (t.double().requires_grad_() for t in (r.f32(48, 24), r.f32(24), r.f32(24)))
    dwf, dbf = r.f32(48, 24).double(), r.f32(48).double()
    ((Wp * g * dwf).sum() + ((Wp @ b) * dbf).sum()).backward()          # Wf = W diag(g), bf = W b
    o = _outs("ln_fold_bwd", dict(w=Wp.detach(), g=g.detach(), b=b.detach(), dwf=dwf, dbf=dbf, dw=None, dg=None,
                                  db=None))
    for name, p in (("dw", Wp), ("dg", g), ("db", b)):
        _grad_check(o[name].ref, p.grad, f"ln_fold_bwd {name}")

    from audio_diffusion_pytorch_b200.utils import _polyphase_bank, resample
    for fi, fo in ((4, 1), (1, 4), (3, 2)):
        bank, half = _polyphase_bank(fi, fo, 0.99, 6, F64, "cpu")
        x = r.f32(1, 3, 480).double().requires_grad_()
        want = resample(x, fi, fo)                       # the host route: the same bank as a strided convolution
        dy = r.f32(*want.shape).double()
        want.backward(dy)
        geom = dict(bank=bank[:, 0], factor_in=fi, factor_out=fo, half=half, t_out=want.shape[-1])
        o = _outs("fir_resample", dict(geom, x=x.detach()[0], adjoint_of=None))
        _grad_check(o["_result"].ref, want.detach()[0], f"resample {fi}->{fo}")
        o = _outs("fir_resample", dict(geom, x=dy[0], adjoint_of=480))
        _grad_check(o["_result"].ref, x.grad[0], f"resample adjoint {fi}->{fo}")


def test_vocoder_front_end_vs_float64_modules():
    """mel_spectrogram against MelSpectrogram's own tensor-op route (torchaudio STFT + MelScale after
    F.pad reflect) in float64, with and without the log; to_flat / to_flat_bwd against
    nn.ConvTranspose1d and its float64 autograd."""
    r = Rand(9)
    for log in (False, True):
        front = _mel_front(log)
        window, fb, band = front._kernel_tables("cpu")
        wave = r.f32(3, 1000).double()
        want = front.double()(wave)
        o = _outs("mel_spectrogram", dict(wave=wave, window=window, fb=fb, band=band, n_fft=MEL["n_fft"],
                                          hop=MEL["hop_length"], pad=front.padding, apply_log=log))
        assert o["mel"].ref.shape == want.shape == (3, MEL["n_mel_channels"], 15)
        _grad_check(o["mel"].ref, want, f"mel_spectrogram (log={log})")

    C, frames, win, hop, pad = (FLAT[k] for k in ("C", "frames", "win", "hop", "pad"))
    conv = torch.nn.ConvTranspose1d(C, 1, win, stride=hop, padding=pad, bias=False).double()
    spec = r.f32(3, C, frames).double().requires_grad_()
    out = conv(spec)
    dout = r.f32(*out.shape).double()
    out.backward(dout)
    w = conv.weight.detach()[:, 0]
    o = _outs("to_flat", dict(spec=spec.detach(), w=w, hop=hop, pad=pad))
    _grad_check(o["out"].ref, out.detach()[:, 0], "to_flat")
    o = _outs("to_flat_bwd", dict(spec=spec.detach(), w=w, dout=dout[:, 0], hop=hop, pad=pad, need_dspec=True,
                                  need_dw=True))
    _grad_check(o["dspec"].ref, spec.grad, "to_flat_bwd dspec")
    _grad_check(o["dw"].ref, conv.weight.grad[:, 0], "to_flat_bwd dw")
    assert set(_outs("to_flat_bwd", dict(spec=spec.detach(), w=w, dout=dout[:, 0], hop=hop, pad=pad,
                                         need_dspec=False, need_dw=True))) == {"dw"}


def test_sampler_steps_vs_float64_formulas():
    """inpaint_blend and arv_step against the reference's formulas (diffusion.py, VInpainter and
    ARVSampler) evaluated directly in float64."""
    from audio_diffusion_pytorch_b200.diffusion import _alpha_beta
    r = Rand(10)
    x, src, noise = (r.f32(2, 2, 500).double() for _ in range(3))
    mask = torch.rand(2, 2, 500, generator=r.g) < 0.4
    sig = torch.tensor([0.7, 0.55], dtype=F64)
    alphas, betas = _alpha_beta(sig)
    ab = torch.stack([alphas[0], betas[0], alphas[1], betas[1]])
    want = x.clone()
    want[mask] = (alphas[1] * src + betas[1] * noise)[mask]
    o = _outs("inpaint_blend", dict(x=x, source=src, noise=noise, mask_u8=mask.to(torch.uint8), ab=ab))
    _grad_check(o["x"].ref, want, "inpaint_blend")
    assert torch.equal(o["x"].keep, ~mask)

    chan = r.f32(3, 3, 300).double()
    chan[:, 2] = torch.rand(3, 300, generator=r.g).double()
    v, sig_next = r.f32(3, 2, 300).double(), torch.rand(3, 300, generator=r.g).double()
    a0, b0 = _alpha_beta(chan[:, 2:])
    a1, b1 = _alpha_beta(sig_next[:, None])
    x_pred, noise_pred = a0 * chan[:, :2] - b0 * v, b0 * chan[:, :2] + a0 * v
    o = _outs("arv_step", dict(chan=chan, v=v, sig_next=sig_next))
    _grad_check(o["chan"].ref, a1 * x_pred + b1 * noise_pred, "arv_step")
    assert torch.equal(o["chan.sigma"].ref, sig_next) and o["chan.sigma"].exact


# ------------------------------------------------------------------------------ mutations
def _roles(kind):
    return lc.ARGS[kind]


_ACC_KINDS = [k for k in DIRECT if k != "stem_out" and _roles(k)[2] and k != "skip_gate"]
_VAL_KINDS = [k for k in DIRECT if _roles(k)[1]]
MUTANTS = ([("acc_stored", k) for k in _ACC_KINDS + ["stem_out"]] +
           [("acc_lost_split", k) for k in _ACC_KINDS + ["stem_out"]] +
           [("scale_largest", k) for k in _VAL_KINDS] +
           [("stale_tile", k) for k in ("gn_silu_bwd", "gn_bwd_apply", "ln_film_bwd", "skip_gate", "skip_gate_bwd",
                                        "narrow_conv_bwd", "stem_out_bwd", "attention_bwd")] +
           [("stats_slot", "skip_gate")] +
           [("outside_view", k) for k in ("wgrad", "ln_film_bwd", "colsum", "skip_gate_bwd", "cond_bwd",
                                          "stem_out_bwd", "attention_bwd", "inpaint_blend", "arv_step")] +
           [("readonly", k) for k in DIRECT] +
           # kind-specific: an alternative operation written over the output
           [("mel_symmetric_pad", "mel_spectrogram"), ("mel_pairs_swapped", "mel_spectrogram"),
            ("to_flat_shifted", "to_flat"), ("to_flat_dw_lost_row", "to_flat_bwd"),
            ("blend_start_level", "inpaint_blend"), ("blend_unmasked_write", "inpaint_blend"),
            ("arv_sigma_kept", "arv_step"), ("arv_v_chan_stride", "arv_step")])
# the variant of each kind whose outputs leave room outside their views (column windows of wider rows)
_VARIANT = {"wgrad": "views", "ln_film_bwd": "film", "attention_bwd": "self", "stem_out_bwd": "adapter",
            "gn_bwd_apply": "dres_colsum", "colsum": "gate", "cond_bwd": "dcond", "stem_in_bwd": "dxin"}


@pytest.mark.parametrize("mutation,kind", MUTANTS, ids=[f"{m}-{k}" for m, k in MUTANTS])
def test_mutation_is_caught(cpu_launches, mutation, kind):
    variant = _VARIANT.get(kind, DIRECT[kind][1][0])
    if (mutation, kind) == ("outside_view", "colsum"):
        variant = "wide"
    run = _launch(kind, variant, seed=100 + MUTANTS.index((mutation, kind)))
    if variant == "wide":                    # the bias gradient of a column window: out wider than C
        r = Rand(9)
        run = lambda: ops.colsum(r.bf(B, T, C), r.acc(2 * C), None)      # noqa: E731
    with lc.Shadow(fake=True, mutate=(kind, lc.MUTATIONS[mutation])) as sh:
        with pytest.raises(lc.CheckError) as err:
            run()
    assert sh.mutate is None, f"{mutation} never applied to a {kind} launch"
    assert f"): {kind}:" in str(err.value), str(err.value)
    print(f"caught {mutation} in {kind}: {err.value}")


def test_acc_bound_is_the_stated_one():
    assert (lc.FP32_REL, lc.FP32_TAU, lc.ACC_EPS, lc.STATS_TOL) == (1e-5, 2.0 ** -14, 2.0 ** -23, 1e-4)
    assert math.isclose(lc.TAU_BF16_OPERAND, 2.0 ** -8) and math.isclose(lc.TAU_FP32_ACC, 2.0 ** -12)
