"""Wide network boundary on the host: UNetV0 with up to 64 input / output channels, in_channels *
factors[0] <= 128 and channels[0] <= 256.  The constructor accepts the envelope's corners and refuses
what lies outside with the limit in the message (LTPlugin on its transformed widths); the C entry
points refuse out-of-envelope sizes before any CUDA call; wide nets' inference, sampling and training
plans build and record on the CPU with level 0 as exactly one stem_in / stem_out (and one
stem_out_bwd / stem_in_bwd); the level-0 SkipCat fold and unfold is exact at wide output widths."""
import ctypes
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from test_launch_programs_cpu import build_net, install  # noqa: E402
from audio_diffusion_pytorch_b200 import _lib, training  # noqa: E402
from audio_diffusion_pytorch_b200.components import LTPlugin  # noqa: E402
from audio_diffusion_pytorch_b200.unet import UNetV0  # noqa: E402

REAL_LIB = _lib.lib                    # the recorder fixture replaces _lib.lib while this module runs
SMALL = dict(channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 1, 1])


def make(**kw):
    return UNetV0(dim=1, **{**SMALL, **kw})


@pytest.mark.parametrize("kw", [
    dict(in_channels=9, out_channels=5),
    dict(in_channels=12, out_channels=6, append_channels=6),            # a 5.1 upsampler
    dict(in_channels=64, out_channels=64),
    dict(in_channels=64, out_channels=64, channels=[128, 256, 256], factors=[2, 4, 4]),   # in * f = 128
    dict(in_channels=32, out_channels=32, factors=[4, 4, 4]),            # in * f = 128
    dict(in_channels=2, channels=[256, 256, 256]),                       # channels[0] = 256
    dict(in_channels=9, out_channels=8, use_modulation=False, use_time_conditioning=False),
])
def test_envelope_accepted(kw):
    net = make(**kw)
    assert net.in_channels == kw["in_channels"]


@pytest.mark.parametrize("kw,msg", [
    (dict(in_channels=65, out_channels=8), "at most 64 input channels"),
    (dict(in_channels=64, out_channels=65, append_channels=0), "at most 64 output channels"),
    (dict(in_channels=12, out_channels=8, append_channels=6), "exceeds the 6 channels of x"),
    (dict(in_channels=43, out_channels=8, factors=[3, 4, 4]), "in_channels * factors[0] = 129"),
    (dict(in_channels=2, channels=[264, 264, 264]), "channels[0]=264"),
])
def test_envelope_refused(kw, msg):
    with pytest.raises(AssertionError, match=msg.replace("[", r"\[").replace("]", r"\]").replace("*", r"\*")):
        make(**kw)


def test_ltplugin_refuses_on_transformed_widths():
    LTPlugin(UNetV0, num_filters=32, window_length=64, stride=32)(dim=1, in_channels=2, **SMALL)
    with pytest.raises(AssertionError, match="at most 64 input channels"):
        LTPlugin(UNetV0, num_filters=33, window_length=64, stride=32)(dim=1, in_channels=2, **SMALL)
    with pytest.raises(AssertionError, match=r"in_channels \* factors\[0\] = 256"):
        LTPlugin(UNetV0, num_filters=32, window_length=64, stride=32)(
            dim=1, in_channels=2, **dict(SMALL, factors=[4, 4, 4]))


def test_entry_points_refuse_out_of_envelope_sizes():
    """Validation runs before any CUDA call, so the refusals are observable without a GPU."""
    from audio_diffusion_pytorch_b200 import _build
    _build.build()
    L = REAL_LIB()
    p = ctypes.c_void_p(256)            # never dereferenced: the size checks fail first

    def refused(rc, what):
        assert rc != 0, what
        assert what in L.adp_last_error().decode()

    sa = _lib.StemInArgs(x=p, w=p, out=p, B=2, T=16, cx=65, ca=0, c0=8, f=1)
    refused(L.adp_stem_in(ctypes.byref(sa), None), "adp_stem_in")             # cx + ca > 64
    sa.cx, sa.f = 33, 4
    refused(L.adp_stem_in(ctypes.byref(sa), None), "adp_stem_in")             # (cx + ca) * f > 128
    sa.cx, sa.f, sa.c0 = 2, 1, 264
    refused(L.adp_stem_in(ctypes.byref(sa), None), "adp_stem_in")             # c0 > 256
    sb = _lib.StemOutArgs(h=p, x=p, w=p, gate=p, B=2, T=16, cx=65, ca=0, c0=8, co=8, f=1)
    refused(L.adp_stem_out(ctypes.byref(sb), None), "adp_stem_out")           # cx + ca > 64
    sb.cx, sb.co = 66, 65
    refused(L.adp_stem_out(ctypes.byref(sb), None), "adp_stem_out")           # co > 64
    sb.cx, sb.co = 4, 6
    refused(L.adp_stem_out(ctypes.byref(sb), None), "adp_stem_out")           # co > cx
    sb.cx, sb.co, sb.c0 = 8, 8, 264
    refused(L.adp_stem_out(ctypes.byref(sb), None), "adp_stem_out")           # c0 > 256
    for name in ("adp_stem_out_bwd", "adp_f32_stem_out_bwd"):
        so = _lib.StemOutBwdArgs(dv=p, h=p, x=p, w=p, gate=p, dh=p, dw=p, dbias=p, dgate=p, B=2, T=16, cx=65,
                                 ca=0, c0=8, co=65, f=1, ld_gate=65, ld_dgate=65)
        if name == "adp_stem_out_bwd":
            refused(getattr(L, name)(ctypes.byref(so), None), name)          # co > 64
            so.cx, so.co, so.c0 = 8, 8, 264
            refused(getattr(L, name)(ctypes.byref(so), None), name)          # c0 > 256
    si = _lib.StemInBwdArgs(dout=p, x=p, dw=p, dbias=p, B=2, T=16, cx=65, ca=0, c0=8, f=1)
    refused(L.adp_stem_in_bwd(ctypes.byref(si), None), "adp_stem_in_bwd")     # cx + ca > 64
    si.cx, si.f = 33, 4
    refused(L.adp_stem_in_bwd(ctypes.byref(si), None), "adp_stem_in_bwd")     # (cx + ca) * f > 128
    si.cx, si.f, si.c0 = 2, 1, 264
    refused(L.adp_stem_in_bwd(ctypes.byref(si), None), "adp_stem_in_bwd")     # c0 > 256
    sf = _lib.StemOutArgs(h=p, x=p, w=p, gate=p, B=2, T=16, cx=65, ca=0, c0=8, co=8, f=1)
    refused(L.adp_f32_stem_out(ctypes.byref(sf), None), "adp_f32_stem_out")   # cx + ca > 64


# ---------------------------------------------------------------- recorded plans (no GPU)
# name -> (net kwargs, B, T, M, inference modes, training (mode, want_dxin) pairs)
WIDE_NETS = {
    "ltplugin_64": (dict(in_channels=64, channels=[128, 256, 256], factors=[1, 4, 4], items=[1, 1, 1]),
                    2, 1024, 0, ("v", "sample"), (("loss", True), ("v", False))),
    "surround_51": (dict(in_channels=6, channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 1, 1]),
                    2, 1024, 0, ("v", "sample"), (("loss", False),)),
    "upsampler_51": (dict(in_channels=12, out_channels=6, append_channels=6, channels=[8, 32, 64],
                          factors=[1, 4, 4], items=[1, 1, 1]),
                     2, 1024, 0, ("v", "sample"), (("loss", True),)),
    "ar_skipcat_9": (dict(in_channels=9, out_channels=8, channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 1, 1],
                          use_modulation=False, use_time_conditioning=False),
                     2, 1024, 0, ("v", "sample"), (("v", True), ("loss", False))),
    "c0_256": (dict(in_channels=2, channels=[256, 256, 256], factors=[2, 2, 2], items=[1, 1, 1]),
               2, 1024, 0, ("v",), (("loss", False),)),
    "cfg_64": (dict(in_channels=64, channels=[128, 256, 256], factors=[1, 4, 4], items=[1, 1, 1],
                    cross_attentions=[0, 1, 1], attention_heads=2, attention_features=64,
                    use_embedding_cfg=True, embedding_max_length=8, embedding_features=32),
               2, 1024, 8, ("v_cfg", "sample_cfg"), ()),
}


@pytest.fixture(scope="module")
def recorder():
    mp = pytest.MonkeyPatch()
    rec = install(mp)
    yield rec
    mp.undo()


def _shape(launch, arg):
    for k, v in launch[1:]:
        if k == arg:
            return v[3] if v else None
    raise KeyError(arg)


def _stems(prog, kinds):
    return [l for l in prog if l[0] in kinds]


@pytest.mark.parametrize("name", sorted(WIDE_NETS))
def test_wide_plans_record(name, recorder):
    kw, B, T, M, modes, trains = WIDE_NETS[name]
    net = build_net(kw, {})
    cin, co, c0, f = net.in_channels, net.out_channels, kw["channels"][0], kw["factors"][0]
    cx = cin - kw.get("append_channels", 0)
    for m in modes:
        cfg = m.endswith("_cfg")
        mode = m[:-4] if cfg else m
        Bh = 2 * B if cfg else B
        plan = net._plan(B, T, Bh, M, mode, (5.0 if cfg else None, False))
        plan.cfg_scale = 5.0 if cfg else None
        recorder.storages, recorder.slots, recorder.keep = {}, {}, []
        for fn in getattr(plan, "pre", []):
            fn()
        recorder.take()
        plan.run_eager()
        prog = recorder.take()
        ins, outs = _stems(prog, ("stem_in",)), _stems(prog, ("stem_out",))
        assert len(ins) == Bh // B and len(outs) == 1, (m, [l[0] for l in prog])
        assert _shape(ins[0], "x") == [B, cx, T] and _shape(ins[0], "w") == [c0, cin, f]
        assert _shape(ins[0], "out") == [B, T // f, c0]
        assert _shape(outs[0], "h") == [Bh, T // f, c0] and _shape(outs[0], "w") == [co, c0, 3]
        assert _shape(outs[0], "gate")[1] >= co
    for mode, want_dxin in trains:
        plan = training.build_train_plan(net, B, T, M, mode, want_dxin)
        recorder.storages, recorder.slots, recorder.keep = {}, {}, []
        for fn in plan.fwd:
            fn()
        fwd = recorder.take()
        plan.backward_program()
        bwd = recorder.take()
        assert [l[0] for l in _stems(fwd, ("stem_in", "stem_out"))] == ["stem_in", "stem_out"]
        assert [l[0] for l in _stems(bwd, ("stem_in_bwd", "stem_out_bwd"))] == ["stem_out_bwd", "stem_in_bwd"]
        so = _stems(bwd, ("stem_out_bwd",))[0]
        assert _shape(so, "dh") == [B, T // f, c0] and _shape(so, "dw") == [co, c0, 3]
        assert _shape(so, "gate")[1] >= co and _shape(so, "dgate")[1] >= co
        assert _shape(_stems(bwd, ("stem_in_bwd",))[0], "dw") == [c0, cin, f]


# --------------------------------------------------------- level-0 SkipCat fold / unfold
D = torch.float64


def _rnd(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=D)


@pytest.mark.parametrize("Co", [6, 64])
@pytest.mark.parametrize("adapter", [False, True])
def test_level0_skipcat_unfold_wide(Co, adapter):
    """As test_train_host_cpu.test_level0_skipcat_unfold at wide output widths: the folded weights
    the stem kernels run reproduce merge(cat([adapter(x) * 2^-0.5, up(h)])), and the unfold turns
    the folded gradients into merge / up / adapter gradients, against float64 autograd."""
    B, T, C = 2, 9, 16
    Ci = Co + 3 if adapter else Co
    torch.manual_seed(19)
    merge = torch.nn.Conv1d(2 * Co, Co, 1).to(D)
    up = torch.nn.Conv1d(C, Co, 3, padding=1).to(D)
    ad = torch.nn.Conv1d(Ci, Co, 1).to(D) if adapter else None
    x, h, dv = _rnd(B, Ci, T, seed=20), _rnd(B, C, T, seed=21), _rnd(B, Co, T, seed=22)
    skip = ad(x) if adapter else x
    ref = merge(torch.cat([skip * 2 ** -0.5, up(h)], 1))
    ref.backward(dv)
    wm = merge.weight.detach()[:, :, 0]
    wc1, wc2 = wm[:, :Co] * 2 ** -0.5, wm[:, Co:]
    fw_up = torch.einsum("om,mck->ock", wc2, up.weight.detach()).requires_grad_()
    fb_up = (wc2 @ up.bias.detach() + merge.bias.detach()).requires_grad_()
    fw_ad = (wc1 @ ad.weight.detach()[:, :, 0] if adapter else wc1).requires_grad_()
    fb_ad = (wc1 @ ad.bias.detach() if adapter else torch.zeros(Co, dtype=D)).requires_grad_()
    folded = F.conv1d(x, fw_ad[:, :, None], fb_ad) + F.conv1d(h, fw_up, fb_up, padding=1)
    assert float((folded - ref).detach().abs().max()) <= 1e-10 * float(ref.detach().abs().max())
    folded.backward(dv)
    g = training.unfold_level0_grads(merge.weight, up.weight, up.bias, fw_up.grad, fb_up.grad, fw_ad.grad,
                                     fb_ad.grad, ad.weight if adapter else None, ad.bias if adapter else None)
    mods = {"merge": merge, "up": up, **({"adapter": ad} if adapter else {})}
    assert sorted(g) == sorted(f"{m}.{p}" for m in mods for p in ("weight", "bias"))
    for name, m in mods.items():
        for pn in ("weight", "bias"):
            got, want = g[f"{name}.{pn}"].reshape(getattr(m, pn).shape), getattr(m, pn).grad
            err = float((got - want).abs().max())
            assert err <= 1e-10 * float(want.abs().max()), f"{name}.{pn}: {err:.3e}"
