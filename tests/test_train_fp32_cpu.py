"""The training program of the fp32 verification mode (B200UNet.verify_fp32), recorded on the CPU with
the recorder of test_launch_programs_cpu.py and compared with the bf16 training program of the same
net: it must be the SAME program -- launch order, gradient-arena layout, flush marks -- with fp32
storage.  The one permitted difference is the C = 8 ConvBlock, which the fp32 mode runs unfused (as
its inference program does):

  forward   narrow_conv      -> gn_silu, conv_gemm
  backward  narrow_conv_bwd  -> wgrad, conv_gemm, gn_silu_bwd
            and, without a ModulationItem, the bias gradient of conv2 as a colsum in front of it
            (the narrow kernel accumulates it itself)

and those blocks' conv weight accumulators are the generic [tap][co][ci] slabs instead of the narrow
kernel's [co][ci][tap] (same arena offsets).  Also: the new fp32 entry points are declared, exported
and refuse bad sizes before launching anything."""
import ctypes
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from test_launch_programs_cpu import NETS, build_net, install  # noqa: E402
from audio_diffusion_pytorch_b200 import _lib, training  # noqa: E402

CASES = ("tiny", "text_cfg", "skipcat_adapter", "inject", "append", "head32_g4", "head128_g4", "readme")

NEW_SYMBOLS = ("adp_f32_attention_lse", "adp_f32_stem_in_train", "adp_f32_stem_out_train", "adp_f32_wgrad",
               "adp_f32_gn_silu_bwd", "adp_f32_gn_bwd_apply", "adp_f32_ln_film_bwd", "adp_f32_colsum",
               "adp_f32_skip_gate", "adp_f32_skip_gate_bwd", "adp_f32_cond_bwd", "adp_f32_stem_out_bwd",
               "adp_f32_stem_in_bwd", "adp_f32_attention_bwd")
REAL_LIB = _lib.lib                    # the recorder fixture replaces _lib.lib while this module runs


@pytest.fixture(scope="module")
def recorder():
    mp = pytest.MonkeyPatch()
    rec = install(mp)
    yield rec
    mp.undo()


def record_train(net, rec, B, T, M, mode, want_dxin):
    plan = training.build_train_plan(net, B, T, M, mode, want_dxin)
    rec.storages, rec.slots, rec.keep = {}, {}, []
    for fn in plan.fwd:
        fn()
    fwd = rec.take()
    marks = []
    plan.on_mark = lambda iv: marks.append(tuple(iv))
    plan.backward_program()
    plan.on_mark = None
    return plan, fwd, rec.take(), marks


def unfused(names, mod):
    """The bf16 launch names with every C = 8 ConvBlock replaced by its unfused composition."""
    out, n_bwd = [], 0
    for n in names:
        if n == "narrow_conv":
            out += ["gn_silu", "conv_gemm"]
        elif n == "narrow_conv_bwd":
            if n_bwd % 2 == 0 and not mod:     # conv2 of the block: its bias gradient
                out.append("colsum")
            out += ["wgrad", "conv_gemm", "gn_silu_bwd"]
            n_bwd += 1
        else:
            out.append(n)
    return out


def tensors(launches):
    for launch in launches:
        for _, v in launch[1:]:
            stack = [v]
            while stack:
                x = stack.pop()
                if isinstance(x, list) and x and x[0] == "T":
                    yield launch[0], x
                elif isinstance(x, list):
                    stack += x


@pytest.mark.parametrize("name", CASES)
def test_fp32_training_program_is_the_bf16_program(name, recorder):
    kw, attrs, B, T, M, _, trains = NETS[name]
    assert trains, name
    for mode, want_dxin in trains:
        net = build_net(kw, attrs)
        names = {id(p): n for n, p in net.named_parameters()}
        narrow = {n for n, p in net.named_parameters() if ".resnet.conv" in n and n.endswith(".weight")
                  and p.shape[0] == 8}
        plan16, fwd16, bwd16, marks16 = record_train(net, recorder, B, T, M, mode, want_dxin)
        net.verify_fp32 = True
        plan32, fwd32, bwd32, marks32 = record_train(net, recorder, B, T, M, mode, want_dxin)
        what = f"{name} train {mode} dxin={want_dxin}"

        for launch, t in tensors(fwd32 + bwd32):
            assert t[5] != "bfloat16", f"{what}: {launch} gets a bf16 tensor"

        mod = net.use_modulation
        assert [x[0] for x in fwd32] == unfused([x[0] for x in fwd16], mod), what + " (forward)"
        assert [x[0] for x in bwd32] == unfused([x[0] for x in bwd16], mod), what + " (backward)"

        assert plan32.flat.numel() == plan16.flat.numel()
        assert marks32 == marks16, what + ": gradient flush marks"
        assert set(plan32.specs) == set(plan16.specs)
        for pid, (start, n, shape, perm) in plan16.specs.items():
            s32 = plan32.specs[pid]
            assert (s32[0], s32[1]) == (start, n), f"{what}: arena slot of {names[pid]}"
            if names[pid] in narrow:             # generic [tap][co][ci] accumulator of a C = 8 conv
                assert (s32[2], s32[3]) == ((3, 8, 8), (1, 2, 0)) and (shape, perm) == ((8, 8, 3), None)
            else:
                assert (s32[2], s32[3]) == (shape, perm), f"{what}: layout of {names[pid]}"
        assert {names[k]: v for k, v in plan32.grads.items()} == {names[k]: v for k, v in plan16.grads.items()}
        assert narrow and any(x[0] == "narrow_conv_bwd" for x in bwd16)    # every net has a C = 8 level
        assert not any(x[0] in ("narrow_conv", "narrow_conv_bwd") for x in fwd32 + bwd32)


def _header():
    with open(os.path.join(ROOT, "include", "adp_b200.h")) as f:
        return f.read()


def test_new_entry_points_are_declared_and_exported():
    from audio_diffusion_pytorch_b200 import _build
    lib = ctypes.CDLL(_build.build())
    header = _header()
    for s in NEW_SYMBOLS:
        assert f"int {s}(" in header, s
        assert hasattr(lib, s), s
        assert s in _lib.EXPORTS, s


def test_new_entry_points_refuse_bad_sizes():
    """Validation runs before any CUDA call, so the refusals are observable without a GPU."""
    from audio_diffusion_pytorch_b200 import _build
    _build.build()
    L = REAL_LIB()
    p = ctypes.c_void_p(256)            # never dereferenced: the size checks fail first

    def refused(rc, what):
        assert rc != 0, what
        assert what in L.adp_last_error().decode()

    a = _lib.WgradArgs(g=p, x=p, dw=p, B=2, T=16, n=8, k=8, ldg=8, ldx=8, ldw=8, g_cols=8, x_cols=8, ntaps=2)
    refused(L.adp_f32_wgrad(ctypes.byref(a), None), "adp_f32_wgrad")
    a.ntaps, a.k = 1, 0
    refused(L.adp_f32_wgrad(ctypes.byref(a), None), "adp_f32_wgrad")
    refused(L.adp_f32_gn_silu_bwd(p, p, p, p, p, p, p, p, p, 2, 16, 12, 8, 1e-5, None), "adp_f32_gn_silu_bwd")
    refused(L.adp_f32_gn_bwd_apply(p, p, p, p, None, p, None, 2, 16, 12, 8, 1e-5, None), "adp_f32_gn_bwd_apply")
    refused(L.adp_f32_ln_film_bwd(p, p, p, 8, p, None, 0, None, None, 2, 16, 8, 1e-6, None), "adp_f32_ln_film_bwd")
    refused(L.adp_f32_colsum(p, None, 0, p, 2, 0, 8, None), "adp_f32_colsum")
    refused(L.adp_f32_skip_gate(p, p, p, 8, p, p, 2, 16, 8, 8, None), "adp_f32_skip_gate")
    refused(L.adp_f32_skip_gate_bwd(p, p, p, 4, p, p, 8, 2, 16, 8, None), "adp_f32_skip_gate_bwd")
    refused(L.adp_f32_cond_bwd(p, 4, p, p, p, p, None, 2, 8, 16, None), "adp_f32_cond_bwd")
    so = _lib.StemOutBwdArgs(dv=p, h=p, x=p, w=p, gate=p, dh=p, dw=p, dbias=p, dgate=p, B=2, T=15, cx=2,
                             ca=0, c0=8, co=2, f=2, ld_gate=8, ld_dgate=8)
    refused(L.adp_f32_stem_out_bwd(ctypes.byref(so), None), "adp_f32_stem_out_bwd")
    si = _lib.StemInBwdArgs(dout=p, x=p, dw=p, dbias=p, B=2, T=16, cx=2, ca=1, c0=8, f=1)
    refused(L.adp_f32_stem_in_bwd(ctypes.byref(si), None), "adp_f32_stem_in_bwd")
    at = _lib.AttentionBwdArgs(q=p, k=p, v=p, o=p, d_o=p, lse=p, delta=p, dq=p, dk=p, dv=p, B=2, H=2, Tq=8, Tk=8,
                               ldq=128, ldk=128, ldv=128, ldo=128, lddo=128, lddq=128, lddk=128, lddv=128,
                               scale=0.125)
    refused(L.adp_f32_attention_bwd(ctypes.byref(at), 96, None), "adp_f32_attention_bwd")
    at.ldk = 64
    refused(L.adp_f32_attention_bwd(ctypes.byref(at), 64, None), "adp_f32_attention_bwd")
    refused(L.adp_f32_attention_lse(p, p, p, p, 2, 2, 64, 8, 8, 64, 128, 128, 128, 0.125, p, None),
            "adp_f32_attention")
    sa = _lib.StemInArgs(x=p, w=p, out=p, noise=p, B=2, T=16, cx=2, ca=0, c0=8, f=4)
    refused(L.adp_f32_stem_in_train(ctypes.byref(sa), None), "adp_f32_stem_in")      # noise without alpha/beta
    refused(L.adp_f32_stem_in(ctypes.byref(sa), None), "adp_f32_stem_in")            # noising is the _train form
    sb = _lib.StemOutArgs(h=p, x=p, w=p, gate=p, dv=p, B=2, T=16, cx=2, ca=0, c0=8, co=2, f=4)
    refused(L.adp_f32_stem_out_train(ctypes.byref(sb), None), "adp_f32_stem_out")    # dv without the loss
    refused(L.adp_f32_stem_out(ctypes.byref(sb), None), "adp_f32_stem_out")
