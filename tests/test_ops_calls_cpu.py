"""What every launching function of `ops` (and the STFT loss in `losses`) passes to the C library,
recorded on the CPU and compared with tests/golden/ops_calls.json.gz.

The library is replaced by a fake whose entry points record (symbol, arguments) and return 0, so
each route of each function -- both dtypes, every optional argument that selects an entry point or
fills one -- runs here without a GPU.  Per call the fixture holds the C functions called in order
and their arguments: a pointer as (index of the tensor whose storage holds it, byte offset into that
storage), where tensors are numbered as passed (a tuple argument such as `gn` in order) and then as
allocated inside the call; None as null; ints as ints; floats by their IEEE bits; a struct passed
by reference field by field.  With it come the trace records' labels, FLOPs and bytes (bench.py's
roofline) and which tensor the function returns.  A change to how `ops` fills an argument list or a
struct, picks an entry point or labels a launch fails here.

    python tests/test_ops_calls_cpu.py --write     # re-record the fixture
"""
import contextlib
import ctypes as C
import gzip
import inspect
import json
import os
import struct
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from audio_diffusion_pytorch_b200 import _lib, losses, ops  # noqa: E402

import launch_check  # noqa: E402

FIXTURE = os.path.join(ROOT, "tests", "golden", "ops_calls.json.gz")

BF, F32, F64, I32, I64, U8 = torch.bfloat16, torch.float32, torch.float64, torch.int32, torch.int64, torch.uint8


def t(*shape, dtype=BF):
    return torch.zeros(*shape, dtype=dtype)


# ------------------------------------------------------------------------------------ the routes
def conv_gemm_case(dt, **kw):
    a, w, out = t(2, 16, 64, dtype=dt), t(32, 192, dtype=dt), t(2, 16, 32, dtype=dt)
    return dict(a=a, w=w, out=out, c_in=64, n_valid=32, taps=(-1, 0, 1), bias=t(32, dtype=F32), **kw)


def conv_gemm_up(dt):
    return dict(a=t(2, 16, 64, dtype=dt), w=t(2 * 32, 128, dtype=dt), out=t(2, 16, 64, dtype=dt), c_in=64,
                n_valid=32, taps=(0,), up_factor=2, bias=t(32, dtype=F32))


def gn_args(dt, **kw):
    return dict(x=t(2, 16, 32, dtype=dt), y=t(2, 16, 32, dtype=dt), stats=t(2, 4, 2, dtype=F64),
                gamma=t(32, dtype=F32), beta=t(32, dtype=F32), groups=4, **kw)


def ln_film_case(dt, **kw):
    return dict(x=t(2, 16, 32, dtype=dt), y=t(2, 16, 32, dtype=dt), **kw)


def attention_case(dt, D=64, lse=False):
    qkv, o = t(2, 16, 3 * 2 * D, dtype=dt), t(2, 16, 2 * D, dtype=dt)
    q, k, v = qkv[..., :2 * D], qkv[..., 2 * D:4 * D], qkv[..., 4 * D:]
    return dict(q=q, k=k, v=v, o=o, heads=2, scale=0.125, lse=t(2, 2, 16, dtype=F32) if lse else None,
                head_dim=D)


def attention_bwd_case(dt, D=64):
    qkv, o, d_o = t(2, 16, 3 * 2 * D, dtype=dt), t(2, 16, 2 * D, dtype=dt), t(2, 16, 2 * D, dtype=dt)
    dqkv = t(2, 16, 3 * 2 * D, dtype=dt)
    return dict(q=qkv[..., :2 * D], k=qkv[..., 2 * D:4 * D], v=qkv[..., 4 * D:], o=o, d_o=d_o,
                lse=t(2, 2, 16, dtype=F32), delta=t(2, 2, 16, dtype=F32), dq=dqkv[..., :2 * D],
                dk=dqkv[..., 2 * D:4 * D], dv=dqkv[..., 4 * D:], heads=2, scale=0.125, head_dim=D)


def stem_in_case(dt, **kw):
    ca = 1 if "append" in kw else 0
    if ca:
        kw["append"] = t(2, 1, 64, dtype=F32)
    return dict(x=t(2, 2, 64, dtype=F32), w=t(8, 2 + ca, 2, dtype=F32), bias=t(8, dtype=F32),
                out=t(2, 32, 8, dtype=dt), f=2, **kw)


def training_inputs(**kw):
    return dict(noise=t(2, 2, 64, dtype=F32), alpha=t(2, dtype=F32), beta=t(2, dtype=F32), **kw)


def stem_out_case(dt, Bh=2, **kw):
    return dict(h=t(Bh, 32, 8, dtype=dt), x=t(2, 2, 64, dtype=F32), w=t(2, 8, 3, dtype=F32),
                bias=t(2, dtype=F32), gate=t(Bh, 16, dtype=F32)[:, 4:], f=2, **kw)


def stem_out_bwd_case(dt, **kw):
    return dict(dv=t(2, 2, 64, dtype=F32), h=t(2, 32, 8, dtype=dt), x=t(2, 2, 64, dtype=F32),
                w=t(2, 8, 3, dtype=F32), bias=t(2, dtype=F32), gate=t(2, 16, dtype=F32), f=2,
                dh=t(2, 32, 8, dtype=dt), dw=t(2, 8, 3, dtype=F32), dbias=t(2, dtype=F32),
                dgate=t(2, 12, dtype=F32), **kw)


def stem_in_bwd_case(dt, **kw):
    return dict(dout=t(2, 32, 8, dtype=dt), x=t(2, 2, 64, dtype=F32), dw=t(8, 2, 2, dtype=F32),
                dbias=t(8, dtype=F32), f=2, **kw)


def wgrad_case(dt, ntaps):
    dw = t(3, 32, 48, dtype=F32) if ntaps == 3 else t(32, 56, dtype=F32)[:, :48]
    return dict(g=t(2, 16, 40, dtype=dt), x=t(2, 16, 64, dtype=dt), dw=dw, n=32, k=48,
                off=-1 if ntaps == 3 else 1, g_col0=8, x_col0=16, ntaps=ntaps)


def gn_bwd_case(dt, **kw):
    return dict(dxh=t(2, 16, 32, dtype=dt), x=t(2, 16, 32, dtype=dt), stats=t(2, 4, 2, dtype=F64),
                S=t(2, 4, 2, dtype=F64), dx=t(2, 16, 32, dtype=dt), groups=4, **kw)


def gn_silu_bwd_case(dt):
    return dict(da=t(2, 16, 32, dtype=dt), x=t(2, 16, 32, dtype=dt), stats=t(2, 4, 2, dtype=F64),
                gamma=t(32, dtype=F32), beta=t(32, dtype=F32), dxh=t(2, 16, 32, dtype=dt),
                dgamma=t(32, dtype=F32), dbeta=t(32, dtype=F32), S=t(2, 4, 2, dtype=F64), groups=4, eps=1e-6)


def ln_film_bwd_case(dt, full):
    kw = dict(dy=t(2, 16, 32, dtype=dt), x=t(2, 16, 32, dtype=dt), scale_shift=None, ss_stride=0,
              dx=t(2, 16, 32, dtype=dt))
    if full:
        kw.update(scale_shift=t(2, 80, dtype=F32), ss_stride=80, dss=t(2, 72, dtype=F32), dss_stride=72,
                  colsum=t(32, dtype=F32), dres=t(2, 16, 32, dtype=dt), eps=1e-5)
    return kw


def skip_gate_case(dt, stats):
    return dict(y=t(2, 16, 32, dtype=dt), skip=t(2, 16, 32, dtype=dt), gate=t(2, 40, dtype=F32),
                out=t(2, 16, 32, dtype=dt), stats=t(2, 4, 2, dtype=F64) if stats else None, groups=4)


def cond_bwd_case(dt, dcond):
    return dict(dss=t(2, 80, dtype=F32)[:, :64], cond=t(2, 24, dtype=F32), w=t(64, 24, dtype=dt),
                dw=t(64, 24, dtype=F32), dbias=t(64, dtype=F32), dcond=t(2, 24, dtype=F32) if dcond else None,
                N=64)


def stft_window():
    # the window losses caches per (n_fft, win_length, device): a tensor the call reads but is not passed
    return losses._window(64, 48, torch.device("cpu"))


def stft_fwd_case(dt, accumulate):
    x, y = t(3, 200, dtype=dt), t(3, 200, dtype=dt)
    return dict(x=x, y=y, res=(64, 16, 48), weights=(1.0, 0.5, 0.25), eps=1e-8, scale=1.0 / 3,
                _known=stft_window(), acc=t(1, dtype=F64), loss=t((), dtype=F32), accumulate=accumulate)


def stft_bwd_case(dt, accumulate, to_bf16):
    x, y = t(3, 200, dtype=dt), t(3, 200, dtype=dt)
    return dict(x=x, y=y, res=(64, 16, 48), weights=(1.0, 0.5, 0.25), eps=1e-8, scale=1.0 / 3,
                _known=stft_window(), stats=t(3, 2, dtype=F64), grad_out=t(1, dtype=F32), dx=t(3, 200, dtype=F32),
                dx_bf16=t(3, 200) if to_bf16 else None, accumulate=accumulate)


def _cases():
    """case id -> (function, builder of its keyword arguments)."""
    c = {}

    def add(name, fn, build):
        c[name] = (fn, build)

    for dn, dt in (("bf16", BF), ("f32", F32)):
        add(f"conv_gemm/plain/{dn}", ops.conv_gemm, lambda dt=dt: conv_gemm_case(dt))
        add(f"conv_gemm/stats/{dn}", ops.conv_gemm,
            lambda dt=dt: conv_gemm_case(dt, stats=t(2, 4, 2, dtype=F64), groups=4, residual=t(2, 16, 32, dtype=dt),
                                         gate=t(2, 48, dtype=F32)))
        add(f"conv_gemm/up2/{dn}", ops.conv_gemm, lambda dt=dt: conv_gemm_up(dt))
        add(f"gn_silu/{dn}", ops.gn_silu, lambda dt=dt: gn_args(dt, eps=1e-6))
        add(f"gn_stats/{dn}", ops.gn_stats, lambda dt=dt: dict(x=t(2, 16, 32, dtype=dt), stats=t(2, 4, 2, dtype=F64),
                                                               groups=4))
        for y2 in (False, True):
            for stats in (False, True):
                def ln(dt=dt, y2=y2, stats=stats):
                    kw = ln_film_case(dt, scale_shift=t(2, 72, dtype=F32), ss_stride=72, eps=1e-5, eps2=1e-6)
                    if y2:
                        kw["y2"] = t(2, 16, 32, dtype=dt)
                    if stats:
                        kw.update(stats_out=t(2, 4, 2, dtype=F64), groups=4)
                    return kw
                add(f"ln_film/{'y2' if y2 else 'y'}{'+stats' if stats else ''}/{dn}", ops.ln_film, ln)
        add(f"ln_film/plain_ln/{dn}", ops.ln_film, lambda dt=dt: ln_film_case(dt))
        for D in (32, 64, 128):
            for lse in (False, True):
                add(f"attention/D{D}{'+lse' if lse else ''}/{dn}", ops.attention,
                    lambda dt=dt, D=D, lse=lse: attention_case(dt, D, lse))
            add(f"attention_bwd/D{D}/{dn}", ops.attention_bwd, lambda dt=dt, D=D: attention_bwd_case(dt, D))
        add(f"skinny_linear/{dn}", ops.skinny_linear,
            lambda dt=dt: dict(x=t(2, 40, dtype=F32)[:, :32], w=t(48, 40, dtype=dt)[:, :32], bias=t(48, dtype=F32),
                               y=t(2, 56, dtype=F32)[:, :48], K=32, N=48, in_act=ops.ACT_SILU, out_act=ops.ACT_GELU))
        add(f"skinny_linear/no_bias/{dn}", ops.skinny_linear,
            lambda dt=dt: dict(x=t(2, 32, dtype=F32), w=t(48, 32, dtype=dt), bias=None, y=t(2, 48, dtype=F32),
                               K=32, N=48))
        add(f"silu_bf16/{dn}", ops.silu_bf16, lambda dt=dt: dict(x=t(2, 64, dtype=F32), y=t(2, 64, dtype=dt)))
        add(f"stem_in/plain/{dn}", ops.stem_in, lambda dt=dt: stem_in_case(dt))
        add(f"stem_in/stats/{dn}", ops.stem_in,
            lambda dt=dt: stem_in_case(dt, append=True, stats=t(2, 4, 2, dtype=F64), groups=4))
        add(f"stem_in/noise/{dn}", ops.stem_in,
            lambda dt=dt: stem_in_case(dt, **training_inputs(stats=t(2, 4, 2, dtype=F64), groups=4)))
        add(f"stem_out/inference/{dn}", ops.stem_out,
            lambda dt=dt: stem_out_case(dt, v_out=t(2, 2, 64, dtype=F32)))
        add(f"stem_out/adapter/{dn}", ops.stem_out,
            lambda dt=dt: stem_out_case(dt, append=t(2, 1, 64, dtype=F32), w_adapt=t(2, 3, dtype=F32),
                                        b_adapt=t(2, dtype=F32), v_out=t(2, 2, 64, dtype=F32)))
        add(f"stem_out/cfg/{dn}", ops.stem_out,
            lambda dt=dt: stem_out_case(dt, Bh=4, v_out=t(2, 2, 64, dtype=F32), cfg_scale=5.0))
        add(f"stem_out/sampler/{dn}", ops.stem_out,
            lambda dt=dt: stem_out_case(dt, x_next=t(2, 2, 64, dtype=F32), ab=t(4, dtype=F32)))
        add(f"stem_out/training/{dn}", ops.stem_out,
            lambda dt=dt: stem_out_case(dt, **training_inputs(loss_sum=t(1, dtype=F64), dv=t(2, 2, 64, dtype=F32))))
        add(f"stem_out/loss_only/{dn}", ops.stem_out,
            lambda dt=dt: stem_out_case(dt, loss_sum=t(1, dtype=F64)))
        for ntaps in (1, 3):
            add(f"wgrad/ntaps{ntaps}/{dn}", ops.wgrad, lambda dt=dt, ntaps=ntaps: wgrad_case(dt, ntaps))
        add(f"gn_silu_bwd/{dn}", ops.gn_silu_bwd, lambda dt=dt: gn_silu_bwd_case(dt))
        add(f"gn_bwd_apply/plain/{dn}", ops.gn_bwd_apply, lambda dt=dt: gn_bwd_case(dt))
        add(f"gn_bwd_apply/dres+colsum/{dn}", ops.gn_bwd_apply,
            lambda dt=dt: gn_bwd_case(dt, dres=t(2, 16, 32, dtype=dt), colsum=t(32, dtype=F32), eps=1e-6))
        for full in (False, True):
            add(f"ln_film_bwd/{'full' if full else 'plain'}/{dn}", ops.ln_film_bwd,
                lambda dt=dt, full=full: ln_film_bwd_case(dt, full))
        add(f"colsum/plain/{dn}", ops.colsum, lambda dt=dt: dict(x=t(2, 16, 32, dtype=dt), out=t(32, dtype=F32)))
        add(f"colsum/gate/{dn}", ops.colsum,
            lambda dt=dt: dict(x=t(2, 16, 32, dtype=dt), out=t(32, dtype=F32), gate=t(2, 40, dtype=F32)))
        for stats in (False, True):
            add(f"skip_gate/{'stats' if stats else 'plain'}/{dn}", ops.skip_gate,
                lambda dt=dt, stats=stats: skip_gate_case(dt, stats))
        add(f"skip_gate_bwd/{dn}", ops.skip_gate_bwd,
            lambda dt=dt: dict(dout=t(2, 16, 32, dtype=dt), y=t(2, 16, 32, dtype=dt), gate=t(2, 40, dtype=F32),
                               dys=t(2, 16, 32, dtype=dt), dgate=t(2, 48, dtype=F32)))
        for dcond in (False, True):
            add(f"cond_bwd/{'dcond' if dcond else 'params'}/{dn}", ops.cond_bwd,
                lambda dt=dt, dcond=dcond: cond_bwd_case(dt, dcond))
        add(f"stem_out_bwd/plain/{dn}", ops.stem_out_bwd, lambda dt=dt: stem_out_bwd_case(dt))
        add(f"stem_out_bwd/full/{dn}", ops.stem_out_bwd,
            lambda dt=dt: stem_out_bwd_case(dt, gscale=t(1, dtype=F32), append=t(2, 1, 64, dtype=F32),
                                            **training_inputs(w_adapt=t(2, 3, dtype=F32), dw_adapt=t(2, 3, dtype=F32),
                                                              db_adapt=t(2, dtype=F32), dxin=t(2, 3, 64, dtype=F32))))
        add(f"stem_in_bwd/plain/{dn}", ops.stem_in_bwd, lambda dt=dt: stem_in_bwd_case(dt))
        add(f"stem_in_bwd/full/{dn}", ops.stem_in_bwd,
            lambda dt=dt: stem_in_bwd_case(dt, append=t(2, 1, 64, dtype=F32), w=t(8, 3, 2, dtype=F32),
                                           dxin=t(2, 3, 64, dtype=F32), **training_inputs()))
        for acc in (False, True):
            add(f"stft_loss_fwd/{'acc' if acc else 'first'}/{dn}", losses._fwd,
                lambda dt=dt, acc=acc: stft_fwd_case(dt, acc))
            add(f"stft_loss_bwd/{'acc' if acc else 'first'}/{dn}", losses._bwd,
                lambda dt=dt, acc=acc: stft_bwd_case(dt, acc, to_bf16=False))
        add(f"stft_loss_bwd/to_bf16/{dn}", losses._bwd, lambda dt=dt: stft_bwd_case(dt, True, to_bf16=True))

    add("conv_gemm/gn/bf16", ops.conv_gemm,
        lambda: conv_gemm_case(BF, gn=(t(2, 4, 2, dtype=F64), t(64, dtype=F32), t(64, dtype=F32), 4, 1e-6),
                               block_n=64))
    add("conv_gemm/out_fp32/bf16", ops.conv_gemm,
        lambda: dict(a=t(2, 1, 64), w=t(48, 64), out=t(2, 1, 48, dtype=F32), c_in=64, n_valid=48))
    add("narrow_conv/plain/bf16", ops.narrow_conv,
        lambda: dict(x=t(2, 16, 8), y=t(2, 16, 8), stats_in=t(2, 4, 2, dtype=F64), gamma=t(8, dtype=F32),
                     beta=t(8, dtype=F32), w=t(8, 8, 3, dtype=F32), bias=t(8, dtype=F32), groups=4))
    add("narrow_conv/full/bf16", ops.narrow_conv,
        lambda: dict(x=t(2, 16, 32), y=t(2, 16, 32), stats_in=t(2, 8, 2, dtype=F64), gamma=t(32, dtype=F32),
                     beta=t(32, dtype=F32), w=t(32, 32, 3, dtype=F32), bias=None, groups=8,
                     residual=t(2, 16, 32), scale_shift=t(2, 72, dtype=F32), ss_stride=72,
                     stats_out=t(2, 8, 2, dtype=F64), gn_eps=1e-6, ln_eps=1e-5, w_packed=t(32, 96)))
    add("narrow_conv_bwd/bf16", ops.narrow_conv_bwd,
        lambda: dict(dy=t(2, 16, 8), x=t(2, 16, 8), stats_in=t(2, 4, 2, dtype=F64), gamma=t(8, dtype=F32),
                     beta=t(8, dtype=F32), w=t(8, 8, 3, dtype=F32), dxh=t(2, 16, 8), dgamma=t(8, dtype=F32),
                     dbeta=t(8, dtype=F32), S=t(2, 4, 2, dtype=F64), dw=t(8, 8, 3, dtype=F32),
                     dbias=t(8, dtype=F32), groups=4, gn_eps=1e-6))
    add("time_features", ops.time_features,
        lambda: dict(sigma=t(2, dtype=F32), freqs=t(8, dtype=F32), out=t(2, 24, dtype=F32)))
    add("sampler_step", ops.sampler_step,
        lambda: dict(x=t(2, 2, 64, dtype=F32), v=t(2, 2, 64, dtype=F32), ab=t(4, dtype=F32),
                     x_next=t(2, 2, 64, dtype=F32)))
    add("step_select", ops.step_select,
        lambda: dict(step=t(1, dtype=I32), ctrl=t(3, dtype=I64), ab_table=t(6, 4, dtype=F32),
                     ab_out=t(4, dtype=F32), ss_out=t(2, 72, dtype=F32)))
    add("step_advance", ops.step_advance, lambda: dict(step=t(1, dtype=I32)))
    add("inpaint_blend", ops.inpaint_blend,
        lambda: dict(x=t(2, 2, 64, dtype=F32), source=t(2, 2, 64, dtype=F32), noise=t(2, 2, 64, dtype=F32),
                     mask_u8=t(2, 2, 64, dtype=U8), ab=t(4, dtype=F32)))
    add("arv_step", ops.arv_step,
        lambda: dict(chan=t(2, 3, 64, dtype=F32), v=t(2, 2, 64, dtype=F32), sig_next=t(2, 64, dtype=F32)))
    add("fir_resample/forward", ops.fir_resample,
        lambda: dict(x=t(2, 64, dtype=F32), bank=t(3, 2 * 5 + 2, dtype=F32), factor_in=2, factor_out=3, half=5,
                     t_out=96))
    add("fir_resample/adjoint", ops.fir_resample,
        lambda: dict(x=t(2, 96, dtype=F32), bank=t(3, 2 * 5 + 2, dtype=F32), factor_in=2, factor_out=3, half=5,
                     t_out=96, adjoint_of=64))
    for log in (False, True):
        add(f"mel_spectrogram/{'log' if log else 'linear'}", ops.mel_spectrogram,
            lambda log=log: dict(wave=t(2, 256, dtype=F32), window=t(64, dtype=F32), fb=t(33, 16, dtype=F32),
                                 band=t(32, dtype=I32), n_fft=64, hop=16, pad=8, apply_log=log,
                                 center_pad=32 if log else 0))
    add("to_flat", ops.to_flat, lambda: dict(spec=t(2, 8, 10, dtype=F32), w=t(8, 32, dtype=F32), hop=16, pad=8))
    for dspec, dw in ((True, True), (True, False), (False, True)):
        add(f"to_flat_bwd/{'dspec' if dspec else ''}{'+' if dspec and dw else ''}{'dw' if dw else ''}",
            ops.to_flat_bwd,
            lambda dspec=dspec, dw=dw: dict(spec=t(2, 8, 10, dtype=F32), w=t(8, 32, dtype=F32),
                                            dout=t(2, 160, dtype=F32), hop=16, pad=8, need_dspec=dspec,
                                            need_dw=dw))
    add("ln_fold_bwd", ops.ln_fold_bwd,
        lambda: dict(w=t(48, 32, dtype=F32), g=t(32, dtype=F32), b=t(32, dtype=F32),
                     dwf=t(48, 40, dtype=F32)[:, :32], dbf=t(48, dtype=F32), dw=t(48, 32, dtype=F32),
                     dg=t(32, dtype=F32), db=t(32, dtype=F32)))
    return c


CASES = _cases()


# --------------------------------------------------------------------------------- the recording
class FakeLib:
    """Every adp_* attribute records its call and returns 0 (success)."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("adp_"):
            raise AttributeError(name)

        def entry(*args):
            self.calls.append((name, args))
            return 0
        return entry


def _float(v):
    return ["f", "%016x" % struct.unpack("<Q", struct.pack("<d", v))[0]]


class Call:
    """One ops call: its known tensors (arguments, then allocations) and the encoding of values."""

    def __init__(self):
        self.tensors = []

    def add(self, v):
        if isinstance(v, torch.Tensor):
            self.tensors.append(v)
        elif isinstance(v, (tuple, list)):
            for x in v:
                self.add(x)

    def pointer(self, p):
        for i, x in enumerate(self.tensors):
            st = x.untyped_storage()
            if st.data_ptr() <= p < st.data_ptr() + st.nbytes():
                return ["P", i, p - st.data_ptr()]
        return None

    def arg(self, v):
        if v is None:
            return None
        if isinstance(v, int):
            p = self.pointer(v)
            assert p is not None or abs(v) < 2 ** 40, f"pointer {v:#x} into no known tensor"
            return v if p is None else p
        if isinstance(v, float):
            return _float(v)
        if hasattr(v, "_obj") and isinstance(v._obj, C.Structure):       # C.byref(args)
            return ["S", type(v._obj).__name__, [[n, self.field(getattr(v._obj, n), ty)]
                                                 for n, ty in v._obj._fields_]]
        raise TypeError(f"unrecorded argument type {type(v)}")

    def field(self, v, ty):
        if ty is C.c_void_p:
            if v is None:
                return None
            p = self.pointer(v)
            assert p is not None, f"struct pointer {v:#x} into no known tensor"
            return p
        if isinstance(v, float):
            return _float(v)
        if isinstance(v, int):
            return v
        return list(v)                                                 # int32_t arrays (tap_off)

    def result(self, r):
        if isinstance(r, torch.Tensor):
            return ["R", next(i for i, x in enumerate(self.tensors) if x is r)]
        if isinstance(r, (tuple, list)):
            return [self.result(x) for x in r]
        assert r is None, type(r)
        return None


@contextlib.contextmanager
def allocations(call):
    """Tensors `ops` and `losses` allocate inside the call join the known tensors in order."""
    mp = pytest.MonkeyPatch()
    for name in ("empty", "zeros", "empty_like", "zeros_like"):
        real = getattr(torch, name)

        def alloc(*a, _real=real, **k):
            x = _real(*a, **k)
            call.tensors.append(x)
            return x
        mp.setattr(torch, name, alloc)
    try:
        yield
    finally:
        mp.undo()


def record(case):
    """(C functions called with their encoded arguments, trace records, encoded result) of one case."""
    fn, build = CASES[case]
    kwargs = build()
    known = kwargs.pop("_known", ())
    fake = FakeLib()
    call = Call()
    b = inspect.signature(fn).bind(**kwargs)
    b.apply_defaults()
    for v in b.arguments.values():
        call.add(v)
    call.add(known)
    mp = pytest.MonkeyPatch()
    mp.setattr(_lib, "lib", lambda: fake)
    mp.setattr(ops, "_stream", lambda: None)
    try:
        with ops.trace() as tr, allocations(call):
            r = fn(**kwargs)
    finally:
        mp.undo()
    return fake.calls, tr.records, call, r


def encode(case):
    calls, records, call, r = record(case)
    return {"calls": [[sym, [call.arg(a) for a in args]] for sym, args in calls],
            "trace": [[rec["name"], rec["flops"], rec["bytes"]] for rec in records],
            "result": call.result(r)}


@pytest.fixture(scope="module")
def fixture():
    with gzip.open(FIXTURE, "rt") as f:
        return json.load(f)


def test_cases_cover_every_launching_function():
    called = {fn.__name__ for fn, _ in CASES.values()}
    missing = sorted(set(launch_check.launching_functions()) - called)
    assert not missing, f"no case calls {missing}"


def test_fixture_covers_every_case(fixture):
    assert sorted(fixture) == sorted(CASES)


@pytest.mark.parametrize("case", sorted(CASES))
def test_ops_call(case, fixture):
    got = json.loads(json.dumps(encode(case)))
    want = fixture[case]
    for part in ("calls", "trace", "result"):
        assert got[part] == want[part], f"{case}: {part}\n  got  {json.dumps(got[part])}\n  want {json.dumps(want[part])}"


def test_trace_symbol_names_the_function_called():
    """Each trace record's `symbol` is the C entry point its launch called (the launch checker's
    Shadow.symbols and the fp32 coverage test read it)."""
    wrong = set()
    for case in sorted(CASES):
        calls, records, _, _ = record(case)
        assert len(calls) == len(records), case
        wrong |= {(rec["symbol"], sym) for (sym, _), rec in zip(calls, records) if rec["symbol"] != sym}
    assert not wrong, "trace symbol != entry point called: " + ", ".join(f"{a} for {b}" for a, b in sorted(wrong))


if __name__ == "__main__" and "--write" in sys.argv:
    data = {case: encode(case) for case in sorted(CASES)}
    with gzip.GzipFile(FIXTURE, "wb", mtime=0) as f:
        f.write(json.dumps(data, separators=(",", ":"), sort_keys=True).encode())
    print(f"{len(data)} cases, {sum(len(v['calls']) for v in data.values())} calls; "
          f"wrote {FIXTURE} ({os.path.getsize(FIXTURE)} bytes)")
