"""The fp32 verification kernels (csrc/verify_f32.cu, verify_f32_bwd.cu) launch by launch on the GPU.

  a. edge launches: each case runs through `ops` once under Shadow(probe=True) and once under
     Shadow(guard=True) with random fp32 data, held to the fp32 bound of tests/launch_check.py
     (err <= 2^-23 |ref| + 10 sqrt(n) 2^-24 absref), at the shapes where index arithmetic goes wrong:
     one- and two-row convs, ragged T, wide output pitches, the residual in place, strided gates,
     the resampling phases, GroupNorm at 1 and 64 groups and at C = 2048, near-constant groups,
     LayerNorm rows of 8 ... 2048 with strided FiLM rows, attention at D = 32 / 64 / 128 over one
     key or one query, q|k|v pitches, the stem envelope corners, and every backward kind;
  b. programs, each under Shadow, then under Shadow(guard=True), then eager / captured / replayed
     with CUDA graphs: the tiny nets (also at T = 4080, B = 3 and at T = 16, innermost length 1), the
     text net at CFG 5 (B = 2 and 3), the README net at 2^13, net (b) of test_widths_gpu.py, the
     64-in / 64-out boundary at c0 = 256, XUNets with a standalone ModulationItem and with SkipAdd,
     the SkipCat DiffusionAR net and the DiffusionUpsampler's net; the tiny 5-step sample; and the
     fp32 training tests of test_train_fp32_gpu.py, test_wide_boundary_gpu.py and test_xunet_gpu.py
     run whole under the checker (their own float64 comparisons included, CUDA graphs off);
  c. the branch v - x of the inference programs against the float64 oracle on the same inputs:
     rel-L2 <= 1e-5 for the tiny, ragged, XUNet, SkipCat and upsampler nets, 1e-4 for the README,
     widths and wide-boundary nets, times |s| + |1 - s| under guidance s; 1e-4 rel-L2 of the sample;
  d. coverage: every adp_f32_* entry point `ops` can call is reached by a checked edge launch, by
     the name ops._launch records for it (the C function called).
"""
import inspect
import re

import pytest
import torch

import launch_check as lc

pytestmark = pytest.mark.gpu

DEV = "cuda"
F32, F64 = torch.float32, torch.float64


@pytest.fixture(scope="module")
def ops():
    from audio_diffusion_pytorch_b200 import ops
    ops.device_check()
    return ops


class R:
    def __init__(self, seed):
        self.g = torch.Generator(device=DEV).manual_seed(seed)

    def n(self, *shape, scale=1.0):
        return torch.randn(*shape, generator=self.g, device=DEV) * scale

    def u(self, *shape):
        return torch.rand(*shape, generator=self.g, device=DEV)


def _conv(ops, r, *, B=2, T=64, c_in=32, n_valid=32, taps=(-1, 0, 1), up=0, ldo=None, residual=False,
          gate_ld=None, stats=False):
    """f32_conv_gemm with weights packed as the fp32 mode packs them."""
    phases = up if up > 1 else 1
    with ops.pack_dtype(F32):
        if up > 1:
            w = ops.pack_upsample_conv(r.n(n_valid, c_in, 3, scale=c_in ** -0.5), up)
        else:
            w = ops.pack_conv(r.n(n_valid, c_in, len(taps), scale=c_in ** -0.5))
    a = r.n(B, T, c_in)
    out = r.n(B, T, ldo or phases * n_valid)
    gate = r.n(B, gate_ld)[:, :n_valid] if gate_ld else None
    st = torch.zeros(B, 8, 2, dtype=F64, device=DEV) if stats else None
    ops.conv_gemm(a, w, out, c_in=c_in, n_valid=n_valid, taps=taps, up_factor=up, bias=r.n(n_valid),
                  residual=out if residual else None, gate=gate, stats=st, groups=8)


def _conv_down(ops, r, f=4, B=2, T=256, ci=32, co=64):
    """The downsample view: [B, T/f, f ci] of the channels-last input, one tap."""
    with ops.pack_dtype(F32):
        w = ops.pack_conv(r.n(co, ci, f, scale=(ci * f) ** -0.5))
    x = r.n(B, T, ci)
    ops.conv_gemm(x.view(B, T // f, f * ci), w, r.n(B, T // f, co), c_in=f * ci, n_valid=co, taps=(0,),
                  bias=r.n(co))


def _gn(ops, r, *, B=2, T=100, C=64, G=8, near_constant=False, silu=True):
    x = r.n(B, T, C)
    if near_constant:
        x = 100.0 + 1e-3 * x                  # var << mean^2
    st = torch.zeros(B, G, 2, dtype=F64, device=DEV)
    ops.gn_stats(x, st, G)
    if silu:
        ops.gn_silu(x, torch.empty_like(x), lc.stats_of(x, G), 1 + 0.1 * r.n(C), 0.1 * r.n(C), G)


def _ln(ops, r, *, B=2, T=37, C=48, ss_pad=0, y2=False, film=True):
    x = r.n(B, T, C) * 3 + 1
    ss = (0.3 * r.n(B, 2 * C + ss_pad)) if film else None
    ops.ln_film(x, torch.empty_like(x), ss, 2 * C + ss_pad if film else 0,
                y2=torch.empty_like(x) if y2 else None)


def _att(ops, r, *, B=2, H=2, D=64, Tq=40, Tk=40, packed=False, lse=False, E=None):
    mid = H * D
    if packed:                                 # q|k|v of one projection: row pitch 3 H D
        qkv = r.n(B, Tq, 3 * mid)
        q, k, v = qkv[..., :mid], qkv[..., mid:2 * mid], qkv[..., 2 * mid:]
    else:
        q, k, v = r.n(B, Tq, mid), r.n(B, Tk, E or mid)[..., :mid], r.n(B, Tk, E or mid)[..., :mid]
    o = torch.empty(B, Tq, mid, device=DEV)
    ops.attention(q, k, v, o, H, D ** -0.5, lse=torch.empty(B, H, Tq, device=DEV) if lse else None, head_dim=D)


def _linear(ops, r, *, B=3, K=96, N=80, ldx=None, in_act=0, out_act=0):
    x = r.n(B, ldx or K)
    ops.skinny_linear(x, r.n(N, K, scale=K ** -0.5), r.n(N), torch.empty(B, N, device=DEV), K, N, in_act, out_act)


def _stem_in(ops, r, *, B=2, cx=2, ca=0, c0=32, f=2, T=64, noise=False, stats=False):
    cin = cx + ca
    ops.stem_in(r.n(B, cx, T), r.n(c0, cin, f, scale=(cin * f) ** -0.5), r.n(c0), torch.empty(B, T // f, c0, device=DEV),
                f, append=r.n(B, ca, T) if ca else None, noise=r.n(B, cx, T) if noise else None,
                alpha=r.u(B) if noise else None, beta=r.u(B) if noise else None,
                stats=torch.zeros(B, 8, 2, dtype=F64, device=DEV) if stats else None)


def _stem_out(ops, r, *, B=2, cx=2, ca=0, co=2, c0=32, f=2, T=64, adapter=False, cfg=None, x_next=False,
              alias=False, loss=False, gate_ld=None):
    cin = cx + ca
    Bh = 2 * B if cfg is not None else B
    x = r.n(B, cx, T)
    kw = dict(append=r.n(B, ca, T) if ca else None)
    if adapter:
        kw.update(w_adapt=r.n(co, cin, scale=cin ** -0.5), b_adapt=r.n(co))
    if x_next:
        kw.update(x_next=x if alias else torch.empty(B, co, T, device=DEV),
                  ab=torch.tensor([0.8, 0.6, 0.9, 0.43589], device=DEV))
    else:
        kw.update(v_out=torch.empty(B, co, T, device=DEV))
    if loss:
        kw.update(noise=r.n(B, cx, T), alpha=r.u(B), beta=r.u(B), loss_sum=torch.zeros(1, dtype=F64, device=DEV),
                  dv=torch.empty(B, co, T, device=DEV))
    gate = r.n(Bh, gate_ld or co)[:, :co]
    ops.stem_out(r.n(Bh, T // f, c0), x, r.n(co, c0, 3, scale=(3 * c0) ** -0.5), r.n(co), gate, f,
                 cfg_scale=cfg, **kw)


# ----------------------------------------------------------------------------- backward
def _wgrad(ops, r, *, B=2, T=50, n=24, k=40, ntaps=1, off=0, g_col0=0, x_col0=0, g_pad=0):
    g = r.n(B, T, g_col0 + n + g_pad)[..., :g_col0 + n + max(0, g_pad - 8)]     # ldg > g_cols when g_pad > 8
    x = r.n(B, T, x_col0 + k)
    dw = r.n(3, n, k + 8)[..., :k] if ntaps == 3 else r.n(n, k + 8)[:, :k]
    ops.wgrad(g, x, dw, n=n, k=k, off=off, g_col0=g_col0, x_col0=x_col0, ntaps=ntaps)


def _gn_bwd(ops, r, *, B=2, T=30, C=64, G=8, dres=False, colsum=False):
    x = r.n(B, T, C) + 0.5
    st = lc.stats_of(x, G)
    gamma, beta = 1 + 0.1 * r.n(C), 0.1 * r.n(C)
    dxh, S = torch.empty_like(x), torch.zeros(B, G, 2, dtype=F64, device=DEV)
    ops.gn_silu_bwd(r.n(B, T, C), x, st, gamma, beta, dxh, r.n(C), r.n(C), S, G)
    ops.gn_bwd_apply(dxh, x, st, S, torch.empty_like(x), G, dres=r.n(B, T, C) if dres else None,
                     colsum=r.n(C + 16)[:C] if colsum else None)


def _ln_bwd(ops, r, *, B=2, T=21, C=48, dss_pad=8, dres=True, colsum=True, film=True):
    x = r.n(B, T, C) * 2 + 1
    ss = 0.3 * r.n(B, 2 * C + 8) if film else None
    ops.ln_film_bwd(r.n(B, T, C), x, ss, 2 * C + 8 if film else 0, torch.empty_like(x),
                    dss=r.n(B, 2 * C + dss_pad) if film else None, dss_stride=2 * C + dss_pad if film else 0,
                    colsum=r.n(C) if colsum else None, dres=r.n(B, T, C) if dres else None)


def _colsum(ops, r, *, B=2, T=17, C=6144, gate=True):
    ops.colsum(r.n(B, T, C), r.n(C), gate=r.n(B, 2 * C)[:, C // 2:C // 2 + C] if gate else None)


def _skip(ops, r, *, B=2, T=33, C=64, stats=True):
    y, skip = r.n(B, T, C), r.n(B, T, C)
    gate = r.n(B, C + 16)[:, :C]
    ops.skip_gate(y, skip, gate, torch.empty_like(y), torch.zeros(B, 8, 2, dtype=F64, device=DEV) if stats else None, 8)
    ops.skip_gate_bwd(r.n(B, T, C), y, gate, torch.empty_like(y), r.n(B, C + 8)[:, :C])


def _cond_bwd(ops, r, *, B=3, N=96, K=72, dcond=True):
    ops.cond_bwd(r.n(B, N + 16)[:, :N], r.n(B, K), r.n(N, K), torch.empty(N, K, device=DEV), torch.empty(N, device=DEV),
                 r.n(B, K) if dcond else None, N)


def _stem_out_bwd(ops, r, *, B=2, cx=3, ca=1, co=2, c0=32, f=2, T=48, adapter=True, noise=True, gscale=True,
                  dxin=True):
    cin = cx + ca
    kw = dict(append=r.n(B, ca, T) if ca else None, gscale=r.u(1) if gscale else None,
              dxin=torch.empty(B, cin, T, device=DEV) if dxin else None)
    if noise:
        kw.update(noise=r.n(B, cx, T), alpha=r.u(B), beta=r.u(B))
    if adapter:
        kw.update(w_adapt=r.n(co, cin), dw_adapt=r.n(co, cin), db_adapt=r.n(co))
    ops.stem_out_bwd(r.n(B, co, T), r.n(B, T // f, c0), r.n(B, cx, T), r.n(co, c0, 3), r.n(co), r.n(B, co + 6)[:, :co],
                     f, torch.empty(B, T // f, c0, device=DEV), r.n(co, c0, 3), r.n(co + 6)[:co],
                     r.n(B, co + 6)[:, :co], **kw)


def _stem_in_bwd(ops, r, *, B=2, cx=2, ca=1, c0=32, f=4, T=64, noise=True, dxin=True):
    cin = cx + ca
    ops.stem_in_bwd(r.n(B, T // f, c0), r.n(B, cx, T), r.n(c0, cin, f), r.n(c0), f, append=r.n(B, ca, T) if ca else None,
                    noise=r.n(B, cx, T) if noise else None, alpha=r.u(B) if noise else None,
                    beta=r.u(B) if noise else None, w=r.n(c0, cin, f) if dxin else None,
                    dxin=r.n(B, cin, T) if dxin else None)


def _att_bwd(ops, r, *, B=2, H=2, D=64, Tq=24, Tk=40):
    mid = H * D
    q, k, v = r.n(B, Tq, mid), r.n(B, Tk, mid), r.n(B, Tk, mid)
    o, lse = torch.empty(B, Tq, mid, device=DEV), torch.empty(B, H, Tq, device=DEV)
    scale = D ** -0.5
    ops.attention(q, k, v, o, H, scale, lse=lse, head_dim=D)      # outside the check: the forward's o and lse
    return lambda: ops.attention_bwd(q, k, v, o, r.n(B, Tq, mid), lse, torch.empty(B * H * Tq + 64, device=DEV),
                                     torch.empty(B, Tq, mid, device=DEV), torch.empty(B, Tk, mid, device=DEV),
                                     torch.empty(B, Tk, mid, device=DEV), H, scale, head_dim=D)


CASES = {
    "conv_k3_T1": lambda o, r: _conv(o, r, B=1, T=1),
    "conv_k3_T2": lambda o, r: _conv(o, r, T=2),
    "conv_k3_T1000_B3": lambda o, r: _conv(o, r, B=3, T=1000, stats=True),
    "conv_k1_wide_ldo": lambda o, r: _conv(o, r, taps=(0,), ldo=80),
    "conv_residual_in_place": lambda o, r: _conv(o, r, residual=True, T=77),
    "conv_gate_ld": lambda o, r: _conv(o, r, gate_ld=64, residual=True),
    "conv_down_f4": lambda o, r: _conv_down(o, r),
    "conv_up_f2": lambda o, r: _conv(o, r, up=2, T=33),
    "conv_up_f4": lambda o, r: _conv(o, r, up=4, T=33, residual=True),
    "conv_n8_pad16": lambda o, r: _conv(o, r, n_valid=8),            # packed rows: round_up(8, 16)
    "conv_cin8": lambda o, r: _conv(o, r, c_in=8, n_valid=32, T=50),
    "gn_groups1": lambda o, r: _gn(o, r, G=1),
    "gn_groups64": lambda o, r: _gn(o, r, G=64, C=128),
    "gn_C2048": lambda o, r: _gn(o, r, C=2048, T=9),
    "gn_near_constant": lambda o, r: _gn(o, r, near_constant=True),
    "ln_C8": lambda o, r: _ln(o, r, C=8),
    "ln_C48_y2": lambda o, r: _ln(o, r, C=48, ss_pad=16, y2=True),
    "ln_C2048": lambda o, r: _ln(o, r, C=2048, T=5, ss_pad=64),
    "ln_plain_y2": lambda o, r: _ln(o, r, C=64, film=False, y2=True),
    "att_D32": lambda o, r: _att(o, r, D=32, H=3),
    "att_D64_lse": lambda o, r: _att(o, r, lse=True),
    "att_D128": lambda o, r: _att(o, r, D=128, H=1, lse=True),
    "att_Tk1": lambda o, r: _att(o, r, Tk=1),
    "att_Tk1_lse": lambda o, r: _att(o, r, Tk=1, lse=True),
    "att_Tq1": lambda o, r: _att(o, r, Tq=1, Tk=7),
    "att_cross_E2048": lambda o, r: _att(o, r, H=16, D=128, Tq=16, Tk=8),
    "att_qkv_pitch": lambda o, r: _att(o, r, packed=True, Tq=33, lse=True),
    "linear_gelu_in": lambda o, r: _linear(o, r, in_act=1),
    "linear_silu_in_gelu_out": lambda o, r: _linear(o, r, in_act=2, out_act=1),
    "linear_silu_out_ldx": lambda o, r: _linear(o, r, out_act=2, ldx=128),
    "linear_cond_table": lambda o, r: _linear(o, r, B=100, K=256, N=12288),    # a guided 50-step table
    "silu": lambda o, r: o.silu_bf16(r.n(3, 77), torch.empty(3, 77, device=DEV)),
    "stem_in_corner_64x2": lambda o, r: _stem_in(o, r, cx=63, ca=1, f=2, c0=256, T=32, stats=True),
    "stem_in_noise_append": lambda o, r: _stem_in(o, r, cx=2, ca=1, f=4, noise=True),
    "stem_out_corner_64": lambda o, r: _stem_out(o, r, cx=64, co=64, c0=256, f=1, T=16),
    "stem_out_adapter_append": lambda o, r: _stem_out(o, r, cx=3, ca=2, co=2, adapter=True, gate_ld=8),
    "stem_out_cfg": lambda o, r: _stem_out(o, r, cfg=5.0),
    "stem_out_x_next_alias": lambda o, r: _stem_out(o, r, x_next=True, alias=True, cfg=3.0),
    "stem_out_loss": lambda o, r: _stem_out(o, r, loss=True, f=4),
    "wgrad_1": lambda o, r: _wgrad(o, r),
    "wgrad_3_cols": lambda o, r: _wgrad(o, r, ntaps=3, off=-1, g_col0=8, x_col0=16, g_pad=24),
    "wgrad_T1": lambda o, r: _wgrad(o, r, T=1, ntaps=3, off=-1),
    "gn_bwd_g1": lambda o, r: _gn_bwd(o, r, G=1, dres=True, colsum=True),
    "gn_bwd_g64": lambda o, r: _gn_bwd(o, r, G=64, C=128),
    "ln_bwd_C8": lambda o, r: _ln_bwd(o, r, C=8),
    "ln_bwd_C48": lambda o, r: _ln_bwd(o, r, C=48, dres=False),
    "ln_bwd_C2048": lambda o, r: _ln_bwd(o, r, C=2048, T=6, dss_pad=64),
    "ln_bwd_plain": lambda o, r: _ln_bwd(o, r, C=64, film=False, colsum=False),
    "colsum_gate_6144": lambda o, r: _colsum(o, r),
    "skip_gate": lambda o, r: _skip(o, r),
    "cond_bwd_dcond": lambda o, r: _cond_bwd(o, r),
    "cond_bwd": lambda o, r: _cond_bwd(o, r, dcond=False),
    "stem_out_bwd_adapter": lambda o, r: _stem_out_bwd(o, r),
    "stem_out_bwd_identity": lambda o, r: _stem_out_bwd(o, r, cx=2, ca=0, adapter=False, noise=False, gscale=False),
    "stem_in_bwd_dxin": lambda o, r: _stem_in_bwd(o, r),
    "stem_in_bwd": lambda o, r: _stem_in_bwd(o, r, ca=0, noise=False, dxin=False),
}
ATT_BWD = {"att_bwd_D32": dict(D=32, H=3), "att_bwd_D64": dict(), "att_bwd_D128": dict(D=128, H=1),
           "att_bwd_Tk1": dict(Tk=1), "att_bwd_Tq1": dict(Tq=1, Tk=9)}


def _run(ops, case, mode, seed):
    r = R(seed)
    if case in ATT_BWD:
        call = _att_bwd(ops, r, **ATT_BWD[case])
    else:
        def call():
            CASES[case](ops, r)
    torch.cuda.synchronize()
    with lc.Shadow(probe=mode == "probe", guard=mode == "guard") as sh:
        call()
    torch.cuda.synchronize()
    assert sh.n_checked == sh.n_launch > 0, sh.table()
    if mode == "guard":
        assert sh.n_guarded == sh.n_launch
    else:
        assert sh.probed
    return sh


ALL = sorted(CASES) + sorted(ATT_BWD)


@pytest.mark.parametrize("mode", ["probe", "guard"])
@pytest.mark.parametrize("case", ALL)
def test_f32_edge_launch(ops, case, mode):
    sh = _run(ops, case, mode, 100 + ALL.index(case))
    print(f"\n{case} ({mode})\n{sh.table()}")


# ------------------------------------------------------------------------------ programs
def rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm())


@pytest.fixture(scope="module")
def adp():
    import audio_diffusion_pytorch_b200 as adp_
    from audio_diffusion_pytorch_b200 import ops
    ops.device_check()
    print("\n" + torch.cuda.get_device_name(0))
    return adp_


TINY = dict(in_channels=2, channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 2, 2],
            attentions=[0, 0, 1], attention_heads=2, attention_features=64)
TINY_TEXT = dict(TINY, cross_attentions=[0, 1, 1], use_embedding_cfg=True, embedding_max_length=8,
                 embedding_features=32)
README = dict(in_channels=2, channels=[8, 32, 64, 128, 256, 512, 512, 1024, 1024],
              factors=[1, 4, 4, 4, 2, 2, 2, 2, 2], items=[1, 2, 2, 2, 2, 2, 2, 4, 4],
              attentions=[0, 0, 0, 0, 0, 1, 1, 1, 1], attention_heads=8, attention_features=64)
BOUNDARY = dict(in_channels=64, channels=[256, 256, 256], factors=[2, 2, 2], items=[1, 1, 1])


def _dbl(kw):
    return {k: (v.double() if torch.is_tensor(v) else
                [None if t is None else t.double() for t in v] if isinstance(v, list) else v) for k, v in kw.items()}


def _dev(kw):
    return {k: (v.to(DEV) if torch.is_tensor(v) else
                [None if t is None else t.to(DEV) for t in v] if isinstance(v, list) else v) for k, v in kw.items()}


def _model(oracle_port, adp, cfg, B, T, seed, scale=None):
    """(oracle, model, x, sigma, kw) of a UNetV0 DiffusionModel config."""
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**cfg)
    model = adp.DiffusionModel(net_t=adp.UNetV0, **cfg).to(DEV)
    model.net.load_reference_parameters(ref.net)
    g = torch.Generator().manual_seed(seed)
    x, sigma = torch.randn(B, cfg["in_channels"], T, generator=g), torch.rand(B, generator=g)
    kw = {}
    if cfg.get("embedding_features"):
        kw = dict(embedding=torch.randn(B, cfg["embedding_max_length"], cfg["embedding_features"], generator=g),
                  embedding_scale=scale or 1.0)
    return ref, model, x, sigma, kw


def _xunet(oracle_port, adp, case):
    from test_xunet_gpu import inputs, oracle_kw, pair
    ref, model = pair(oracle_port, adp, case)
    x, sigma, emb, channels = inputs(case, seed=9)
    return ref, model, x, sigma, oracle_kw(emb, channels)


def _skipcat_ar(oracle_port, adp):
    """DiffusionAR's net: use_modulation=False (SkipCat merges), x | per-position sigma in."""
    from test_train_fp32_gpu import ATT
    cfg = dict(ATT, in_channels=2, length=4096, num_splits=4)
    torch.manual_seed(0)
    ref = oracle_port.DiffusionARPort(**cfg)
    model = adp.DiffusionAR(net_t=adp.UNetV0, **cfg).to(DEV)
    model.net.load_reference_parameters(ref.net)
    g = torch.Generator().manual_seed(12)
    sig = torch.rand(2, 1, 4, generator=g).repeat_interleave(1024, dim=2)
    return ref, model, torch.cat([torch.randn(2, 2, 4096, generator=g), sig], 1), None, {}


def _upsampler(oracle_port, adp):
    from test_train_fp32_gpu import CFG
    cfg = {k: v for k, v in CFG.items() if k != "in_channels"}
    torch.manual_seed(0)
    ref = oracle_port.DiffusionUpsamplerPort(upsample_factor=16, in_channels=2, **cfg)
    model = adp.DiffusionUpsampler(net_t=adp.UNetV0, upsample_factor=16, in_channels=2, **cfg).to(DEV)
    model.net.load_reference_parameters(ref.net)
    g = torch.Generator().manual_seed(13)
    x, sigma = torch.randn(2, 2, 4096, generator=g), torch.rand(2, generator=g)
    return ref, model, x, sigma, dict(append_channels=ref.reupsample(torch.randn(2, 2, 4096, generator=g)))


def _widths_b():
    from test_widths_gpu import NET_B
    return NET_B


# name -> (builder(oracle_port, adp) -> (oracle, model, x, sigma or None, kw), branch bound at scale 1)
PROGRAMS = {
    "tiny": (lambda o, a: _model(o, a, TINY, 2, 4096, 11), 1e-5),
    "tiny_T4080_B3": (lambda o, a: _model(o, a, TINY, 3, 4080, 11), 1e-5),
    "tiny_T16": (lambda o, a: _model(o, a, TINY, 1, 16, 11), 1e-5),
    "text_cfg5": (lambda o, a: _model(o, a, TINY_TEXT, 2, 4096, 11, 5.0), 1e-5),
    "text_cfg5_B3": (lambda o, a: _model(o, a, TINY_TEXT, 3, 2048, 11, 5.0), 1e-5),
    "readme_2e13": (lambda o, a: _model(o, a, README, 1, 2 ** 13, 11), 1e-4),
    "widths_b_T1024": (lambda o, a: _model(o, a, _widths_b(), 2, 1024, 11), 1e-4),
    "boundary_64x64_c0_256": (lambda o, a: _model(o, a, BOUNDARY, 2, 1024, 11), 1e-4),
    "xunet_mod_first": (lambda o, a: _xunet(o, a, "mod_first"), 1e-5),
    "xunet_skipadd": (lambda o, a: _xunet(o, a, "skipadd"), 1e-5),
    "skipcat_ar": (_skipcat_ar, 1e-5),
    "upsampler": (_upsampler, 1e-5),
}


def _call(net, x, sigma, kw):
    return net(x, sigma, **kw) if sigma is not None else net(x, **kw)


@pytest.mark.parametrize("name", sorted(PROGRAMS))
def test_f32_inference_program(adp, oracle_port, name):
    """v under Shadow, then under Shadow(guard=True), then eager / capture / replay; the branch
    v - x (x: the channels the net's output skips over) against the float64 oracle."""
    build, tol = PROGRAMS[name]
    ref, model, x, sigma, kw = build(oracle_port, adp)
    ref.double()
    net = model.net
    net.verify_fp32 = True
    s = kw.get("embedding_scale")
    s = s if s not in (None, 1.0) else None
    with torch.no_grad():
        want = _call(ref.net, x.double(), None if sigma is None else sigma.double(), _dbl(kw))
        args = (x.to(DEV), None if sigma is None else sigma.to(DEV), _dev(kw))
        net.use_cuda_graph = False
        runs = []
        for guard in (False, True):
            with lc.Shadow(guard=guard) as sh:
                runs.append(_call(net, *args).clone())
            torch.cuda.synchronize()
            print(f"\n{name} fp32 v (guard={guard})\n{sh.table()}")
            assert sh.n_checked == sh.n_launch > 0
            assert not guard or sh.n_guarded == sh.n_launch
        net.use_cuda_graph = True
        for _ in range(3):                      # eager, capture + replay, replay
            v = _call(net, *args)
    bound = tol * ((abs(s) + abs(1 - s)) if s is not None else 1.0)
    skip = x.double()[:, :want.shape[1]]
    for what, got in (("checked", runs[0]), ("guarded", runs[1]), ("replay", v)):
        e = rel_l2(got.cpu().double() - skip, want - skip)
        print(f"{name}: fp32 branch rel-L2 vs float64 ({what}) {e:.3e} (bound {bound:.1e})")
        assert e <= bound


def test_f32_sample_program(adp, oracle_port):
    """The tiny 5-step sample under Shadow, under guard bands, then eager / capture / replay."""
    ref, model, _, _, _ = _model(oracle_port, adp, TINY, 2, 4096, 11)
    ref.double()
    model.net.verify_fp32 = True
    model.net.use_cuda_graph = False
    noise = torch.randn(2, 2, 4096, generator=torch.Generator().manual_seed(4))
    want = ref.sample(noise.double(), num_steps=5)
    for guard in (False, True):
        with torch.no_grad(), lc.Shadow(guard=guard) as sh:
            got = model.sample(noise.to(DEV), num_steps=5)
        torch.cuda.synchronize()
        assert sh.n_checked == sh.n_launch > 0 and (not guard or sh.n_guarded == sh.n_launch)
        e = rel_l2(got, want)
        print(f"tiny fp32 5-step sample (guard={guard}): rel-L2 vs float64 {e:.3e}\n{sh.table()}")
        assert e <= 1e-4
    model.net.use_cuda_graph = True
    for call in range(3):
        got = model.sample(noise.to(DEV), num_steps=5)
        e = rel_l2(got, want)
        print(f"tiny fp32 5-step sample, graph call {call}: rel-L2 vs float64 {e:.3e}")
        assert e <= 1e-4


# The fp32 training tests of the other files, run whole under the checker: each already compares the
# loss, every parameter gradient and its input / encoder / embedding gradients with autograd through
# the float64 oracle.  id -> (module, test, keyword arguments besides the fixtures)
TRAINING = {
    "attention_free_and_golden": ("test_train_fp32_gpu", "test_attention_free_net_and_golden_gradients", {}),
    "upsampler": ("test_train_fp32_gpu", "test_upsampler", {}),
    "head_dim_32": ("test_train_fp32_gpu", "test_self_attention_head_dims", {"head_dim": 32}),
    "head_dim_128": ("test_train_fp32_gpu", "test_self_attention_head_dims", {"head_dim": 128}),
    "groups_1": ("test_train_fp32_gpu", "test_resnet_groups", {"groups": 1}),
    "groups_4": ("test_train_fp32_gpu", "test_resnet_groups", {"groups": 4}),
    "embedding_gradient": ("test_train_fp32_gpu", "test_cross_attention_embedding_gradient_and_guidance", {}),
    "input_gradients": ("test_train_fp32_gpu", "test_custom_loss_with_input_gradients", {}),
    "autoencoder_encoder": ("test_train_fp32_gpu", "test_autoencoder_encoder_gradient", {}),
    "skipcat_ar": ("test_train_fp32_gpu", "test_autoregressive_skipcat", {}),
    "wide_boundary_c0_256": ("test_wide_boundary_gpu", "test_training", {"kind": "c0_256", "fp32": True}),
    "xunet_skipadd": ("test_xunet_gpu", "test_fp32_verification_mode", {"case": "skipadd"}),
}


@pytest.mark.parametrize("guard", [False, True], ids=["checked", "guarded"])
@pytest.mark.parametrize("name", sorted(TRAINING))
def test_f32_training_under_checker(adp, oracle_port, golden_dir, monkeypatch, name, guard):
    import importlib
    module, test, kw = TRAINING[name]
    fn = getattr(importlib.import_module(module), test)
    init = adp.B200UNet._init_runtime           # every net (UNetV0, XUNet) sets its runtime up here

    def eager_init(self):                       # the checker synchronises around every launch
        init(self)
        self.use_cuda_graph = False
    monkeypatch.setattr(adp.B200UNet, "_init_runtime", eager_init)
    fixtures = {"adp": adp, "oracle_port": oracle_port, "golden_dir": golden_dir}
    kw = dict(kw, **{k: v for k, v in fixtures.items() if k in inspect.signature(fn).parameters})
    with lc.Shadow(guard=guard) as sh:
        fn(**kw)
    torch.cuda.synchronize()
    print(f"\n{name} (guard={guard})\n{sh.table()}")
    assert sh.n_checked == sh.n_launch > 0 and (not guard or sh.n_guarded == sh.n_launch)
    assert {"wgrad", "gn_silu_bwd", "stem_out_bwd"} <= {k.split(".")[0] for k in sh.records}


def test_every_f32_entry_point_is_checked(ops):
    """One probe pass over every edge case: the C entry points its checked launches call."""
    src = inspect.getsource(ops)
    callable_ = set(re.findall(r'"(adp_f32_\w+)"', src))   # the symbols ops._launch calls and records
    reached = set()
    for case in ALL:
        reached |= _run(ops, case, "probe", 100 + ALL.index(case)).symbols
    missing = sorted(callable_ - reached)
    print(f"f32 entry points reached: {sorted(reached & callable_)}")
    assert not missing, f"no checked launch reaches {missing}"
