"""Conv GEMM tile plan: every launch the plan gives 256-row tiles writes the same bits as the
128-row tiles (adp_debug_set(4, 128)) and GroupNorm statistics that agree within fp32 summation
order.  Each output element sums its products in the same (chunk, tap, k16) order under both
plans, so only the statistics' summation order differs."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


@pytest.fixture(scope="module")
def ops():
    from audio_diffusion_pytorch_b200 import ops
    ops.device_check()
    return ops


def debug_set(key, value):
    from audio_diffusion_pytorch_b200 import _lib
    _lib.check(_lib.lib().adp_debug_set(key, value), "adp_debug_set")


# (name, kind, B, T, c_in, c_out, groups or 0 = no statistics, residual, gate, fp32 output);
# kind: k3, k1, up<f> (nearest upsample + conv3) or down<f> (k = s = f conv over the [B, T/f, f*C] view)
_CASES = [
    # cfg2 (B = 8, T = 2^18) and cfg3 (B = 32) deep-level launches
    ("L3-k3", "k3", 8, 4096, 128, 128, 8, True, False, False),
    ("L3-k1", "k1", 8, 4096, 256, 128, 8, True, False, False),
    ("L4-k3", "k3", 8, 2048, 256, 256, 8, True, False, False),
    ("L5-k3", "k3", 8, 1024, 512, 512, 8, True, False, False),
    ("L6-k3", "k3", 8, 512, 512, 512, 8, True, False, False),
    ("L7-k3", "k3", 8, 256, 1024, 1024, 8, True, False, False),
    ("L5-qkv", "k1", 8, 1024, 512, 1536, 0, False, False, False),
    ("L6-qkv", "k1", 8, 512, 512, 1536, 0, False, False, False),
    ("L5-out", "k1", 8, 1024, 512, 512, 8, True, False, False),
    ("L7-out", "k1", 8, 256, 512, 1024, 8, True, False, False),
    ("cfg3-L5-k3", "k3", 32, 1024, 512, 512, 8, True, False, False),
    ("cfg3-L7-k3", "k3", 32, 256, 1024, 1024, 8, True, False, False),
    ("cfg3-L7-qkv", "k1", 32, 256, 1024, 1536, 0, False, False, False),
    # edge cases: T not a multiple of 256 (ragged last tile, zero-filled A rows past T), bias
    # only, gate, fp32 output, group sizes 8, 24 and 64 at 5 groups, upsample phases, downsample
    ("ragged-k3", "k3", 3, 1000, 128, 256, 8, True, False, False),
    ("ragged-300", "k3", 2, 300, 64, 64, 8, False, False, False),
    ("gate", "k1", 4, 768, 256, 512, 8, False, True, False),
    ("fp32-out", "k3", 4, 520, 128, 128, 0, False, False, True),
    ("group8", "k3", 4, 1024, 256, 64, 8, True, False, False),
    ("group24", "k3", 4, 1024, 256, 192, 8, True, False, False),
    ("groups5", "k3", 4, 1024, 256, 320, 5, True, False, False),
    ("up4", "up4", 4, 512, 128, 64, 8, True, False, False),
    ("up2", "up2", 3, 700, 256, 128, 8, True, False, False),
    ("down4", "down4", 4, 4096, 64, 128, 8, False, False, False),
    ("short-T", "k3", 4, 200, 256, 256, 8, True, False, False),   # T < 256: 128 rows only
]


def _launch(ops, case, plan):
    _, kind, B, T, ci, co, groups, has_res, has_gate, fp32 = case
    if kind.startswith("down"):
        f = int(kind[4:])
        x = rnd(B, T, ci, seed=1).bfloat16()
        w = rnd(co, ci, f, scale=(f * ci) ** -0.5, seed=2).bfloat16()
        a, wp, T_a, kw = x.view(B, T // f, f * ci), ops.pack_conv(w), T // f, dict(c_in=f * ci)
        out_shape = (B, T // f, co)
    elif kind.startswith("up"):
        f = int(kind[2:])
        a = rnd(B, T, ci, seed=1).bfloat16()
        wp = ops.pack_upsample_conv(rnd(co, ci, 3, scale=(3 * ci) ** -0.5, seed=2).bfloat16(), f)
        T_a, kw, out_shape = T, dict(c_in=ci, up_factor=f), (B, T * f, co)
    else:
        taps = 3 if kind == "k3" else 1
        a = rnd(B, T, ci, seed=1).bfloat16()
        wp = ops.pack_conv(rnd(co, ci, taps, scale=(taps * ci) ** -0.5, seed=2).bfloat16())
        T_a, kw, out_shape = T, dict(c_in=ci, taps=(-1, 0, 1) if taps == 3 else (0,)), (B, T, co)
    f = int(kind[2:]) if kind.startswith("up") else 1
    if has_res:
        kw["residual"] = rnd(*out_shape, seed=3).bfloat16().view(B, T_a, f * co)
    if has_gate:
        kw["gate"] = rnd(B, co, seed=4)
    stats = torch.zeros(B, groups, 2, dtype=torch.float64, device=DEV) if groups else None
    out = torch.full(out_shape, float("nan"), device=DEV, dtype=torch.float32 if fp32 else torch.bfloat16)
    debug_set(4, plan)
    try:
        ops.conv_gemm(a, wp, out.view(B, T_a, f * co), n_valid=co, bias=rnd(co, seed=5), stats=stats,
                      groups=groups or 8, **kw)
    finally:
        debug_set(4, 0)
    torch.cuda.synchronize()
    return out, stats


@pytest.mark.parametrize("case", _CASES, ids=[c[0] for c in _CASES])
def test_tile_plans_agree(ops, case):
    """The plan's launch, and a launch forced onto 256-row tiles where they exist, against the
    128-row tiles: bitwise-equal outputs, statistics within the fp32 summation-order bound."""
    ref, ref_stats = _launch(ops, case, 128)
    assert not ref.isnan().any()
    plans = [0]
    T_rows = case[3] // int(case[1][4:]) if case[1].startswith("down") else case[3]
    if T_rows >= 256:
        plans.append(256)
    else:       # tiles never span batch elements: no 256-row tile below T = 256
        with pytest.raises(RuntimeError, match="256-row"):
            _launch(ops, case, 256)
    for plan in plans:
        out, stats = _launch(ops, case, plan)
        assert torch.equal(out, ref), f"{case[0]} plan {plan}: outputs differ from the 128-row tiles"
        if stats is not None:
            torch.testing.assert_close(stats, ref_stats, rtol=1e-4, atol=1e-2)
