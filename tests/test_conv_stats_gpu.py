"""GroupNorm statistics fused into the conv GEMM epilogue, checked against a float64 sum of the
output it wrote (same helpers as test_ops_gpu.py)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda"
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def bf(t):
    return t.to(torch.bfloat16)


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def assert_close(got, ref, rtol, atol, what):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    bad = err > atol + rtol * ref.abs()
    msg = (f"{what}: max abs err {err.max().item():.4e}, ref max {ref.abs().max().item():.3e}, "
           f"violations {int(bad.sum())}/{bad.numel()}")
    print(msg)
    assert not bad.any(), msg


def stats_of(y, groups):
    """(sum, sumsq) per (batch, group) of a channels-last tensor."""
    B, T, Cc = y.shape
    yg = y.double().reshape(B, T, groups, Cc // groups)
    return torch.stack([yg.sum(dim=(1, 3)), (yg * yg).sum(dim=(1, 3))], dim=-1)


@pytest.fixture(scope="module")
def ops():
    from audio_diffusion_pytorch_b200 import ops
    ops.device_check()
    return ops


@pytest.mark.parametrize("kind,B,T,ci,co", [
    ("down", 2, 1024, 8, 8),       # group size 1
    ("down", 2, 1024, 8, 16),      # group size 2
    ("down", 2, 1024, 8, 32),      # group size 4
    ("down", 3, 80000, 8, 32),     # 157 ragged 128-row tiles per batch element
    ("up", 2, 256, 32, 16),        # group size 2
    ("up", 3, 8500, 32, 8),        # group size 1, 4 x 67 tiles per batch element
    ("linear", 3, 1000, 64, 16),   # group size 2, ragged T
    ("conv3", 2, 300, 32, 16),     # group size 2
    ("conv3", 2, 300, 32, 24),     # group size 3 (not a power of two)
    ("conv3", 2, 300, 32, 48),     # group size 6
])
def test_conv_gemm_narrow_group_stats(ops, kind, B, T, ci, co):
    """GroupNorm statistics fused into the conv GEMM epilogue for groups narrower than 8 channels.
    The large shapes give each persistent CTA a tile range that straddles a batch boundary (tile
    counts per batch element that the tiles per CTA do not divide).  Two launches on the same
    input write the same bits."""
    groups = 8
    f = 4
    if kind == "down":
        x = bf(rnd(B, T, ci, seed=70))
        w = bf(rnd(co, ci, f, scale=(f * ci) ** -0.5, seed=71))
        a, wp, T_out, kw = x.view(B, T // f, f * ci), ops.pack_conv(w), T // f, dict(c_in=f * ci)
        ref = F.conv1d(x.float().transpose(1, 2), w.float(), stride=f).transpose(1, 2)
    elif kind == "up":
        x = bf(rnd(B, T, ci, seed=72))
        w = bf(rnd(co, ci, 3, scale=(3 * ci) ** -0.5, seed=73))
        skip = bf(rnd(B, T * f, co, seed=74))
        a, wp, T_out = x, ops.pack_upsample_conv(w, f), T * f
        kw = dict(c_in=ci, up_factor=f, residual=skip.view(B, T, f * co))
        up = F.interpolate(x.float().transpose(1, 2), scale_factor=f, mode="nearest")
        ref = skip.float() + F.conv1d(up, w.float(), padding=1).transpose(1, 2)
    elif kind == "linear":
        x = bf(rnd(B, T, ci, seed=75))
        w = bf(rnd(co, ci, scale=ci ** -0.5, seed=76))
        a, wp, T_out, kw = x, ops.pack_linear(w), T, dict(c_in=ci)
        ref = x.float() @ w.float().t()
    else:
        x = bf(rnd(B, T, ci, seed=77))
        w = bf(rnd(co, ci, 3, scale=(3 * ci) ** -0.5, seed=78))
        res = bf(rnd(B, T, co, seed=79))
        a, wp, T_out, kw = x, ops.pack_conv(w), T, dict(c_in=ci, taps=(-1, 0, 1), residual=res)
        ref = F.conv1d(x.float().transpose(1, 2), w.float(), padding=1).transpose(1, 2) + res.float()
    bias = rnd(co, seed=80)
    ref = ref + bias
    outs = []
    for _ in range(2):
        stats = torch.zeros(B, groups, 2, dtype=torch.float64, device=DEV)
        out = torch.empty(B, T_out, co, dtype=torch.bfloat16, device=DEV)
        view = out.view(B, T, f * co) if kind == "up" else out
        ops.conv_gemm(a, wp, view, n_valid=co, bias=bias, stats=stats, groups=groups, **kw)
        assert_close(stats, stats_of(out, groups), 1e-4, 1e-2, f"{kind} B{B} T{T} co{co} stats")
        outs.append(out)
    assert torch.equal(outs[0], outs[1])
    assert_close(outs[0], ref, 2 ** -6, 3e-2, f"{kind} B{B} T{T} co{co}")
