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


# (kind, B, T, ci, co, groups, upsample factor / downsample stride, forced N tile or 0)
_CASES = [
    ("down", 2, 1024, 8, 8, 8, 4, 0),        # group size 1
    ("down", 2, 1024, 8, 16, 8, 4, 0),       # group size 2
    ("down", 2, 1024, 8, 32, 8, 4, 0),       # group size 4
    ("down", 3, 80000, 8, 32, 8, 4, 0),      # 157 ragged 128-row tiles per batch element
    ("up", 2, 256, 32, 16, 8, 4, 0),         # group size 2
    ("up", 3, 8500, 32, 8, 8, 4, 0),         # group size 1, 4 x 67 tiles per batch element
    ("linear", 3, 1000, 64, 16, 8, 4, 0),    # group size 2, ragged T
    ("conv3", 2, 300, 32, 16, 8, 4, 0),      # group size 2
    ("conv3", 2, 300, 32, 24, 8, 4, 0),      # group size 3 (not a power of two)
    ("conv3", 2, 300, 32, 48, 8, 4, 0),      # group size 6
    # fewer groups: the per-lane narrow path at other (lane, block) -> group layouts, and
    # power-of-two sizes >= 8 (warp-uniform group per 8-column block) at n_valid <= 32
    ("down", 2, 1024, 8, 8, 1, 4, 0),        # group size 8
    ("down", 2, 1024, 8, 8, 2, 4, 0),        # group size 4
    ("down", 2, 1024, 8, 8, 4, 4, 0),        # group size 2
    ("down", 2, 1024, 8, 16, 1, 4, 0),       # group size 16
    ("down", 2, 1024, 8, 16, 2, 4, 0),       # group size 8
    ("down", 2, 1024, 8, 16, 4, 4, 0),       # group size 4
    ("down", 2, 1024, 8, 32, 1, 4, 0),       # group size 32
    ("down", 2, 1024, 8, 32, 2, 4, 0),       # group size 16
    ("down", 2, 1024, 8, 32, 4, 4, 0),       # group size 8
    ("down", 3, 80000, 8, 32, 2, 4, 0),      # ragged tiles straddling batch elements, size 16
    ("up", 3, 8500, 32, 8, 2, 4, 0),         # ragged, group size 4
    ("up", 3, 8500, 32, 8, 4, 4, 0),         # ragged, group size 2
    ("up", 2, 256, 32, 16, 4, 2, 0),         # f = 2, group size 4
    ("up", 3, 700, 64, 32, 2, 2, 0),         # f = 2, group size 16, ragged
    ("linear", 3, 1000, 64, 16, 1, 4, 0),    # group size 16
    ("conv3", 2, 300, 32, 24, 1, 4, 0),      # group size 24 (per-block path)
    ("conv3", 2, 300, 32, 48, 4, 4, 0),      # group size 12
    # n_valid = 1024: a 1024 / G-channel group spans several N tiles (and CTAs)
    ("conv3", 3, 1000, 64, 1024, 8, 4, 0),
    ("conv3", 3, 1000, 64, 1024, 1, 4, 0),
    ("conv3", 3, 1000, 64, 1024, 2, 4, 0),
    ("conv3", 3, 1000, 64, 1024, 4, 4, 0),
    ("conv3", 3, 1000, 64, 1024, 4, 4, 64),
    ("linear", 3, 1000, 64, 1024, 4, 4, 256),   # a 3-tap stage of 256 columns exceeds shared memory
]


def _case_id(c):
    kind, B, T, ci, co, groups, f, block_n = c
    return (f"{kind}-{B}-{T}-{ci}-{co}" + ("" if groups == 8 else f"-g{groups}")
            + ("" if f == 4 else f"-f{f}") + (f"-bn{block_n}" if block_n else ""))


@pytest.mark.parametrize("kind,B,T,ci,co,groups,f,block_n", _CASES, ids=[_case_id(c) for c in _CASES])
def test_conv_gemm_narrow_group_stats(ops, kind, B, T, ci, co, groups, f, block_n):
    """GroupNorm statistics fused into the conv GEMM epilogue, for groups narrower than 8 channels
    and for group counts other than 8 (up to groups spanning several N tiles).
    The large shapes give each persistent CTA a tile range that straddles a batch boundary (tile
    counts per batch element that the tiles per CTA do not divide).  Two launches on the same
    input write the same bits."""
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
        ops.conv_gemm(a, wp, view, n_valid=co, bias=bias, stats=stats, groups=groups, block_n=block_n, **kw)
        assert_close(stats, stats_of(out, groups), 1e-4, 1e-2, f"{kind} B{B} T{T} co{co} G{groups} stats")
        outs.append(out)
    assert torch.equal(outs[0], outs[1])
    assert_close(outs[0], ref, 2 ** -6, 3e-2, f"{kind} B{B} T{T} co{co} G{groups}")
