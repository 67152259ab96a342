"""The conv GEMM's BN <= 64 tiles without the narrow-group statistics registers against the
variant that has them (adp_debug_set(7, 1) sends every such launch to it).  Both run the same
MMAs in the same order on the same tiles, so the outputs must be bitwise equal; the GroupNorm
sums may differ only by the order of the fp64 atomics that combine the per-CTA partials."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"


@pytest.fixture(scope="module")
def ops():
    from audio_diffusion_pytorch_b200 import _lib, ops
    ops.device_check()
    yield ops
    _lib.check(_lib.lib().adp_debug_set(7, 0), "adp_debug_set")


def _force_narrow(on):
    from audio_diffusion_pytorch_b200 import _lib
    _lib.check(_lib.lib().adp_debug_set(7, 1 if on else 0), "adp_debug_set")


def _rnd(*shape, g, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


# (name, B, T, c_in, c_out, kind, groups, block_n, residual, gate); kind: k3, k1 or upF.
# The deep shapes are those of the README net at T = 2^18 (cfg2: B = 8, cfg3: B = 16).
_CASES = [
    ("L8 k3", 8, 128, 1024, 1024, "k3", 8, 0, True, False),
    ("L8 k3 cfg3", 16, 128, 1024, 1024, "k3", 8, 0, False, True),
    ("L8 out", 8, 128, 512, 1024, "k1", 8, 0, True, False),
    ("L8 up2", 8, 128, 1024, 1024, "up2", 8, 64, False, False),
    ("dgrad L8->L7", 4, 128, 1024, 1024, "k3", 0, 64, False, False),
    ("odd M tiles", 1, 384, 256, 256, "k3", 8, 64, False, False),
    ("ragged T", 2, 1000, 256, 512, "k3", 8, 64, True, True),
    ("T <= 128", 4, 100, 512, 512, "k3", 8, 64, True, False),
    ("up4 phases", 4, 300, 256, 128, "up4", 8, 64, True, False),
    ("BN 32 groups of 3", 2, 300, 64, 24, "k3", 8, 0, False, False),
    ("BN 32 groups of 16", 4, 512, 64, 128, "k3", 8, 32, False, False),
    ("BN 16 groups of 8", 4, 512, 128, 64, "k1", 8, 16, True, False),
    ("BN 64 no statistics", 4, 512, 128, 256, "k1", 0, 64, False, True),
]


def _run_case(ops, case, narrow):
    name, B, T, ci, co, kind, groups, bn, with_res, with_gate = case
    g = torch.Generator().manual_seed(7)
    x = _rnd(B, T, ci, g=g).bfloat16()
    up = int(kind[2:]) if kind.startswith("up") else 0
    taps = (-1, 0, 1) if kind == "k3" else (0,)
    w = _rnd(co, ci, 1 if kind == "k1" else 3, g=g, scale=(3 * ci) ** -0.5)
    wp = ops.pack_upsample_conv(w, up) if up else ops.pack_conv(w)
    phases = up if up else 1
    bias = _rnd(co, g=g)
    res = _rnd(B, T, phases * co, g=g).bfloat16() if with_res else None
    gate = _rnd(B, phases * co, g=g) if with_gate else None
    st = torch.zeros(B, groups, 2, device=DEV, dtype=torch.float64) if groups else None
    out = torch.empty(B, T, phases * co, device=DEV, dtype=torch.bfloat16)
    _force_narrow(narrow)
    try:
        ops.conv_gemm(x, wp, out, c_in=ci, n_valid=co, taps=taps, up_factor=up, bias=bias,
                      residual=res, gate=gate, stats=st, groups=groups or 8, block_n=bn)
        torch.cuda.synchronize()
    finally:
        _force_narrow(False)
    return out, st


@pytest.mark.parametrize("case", _CASES, ids=[c[0] for c in _CASES])
def test_narrow_variant_bitwise(ops, case):
    out_a, st_a = _run_case(ops, case, False)
    out_b, st_b = _run_case(ops, case, True)
    diff = int((out_a.view(torch.int16) != out_b.view(torch.int16)).sum())
    assert diff == 0, f"{case[0]}: {diff} of {out_a.numel()} outputs differ"
    if st_a is None:
        return
    B, T, N = out_a.shape
    og = out_a.double().reshape(B, T, st_a.shape[1], N // st_a.shape[1])
    scale = torch.stack([og.abs().sum(dim=(1, 3)), (og * og).sum(dim=(1, 3))], dim=-1)
    err = float(((st_a - st_b).abs() / scale.clamp_min(1e-30)).max())
    print(f"{case[0]}: statistics differ by {err:.2e} of sum|x| / sum x^2")
    assert err <= 1e-12, f"{case[0]}: statistics differ by {err:.3e}"
