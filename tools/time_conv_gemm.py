"""Times the deep-level conv GEMM launches of cfg2 (README net, B = 8, T = 2^18) and cfg3
(B = 32 under CFG) in isolation, interleaved in one process, under three tile plans
(adp_debug_set(4, ...)): `rows128` (128-row tiles only, the plan before 256-row tiles),
`rows256` (256 x 64 wherever the kernel has it) and `plan` (the tile plan adp_conv_gemm
picks).  `--plan` times `rows128` and `plan` only.

For each shape it prints the median time of a launch, TFLOP/s and the L2 -> SM bytes that the
tile implies (every CTA loads its A box(es) of 128 + span rows and its BN-row weight slice per
tile) over the launch time.

usage: python tools/time_conv_gemm.py [--plan] [--launches N] [--rounds R] [--json PATH]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audio_diffusion_pytorch_b200 import _lib, ops  # noqa: E402

# (label, B, M = B*T, K, N, taps, GroupNorm statistics + residual): ResnetBlock k=3 convs and
# k=1 convs of L3-L8, q|k|v and out projections of L5-L8 (cfg2), and the deep shapes of cfg3
SHAPES = [
    ("L3 k3", 8, 32768, 128, 128, 3, True),
    ("L3 k1", 8, 32768, 256, 128, 1, True),
    ("L4 k3", 8, 16384, 256, 256, 3, True),
    ("L5 k3", 8, 8192, 512, 512, 3, True),
    ("L6 k3", 8, 4096, 512, 512, 3, True),
    ("L7 k3", 8, 2048, 1024, 1024, 3, True),
    ("L8 k3", 8, 1024, 1024, 1024, 3, True),
    ("L5 qkv", 8, 8192, 512, 1536, 1, False),
    ("L6 qkv", 8, 4096, 512, 1536, 1, False),
    ("L7 qkv", 8, 2048, 1024, 1536, 1, False),
    ("L8 qkv", 8, 1024, 1024, 1536, 1, False),
    ("L5 out", 8, 8192, 512, 512, 1, True),
    ("L7 out", 8, 2048, 512, 1024, 1, True),
    ("L8 out", 8, 1024, 512, 1024, 1, True),
    ("cfg3 L5 k3", 32, 32768, 512, 512, 3, True),
    ("cfg3 L6 k3", 32, 16384, 512, 512, 3, True),
    ("cfg3 L7 k3", 32, 8192, 1024, 1024, 3, True),
    ("cfg3 L8 k3", 32, 4096, 1024, 1024, 3, True),
    ("cfg3 L7 qkv", 32, 8192, 1024, 1536, 1, False),
    ("cfg3 L8 qkv", 32, 4096, 1024, 1536, 1, False),
]
MODES = {"rows128": 128, "rows256": 256, "plan": 0}


def block_n(M: int, K: int, N: int, taps: int) -> int:
    """The N tile of the 128-row tiles adp_conv_gemm picks (block_n = 0, no A transform)."""
    m_tiles = (M + 127) // 128
    for cand in (128, 64, 32, 16):
        if N % cand or (cand == 128 and taps * K <= 1024):
            continue
        if m_tiles * (N // cand) >= 96 or cand <= 64:
            return cand
    return 16


def tile_of(mode: str, B: int, M: int, K: int, N: int, taps: int):
    """(BM, BN) the mode runs, or None where the kernel has no such tile."""
    bn = block_n(M, K, N, taps)
    has256 = K % 64 == 0 and N % 64 == 0 and M // B >= 256
    if mode == "rows128":
        return 128, bn
    if mode == "rows256":
        return (256, 64) if has256 else None
    return (256, 64) if has256 and bn == 128 else (128, bn)


def l2_bytes(B: int, M: int, K: int, N: int, taps: int, bm: int, bn: int) -> float:
    tiles = B * ((M // B + bm - 1) // bm) * (N // bn)
    return tiles * ((bm // 128) * (128 + taps - 1) * K * 2 + bn * taps * K * 2)


def time_launches(fn, launches: int) -> float:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / launches   # us per launch


def card() -> dict:
    info = {"name": torch.cuda.get_device_name()}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        info["power_limit_and_max_sm_clock"] = "unavailable"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--plan", action="store_true", help="time rows128 and plan only")
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_conv_gemm.py needs a CUDA device")
    dev = "cuda"
    lib = _lib.lib()
    g = torch.Generator(device=dev).manual_seed(0)
    info = card()
    print(json.dumps(info))
    modes = {m: k for m, k in MODES.items() if not (args.plan and m == "rows256")}
    rows = []
    for label, B, M, K, N, taps, epi in SHAPES:
        x = torch.randn(B, M // B, K, device=dev, generator=g).bfloat16()
        w = ops.pack_conv(torch.randn(N, K, taps, device=dev, generator=g) * (K * taps) ** -0.5)
        out = torch.empty(B, M // B, N, device=dev, dtype=torch.bfloat16)
        bias = torch.randn(N, device=dev, generator=g)
        res = torch.randn(B, M // B, N, device=dev, generator=g).bfloat16() if epi else None
        st = torch.zeros(B, 8, 2, device=dev, dtype=torch.float64) if epi else None
        tp = (-1, 0, 1) if taps == 3 else (0,)

        def run():
            ops.conv_gemm(x, w, out, c_in=K, n_valid=N, taps=tp, bias=bias, residual=res, stats=st)

        tiles = {m: tile_of(m, B, M, K, N, taps) for m in modes}
        times = {m: [] for m in modes if tiles[m]}
        try:
            for r in range(args.rounds):
                for m in times:
                    _lib.check(lib.adp_debug_set(4, modes[m]), "adp_debug_set")
                    if r == 0:
                        time_launches(run, 20)
                    times[m].append(time_launches(run, args.launches))
        finally:
            _lib.check(lib.adp_debug_set(4, 0), "adp_debug_set")
        flops = 2.0 * M * K * N * taps
        row = {"shape": f"{label} M={M} K={K} N={N}"}
        for m in times:
            us = statistics.median(times[m])
            bm, bn = tiles[m]
            row[m] = {"tile": f"{bm}x{bn}", "us": round(us, 2),
                      "spread_us": round(max(times[m]) - min(times[m]), 2),
                      "tflops": round(flops / us * 1e-6, 1),
                      "l2_mb_per_us": round(l2_bytes(B, M, K, N, taps, bm, bn) / 1e6 / us, 2)}
        rows.append(row)
        print(f"{row['shape']:34s} " + "  ".join(
            f"{m} {row[m]['tile']:>7s} {row[m]['us']:7.2f}us (spread {row[m]['spread_us']:.2f}) "
            f"{row[m]['tflops']:5.0f}TF/s {row[m]['l2_mb_per_us']:5.2f}MB/us" for m in times), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
