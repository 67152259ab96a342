"""Times the attention kernels at head dims 32, 64 and 128 with heads * D = 512.

Self-attention on a packed q|k|v buffer (as the fused projection writes it), B = 8, at the
README net's attention levels (N = 1024, 512, 256, 128 tokens) plus N = 4096.  Forward
(adp_attention) and forward + backward (adp_attention with lse, then adp_attention_bwd) are
timed with CUDA events around `--iters` back-to-back launches after `--warmup` launches.
FLOPs are those ops.attention / ops.attention_bwd report (4 and 14 x B H N^2 D; the backward
count includes recomputing S and dP in both of its kernels); the fraction is of the H100 SXM
data-sheet dense BF16 rate, 989 TFLOP/s.

    python tools/time_attention.py [--iters 200] [--warmup 20] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audio_diffusion_pytorch_b200 import ops  # noqa: E402

PEAK_TFLOPS = 989.0
DIMS = (32, 64, 128)
TOKENS = (1024, 512, 256, 128, 4096)


def card() -> str:
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit unknown"
    return f"{name} ({q})"


def time_ms(fn, iters: int, warmup: int) -> float:
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def measure(D: int, N: int, B: int, width: int, iters: int, warmup: int) -> dict:
    H = width // D
    mid = H * D
    g = torch.Generator(device="cpu").manual_seed(0)
    qkv = torch.randn(B, N, 3 * mid, generator=g).to("cuda", torch.bfloat16)
    q, k, v = qkv[..., :mid], qkv[..., mid:2 * mid], qkv[..., 2 * mid:]
    o = torch.empty(B, N, mid, dtype=torch.bfloat16, device="cuda")
    d_o = torch.randn(B, N, mid, generator=g).to("cuda", torch.bfloat16)
    dqkv = torch.empty_like(qkv)
    lse = torch.empty(B, H, N, device="cuda")
    delta = torch.empty(B, H, N, device="cuda")
    scale = D ** -0.5

    def fwd():
        ops.attention(q, k, v, o, H, scale, head_dim=D)

    def fwd_bwd():
        ops.attention(q, k, v, o, H, scale, lse=lse, head_dim=D)
        ops.attention_bwd(q, k, v, o, d_o, lse, delta, dqkv[..., :mid], dqkv[..., mid:2 * mid],
                          dqkv[..., 2 * mid:], H, scale, head_dim=D)

    t_f = time_ms(fwd, iters, warmup)
    t_fb = time_ms(fwd_bwd, iters, warmup)
    f_f = 4.0 * B * H * N * N * D
    f_fb = f_f + 14.0 * B * H * N * N * D
    return dict(D=D, H=H, B=B, N=N, fwd_us=t_f * 1e3, fwd_tflops=f_f / t_f / 1e9,
                fwdbwd_us=t_fb * 1e3, fwdbwd_tflops=f_fb / t_fb / 1e9)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--width", type=int, default=512, help="heads * head_dim")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_attention.py measures on the GPU"
    ops.device_check()
    dev = card()
    print(f"# {dev}; B={a.batch}, heads*D={a.width}, {a.iters} timed launches after {a.warmup}")
    print(f"{'N':>5} {'D':>4} {'H':>3} | {'fwd us':>9} {'TF/s':>7} {'%peak':>6} | "
          f"{'fwd+bwd us':>10} {'TF/s':>7} {'%peak':>6}")
    rows = []
    for N in TOKENS:
        for D in DIMS:
            r = measure(D, N, a.batch, a.width, a.iters, a.warmup)
            rows.append(r)
            print(f"{N:>5} {D:>4} {r['H']:>3} | {r['fwd_us']:>9.1f} {r['fwd_tflops']:>7.1f} "
                  f"{100 * r['fwd_tflops'] / PEAK_TFLOPS:>5.1f}% | {r['fwdbwd_us']:>10.1f} "
                  f"{r['fwdbwd_tflops']:>7.1f} {100 * r['fwdbwd_tflops'] / PEAK_TFLOPS:>5.1f}%")
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(dict(device=dev, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
