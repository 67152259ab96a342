"""Times the LayerNorm row kernels at level widths that do not fill a power of two of lanes or
exceed 1024 channels, next to their power-of-two neighbours, and one evaluation and one training
step of a wide net with the share of it spent in the row kernels.

    python tools/time_widths.py [--T 262144] [--B 8] [--no-net]

Per launch: CUDA events around 50 back-to-back launches after a warm-up, bytes moved (x read, y
written, y2 written for the dual pass; x and dy read, dx written for the backward) over the
time, against the H100 SXM's 3.35 TB/s.  The net: UNetV0 channels [8, 64, 384, 1536, 2048],
16 heads x 64 self- and cross-attention on a 2048-wide embedding, CFG off; the eval is a graph
replay of net(x, sigma), the training step fused_v_loss + backward; kernel shares come from a
torch.profiler run of its own.
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import audio_diffusion_pytorch_b200 as adp  # noqa: E402
from audio_diffusion_pytorch_b200 import ops  # noqa: E402

HBM = 3.35e12
# (new width, its power-of-two neighbours)
GROUPS = [(48, 32, 64), (96, 64, 128), (192, 128, 256), (320, 256, 512), (384, 256, 512), (640, 512, 1024),
          (1280, 1024, 2048), (1536, 1024, 2048)]
NET_B = dict(in_channels=2, channels=[8, 64, 384, 1536, 2048], factors=[1, 4, 4, 2, 2], items=[1, 1, 1, 1, 1],
             attentions=[0, 0, 0, 1, 1], cross_attentions=[0, 0, 0, 1, 1], attention_heads=16,
             attention_features=64, use_embedding_cfg=True, embedding_max_length=64, embedding_features=2048)
ROW_KERNELS = ("ln_film", "gn_silu_bwd", "gn_bwd_apply", "skip_gate", "colsum")


def timed(fn, n=50):
    for _ in range(5):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n * 1e3          # microseconds


def row_kernels(B, T):
    print(f"{'C':>6} {'kernel':>12} {'us':>9} {'GB/s':>8} {'of HBM':>7}")
    done = set()
    for group in GROUPS:
        for C in group:
            if C in done:
                continue
            done.add(C)
            rows = max(1, (B * T * 16) // C)        # the same bytes per launch at every width
            x = (torch.randn(1, rows, C, device="cuda") * 2 + 0.5).bfloat16()
            y, y2, dx = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
            dy = torch.randn_like(x)
            ss = torch.randn(1, 2 * C, device="cuda") * 0.3
            stats = torch.zeros(1, 8, 2, dtype=torch.float64, device="cuda")
            dss, cs = torch.zeros(1, 2 * C, device="cuda"), torch.zeros(C, device="cuda")
            nbytes = x.numel() * 2
            cases = {
                "ln_film": (lambda: ops.ln_film(x, y, ss, 2 * C, stats, 8, 1e-6), 2 * nbytes),
                "ln_film_dual": (lambda: ops.ln_film(x, y, ss, 2 * C, stats, 8, 1e-6, y2=y2), 3 * nbytes),
                "ln_film_bwd": (lambda: ops.ln_film_bwd(dy, x, ss, 2 * C, dx, dss=dss, dss_stride=2 * C,
                                                        colsum=cs), 3 * nbytes),
            }
            for name, (fn, moved) in cases.items():
                us = timed(fn)
                rate = moved / (us * 1e-6)
                print(f"{C:>6} {name:>12} {us:9.2f} {rate / 1e9:8.0f} {rate / HBM:7.1%}")


def net_b(B, T):
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    torch.manual_seed(0)
    model = adp.DiffusionModel(net_t=adp.UNetV0, **NET_B).cuda()
    net = model.net
    x, noise = torch.randn(B, 2, T, device="cuda"), torch.randn(B, 2, T, device="cuda")
    sigma, emb = torch.rand(B, device="cuda"), torch.randn(B, 64, 2048, device="cuda")

    def evaluate():
        with torch.no_grad():
            net(x, sigma, embedding=emb)

    def train():
        fused_v_loss(net, x, noise, sigma, embedding=emb, embedding_mask_proba=0.0).backward()

    for name, fn in (("eval", evaluate), ("train step", train)):
        ms = timed(fn, n=10) / 1e3
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        total = row = 0.0
        for ev in prof.key_averages():
            t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                total += t
                if any(k in ev.key for k in ROW_KERNELS):
                    row += t
        print(f"net (b) B={B} T={T} {name}: {ms:.2f} ms; row kernels {row / max(total, 1e-9):.1%} of kernel time")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=2 ** 18)
    ap.add_argument("--B", type=int, default=8)
    ap.add_argument("--no-net", action="store_true")
    a = ap.parse_args()
    ops.device_check()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    row_kernels(a.B, a.T)
    if not a.no_net:
        net_b(a.B, a.T)


if __name__ == "__main__":
    main()
