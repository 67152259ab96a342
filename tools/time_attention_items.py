"""Times the README net with two self-attention items per repetition at its attention levels
(attentions=[0, 0, 0, 0, 0, 2, 2, 2, 2]) against one ([..., 1, 1, 1, 1]): one evaluation (a graph
replay of net(x, sigma)) and one training step (fused_v_loss + backward), B = 8, T = 2^18.

    python tools/time_attention_items.py [--runs 3] [--B 8] [--T 262144]

Each measurement runs in a fresh process, the two configs alternating; per process: warm-up, then
CUDA events around 20 evaluations and 10 training steps.  Prints the card and its power limit.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
README = dict(in_channels=2, channels=[8, 32, 64, 128, 256, 512, 512, 1024, 1024],
              factors=[1, 4, 4, 4, 2, 2, 2, 2, 2], items=[1, 2, 2, 2, 2, 2, 2, 4, 4],
              attention_heads=8, attention_features=64)


def timed(fn, n, warmup=3):
    for _ in range(warmup):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


def one(att: int, B: int, T: int) -> dict:
    sys.path.insert(0, ROOT)
    import audio_diffusion_pytorch_b200 as adp
    from audio_diffusion_pytorch_b200 import ops
    from audio_diffusion_pytorch_b200.training import fused_v_loss
    ops.device_check()
    torch.manual_seed(0)
    model = adp.DiffusionModel(net_t=adp.UNetV0, attentions=[0] * 5 + [att] * 4, **README).cuda()
    net = model.net
    g = torch.Generator(device="cuda").manual_seed(1)
    x, noise = torch.randn(B, 2, T, device="cuda", generator=g), torch.randn(B, 2, T, device="cuda", generator=g)
    sigma = torch.rand(B, device="cuda", generator=g)

    def evaluate():
        with torch.no_grad():
            net(x, sigma)

    def train():
        fused_v_loss(net, x, noise, sigma).backward()

    out = {"attentions": att, "B": B, "T": T, "eval_ms": timed(evaluate, 20), "train_ms": timed(train, 10),
           "params": sum(p.numel() for p in net.parameters())}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--B", type=int, default=8)
    ap.add_argument("--T", type=int, default=2 ** 18)
    ap.add_argument("--one", type=int, default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.one is not None:
        print(json.dumps(one(a.one, a.B, a.T)))
        return
    assert torch.cuda.is_available(), "time_attention_items.py measures on the GPU"
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    res = {1: [], 2: []}
    for _ in range(a.runs):
        for att in (1, 2):
            p = subprocess.run([sys.executable, __file__, "--one", str(att), "--B", str(a.B), "--T", str(a.T)],
                               capture_output=True, text=True, check=True)
            r = json.loads(p.stdout.strip().splitlines()[-1])
            print(json.dumps(r), flush=True)
            res[att].append(r)
    for att in (1, 2):
        ev = sorted(r["eval_ms"] for r in res[att])
        tr = sorted(r["train_ms"] for r in res[att])
        print(f"attentions {att} at levels 5..8: eval {ev[0]:.2f}-{ev[-1]:.2f} ms (median {ev[len(ev) // 2]:.2f}), "
              f"train step {tr[0]:.2f}-{tr[-1]:.2f} ms (median {tr[len(tr) // 2]:.2f})")


if __name__ == "__main__":
    main()
