"""Times DPMSolverSampler against VSampler on the README U-Net at the benchmark's cfg2 shape
(noise [8, 2, 2^18], unconditional), and the adp_dpm_step kernel on its own.

    python tools/time_dpm_sampler.py [--B 8] [--T 262144] [--steps 50] [--reps 5] [--out DIR]

Per step: CUDA events around whole `sampler(noise, num_steps)` calls (the conditioning table, the
staging and every step graph included), divided by the steps; the two samplers alternate in one
process after a warm-up call each, and the median over --reps calls is reported.  The kernel: a
torch.profiler run of its own over one DPMSolverSampler call, the mean device time of the
dpm_step_kernel launches, and the bytes it moves (x, v and the history read, x and the history
written, fp32) over that time.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import audio_diffusion_pytorch_b200 as adp  # noqa: E402

README = dict(in_channels=2, channels=[8, 32, 64, 128, 256, 512, 512, 1024, 1024],
              factors=[1, 4, 4, 4, 2, 2, 2, 2, 2], items=[1, 2, 2, 2, 2, 2, 2, 4, 4],
              attentions=[0, 0, 0, 0, 0, 1, 1, 1, 1], attention_heads=8, attention_features=64)


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


def call_ms(sampler, noise, steps) -> float:
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    sampler(noise, num_steps=steps)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=8)
    ap.add_argument("--T", type=int, default=2 ** 18)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for dpm_sampler.json")
    args = ap.parse_args()
    torch.manual_seed(0)
    net = adp.UNetV0(dim=1, **README).cuda()
    samplers = {"VSampler": adp.VSampler(net), "DPMSolverSampler": adp.DPMSolverSampler(net)}
    noise = torch.randn(args.B, 2, args.T, device="cuda")
    with torch.no_grad():
        for sampler in samplers.values():          # plans, graphs and the conditioning pass warmed up
            call_ms(sampler, noise, args.steps)
            call_ms(sampler, noise, args.steps)
        times = {name: [] for name in samplers}
        for _ in range(args.reps):
            for name, sampler in samplers.items():
                times[name].append(call_ms(sampler, noise, args.steps) / args.steps)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            samplers["DPMSolverSampler"](noise, num_steps=args.steps)
            torch.cuda.synchronize()
    kernel = [e for e in prof.events() if "dpm_step_kernel" in e.name and e.device_type.name == "CUDA"]
    kernel_us = statistics.mean(e.device_time for e in kernel) if kernel else float("nan")
    n = noise.numel()
    moved = 5 * 4 * n                                # x, v, history read; x, history written
    per_step = {name: statistics.median(t) for name, t in times.items()}
    result = {
        "card": card(), "B": args.B, "T": args.T, "steps": args.steps, "reps": args.reps,
        "ms_per_step": per_step, "ms_per_step_all": times,
        "dpm_minus_v_ms_per_step": per_step["DPMSolverSampler"] - per_step["VSampler"],
        "dpm_step_kernel_us": kernel_us, "dpm_step_kernel_launches": len(kernel),
        "dpm_step_bytes": moved, "dpm_step_GBps": moved / (kernel_us * 1e-6) / 1e9 if kernel else None,
        "dpm_step_share_of_step": kernel_us * 1e-3 / per_step["DPMSolverSampler"],
    }
    print(json.dumps(result))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "dpm_sampler.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
