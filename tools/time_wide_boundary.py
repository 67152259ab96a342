"""Wide network boundary on one GPU: the time of a whole evaluation of v, of one training step
(loss + backward), and the in-graph time of each stem kernel within them, for
  (a) LTPlugin(UNetV0, num_filters=32, window_length=64, stride=32) on stereo: a 64-channel boundary at
      1/32 of the rate, channels=[128, 256, 512, 512, 1024, 1024], T = 2^18, B = 8;
  (b) a 5.1 DiffusionModel with the README channels, T = 2^18, B = 8.
Prints the card name and power limit of the run.  usage: python tools/time_wide_boundary.py [a|b ...]"""
import os
import subprocess
import sys
from collections import defaultdict

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import audio_diffusion_pytorch_b200 as adp  # noqa: E402
from audio_diffusion_pytorch_b200 import _lib  # noqa: E402

B, T = 8, 2 ** 18
README = dict(channels=[8, 32, 64, 128, 256, 512, 512, 1024, 1024], factors=[1, 4, 4, 4, 2, 2, 2, 2, 2],
              items=[1, 2, 2, 2, 2, 2, 2, 4, 4], attentions=[0, 0, 0, 0, 0, 1, 1, 1, 1], attention_heads=8,
              attention_features=64)
LT_NET = dict(channels=[128, 256, 512, 512, 1024, 1024], factors=[1, 2, 2, 2, 2, 2], items=[2, 2, 2, 2, 2, 2],
              attentions=[0, 0, 0, 1, 1, 1], attention_heads=8, attention_features=64)


def build(which):
    if which == "a":
        lt = adp.LTPlugin(adp.UNetV0, num_filters=32, window_length=64, stride=32)
        return adp.DiffusionModel(net_t=lt, in_channels=2, **LT_NET).cuda(), 2
    return adp.DiffusionModel(net_t=adp.UNetV0, in_channels=6, **README).cuda(), 6


def timed(fn, n):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(n):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / n


def kernel_table(fn, what):
    """adp kernel time of one call of fn (PDL off so that kernel intervals do not overlap)."""
    _lib.lib().adp_debug_set(6, 0)
    try:
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
    finally:
        _lib.lib().adp_debug_set(6, 1)
    agg = defaultdict(lambda: [0, 0.0])
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "adp::" in e.name:
            name = e.name.split("adp::")[1].split("(")[0].split("<")[0]
            agg[name][0] += 1
            agg[name][1] += e.time_range.end - e.time_range.start
    total = sum(v[1] for v in agg.values())
    stems = {k: v for k, v in agg.items() if "stem" in k}
    st = sum(v[1] for v in stems.values())
    print(f"  {what}: adp kernel time {total / 1e3:.2f} ms, stem kernels {st / 1e3:.3f} ms "
          f"({100 * st / max(total, 1e-9):.1f} %)")
    for k, (n, us) in sorted(stems.items(), key=lambda kv: -kv[1][1]):
        print(f"    {k:40s} x{n:<3d} {us:9.1f} us")


def run(which):
    torch.manual_seed(0)
    model, C = build(which)
    x = torch.randn(B, C, T, device="cuda")
    sigma = torch.rand(B, device="cuda")
    print(f"config ({which}): {'LTPlugin stereo x 32 filters' if which == 'a' else '5.1 DiffusionModel'}, "
          f"B={B}, T=2^18, {sum(p.numel() for p in model.parameters()) / 1e6:.1f} M parameters")

    def evaluate():
        with torch.no_grad():
            model.net(x, sigma)

    def train_step():
        model.zero_grad(set_to_none=True)
        model(x).backward()

    for _ in range(3):
        evaluate()
        train_step()
    print(f"  evaluation of v: {timed(evaluate, 10):.2f} ms   training step: {timed(train_step, 5):.2f} ms")
    kernel_table(evaluate, "evaluation")
    kernel_table(train_step, "training step")
    del model
    torch.cuda.empty_cache()


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(f"card: {torch.cuda.get_device_name(0)}; nvidia-smi: {q.stdout.strip() or q.stderr.strip()}")
    for which in sys.argv[1:] or ["a", "b"]:
        run(which)


if __name__ == "__main__":
    main()
