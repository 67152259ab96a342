"""Where a cfg4 training step (DiffusionUpsampler, B=4 x [2,2^18], fwd + bwd + AdamW) spends its
time: host-timed phases + in-graph kernel durations of the forward and backward graphs (CUPTI,
aggregated per kernel + shape label).  usage: python tools/time_train.py [batch]"""
import os, sys, time
from collections import defaultdict
import torch
from torch.profiler import ProfilerActivity, profile
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import audio_diffusion_pytorch_b200 as adp
from audio_diffusion_pytorch_b200 import ops, _lib
from bench import UPSAMPLER, LENGTH
_lib.lib().adp_debug_set(6, 0)        # PDL off: kernel durations must not overlap in the profile
B = int(sys.argv[1]) if len(sys.argv) > 1 else 4
dev = torch.device("cuda")
model = adp.DiffusionUpsampler(net_t=adp.UNetV0, **UPSAMPLER).to(dev)
opt = torch.optim.AdamW(model.parameters(), lr=1e-4, fused=True)
audio = torch.randn(B, 2, LENGTH, device=dev)
def step():
    opt.zero_grad(set_to_none=True); loss = model(audio); loss.backward(); opt.step()
for _ in range(4): step()
torch.cuda.synchronize()
net = model.net
def timeit(name, fn, n=5):
    torch.cuda.synchronize(); t0 = time.perf_counter()
    for _ in range(n): fn()
    torch.cuda.synchronize(); print(f"{name:30s} {(time.perf_counter()-t0)/n*1e3:8.2f} ms", flush=True)
plan = next(p for k, p in net._plans.items() if k[0] == "train")
timeit("full step", step)
def repack():
    net._packed_version = -1; net.packed()
    with torch.no_grad():
        for r in plan.refreshers: r()
timeit("repack fwd+dgrad weights", repack)
timeit("forward graph", lambda: plan.forward.graph.replay())
timeit("backward graph", lambda: plan.backward.graph.replay())
timeit("finals", lambda: [f() for f in plan.finals])
timeit("optimizer step", lambda: opt.step())
timeit("reupsample", lambda: model.reupsample(audio))

def graph_table(which):
    graphed = plan.forward if which == "f" else plan.backward
    prog, graph = graphed.run, graphed.graph
    with ops.trace() as tr:
        prog()
    torch.cuda.synchronize()
    labels = []
    for r in tr.records:        # adp_attention_bwd = 3 kernels per record
        labels += [r] * (3 if r["name"].startswith("attention_bwd") else 1)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        graph.replay(); torch.cuda.synchronize()
    ks = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "adp::" in e.name),
                key=lambda e: e.time_range.start)
    assert len(ks) == len(labels), (len(ks), len(labels))
    agg = defaultdict(lambda: [0, 0.0, 0.0, 0.0])
    for e, r in zip(ks, labels):
        a = agg[r["name"]]; a[0] += 1; a[1] += e.time_range.end - e.time_range.start; a[2], a[3] = r["flops"], r["bytes"]
    tot = sum(a[1] for a in agg.values())
    print(f"--- {'forward' if which == 'f' else 'backward'} graph: {len(ks)} adp kernels, kernel-busy {tot / 1e3:.2f} ms")
    fam = defaultdict(float)
    for k, a in agg.items():
        fam[k.split("[")[0]] += a[1]
    print("by family: " + ", ".join(f"{k} {v / 1e3:.2f} ms" for k, v in sorted(fam.items(), key=lambda kv: -kv[1])))
    for k, a in sorted(agg.items(), key=lambda kv: -kv[1][1])[:28]:
        us = a[1] / a[0]
        print(f"  {k[:60]:60s} x{a[0]:3d} avg {us:8.1f} us total {a[1] / 1e3:7.3f} ms  {a[2] / us / 1e6:7.1f} TF/s {a[3] / us / 1e3:7.1f} GB/s")
graph_table("f")
graph_table("b")
