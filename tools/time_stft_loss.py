"""Times MultiResolutionSTFTLoss forward + backward (csrc/stft_loss.cu) against the same definition
in torch ops (torch.stft on cuFFT, autograd), on a B = 4, C = 2, T = 2^18 batch with the default
resolutions (1024/120/600, 2048/240/1200, 512/50/240), CUDA events around many calls, the two routes
alternating round by round in one process.  Also times each route's forward alone and prints how
far each is from a float64 evaluation.  Prints the card and its power limit.

    python tools/time_stft_loss.py [--rounds 5] [--calls 20]
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, CH, T = 4, 2, 2 ** 18


def timed(fn, calls):
    fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(calls):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_stft_loss.py measures on the GPU"
    sys.path.insert(0, ROOT)
    from audio_diffusion_pytorch_b200 import losses, ops
    ops.device_check()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    print(f"B {B} x C {CH} x T {T}, default resolutions, {a.calls} calls per timing, {a.rounds} rounds")
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(B, CH, T, device="cuda", generator=g)
    y = torch.randn(B, CH, T, device="cuda", generator=g)
    mod = losses.MultiResolutionSTFTLoss()
    res = [(f.fft_size, f.hop_size, f.win_length) for f in mod.stft_losses]
    weights = (1.0, 1.0, 0.0)

    def kernel_fwd():
        return mod(x, y)

    def torch_fwd(v=x):
        return losses._host_loss(v, y, res, weights, 1e-8)      # the definition in torch ops

    def step(fwd):
        def run():
            xg = x.detach().requires_grad_(True)
            fwd(xg).backward()
            return xg.grad
        return run

    runs = {"kernels fwd+bwd": step(lambda v: mod(v, y)), "torch ops fwd+bwd": step(torch_fwd),
            "kernels fwd": lambda: mod(x, y), "torch ops fwd": torch_fwd}
    x64 = x.double().requires_grad_(True)
    want = losses._host_loss(x64, y.double(), res, weights, 1e-8)
    want.backward()
    for name, fwd in (("kernels", lambda v: mod(v, y)), ("torch ops", torch_fwd)):
        xg = x.detach().requires_grad_(True)
        loss = fwd(xg)
        loss.backward()
        e_l = abs(float(loss.detach()) - float(want.detach())) / float(want.detach())
        e_dx = float((xg.grad.double() - x64.grad).norm() / x64.grad.norm())
        print(f"{name:10s} loss rel err {e_l:.2e}, dx rel-L2 {e_dx:.2e} against float64")
    times = {k: [] for k in runs}
    for _ in range(a.rounds):
        for k, fn in runs.items():
            times[k].append(timed(fn, a.calls))
    for k, ts in times.items():
        ts = sorted(ts)
        print(f"{k:20s} median {ts[len(ts) // 2]:8.3f} ms  range {ts[0]:.3f}-{ts[-1]:.3f} ms")
    with ops.trace(timing=True) as tr:
        step(lambda v: mod(v, y))()
    for row in tr.table().values():
        print(f"  {row['name']:28s} {row['ms_avg'] * 1e3:8.1f} us")


if __name__ == "__main__":
    main()
