"""Times the mel front-end kernel (adp_mel_spectrogram) on the shape of a cfg5-sized training batch:
16 rows (8 stereo clips) of t = 2^18 samples, CUDA events around many launches.

    python tools/time_mel.py [--rounds 5] [--launches 50] [--parent-lib PATH]

Sizes: n_fft 1024 / hop 256 / 80 mels (the vocoder's default), then 400, 1200, 1920 and 8192 (hop
n_fft / 4), each also through torchaudio's CUDA route (torch.stft + MelScale on the GPU) as a
yardstick.  With --parent-lib, a libadp_b200.so built from the commit before `center_pad` joined the
C ABI (the radix-2 kernel, n_fft a power of two) is timed at n_fft 1024 against this build, the two
alternating round by round in one process, and their outputs are compared.  Prints the card and its
power limit.
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROWS, T = 16, 2 ** 18
SIZES = [(1024, 256, 80), (400, 100, 80), (1200, 300, 80), (1920, 480, 128), (8192, 2048, 128)]


def timed(fn, launches):
    fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(launches):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / launches


def parent_launcher(path):
    """adp_mel_spectrogram of a library without center_pad: 5 pointers, 8 ints, the stream."""
    lib = C.CDLL(path)
    fn = lib.adp_mel_spectrogram
    fn.argtypes = [C.c_void_p] * 5 + [C.c_int] * 8 + [C.c_void_p]
    fn.restype = C.c_int

    def mel(wave, window, fb, band, n_fft, hop, pad, apply_log):
        rows, t = wave.shape
        n_mels = fb.shape[1]
        frames = 1 + (t + 2 * pad - n_fft) // hop
        out = torch.empty(rows, n_mels, frames, device=wave.device)
        rc = fn(wave.data_ptr(), window.data_ptr(), fb.data_ptr(), band.data_ptr(), out.data_ptr(), rows, t, n_fft,
                hop, pad, frames, n_mels, int(apply_log), torch.cuda.current_stream().cuda_stream)
        assert rc == 0, "parent adp_mel_spectrogram failed"
        return out
    return mel


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--parent-lib", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_mel.py measures on the GPU"
    sys.path.insert(0, ROOT)
    from audio_diffusion_pytorch_b200 import ops
    from audio_diffusion_pytorch_b200.components import MelSpectrogram
    ops.device_check()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    print(f"{ROWS} rows x {T} samples, {a.launches} launches per timing, {a.rounds} rounds")
    wave = torch.randn(ROWS, T, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
    parent = parent_launcher(a.parent_lib) if a.parent_lib else None
    for n_fft, hop, n_mels in SIZES:
        front = MelSpectrogram(n_fft=n_fft, hop_length=hop, win_length=n_fft, sample_rate=48000,
                               n_mel_channels=n_mels, normalize_log=True).cuda()
        window, fb, band = front._kernel_tables(wave.device)
        pad = front.padding
        runs = {"kernel": lambda: ops.mel_spectrogram(wave, window, fb, band, n_fft, hop, pad, apply_log=True),
                "torch.stft+MelScale": lambda: torch.log(torch.clamp(front.to_mel_scale(torch.abs(
                    front.to_spectrogram(F.pad(wave, [pad] * 2, mode="reflect")))), min=1e-5))}
        if parent is not None and n_fft == 1024:
            runs = {"parent kernel": lambda: parent(wave, window, fb, band, n_fft, hop, pad, True), **runs}
            e = float((runs["kernel"]() - runs["parent kernel"]()).abs().max())
            print(f"n_fft {n_fft}: max |this build - parent| of the log-mel: {e:.3e}")
        times = {k: [] for k in runs}
        for _ in range(a.rounds):
            for k, fn in runs.items():
                times[k].append(timed(fn, a.launches))
        for k, ts in times.items():
            ts = sorted(ts)
            print(f"n_fft {n_fft:5d} hop {hop:4d} mels {n_mels:3d}  {k:22s} median {ts[len(ts) // 2] * 1e3:8.1f} us  "
                  f"range {ts[0] * 1e3:.1f}-{ts[-1] * 1e3:.1f} us")


if __name__ == "__main__":
    main()
