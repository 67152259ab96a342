"""Every launch of the vocoder, inpainting and autoregressive programs checked against an fp64
restatement (tests/launch_check.py), and the front-end kernels at the sizes where they go wrong:

  * cfg5, the benchmark's vocoder sample (16 rows, 80 mels x 1024 frames -> 2^18 samples): to_flat,
    then the sampling program;
  * a vocoder training step at cfg5's shape: mel_spectrogram and to_flat forward, the loss, and the
    backward with to_flat_bwd's weight gradient;
  * VInpainter on the README net (2 steps x 2 resamples): the alpha / beta row every inpaint_blend is
    handed is the one the reference uses -- the launch check verifies a launch against the operands
    it is given and cannot see the device step selector pass the wrong row;
  * DiffusionAR on the README widths (the SkipCat net, no time conditioning): the start window and
    five ladder passes, each arv_step handed sigma_{i+1};
  * direct launches of mel_spectrogram, to_flat / to_flat_bwd, inpaint_blend and arv_step at edge
    sizes, with distinct rows so that a row-stride error shows.

Each program's checked eager run is followed by the same call three times with the CUDA graph on,
compared on a well-conditioned output (a one-step sample: x_1 = -v at sigma = 1; see
test_launch_check_gpu.py).  Run with -s for the per-kind tables."""
import gc
import time

import pytest
import torch

import launch_check as lc

pytestmark = pytest.mark.gpu

DEV = "cuda"
T_FULL = 2 ** 18
UNET9 = dict(channels=[8, 32, 64, 128, 256, 512, 512, 1024, 1024],
             factors=[1, 4, 4, 4, 2, 2, 2, 2, 2], items=[1, 2, 2, 2, 2, 2, 2, 4, 4])
README = dict(in_channels=2, attentions=[0, 0, 0, 0, 0, 1, 1, 1, 1], attention_heads=8, attention_features=64,
              **UNET9)
# the benchmark's cfg5 (bench.py)
VOCODER = dict(mel_n_fft=1024, mel_channels=80, mel_sample_rate=48000, mel_normalize_log=True, **UNET9)
# Graph replay against the checked eager run, observed on an H100 80GB HBM3 (700 W limit):
#   * vocoder training step: the loss bit-equal (bound 1e-6 relative, as for cfg4) and
#     to_flat.weight.grad 3.6e-7 and 3.9e-7 rel-L2 in two runs (an eager rerun: 3.4e-7, 3.9e-7);
#     bound 2e-6, ~5x the observed;
#   * the SkipCat net of DiffusionAR has no identity skip (SkipCat merges x through a 1x1 conv), so
#     v = -x_1 is all branch and carries any run-to-run jitter of the GroupNorm statistics undiluted:
#     1.6e-4 rel-L2 graph against checked run and replay against replay alike while narrow_conv added
#     its warps' partial sums with fp32 shared-memory atomics (3.2e-3 on some runs); bitwise equal
#     since it adds them in a fixed order.  Bound 1e-3 (the 1e-4 of the other programs assumes
#     v = skip + a branch of ~1 % of it).
FLAT_GRAD_TOL, SKIPCAT_REPLAY_TOL = 2e-6, 1e-3


@pytest.fixture(scope="module")
def adp():
    import audio_diffusion_pytorch_b200 as adp
    from audio_diffusion_pytorch_b200 import ops
    ops.device_check()
    print("\n" + torch.cuda.get_device_name(0))
    return adp


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _checked(call, what):
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    with lc.Shadow() as sh:
        out = call().clone()
    torch.cuda.synchronize()
    print(f"\n{what}: {time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB"
          f"\n{sh.table()}")
    print(f"{what}: n_checked {sh.n_checked} == n_launch {sh.n_launch}")
    assert sh.n_checked == sh.n_launch > 0
    return out, sh


def _graph_vs_checked(net, call, what, tol=1e-4):
    """call() checked once (eager), then three times unwrapped with the CUDA graph on."""
    net.use_cuda_graph = False
    out, _ = _checked(call, what)
    net.use_cuda_graph = True
    net._plans.clear()
    runs = [call().clone() for _ in range(3)]
    e = rel_l2(runs[2], out)
    print(f"{what}: graph replay vs checked eager run: rel-L2 {e:.3e} "
          f"(replay vs replay {rel_l2(runs[2], runs[1]):.3e})")
    assert e <= tol, f"{what}: the captured graph disagrees with the checked run ({e:.3e})"
    net.use_cuda_graph = False
    return out


def _kinds(sh):
    return {k.split(".")[0] for k in sh.records}


def test_cfg5_sample(adp):
    """The benchmark's vocoder sample: mel [8, 2, 80, 1024] -> 16 rows of 2^18 samples, 2 steps."""
    t0 = time.perf_counter()
    torch.manual_seed(1234)
    model = adp.DiffusionVocoder(net_t=adp.UNetV0, **VOCODER).to(DEV)
    mel = torch.randn(8, 2, 80, T_FULL // 256, generator=torch.Generator().manual_seed(0)).to(DEV)
    try:
        with torch.no_grad():
            model.net.use_cuda_graph = False
            out, sh = _checked(lambda: model.sample(mel, num_steps=2, generator=torch.Generator().manual_seed(7)),
                               "cfg5 sample(num_steps=2) 16 rows")
            assert out.shape == (8, 2, T_FULL)
            assert sh.records["to_flat.out"].count == 1 and {"stem_in", "stem_out", "conv_gemm"} <= _kinds(sh)
            one = _graph_vs_checked(model.net, lambda: model.sample(mel, num_steps=1,
                                                                    generator=torch.Generator().manual_seed(7)),
                                    "cfg5 sample(num_steps=1), for the graph comparison")
            assert torch.isfinite(one).all()
    finally:
        del model
        _free()
    print(f"test_cfg5_sample: {time.perf_counter() - t0:.1f} s")


def test_vocoder_training_step(adp):
    """DiffusionVocoder's training step at cfg5's shape: audio [4, 2, 2^18] -> mel_spectrogram (log),
    to_flat, the net, the fused loss, the backward and to_flat_bwd (dw only: the audio needs no
    gradient); then the same step with CUDA graphs."""
    from test_launch_check_train_gpu import _room, _step_and_compare
    t0 = time.perf_counter()
    _room(16)
    torch.manual_seed(1234)
    model = adp.DiffusionVocoder(net_t=adp.UNetV0, **VOCODER).to(DEV)
    audio = torch.randn(4, 2, T_FULL, generator=torch.Generator().manual_seed(3)).to(DEV)
    seen = []                     # (loss, to_flat.weight.grad) of every step: checked, rerun, 3 graph runs

    def step():
        model.zero_grad(set_to_none=True)
        torch.manual_seed(77)
        loss = model(audio)
        loss.backward()
        seen.append((loss.detach().clone(), model.to_flat.weight.grad.clone()))
        return loss.detach().clone(), [p.grad.clone() for p in model.parameters()]
    try:
        sh = _step_and_compare(model, step, "vocoder training step 8 rows T=2^18")
        assert {"mel_spectrogram", "to_flat", "to_flat_bwd", "stem_out", "stem_in_bwd"} <= _kinds(sh)
        assert sh.records["mel_spectrogram.mel"].count == sh.records["to_flat_bwd.dw"].count == 1
        assert "to_flat_bwd.dspec" not in sh.records
        (loss0, g0), (loss_g, g_g) = seen[0], seen[-1]
        e_loss, e_w = abs(float(loss_g) - float(loss0)) / abs(float(loss0)), rel_l2(g_g, g0)
        print(f"vocoder step: graph replay vs checked run: loss {float(loss0):.6f} (relative difference "
              f"{e_loss:.3e}), to_flat.weight.grad rel-L2 {e_w:.3e} (eager rerun {rel_l2(seen[1][1], g0):.3e})")
        assert e_loss <= 1e-6 and e_w <= FLAT_GRAD_TOL
    finally:
        del model
        _free()
    print(f"test_vocoder_training_step: {time.perf_counter() - t0:.1f} s")


def test_inpainter_readme(adp):
    """VInpainter around the README net, B = 2, T = 2^18, 2 steps x 2 resamples: the "stay" and
    "advance" alpha / beta rows both occur, and every inpaint_blend is handed the reference's row."""
    from audio_diffusion_pytorch_b200 import ops
    from audio_diffusion_pytorch_b200.diffusion import LinearSchedule, _alpha_beta
    t0 = time.perf_counter()
    torch.manual_seed(1234)
    model = adp.DiffusionModel(net_t=adp.UNetV0, **README).to(DEV)
    g = torch.Generator().manual_seed(4)
    source = torch.randn(2, 2, T_FULL, generator=g).to(DEV)
    mask = torch.zeros(2, 2, T_FULL, dtype=torch.bool)
    mask[0, :, : T_FULL // 3] = True
    mask[1, :, T_FULL // 2: T_FULL // 2 + 40000] = True
    mask = mask.to(DEV)
    inpainter = adp.VInpainter(net=model.net)
    steps, resamples = 2, 2

    def inpaint(num_steps, num_resamples):
        torch.manual_seed(9)
        return inpainter(source, mask, num_steps=num_steps, num_resamples=num_resamples)
    try:
        with torch.no_grad():
            model.net.use_cuda_graph = False
            handed = []
            with lc.Shadow() as sh:
                checked = ops.inpaint_blend

                def recording(x, src, noise, mask_u8, ab):
                    handed.append(ab.clone())
                    return checked(x, src, noise, mask_u8, ab)
                ops.inpaint_blend = recording            # Shadow puts the real function back on exit
                inpaint(steps, resamples)
            print(f"\nVInpainter README B=2 T=2^18 {steps} steps x {resamples} resamples\n{sh.table()}")
            print(f"VInpainter: n_checked {sh.n_checked} == n_launch {sh.n_launch}")
            assert sh.n_checked == sh.n_launch > 0
            assert sh.records["inpaint_blend.x"].count == steps * resamples
            sig = LinearSchedule()(steps + 1, device=DEV)
            a, b = (t.float() for t in _alpha_beta(sig))
            want = [torch.stack([a[i], b[i], a[i + j], b[i + j]]) for i in range(steps)
                    for j in (int(r == resamples - 1) for r in range(resamples))]
            assert len(handed) == len(want)
            for k, (h, w) in enumerate(zip(handed, want)):
                assert torch.equal(h, w), \
                    f"evaluation {k}: inpaint_blend handed {h.tolist()}, the schedule's row is {w.tolist()}"
            one = _graph_vs_checked(model.net, lambda: inpaint(1, 1),
                                    "VInpainter 1 step x 1 resample, for the graph comparison")
            assert torch.equal(one[mask], source[mask])      # sigma = 0: the known region is the source
    finally:
        del model, inpainter
        _free()
    print(f"test_inpainter_readme: {time.perf_counter() - t0:.1f} s")


def test_autoregressive_readme(adp):
    """DiffusionAR on the README widths (in_channels 2, length 2^16, 4 splits): the start window (4
    steps, one sigma for the window) and five ladder passes (one step each, a sigma per position) --
    the SkipCat net under Shadow; every arv_step is handed sigma_{i+1} of its ladder."""
    from audio_diffusion_pytorch_b200 import ops
    t0 = time.perf_counter()
    length, n = 2 ** 16, 4
    torch.manual_seed(1234)
    model = adp.DiffusionAR(net_t=adp.UNetV0, length=length, num_splits=n, **README).to(DEV)
    sampler = model.sampler
    try:
        with torch.no_grad():
            model.net.use_cuda_graph = False
            handed = []
            with lc.Shadow() as sh:
                checked = ops.arv_step

                def recording(chan, v, sig_next):
                    handed.append(sig_next.clone())
                    return checked(chan, v, sig_next)
                ops.arv_step = recording
                torch.manual_seed(5)
                out = model.sample(num_items=2, num_chunks=5, num_steps=4)
            print(f"\nDiffusionAR README widths T=2^16, 5 chunks x 4 steps\n{sh.table()}")
            print(f"DiffusionAR: n_checked {sh.n_checked} == n_launch {sh.n_launch}")
            assert sh.n_checked == sh.n_launch > 0 and out.shape == (2, 2, 5 * length // n)
            assert {"conv_gemm", "attention", "arv_step"} <= _kinds(sh)
            start = torch.linspace(1, 0, 5, device=DEV)
            ladder = sampler.get_sigmas_ladder(num_items=2, num_steps_per_split=1).float()
            want = [start[i].expand(2, length) for i in range(1, 5)] + [ladder[1].reshape(2, length)] * 5
            assert len(handed) == len(want) == sh.records["arv_step.chan"].count
            for k, (h, w) in enumerate(zip(handed, want)):
                assert torch.equal(h, w), f"step {k}: arv_step handed another sigma row than sigma_(i+1)"
            current = torch.randn(2, 2, length, generator=torch.Generator().manual_seed(6)).to(DEV)
            sig = torch.tensor([1.0, 0.0], device=DEV)[:, None, None, None].expand(2, 2, 1, length)
            _graph_vs_checked(model.net, lambda: sampler.sample_loop(current, sig),
                              "DiffusionAR one-step window sigma 1 -> 0, for the graph comparison",
                              tol=SKIPCAT_REPLAY_TOL)
    finally:
        del model, sampler
        _free()
    print(f"test_autoregressive_readme: {time.perf_counter() - t0:.1f} s")


# ------------------------------------------------------------------------- edge launches
def _rows(g, rows, t):
    """Distinct rows: row r scaled by 1 + r."""
    return (torch.randn(rows, t, generator=g) * torch.arange(1, rows + 1)[:, None]).to(DEV)


# (n_fft, hop, win_length, n_mels, sample_rate, t, pad or None for (n_fft - hop) // 2, log)
MEL_EDGES = {
    "n_fft32": (32, 8, 32, 8, 16000, 1000, None, False),
    "n_fft1024": (1024, 256, 1024, 80, 48000, 2 ** 14, None, True),
    "n_fft4096": (4096, 1024, 4096, 128, 48000, 2 ** 16, None, True),       # the kernel's maximum, ~70 KB smem
    "win_lt_n_fft": (256, 64, 160, 24, 16000, 5000, None, False),
    "frames1": (256, 64, 256, 24, 16000, 100, None, True),
    "frames7": (256, 64, 256, 24, 16000, 465, None, True),
    "frames9": (256, 64, 256, 24, 16000, 581, None, True),
    "prime_frames_2e18": (1024, 241, 1024, 80, 48000, 2 ** 18, None, True),  # 1087 frames
    "pad0": (256, 256, 256, 24, 16000, 2660, 0, False),
    "just_long_enough": (256, 64, 256, 24, 16000, 97, None, False),          # t = pad + 1: both ends reflect
    "n_mels512": (2048, 512, 2048, 512, 48000, 2 ** 15, None, True),
    "empty_filters": (256, 64, 256, 128, 16000, 4000, None, True),            # 128 mels over 129 bins
}


def test_mel_spectrogram_edges(adp):
    from audio_diffusion_pytorch_b200 import ops
    from audio_diffusion_pytorch_b200.components import MelSpectrogram
    t0 = time.perf_counter()
    g = torch.Generator().manual_seed(8)
    with lc.Shadow() as sh:
        for name, (n_fft, hop, win, n_mels, sr, t, pad, log) in MEL_EDGES.items():
            front = MelSpectrogram(n_fft=n_fft, hop_length=hop, win_length=win, sample_rate=sr, n_mel_channels=n_mels)
            window, fb, band = front._kernel_tables(DEV)
            pad = front.padding if pad is None else pad
            mel = ops.mel_spectrogram(_rows(g, 3, t), window, fb, band, n_fft, hop, pad, apply_log=log)
            frames = mel.shape[-1]
            if name.startswith("frames"):
                assert frames == int(name[6:]), name
            if name == "prime_frames_2e18":
                assert frames == 1087
            if name == "just_long_enough":
                assert frames == 1 and t == pad + 1
            if name == "empty_filters":
                empty = band[:, 0] == band[:, 1]
                assert bool(empty.any()), "the filterbank has no empty filter"
                print(f"mel_spectrogram {name}: {int(empty.sum())} empty filters of {n_mels}")
    print(f"\nmel_spectrogram edges: {time.perf_counter() - t0:.1f} s\n{sh.table()}")
    assert sh.n_checked == sh.n_launch == len(MEL_EDGES)


# (C, frames, win, hop, pad or None for (win - hop) // 2)
FLAT_EDGES = {
    "hop_not_dividing_win": (20, 50, 100, 30, None),
    "hop_gt_win_pad0": (16, 20, 64, 100, 0),          # output samples no frame reaches
    "frames1": (80, 1, 1024, 256, None),
    "win12288": (16, 10, 12288, 3072, None),          # dspec's 48 KB shared-memory window
    "C13": (13, 40, 256, 64, None),                   # dspec: a warp per channel, strided by 8
    "cfg5": (80, 1024, 1024, 256, None),
}


def test_to_flat_edges(adp):
    from audio_diffusion_pytorch_b200 import ops
    t0 = time.perf_counter()
    g = torch.Generator().manual_seed(9)
    with lc.Shadow(probe=True) as sh:
        for name, (C, frames, win, hop, pad) in FLAT_EDGES.items():
            pad = (win - hop) // 2 if pad is None else pad
            spec = (torch.randn(3, C, frames, generator=g) * torch.arange(1, 4)[:, None, None]).to(DEV)
            w = (torch.randn(C, win, generator=g) / C).to(DEV)
            out = ops.to_flat(spec, w, hop, pad)
            dout = _rows(g, 3, out.shape[1])
            for need_dspec, need_dw in ((True, True), (True, False), (False, True)):
                ops.to_flat_bwd(spec, w, dout, hop, pad, need_dspec, need_dw)
    print(f"\nto_flat edges: {time.perf_counter() - t0:.1f} s\n{sh.table()}")
    assert sh.n_checked == sh.n_launch == 4 * len(FLAT_EDGES)
    assert sh.records["to_flat_bwd.dspec"].count == sh.records["to_flat_bwd.dw"].count == 2 * len(FLAT_EDGES)


def test_sampler_step_edges(adp):
    from audio_diffusion_pytorch_b200 import ops
    t0 = time.perf_counter()
    g = torch.Generator().manual_seed(10)
    ab = torch.tensor([0.8, 0.6, 0.9, 0.43589], device=DEV)
    with lc.Shadow(probe=True) as sh:
        n = 100003                                      # not a multiple of any grid stride
        x = _rows(g, 6, n).reshape(3, 2, n)
        mask = torch.rand(3, 2, n, generator=g) < 0.5
        ops.inpaint_blend(x, _rows(g, 6, n).reshape(3, 2, n), _rows(g, 6, n).reshape(3, 2, n),
                          mask.to(torch.uint8).to(DEV), ab)
        iso = torch.zeros(3 * 2 * n, dtype=torch.uint8)
        iso[::7] = 1                                    # isolated single elements
        ops.inpaint_blend(x, _rows(g, 6, n).reshape(3, 2, n), _rows(g, 6, n).reshape(3, 2, n),
                          iso.reshape(3, 2, n).to(DEV), ab)
        for B, C, T in ((3, 1, 1000), (4, 2, 2 ** 16 + 3)):
            chan = _rows(g, B * (C + 1), T).reshape(B, C + 1, T)
            chan[:, C] = torch.rand(B, T, generator=g).to(DEV)
            sig_next = chan[:, C] * torch.rand(B, T, generator=g).to(DEV)
            ops.arv_step(chan, _rows(g, B * C, T).reshape(B, C, T), sig_next.contiguous())
    print(f"\nsampler step edges: {time.perf_counter() - t0:.1f} s\n{sh.table()}")
    assert sh.n_checked == sh.n_launch == 4
