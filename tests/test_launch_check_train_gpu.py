"""Every kernel launch of a full-size training step -- forward, loss and backward -- checked
against an fp64 restatement (tests/launch_check.py): each launch on the activations and gradients
the real step gives it, into the real gradient arena (every accumulator is a view of one storage,
and no byte of it outside the written view may change), held to its own bound.

  * cfg4, the benchmark's training step: DiffusionUpsampler, batch 4, 2^18 samples;
  * the text-conditional README net at batch 2, 2^18 samples, through the differentiable forward with
    input and embedding gradients: self-attention backward at 1024 ... 128 positions, cross-attention
    backward over 64 tokens, the folded LayerNorm projections, the dxin paths of the stems;
  * one step after an AdamW update (2^14 samples): the launches then read the weight packs refreshed
    in place; and that step against the same step on packs and plans built afresh;
  * direct launches of wgrad (single split, both store paths; split over 2^20 rows), colsum and
    gn_silu_bwd into accumulators that hold something, as views inside a larger non-zero arena: in a
    training step every accumulator is zero before its one launch, so a launch that stored instead
    of adding would pass there.

The wrapped steps are eager and synchronised.  Each test then runs the same model and inputs
unwrapped with CUDA graphs on (eager, capture + replay, replay) and requires the replayed loss and
every gradient to agree with the checked run: the fp32 split-K and bin atomics land in another
order, nothing else may differ.  Run with -s for the per-kind tables."""
import gc
import time

import pytest
import torch

import launch_check as lc

pytestmark = pytest.mark.gpu

DEV = "cuda"
T_FULL = 2 ** 18
# the benchmark's workloads (bench.py)
UNET9 = dict(channels=[8, 32, 64, 128, 256, 512, 512, 1024, 1024],
             factors=[1, 4, 4, 4, 2, 2, 2, 2, 2], items=[1, 2, 2, 2, 2, 2, 2, 4, 4])
UPSAMPLER = dict(upsample_factor=16, in_channels=2, **UNET9)
CFG3 = dict(in_channels=2, attentions=[0, 0, 0, 0, 0, 1, 1, 1, 1], attention_heads=8, attention_features=64,
            cross_attentions=[0, 0, 0, 1, 1, 1, 1, 1, 1], use_embedding_cfg=True, embedding_max_length=64,
            embedding_features=768, **UNET9)
BACKWARD = {"wgrad", "gn_silu_bwd", "gn_bwd_apply", "ln_film_bwd", "colsum", "skip_gate_bwd", "cond_bwd",
            "narrow_conv_bwd", "stem_out_bwd", "stem_in_bwd"}       # of a net without attention
# Graph replay against the checked eager run, worst parameter rel-L2.  Observed on an H100 80GB HBM3
# (700 W limit): 1.5e-3 for cfg4 and 1.6e-2 for the text net, both on a parameter of the deepest
# levels, whose gradients in an untrained net are ~1e-15 and follow every bf16 rounding flip of the
# long chain above them -- and the SAME size as an eager rerun against the eager run (1.2e-3, 1.7e-2),
# which the test prints next to it.  Level 0 .. 2 agree to ~1e-5.  The bound is 3 x the largest
# observed; the loss differed by 0 (cfg4).
# observed.  It holds for every parameter; those whose gradient rms is at least SMALL_RMS of the
# largest one (levels 0 .. 2 of the untrained nets) are held to a bound per test: 2e-4 for the loss
# steps (observed 1.7e-5 against the graph, 4.1e-5 between two eager runs), 1e-2 for the text step,
# whose loss sum(v w) with a random w of size 1/T leaves gradients that two eager runs already
# reproduce only to 3.3e-3 at level 1.  The eager rerun must meet the same bounds.
GRAD_REPLAY_TOL, SMALL_RMS, LOSS_REPLAY_TOL = 5e-2, 1e-4, 1e-6


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


def _room(gib):
    free = torch.cuda.mem_get_info()[0] / 2 ** 30
    assert free >= gib, f"{free:.1f} GiB of device memory free, this test needs about {gib} GiB"


def _kinds(sh):
    return {k.split(".")[0] for k in sh.records}


def _step_and_compare(model, step, what, extra=(), names=None, large_tol=2e-4):
    """step() -> (loss or None, [gradients]) once under Shadow (eager), then three times unwrapped
    with CUDA graphs on and fresh plans; returns the Shadow."""
    net = model.net
    net.use_cuda_graph = False
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    with lc.Shadow() as sh:
        loss, grads = step()
        for fn in extra:
            fn()
    torch.cuda.synchronize()
    print(f"\n{what}: {time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB"
          f"\n{sh.table()}")
    assert sh.n_checked == sh.n_launch > 0
    names = names or [n for n, _ in model.named_parameters()]
    assert len(names) == len(grads)
    # conv1.bias of a level with one channel per GroupNorm group (level 0: 8 channels, 8 groups) feeds
    # nothing but that GroupNorm, which removes it: its exact gradient is zero and what the step
    # computes is the rounding noise of a sum that cancels (rms ~1e-10 next to 0.3 for its peers)
    zero_grads = {n for n in names if n.endswith("resnet.conv1.bias") and n.count("inner") == 0
                  and net.groups == UNET9["channels"][0]}
    assert len(zero_grads) == 2 * UNET9["items"][0]

    rms = [float(w.double().norm()) / w.numel() ** 0.5 for w in grads]

    def worst_of(got):
        """(worst rel-L2 / its bound, rel-L2, name) over the parameters."""
        worst = (0.0, 0.0, "")
        for n, g, w, r in zip(names, got, grads, rms):
            if n in zero_grads:
                continue
            e = rel_l2(g, w)
            tol = large_tol if r >= SMALL_RMS * max(rms) else GRAD_REPLAY_TOL
            worst = max(worst, (e / tol, e, n))
        return worst
    # the run-to-run spread of the eager step itself (same plans, same inputs): what atomics' order does
    rerun = worst_of(step()[1])
    print(f"{what}: eager rerun vs checked eager run: worst gradient rel-L2 / bound {rerun[0]:.3f} "
          f"(rel-L2 {rerun[1]:.3e}, {rerun[2]})")
    assert rerun[0] <= 1.0, "the eager step does not reproduce itself within the replay bounds"
    net.use_cuda_graph = True
    net._plans.clear()
    for _ in range(3):                       # eager, capture + replay, replay
        loss_g, grads_g = step()
    worst, e_worst, worst_name = worst_of(grads_g)
    line = (f"{what}: graph replay vs checked eager run: worst gradient rel-L2 / bound {worst:.3f} "
            f"(rel-L2 {e_worst:.3e}, {worst_name}) of {len(grads)}")
    if loss is not None:
        e_loss = abs(float(loss_g) - float(loss)) / abs(float(loss))
        line += f", loss {float(loss):.6f}, relative difference {e_loss:.3e}"
        assert e_loss <= LOSS_REPLAY_TOL, line
    print(line)
    assert len(grads) == len(grads_g) > 0 and worst <= 1.0, line
    return sh


def _free(*objs):
    del objs
    gc.collect()
    torch.cuda.empty_cache()


def _loss_step(model, audio, seed=77):
    def step():
        model.zero_grad(set_to_none=True)
        torch.manual_seed(seed)              # the same sigmas and noise for every run
        loss = model(audio)
        loss.backward()
        return loss.detach().clone(), [p.grad.clone() for p in model.parameters()]
    return step


def test_cfg4_training_step(adp):
    """The benchmark's train_step: DiffusionUpsampler, batch 4, 2^18 samples, fused loss."""
    from audio_diffusion_pytorch_b200 import ops
    from audio_diffusion_pytorch_b200.utils import _polyphase_bank
    _room(16)
    torch.manual_seed(1234)
    model = adp.DiffusionUpsampler(net_t=adp.UNetV0, **UPSAMPLER).to(DEV)
    audio = torch.randn(4, 2, T_FULL, generator=torch.Generator().manual_seed(0)).to(DEV)

    def adjoint():       # the clip does not require grad, so the step never runs the resampler's backward
        bank, half = _polyphase_bank(16, 1, 0.99, 6, torch.float32, DEV)
        dy = torch.randn(8, T_FULL // 16, generator=torch.Generator().manual_seed(5)).to(DEV)
        ops.fir_resample(dy, bank[:, 0].contiguous(), 16, 1, half, T_FULL // 16, adjoint_of=T_FULL)
    try:
        sh = _step_and_compare(model, _loss_step(model, audio), "cfg4 training step B=4 T=2^18", extra=[adjoint])
        assert BACKWARD | {"fir_resample", "skip_gate", "stem_out", "stem_in", "conv_gemm"} <= _kinds(sh)
        assert {"stem_out.loss_sum", "stem_out.dv", "wgrad.dw"} <= set(sh.records)
        assert sh.records["fir_resample._result"].count == 3       # down, up, and the adjoint
    finally:
        _free(model)


def test_text_training_step(adp):
    """Text-conditional README net, batch 2, 2^18 samples, gradients of the input and the embedding."""
    _room(16)
    torch.manual_seed(1234)
    model = adp.DiffusionModel(net_t=adp.UNetV0, **CFG3).to(DEV)
    g = torch.Generator().manual_seed(1)
    x0, sigma = torch.randn(2, 2, T_FULL, generator=g).to(DEV), torch.rand(2, generator=g).to(DEV)
    emb0 = torch.randn(2, 64, 768, generator=g).to(DEV)
    wgt = (torch.randn(2, 2, T_FULL, generator=g) / T_FULL).to(DEV)

    def step():
        model.zero_grad(set_to_none=True)
        x, emb = x0.clone().requires_grad_(), emb0.clone().requires_grad_()
        v = model.net(x, sigma, embedding=emb)
        (v * wgt).sum().backward()
        # the fixed (masked) embedding takes no part at mask probability 0: no gradient
        return None, [x.grad.clone(), emb.grad.clone()] + [torch.zeros_like(p) if p.grad is None else p.grad.clone()
                                                           for p in model.parameters()]
    try:
        sh = _step_and_compare(model, step, "text training step B=2 T=2^18",
                               names=["x", "embedding"] + [n for n, _ in model.named_parameters()], large_tol=1e-2)
        assert (BACKWARD - {"narrow_conv_bwd"}) | {"attention_bwd", "ln_fold_bwd", "attention"} <= _kinds(sh)
        assert {"attention.lse", "attention_bwd.delta", "stem_out_bwd.dxin", "stem_in_bwd.dxin"} <= set(sh.records)
        labels = " ".join(sh.labels)
        for shape in ("Tq=1024 Tk=1024", "Tq=128 Tk=128", "Tq=1024 Tk=64", "Tq=128 Tk=64"):
            assert f"attention_bwd[B=2 H=8 {shape}]" in labels, shape
    finally:
        _free(model)


def _after_update(adp):
    torch.manual_seed(1234)
    model = adp.DiffusionUpsampler(net_t=adp.UNetV0, **UPSAMPLER).to(DEV)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-3, fused=True)
    audio = torch.randn(4, 2, 2 ** 14, generator=torch.Generator().manual_seed(2)).to(DEV)
    model.net.use_cuda_graph = False
    _loss_step(model, audio, seed=3)()
    opt.step()
    return model, audio


def test_step_after_an_optimizer_update(adp):
    """The second step's launches read the forward and dgrad packs refreshed in place by the first:
    every launch against its restatement."""
    model, audio = _after_update(adp)
    try:
        with lc.Shadow() as sh:
            _loss_step(model, audio)()
        print(f"\ncfg4 step after AdamW B=4 T=2^14\n{sh.table()}")
        assert sh.n_checked == sh.n_launch > 0 and BACKWARD <= _kinds(sh)
    finally:
        _free(model)


def test_refreshed_plan_matches_fresh_plan(adp):
    """After a fused AdamW step (which bumps no tensor version counter) the plan refreshed in place
    and plans built afresh from the same weights give the same loss and gradients: the packs of the
    forward and of the data-gradient GEMMs follow the update."""
    model, audio = _after_update(adp)
    try:
        step = _loss_step(model, audio)
        loss_r, refreshed = step()
        model.net._plans.clear()
        model.net.invalidate()                   # fresh forward packs too
        loss_f, fresh = step()
        assert abs(float(loss_r) - float(loss_f)) <= LOSS_REPLAY_TOL * abs(float(loss_f)), (loss_r, loss_f)
        names = [n for n, _ in model.named_parameters()]
        worst = max((rel_l2(g, w), n) for n, g, w in zip(names, refreshed, fresh)
                    if not (n.endswith("resnet.conv1.bias") and "inner" not in n))
        print(f"\nrefreshed plan vs fresh plan after AdamW: worst gradient rel-L2 {worst[0]:.3e} ({worst[1]})")
        assert worst[0] <= GRAD_REPLAY_TOL
    finally:
        _free(model)


def test_accumulators_with_a_non_zero_before(adp):
    """In the training step the arena is zeroed first and every accumulator receives one launch, so
    after - before = after.  Here the accumulators hold values and sit inside a larger arena."""
    from audio_diffusion_pytorch_b200 import ops
    _room(16)
    g = torch.Generator().manual_seed(11)

    def bf(*shape):
        return torch.randn(*shape, generator=g).to(DEV).to(torch.bfloat16)

    def arena(*shape, dtype=torch.float32):
        return (torch.randn(*shape, generator=g) * 50).to(DEV).to(dtype)
    with lc.Shadow() as sh:
        # a deep level's k = 3 conv (M = 512, 1024 x 1024 x 3: one split): odd row pitch -> the scalar
        # read-modify-write path, even pitch -> the paired one
        gd, xd = bf(4, 128, 1024), bf(4, 128, 1024)
        ops.wgrad(gd, xd, arena(3, 1024, 1031)[..., 3:1027], n=1024, k=1024, off=-1, ntaps=3)
        ops.wgrad(gd, xd, arena(3, 1024, 1032)[..., 4:1028], n=1024, k=1024, off=-1, ntaps=3)
        ops.wgrad(gd, xd[..., :1016], arena(1024, 1024)[:, :1015], n=1024, k=1015)      # odd width, one tap
        # level-1 sized channels over 2^20 rows: split-K at the caps, atomics
        gl, xl = bf(4, T_FULL, 32), bf(4, T_FULL, 32)
        ops.wgrad(gl, xl, arena(3, 32, 64)[..., 16:48], n=32, k=32, off=-1, ntaps=3)
        ops.colsum(gl, arena(64)[:32])
        st = lc.stats_of(xl, 8)
        ops.gn_silu_bwd(gl, xl, st, arena(32) / 50, arena(32) / 50, torch.empty_like(xl), arena(96)[32:64],
                        arena(96)[:32], arena(4, 8, 2, dtype=torch.float64), 8)
    print(f"\naccumulators with a non-zero before\n{sh.table()}")
    assert sh.n_checked == sh.n_launch == 6
    assert any("x3" in lab and "M=512" in lab for lab in sh.labels)
