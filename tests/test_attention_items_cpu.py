"""Repeated attention items on the CPU: UNetV0(attentions=[..., n], cross_attentions=[..., m]) builds
each repetition of a level as a_unet does, [ResnetItem, ModulationItem?, InjectChannelsItem?] +
[AttentionItem] * n + [CrossAttentionItem] * m.

  * the parameter tree equals the oracle's (count and shapes in order) for every config of the table
    below, reference weights load by position and reference checkpoints by `load_reference_state_dict`;
    a count of True is one item, and 0, False or a negative count none;
  * a net with counts <= 1 keeps the state_dict key names it had before counts above 1 were supported;
  * the inference, 3-step sampling and guidance-5 programs of each config run with fake kernels that
    write the launch checker's fp64 restatements (tests/launch_check.py), against the CPU oracle;
  * the training programs of each config build and run under the same checker, with the gradient
    arena laid out in forward build order.
"""
import pytest
import torch

import launch_check as lc
from audio_diffusion_pytorch_b200 import _lib, ops, training
from audio_diffusion_pytorch_b200.diffusion import VSampler
from audio_diffusion_pytorch_b200.models import DiffusionModel
from audio_diffusion_pytorch_b200.unet import UNetV0
from test_launch_check_cpu import rel_l2

V_TOL, BRANCH_TOL = 1e-4, 1.2e-2
CFG_V_TOL, CFG_BRANCH_TOL = 3e-4, 2.5 * BRANCH_TOL
SAMPLE_TOL = 5e-3
SKIPCAT_V_TOL = 5e-3

BASE = dict(in_channels=2, channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 2, 2], attention_heads=2,
            attention_features=32)
TEXT = dict(use_embedding_cfg=True, embedding_max_length=8, embedding_features=32)
# also run on the GPU (tests/test_attention_items_gpu.py)
CONFIGS = {
    "self_2": dict(BASE, attentions=[0, 0, 2]),
    "cross_2_cfg": dict(BASE, cross_attentions=[0, 0, 2], **TEXT),
    "mixed": dict(BASE, attentions=[0, 1, 3], cross_attentions=[0, 2, 1], **TEXT),
    # DiffusionAE's net: an InjectChannelsItem before the two attentions of the same level
    "inject_2": dict(BASE, attentions=[0, 0, 2], context_channels=[0, 0, 4]),
    # DiffusionAR's net: no ModulationItem, so the first attention runs its own LayerNorm too
    "skipcat_2": dict(BASE, attentions=[0, 0, 2], use_modulation=False, use_time_conditioning=False),
}

# state_dict() keys of a net with counts of 1, recorded before counts above 1 were supported
KEYS_CFG = dict(in_channels=2, channels=[8, 32], factors=[1, 2], items=[1, 1], attentions=[0, 1],
                cross_attentions=[0, True], context_channels=[0, 4], attention_heads=1, attention_features=32,
                embedding_features=32, use_embedding_cfg=True, embedding_max_length=4)
_RESNET = ["resnet.gn1.weight", "resnet.gn1.bias", "resnet.conv1.weight", "resnet.conv1.bias", "resnet.gn2.weight",
           "resnet.gn2.bias", "resnet.conv2.weight", "resnet.conv2.bias", "modulation.proj.weight",
           "modulation.proj.bias"]
_ATTN = ["norm.weight", "norm.bias", "norm_context.weight", "norm_context.bias", "to_q.weight", "to_kv.weight",
         "to_out.weight"]
KEYS_AT_COUNT_1 = [
    'time.weights', 'time.to_out.weight', 'time.to_out.bias', 'time.mlp.weight', 'time.mlp.bias',
    'fixed_embedding.weight', 'net.down.weight', 'net.down.bias',
    'net.items_down.0.resnet.gn1.weight', 'net.items_down.0.resnet.gn1.bias', 'net.items_down.0.resnet.conv1.weight',
    'net.items_down.0.resnet.conv1.bias', 'net.items_down.0.resnet.gn2.weight', 'net.items_down.0.resnet.gn2.bias',
    'net.items_down.0.resnet.conv2.weight', 'net.items_down.0.resnet.conv2.bias',
    'net.items_down.0.modulation.proj.weight', 'net.items_down.0.modulation.proj.bias',
    'net.inner.down.weight', 'net.inner.down.bias',
    'net.inner.items_down.0.resnet.gn1.weight', 'net.inner.items_down.0.resnet.gn1.bias',
    'net.inner.items_down.0.resnet.conv1.weight', 'net.inner.items_down.0.resnet.conv1.bias',
    'net.inner.items_down.0.resnet.gn2.weight', 'net.inner.items_down.0.resnet.gn2.bias',
    'net.inner.items_down.0.resnet.conv2.weight', 'net.inner.items_down.0.resnet.conv2.bias',
    'net.inner.items_down.0.modulation.proj.weight', 'net.inner.items_down.0.modulation.proj.bias',
    'net.inner.items_down.0.inject.weight', 'net.inner.items_down.0.inject.bias',
    'net.inner.items_down.0.attention.norm.weight', 'net.inner.items_down.0.attention.norm.bias',
    'net.inner.items_down.0.attention.norm_context.weight', 'net.inner.items_down.0.attention.norm_context.bias',
    'net.inner.items_down.0.attention.to_q.weight', 'net.inner.items_down.0.attention.to_kv.weight',
    'net.inner.items_down.0.attention.to_out.weight',
    'net.inner.items_down.0.cross.norm.weight', 'net.inner.items_down.0.cross.norm.bias',
    'net.inner.items_down.0.cross.norm_context.weight', 'net.inner.items_down.0.cross.norm_context.bias',
    'net.inner.items_down.0.cross.to_q.weight', 'net.inner.items_down.0.cross.to_kv.weight',
    'net.inner.items_down.0.cross.to_out.weight',
    'net.inner.items_up.0.resnet.gn1.weight', 'net.inner.items_up.0.resnet.gn1.bias',
    'net.inner.items_up.0.resnet.conv1.weight', 'net.inner.items_up.0.resnet.conv1.bias',
    'net.inner.items_up.0.resnet.gn2.weight', 'net.inner.items_up.0.resnet.gn2.bias',
    'net.inner.items_up.0.resnet.conv2.weight', 'net.inner.items_up.0.resnet.conv2.bias',
    'net.inner.items_up.0.modulation.proj.weight', 'net.inner.items_up.0.modulation.proj.bias',
    'net.inner.items_up.0.inject.weight', 'net.inner.items_up.0.inject.bias',
    'net.inner.items_up.0.attention.norm.weight', 'net.inner.items_up.0.attention.norm.bias',
    'net.inner.items_up.0.attention.norm_context.weight', 'net.inner.items_up.0.attention.norm_context.bias',
    'net.inner.items_up.0.attention.to_q.weight', 'net.inner.items_up.0.attention.to_kv.weight',
    'net.inner.items_up.0.attention.to_out.weight',
    'net.inner.items_up.0.cross.norm.weight', 'net.inner.items_up.0.cross.norm.bias',
    'net.inner.items_up.0.cross.norm_context.weight', 'net.inner.items_up.0.cross.norm_context.bias',
    'net.inner.items_up.0.cross.to_q.weight', 'net.inner.items_up.0.cross.to_kv.weight',
    'net.inner.items_up.0.cross.to_out.weight',
    'net.inner.up.weight', 'net.inner.up.bias', 'net.inner.merge.weight', 'net.inner.merge.bias',
    'net.items_up.0.resnet.gn1.weight', 'net.items_up.0.resnet.gn1.bias', 'net.items_up.0.resnet.conv1.weight',
    'net.items_up.0.resnet.conv1.bias', 'net.items_up.0.resnet.gn2.weight', 'net.items_up.0.resnet.gn2.bias',
    'net.items_up.0.resnet.conv2.weight', 'net.items_up.0.resnet.conv2.bias',
    'net.items_up.0.modulation.proj.weight', 'net.items_up.0.modulation.proj.bias',
    'net.up.weight', 'net.up.bias', 'net.merge.weight', 'net.merge.bias',
]


def n_items(cfg, key):
    return sum(max(0, int(a)) * 2 * n for a, n in zip(cfg.get(key, [0] * 3), cfg["items"]))


def inputs(cfg, B=2, T=1024, seed=3):
    """(x, sigma or None, embedding or None, context channels or None) for a config."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, cfg["in_channels"], T, generator=g)
    sigma = torch.rand(B, generator=g) if cfg.get("use_time_conditioning", True) else None
    emb = (torch.randn(B, 8, cfg["embedding_features"], generator=g)
           if any(cfg.get("cross_attentions", [])) else None)
    channels = None
    if "context_channels" in cfg:
        channels, t = [], T
        for c, f in zip(cfg["context_channels"], cfg["factors"]):
            t //= f
            channels.append(torch.randn(B, c, t, generator=g) if c else None)
    return x, sigma, emb, channels


def oracle_kw(emb, channels, scale=1.0):
    kw = {}
    if emb is not None:
        kw.update(embedding=emb, embedding_scale=scale)
    if channels is not None:
        kw["channels"] = channels
    return kw


@pytest.fixture
def cpu_launches(monkeypatch):
    monkeypatch.setattr(ops, "device_check", lambda: None)
    monkeypatch.setattr(ops, "require_cuda", lambda x: None)

    def no_library():
        raise AssertionError("a launch reached the CUDA library")
    monkeypatch.setattr(_lib, "lib", no_library)


def pair(oracle_port, cfg):
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**cfg)
    model = DiffusionModel(net_t=UNetV0, **cfg)
    model.net.load_reference_parameters(ref.net)
    model.net.use_cuda_graph = False           # every call runs the plan's launches eagerly
    return ref, model.net


# ------------------------------------------------------------------------------ parameter tree
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_parameter_tree_matches_oracle(oracle_port, name):
    cfg = CONFIGS[name]
    torch.manual_seed(0)
    ref = oracle_port.build_unet_v0(dim=1, **cfg)
    net = UNetV0(dim=1, **cfg)
    assert [tuple(p.shape) for p in net.parameters()] == [tuple(p.shape) for p in ref.parameters()]
    net.load_reference_parameters(ref)
    for a, b in zip(net.parameters(), ref.parameters()):
        assert torch.equal(a, b)
    items = [it for lv in net.levels() for it in (*lv.items_down, *lv.items_up)]
    assert sum(len(it.attentions()) for it in items) == n_items(cfg, "attentions")
    assert sum(len(it.crosses()) for it in items) == n_items(cfg, "cross_attentions")


@pytest.mark.parametrize("count,same_as", [(True, 1), (False, 0), (-1, 0), (-3, 0), (2, 2)])
def test_counts_are_a_unet_item_counts(oracle_port, count, same_as):
    """`[Item] * count`: True is one item, False and negative counts none."""
    def shapes(net):
        return [tuple(p.shape) for p in net.parameters()]
    for key in ("attentions", "cross_attentions"):
        cfg = dict(BASE, **TEXT, **{key: [0, 0, count]})
        ours = UNetV0(dim=1, **cfg)
        assert shapes(ours) == shapes(oracle_port.build_unet_v0(dim=1, **cfg))
        assert shapes(ours) == shapes(UNetV0(dim=1, **dict(cfg, **{key: [0, 0, same_as]})))


def test_counts_of_one_keep_their_state_dict_keys():
    assert list(UNetV0(dim=1, **KEYS_CFG).state_dict().keys()) == KEYS_AT_COUNT_1


def test_repeated_items_register_after_the_first():
    net = UNetV0(dim=1, **CONFIGS["mixed"])
    keys = [k[len("net.inner.inner.items_down.0."):] for k in net.state_dict()
            if k.startswith("net.inner.inner.items_down.0.")]
    want = (_RESNET + [f"attention.{k}" for k in _ATTN] + [f"extra_attention.{i}.{k}" for i in (0, 1) for k in _ATTN]
            + [f"cross.{k}" for k in _ATTN])
    assert keys == want
    keys = [k[len("net.inner.items_up.1."):] for k in net.state_dict() if k.startswith("net.inner.items_up.1.")]
    assert keys == (_RESNET + [f"attention.{k}" for k in _ATTN] + [f"cross.{k}" for k in _ATTN]
                    + [f"extra_cross.0.{k}" for k in _ATTN])


@pytest.mark.parametrize("name", ["mixed", "inject_2"])
def test_reference_checkpoint_loads(oracle_port, tmp_path, name):
    cfg = CONFIGS[name]
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**cfg)
    model = DiffusionModel(net_t=UNetV0, **cfg)
    torch.save(ref.state_dict(), tmp_path / "ref.pt")
    model.load_reference_state_dict(torch.load(tmp_path / "ref.pt"))
    for a, b in zip(model.net.parameters(), ref.net.parameters()):
        assert torch.equal(a, b)
    # a checkpoint of the same net with one attention per item has fewer tensors: refused
    fewer = oracle_port.DiffusionModelPort(**dict(cfg, attentions=[min(1, a) for a in cfg["attentions"]]))
    with pytest.raises(AssertionError, match="tensors"):
        model.load_reference_state_dict(fewer.state_dict())


# ------------------------------------------------------------------------------ programs
def _oracle_v(ref, x, sigma, kw):
    return ref.net(x, sigma, **kw) if sigma is not None else ref.net(x, **kw)


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_program_vs_oracle(cpu_launches, oracle_port, name):
    cfg = CONFIGS[name]
    ref, net = pair(oracle_port, cfg)
    x, sigma, emb, channels = inputs(cfg)
    cases = [(1.0, V_TOL, BRANCH_TOL)] + ([(5.0, CFG_V_TOL, CFG_BRANCH_TOL)] if emb is not None else [])
    if not cfg.get("use_modulation", True):
        # SkipCat merges x through a 1x1 conv: v has no identity part, and is held to DiffusionAR's v
        # bound of test_net_gpu.py (its bf16 error, ~2e-3, is the same at attention counts 0, 1 and 2)
        cases = [(1.0, SKIPCAT_V_TOL, BRANCH_TOL)]
    with torch.no_grad():
        for scale, v_tol, b_tol in cases:
            want = _oracle_v(ref, x, sigma, oracle_kw(emb, channels, scale))
            with lc.Shadow(fake=True) as sh:
                v = net(x, sigma, **oracle_kw(emb, channels, scale))
            assert sh.n_checked == sh.n_launch > 0
            assert sh.records["attention.o"].count == n_items(cfg, "attentions") + n_items(cfg, "cross_attentions")
            e_v, e_b = rel_l2(v, want), rel_l2(v - x[:, :v.shape[1]], want - x[:, :v.shape[1]])
            print(f"{name} scale {scale}: rel-L2(v) {e_v:.3e} rel-L2(branch) {e_b:.3e}")
            assert e_v <= v_tol and e_b <= b_tol


@pytest.mark.parametrize("name", sorted(n for n in CONFIGS if CONFIGS[n].get("use_time_conditioning", True)))
def test_sampling_program_vs_oracle(cpu_launches, oracle_port, name):
    cfg = CONFIGS[name]
    ref, net = pair(oracle_port, cfg)
    noise, _, emb, channels = inputs(cfg, seed=4)
    with torch.no_grad():
        want = ref.sample(noise, num_steps=3, **oracle_kw(emb, channels))
        with lc.Shadow(fake=True) as sh:
            s = VSampler(net=net)(noise, num_steps=3, **oracle_kw(emb, channels))
    assert sh.n_checked == sh.n_launch > 0
    e = rel_l2(s, want)
    print(f"{name} 3-step sample: rel-L2 {e:.3e}")
    assert e <= SAMPLE_TOL


@pytest.mark.parametrize("name", ["cross_2_cfg", "mixed"])
def test_each_cross_item_projects_the_context_once_per_sample(cpu_launches, name):
    """The sampling plan's step-invariant part: one LayerNorm of the embedding, shared, and one
    K|V projection per cross-attention item; the step program itself projects no context."""
    from test_launch_programs_cpu import install
    mp = pytest.MonkeyPatch()
    try:
        rec = install(mp)
        torch.manual_seed(0)
        net = UNetV0(dim=1, **CONFIGS[name])
        plan = net._plan(2, 1024, 2, 8, "sample", (None, False))
        for fn in plan.pre:
            fn()
        pre = [k[0] for k in rec.take()]
        plan.run_eager()
        prog = rec.take()
    finally:
        mp.undo()
    assert pre == ["ln_film"] + ["conv_gemm"] * n_items(CONFIGS[name], "cross_attentions")
    assert sum(1 for k in prog if k[0] == "attention") == (n_items(CONFIGS[name], "attentions")
                                                          + n_items(CONFIGS[name], "cross_attentions"))


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_training_program_runs_under_the_checker(cpu_launches, name):
    """Forward and backward of the training plan with fake kernels, every launch checked; one
    attention_bwd per attention item, and every attention parameter's gradient in the arena in
    forward build order."""
    cfg = CONFIGS[name]
    torch.manual_seed(0)
    net = UNetV0(dim=1, **cfg)
    x, _, emb, channels = inputs(cfg, B=2, T=1024, seed=5)
    M = 8 if emb is not None else 0
    plan = training.build_train_plan(net, 2, 1024, M, "loss", True)
    plan.x.copy_(x[:, :net.x_channels])
    plan.noise.normal_()
    plan.alpha.fill_(0.8)
    plan.beta.fill_(0.6)
    plan.cond.normal_()
    if M:
        plan.embedding.copy_(emb)
    for d, c in plan.ctx.items():
        c[:, :, :channels[d].shape[1]].copy_(channels[d].transpose(1, 2))
    with lc.Shadow(fake=True) as sh:
        for fn in plan.fwd:
            fn()
        plan.backward_program()
    assert sh.n_checked == sh.n_launch > 0
    n_att = n_items(cfg, "attentions") + n_items(cfg, "cross_attentions")
    assert sh.records["attention_bwd.dq"].count == n_att
    starts = [plan.specs[id(p)][0] for lv in net.levels() for it in (*lv.items_down, *lv.items_up)
              for am in it.attentions() + it.crosses() for p in am.parameters()]
    assert len(starts) == 7 * n_att
    # forward build order is the recursive level order, not the flat one: compare per item chain, one
    # entry per attention item (its own accumulators follow the backward's order)
    for lv in net.levels():
        for items in (lv.items_down, lv.items_up):
            s = [min(plan.specs[id(p)][0] for p in am.parameters()) for it in items
                 for am in it.attentions() + it.crosses()]
            assert s == sorted(s)
    if M:
        assert plan.demb.float().abs().sum() > 0
