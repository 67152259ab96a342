"""XUNet (a_unet's U-Net builder over XBlock item lists) on the CPU:

  * the parameter tree against the oracle's XUNet built from the same blocks, for item lists in
    other orders than UNetV0's (attention before the ResnetItem, a ModulationItem with no ResnetItem
    before it, a level with no ResnetItem, items_up != items, InjectChannelsItem at one depth) and
    each skip merge (SkipModulate, SkipCat, SkipAdd);
  * a reference-style checkpoint of the oracle loaded with load_reference_state_dict;
  * the refusals, each naming its option;
  * an XUNet built from the XBlocks that UNetV0 builds emits UNetV0's launch programs (inference,
    sampling, conditioning and training), recorded with the launch recorder of
    tests/test_launch_programs_cpu.py."""
import json

import pytest
import torch

import test_launch_programs_cpu as tlp
from audio_diffusion_pytorch_b200 import apex
from audio_diffusion_pytorch_b200 import ClassifierFreeGuidancePlugin, TimeConditioningPlugin, UNetV0, XUNet

# name -> skip merge, plugins from the outside in, blocks as (channels, factor, items, items_up or None,
# context_channels) with items spelled R(esnet) M(odulation) I(nject) A(ttention) C(ross-attention)
CASES = {
    "att_first": ("modulate", ("time",), [(8, 1, "RM", None, None), (32, 4, "ARM", None, None),
                                          (64, 4, "RMA", "RRA", None)]),
    "mod_first": ("modulate", ("time",), [(8, 1, "MR", None, None), (32, 4, "MA", "RM", None),
                                          (64, 4, "RMMA", None, None)]),
    "no_resnet_level": ("modulate", ("time",), [(8, 1, "RM", None, None), (32, 4, "A", "MA", None),
                                                (64, 4, "RA", "", None)]),
    "skipadd": ("add", ("time",), [(8, 1, "RM", None, None), (32, 4, "RMA", "RR", None),
                                   (64, 4, "RMA", None, None)]),
    "skipadd_plain": ("add", (), [(8, 1, "R", None, None), (32, 4, "RA", None, None), (64, 4, "R", "", None)]),
    "skipcat": ("cat", (), [(8, 1, "R", None, None), (32, 4, "RR", "R", None), (64, 4, "AR", None, None)]),
    "inject": ("modulate", ("time",), [(8, 1, "RM", None, None), (32, 4, "RMI", "IRM", 4),
                                       (64, 4, "RM", None, None)]),
    "cross_cfg": ("modulate", ("time", "cfg"), [(8, 1, "RM", None, None), (32, 4, "RMC", None, None),
                                                (64, 4, "CRMA", "RMAC", None)]),
    # the time plugin on nets with no ModulationItem and no SkipModulate: a_unet computes the time
    # features and nothing reads them
    "skipadd_time_only": ("add", ("time",), [(8, 1, "R", None, None), (32, 4, "RA", "R", None),
                                             (64, 4, "R", None, None)]),
    "skipcat_time_only": ("cat", ("time",), [(8, 1, "R", None, None), (32, 4, "R", "AR", None)]),
    # the guidance plugin outside the time plugin registers fixed_embedding first (its forward takes
    # `embedding` as the second positional argument, so the GPU tests call the other order)
    "cfg_outer": ("modulate", ("cfg", "time"), [(8, 1, "RM", None, None), (32, 4, "RC", "CR", None)]),
}
EMBEDDING_MAX_LENGTH = 8


def oracle_modules(oracle_port):
    import a_unet
    from a_unet import apex as oapex
    return a_unet, oapex


def xunet_t(top, ap, case: str):
    """(net_t, kwargs) of a case: top provides the plugins, ap the apex names."""
    skip, plugins, blocks = CASES[case]
    kinds = {"R": ap.ResnetItem, "M": ap.ModulationItem, "I": ap.InjectChannelsItem, "A": ap.AttentionItem,
             "C": ap.CrossAttentionItem}
    xblocks = [ap.XBlock(channels=c, factor=f, items=[kinds[k] for k in items],
                         items_up=None if up is None else [kinds[k] for k in up], context_channels=ctx)
               for c, f, items, up, ctx in blocks]
    net_t = ap.XUNet
    for p in reversed(plugins):
        net_t = (top.TimeConditioningPlugin(net_t) if p == "time"
                 else top.ClassifierFreeGuidancePlugin(net_t, EMBEDDING_MAX_LENGTH))
    kw = dict(in_channels=2, blocks=xblocks, resnet_groups=8, attention_features=64, attention_heads=2,
              skip_t={"modulate": ap.SkipModulate, "cat": ap.SkipCat, "add": ap.SkipAdd}[skip])
    if skip == "modulate" or "time" in plugins or any("M" in b[2] + (b[3] or "") for b in blocks):
        kw["modulation_features"] = 1024
    if "cfg" in plugins or any("C" in b[2] + (b[3] or "") for b in blocks):
        kw["embedding_features"] = 32
    return net_t, kw


def ours(case: str):
    import audio_diffusion_pytorch_b200 as adp
    net_t, kw = xunet_t(adp, apex, case)
    return net_t(dim=1, **kw)


def theirs(oracle_port, case: str):
    top, oapex = oracle_modules(oracle_port)
    net_t, kw = xunet_t(top, oapex, case)
    return net_t(dim=1, **kw)


def shapes(m):
    return [tuple(p.shape) for p in m.parameters()]


@pytest.mark.parametrize("case", sorted(CASES))
def test_parameter_tree_matches_oracle(oracle_port, case):
    torch.manual_seed(0)
    net, ref = ours(case), theirs(oracle_port, case)
    assert isinstance(net, XUNet)
    assert shapes(net) == shapes(ref)


@pytest.mark.parametrize("case", sorted(CASES))
def test_reference_state_dict(oracle_port, case):
    torch.manual_seed(0)
    ref = theirs(oracle_port, case)
    net = ours(case)
    net.load_reference_state_dict(ref.state_dict())
    for a, b in zip(net.parameters(), ref.parameters()):
        assert torch.equal(a, b)
    net2 = ours(case)
    net2.load_reference_parameters(ref)
    for a, b in zip(net2.parameters(), ref.parameters()):
        assert torch.equal(a, b)


def blocks(items=(apex.ResnetItem,), **kw):
    return [apex.XBlock(channels=8, factor=1, items=list(items), **kw),
            apex.XBlock(channels=32, factor=4, items=list(items))]


BASE = dict(dim=1, in_channels=2, resnet_groups=8)


@pytest.mark.parametrize("kw, match", [
    (dict(dim=2), "dim=2"),
    (dict(downsample_t=apex.ResnetItem), "downsample_t"),
    (dict(upsample_t=apex.ResnetItem), "upsample_t"),
    (dict(skip_adapter_t=apex.ResnetItem), "skip_adapter_t"),
    (dict(resnet_kernel_size=5), "resnet_kernel_size"),
    (dict(skip_t=apex.ResnetItem), "skip_t"),
])
def test_refusals_name_the_option(kw, match):
    with pytest.raises((NotImplementedError, TypeError), match=match):
        XUNet(blocks=blocks(), **{**BASE, **kw})


def test_block_refusals_name_the_option():
    with pytest.raises(NotImplementedError, match="resnet_kernel_size"):
        apex.XBlock(channels=8, factor=1, items=[apex.ResnetItem], resnet_kernel_size=5)
    with pytest.raises(NotImplementedError, match="downsample_t"):
        apex.XBlock(channels=8, factor=1, items=[apex.ResnetItem], downsample_t=apex.ResnetItem)
    with pytest.raises(NotImplementedError, match=r"blocks\[1\]\.items: str is not an item type"):
        XUNet(blocks=[apex.XBlock(channels=8, factor=1), apex.XBlock(channels=32, factor=4, items=[str])], **BASE)
    with pytest.raises(NotImplementedError, match=r"blocks\[0\]\.items_up: SkipAdd"):
        XUNet(blocks=blocks(items_up=[apex.SkipAdd]), **BASE)
    with pytest.raises(NotImplementedError, match="num_layers=3"):
        TimeConditioningPlugin(XUNet, num_layers=3)
    with pytest.raises(NotImplementedError, match="wraps XUNet"):
        ClassifierFreeGuidancePlugin(UNetV0, 8)


@pytest.mark.parametrize("kw", [
    dict(resnet_groups=16),
    dict(attention_features=48, attention_heads=2),
    dict(in_channels=65),
])
def test_envelope_messages_match_unet_v0(kw):
    """The same limits as UNetV0, checked by the same code with the same messages."""
    items = [apex.ResnetItem, apex.AttentionItem] if "attention_features" in kw else [apex.ResnetItem]
    with pytest.raises(AssertionError) as got:
        XUNet(blocks=[apex.XBlock(channels=16, factor=1, items=items),
                      apex.XBlock(channels=32, factor=4, items=items)], **{**BASE, **kw})
    v0 = dict(dim=1, in_channels=2, channels=[16, 32], factors=[1, 4], items=[1, 1], use_modulation=False,
              use_time_conditioning=False, resnet_groups=8)
    if "attention_features" in kw:
        v0["attentions"] = [1, 1]
    with pytest.raises(AssertionError) as want:
        UNetV0(**{**v0, **kw})
    assert str(got.value) == str(want.value)


# ------------------------------------------------------------------ UNetV0's blocks, UNetV0's program
def unet_v0_as_xunet(kw):
    """XUNet + plugins built from the XBlocks UNetV0 builds (reference components.py:55-105)."""
    n = len(kw["channels"])
    att, cross = kw.get("attentions", [0] * n), kw.get("cross_attentions", [0] * n)
    ctx = kw.get("context_channels", [0] * n)
    mod = kw.get("use_modulation", True)
    xblocks = [apex.XBlock(channels=c, factor=f, context_channels=cc,
                           items=([apex.ResnetItem] + [apex.ModulationItem] * mod +
                                  [apex.InjectChannelsItem] * (cc > 0) + [apex.AttentionItem] * a +
                                  [apex.CrossAttentionItem] * x) * it)
               for c, f, it, a, x, cc in zip(kw["channels"], kw["factors"], kw["items"], att, cross, ctx)]
    net_t = XUNet
    if kw.get("use_embedding_cfg", False):
        net_t = ClassifierFreeGuidancePlugin(net_t, kw["embedding_max_length"])
    if kw.get("use_time_conditioning", True):
        net_t = TimeConditioningPlugin(net_t)
    extra = {k: kw[k] for k in ("attention_features", "attention_heads", "embedding_features", "resnet_groups",
                                "modulation_features") if k in kw}
    return net_t(dim=1, in_channels=kw["in_channels"], out_channels=kw.get("out_channels"), blocks=xblocks,
                 skip_t=apex.SkipModulate if mod else apex.SkipCat, modulation_features=1024,
                 **{**{"resnet_groups": 8}, **extra})


SAME_PROGRAM = ("tiny", "tiny_fp32", "text_cfg", "skipcat_adapter", "inject", "att_narrow", "head32_g4",
                "factor1_c128")


@pytest.mark.parametrize("name", SAME_PROGRAM)
def test_unet_v0_blocks_emit_unet_v0_program(name, monkeypatch):
    rec = tlp.install(monkeypatch)
    want = json.loads(json.dumps(tlp.record_case(name, rec)))
    v0_names = [n for n, _ in tlp.build_net(*tlp.NETS[name][:2]).named_parameters()]

    def build_xunet(kw, attrs):
        torch.manual_seed(0)
        net = unet_v0_as_xunet(kw)
        for k, v in attrs.items():
            setattr(net, k, v)
        return net
    monkeypatch.setattr(tlp, "build_net", build_xunet)
    got = json.loads(json.dumps(tlp.record_case(name, rec)))
    # the gradient specs are keyed by parameter name: XUNet's names, mapped to UNetV0's by position
    x_names = [n for n, _ in build_xunet(*tlp.NETS[name][:2]).named_parameters()]
    rename = dict(zip(x_names, v0_names))
    assert len(x_names) == len(v0_names)
    for prog in got.values():
        for key in ("specs", "grads"):
            if key in prog:
                prog[key] = {rename[k]: v for k, v in prog[key].items()}
    d = tlp.first_difference(got, want, name)
    assert d is None, "XUNet's launch program differs from UNetV0's at " + d


@pytest.mark.parametrize("case", sorted(CASES))
def test_programs_build_for_every_case(case, monkeypatch):
    """Every case's inference, sampling and training programs build and run on the recorder."""
    rec = tlp.install(monkeypatch)
    torch.manual_seed(0)
    net = ours(case)
    cfg = net.use_embedding_cfg
    M = 8 if any(net.cross_attentions) else 0
    for mode, Bh in (("v", 2), ("sample", 2)) + ((("v", 4),) if cfg else ()):
        plan = net._plan(2, 4096, Bh, M, mode, (5.0 if Bh == 4 else None, False))
        for fn in plan.pre:
            fn()
        plan.run_eager()
        assert rec.take()
    from audio_diffusion_pytorch_b200 import training
    for mode in ("loss", "v"):
        plan = training.build_train_plan(net, 2, 4096, M, mode, True)
        for fn in plan.fwd:
            fn()
        marks = []
        plan.on_mark = marks.append
        plan.backward_program()
        assert rec.take() and marks
        for fin in plan.finals:
            fin()
        routed = set(plan.specs) | set(plan.grads)
        missing = [n for n, p in net.named_parameters() if id(p) not in routed
                   and any(p is q for q in training._net_params(net))]
        assert not missing, f"parameters without a gradient: {missing}"


@pytest.mark.parametrize("items", [
    ("R", "A", "A"),                      # attention levels with no ResnetItem
    ("R", "CAC", "AAR"),                  # attention items ahead of a level's ResnetItem
])
def test_gradient_arena_with_wide_attention_before_any_resnet(items, monkeypatch):
    """Every attention item ahead of a chain's first ResnetItem reserves its projection-gradient
    scratch: narrow levels under wide attention (8 heads x 64) build their training plans."""
    from audio_diffusion_pytorch_b200 import training
    tlp.install(monkeypatch)
    kinds = {"R": apex.ResnetItem, "A": apex.AttentionItem, "C": apex.CrossAttentionItem}
    torch.manual_seed(0)
    net = XUNet(dim=1, in_channels=2, resnet_groups=8, attention_features=64, attention_heads=8,
                embedding_features=32,
                blocks=[apex.XBlock(channels=c, factor=f, items=[kinds[k] for k in it])
                        for c, f, it in zip((16, 128, 256), (1, 4, 4), items)])
    M = 8 if any(net.cross_attentions) else 0
    for mode in ("loss", "v"):
        plan = training.build_train_plan(net, 2, 4096, M, mode, True)
        for fn in plan.fwd:
            fn()
        plan.backward_program()
