"""a_unet's general U-Net builder on the CUDA path: `XUNet` over `XBlock` item lists, the item and
skip-merge types it takes, and the time-conditioning and classifier-free-guidance plugins.

    net = XUNet(dim=1, in_channels=2, skip_t=SkipCat, resnet_groups=8, attention_features=64,
                attention_heads=8, modulation_features=1024,
                blocks=[XBlock(channels=32, factor=4, items=[ResnetItem, ModulationItem],
                               items_up=[ResnetItem, ResnetItem]), ...])
    v = net(x, features=f)                                   # a_unet XUNet.forward

Each block's `items` and `items_up` (default: `items`) may hold the five item types below in any
order and number, zero included.  The net runs the same sm_90a kernels as UNetV0 (`B200UNet`),
whose program builder takes each chain as a list of items; UNetV0 is one such list per level.
Parameters are registered in a_unet's module order, so `load_reference_parameters` and
`load_reference_state_dict` copy a net that a_unet built from the same blocks.

Under TimeConditioningPlugin, a net with no ModulationItem and no SkipModulate runs as a_unet runs it:
nothing reads the time features, so the time MLP is not evaluated and gets no gradient.

Outside the kernels' envelope (the limits of UNetV0: level widths, boundary, resnet_groups <= 8,
head dims 32 / 64 / 128) and outside a_unet's 1-D U-Net with its default down / upsampling, skip
adapter and kernel size 3, the constructor raises and names the option."""
from typing import Callable, Optional, Sequence

from torch import nn

from .unet import AttentionParams, B200UNet, LevelParams, ModulationParams, ResnetParams, TimeParams, exists


# ------------------------------------------------------------------------------ item and merge types
class ResnetItem:
    """(GroupNorm, SiLU, Conv1d k3) x 2 + x."""


class ModulationItem:
    """LayerNorm(x) (1 + scale) + shift, (scale, shift) = Linear(SiLU(features))."""


class InjectChannelsItem:
    """Conv1d k1 over cat([x, channels[depth]]) + x; the block gives `context_channels`."""


class AttentionItem:
    """x + self-attention over LayerNorm(x)."""


class CrossAttentionItem:
    """x + attention from LayerNorm(x) to LayerNorm(embedding)."""


class SkipModulate:
    """skip + Linear(SiLU(features)) * y."""


class SkipCat:
    """Conv1d k1 over cat([skip * 2^-0.5, y])."""


class SkipAdd:
    """skip + y (a_unet's default merge)."""


_KINDS = {ResnetItem: "resnet", ModulationItem: "mod", InjectChannelsItem: "inj", AttentionItem: "att",
          CrossAttentionItem: "cross"}
_MERGES = {SkipModulate: "modulate", SkipCat: "cat", SkipAdd: "add"}

# a_unet options whose other values the kernels do not implement: accepted at their default only
_FIXED = {"downsample_t": None, "upsample_t": None, "skip_adapter_t": None, "resnet_kernel_size": 3}


def _check_fixed(kwargs, where: str) -> None:
    for k, v in kwargs.items():
        if k not in _FIXED:
            raise TypeError(f"{where}: unexpected option {k}")
        if v != _FIXED[k]:
            raise NotImplementedError(
                f"{where}: {k}={getattr(v, '__name__', v)} is not supported (XUNet runs a_unet's strided-conv "
                f"downsample, nearest + conv3 upsample, conv1x1 skip adapter and kernel size 3)")


class XBlock:
    """One U-Net level: `channels` wide, downsampled by `factor`, with the item chains `items` (down)
    and `items_up` (default: `items`).  `context_channels`: channels of `channels[depth]` read by
    the block's InjectChannelsItems."""

    def __init__(self, channels: int, factor: int, items: Sequence = (), items_up: Optional[Sequence] = None,
                 context_channels: Optional[int] = None, **kwargs):
        _check_fixed(kwargs, "XBlock")
        self.channels, self.factor, self.context_channels = channels, factor, context_channels
        self.items = list(items)
        self.items_up = list(items) if items_up is None else list(items_up)


class XLevelParams(LevelParams):
    """a_unet Block of an XUNet: registration order skip_adapter, (down, items, inner, items_up,
    up), merge, with one module per item of each chain."""

    def __init__(self, in_ch: int, out_ch: int, ch: int, factor: int, kinds_down: Sequence[str],
                 kinds_up: Sequence[str], inner, merge: str, groups: int, features: int,
                 head_features: Optional[int], heads: Optional[int], embedding_features: Optional[int],
                 context: int):
        nn.Module.__init__(self)

        def item(kind: str) -> nn.Module:
            if kind == "resnet":
                return ResnetParams(ch, groups)
            if kind == "mod":
                return ModulationParams(ch, features)
            if kind == "inj":
                return nn.Conv1d(ch + context, ch, 1)
            return AttentionParams(ch, head_features, heads, embedding_features if kind == "cross" else None)
        self.adapter = nn.Conv1d(in_ch, out_ch, 1) if in_ch != out_ch else None
        self.down = nn.Conv1d(in_ch, ch, factor, stride=factor)
        self.items_down = nn.ModuleList([item(k) for k in kinds_down])
        self.inner = inner
        self.items_up = nn.ModuleList([item(k) for k in kinds_up])
        self.up = nn.Conv1d(ch, out_ch, 3, padding=1)
        if merge == "modulate":
            self.merge = nn.Linear(features, out_ch)
        elif merge == "cat":
            self.merge = nn.Conv1d(2 * out_ch, out_ch, 1)
        else:
            self.merge = None
        self.kinds_down, self.kinds_up = list(kinds_down), list(kinds_up)
        self.in_ch, self.out_ch, self.ch, self.factor = in_ch, out_ch, ch, factor

    def chain(self, up: bool):
        return list(zip(self.kinds_up, self.items_up) if up else zip(self.kinds_down, self.items_down))


class XUNet(B200UNet):
    """a_unet XUNet(in_channels, blocks, out_channels=None, **kwargs) on the CUDA path; see the
    module docstring.  `forward(x, *, features=None, embedding=None, channels=None)`, plus `time`
    under TimeConditioningPlugin and `embedding_scale` / `embedding_mask_proba` under
    ClassifierFreeGuidancePlugin."""

    def __init__(self, in_channels: int, blocks: Sequence[XBlock], out_channels: Optional[int] = None, *,
                 dim: Optional[int] = None, skip_t: Callable = SkipAdd,
                 attention_features: Optional[int] = None, attention_heads: Optional[int] = None,
                 embedding_features: Optional[int] = None, modulation_features: Optional[int] = None,
                 resnet_groups: Optional[int] = None, _plugins: Sequence[tuple] = (), **kwargs):
        nn.Module.__init__(self)
        _check_fixed(kwargs, "XUNet")
        if dim != 1:
            raise NotImplementedError(f"dim={dim}: XUNet runs the 1-D (waveform) U-Net")
        if skip_t not in _MERGES:
            raise NotImplementedError(f"skip_t={getattr(skip_t, '__name__', skip_t)}: XUNet merges with "
                                      f"SkipModulate, SkipCat or SkipAdd")
        merge = _MERGES[skip_t]
        chains = []
        for i, b in enumerate(blocks):
            if not isinstance(b, XBlock):
                raise TypeError(f"blocks[{i}]: an XBlock is expected")
            kinds = []
            for name in ("items", "items_up"):
                for it in getattr(b, name):
                    if it not in _KINDS:
                        raise NotImplementedError(
                            f"blocks[{i}].{name}: {getattr(it, '__name__', it)} is not an item type of XUNet "
                            f"({', '.join(t.__name__ for t in _KINDS)})")
                kinds.append([_KINDS[it] for it in getattr(b, name)])
            chains.append(kinds)
        every = [k for down, up in chains for k in down + up]
        if "resnet" in every:
            assert exists(resnet_groups), "ResnetItem requires dim, channels, and resnet_groups"
        uses_features = "mod" in every or merge == "modulate" or any(p[0] == "time" for p in _plugins)
        if uses_features:
            assert exists(modulation_features), "ModulationItem requires channels, modulation_features"
        context = []
        for i, ((down, up), b) in enumerate(zip(chains, blocks)):
            if "inj" in down + up:
                assert exists(b.context_channels), "InjectChannelsItem requires dim, depth, channels, context_channels"
            context.append(b.context_channels if "inj" in down + up else 0)
        channels = [b.channels for b in blocks]
        self._setup(in_channels, out_channels, 0, channels, [b.factor for b in blocks],
                    [len(down) for down, _ in chains],
                    [(down + up).count("att") for down, up in chains],
                    [(down + up).count("cross") for down, up in chains], context,
                    attention_features, attention_heads, embedding_features,
                    resnet_groups if exists(resnet_groups) else 8, "mod" in every or merge == "modulate", merge,
                    modulation_features if exists(modulation_features) else 1024,
                    any(p[0] == "time" for p in _plugins), any(p[0] == "cfg" for p in _plugins))

        # registration order mirrors a_unet: the plugins from the outside in, then the blocks
        self.time = self.fixed_embedding = None
        for p in _plugins:
            if p[0] == "time":
                self.time = TimeParams(self.features)
            else:
                assert exists(embedding_features), "ClassifierFreeGuidancePlugin requires embedding_features"
                self.fixed_embedding = nn.Embedding(p[1], embedding_features)

        def build(i: int):
            if i == len(blocks):
                return None
            in_ch = in_channels if i == 0 else channels[i - 1]
            out_ch = self.out_channels if i == 0 else in_ch
            return XLevelParams(in_ch, out_ch, channels[i], blocks[i].factor, chains[i][0], chains[i][1],
                                build(i + 1), merge, self.groups, self.features, attention_features,
                                attention_heads, embedding_features, context[i])

        self.net = build(0)
        self._init_runtime()


# -------------------------------------------------------------------------------------- plugins
def _wrap(net_t: Callable, plugin: str, Net: Callable) -> Callable:
    if net_t is not XUNet and not getattr(net_t, "_wraps_xunet", False):
        raise NotImplementedError(f"{plugin} wraps XUNet (UNetV0 has use_time_conditioning= and "
                                  f"use_embedding_cfg= for the same plugins)")
    Net._wraps_xunet = True
    return Net


def TimeConditioningPlugin(net_t: Callable, num_layers: int = 2) -> Callable:
    """a_unet TimeConditioningPlugin: features += MLP(GELU(NumberEmbedder(time))), the MLP's one
    Linear + GELU applied num_layers = 2 times; `net(x, time, ...)`."""
    if num_layers != 2:
        raise NotImplementedError(f"num_layers={num_layers}: the time conditioning applies its Linear twice")

    def Net(modulation_features: Optional[int] = None, _plugins: Sequence[tuple] = (), **kwargs):
        assert exists(modulation_features), "TimeConditioningPlugin requires modulation_features"
        return net_t(modulation_features=modulation_features, _plugins=(*_plugins, ("time",)), **kwargs)
    return _wrap(net_t, "TimeConditioningPlugin", Net)


def ClassifierFreeGuidancePlugin(net_t: Callable, embedding_max_length: int) -> Callable:
    """a_unet ClassifierFreeGuidancePlugin: a learned mask embedding of embedding_max_length tokens;
    `net(x, embedding=..., embedding_scale=s, embedding_mask_proba=p)`."""
    def Net(embedding_features: int, _plugins: Sequence[tuple] = (), **kwargs):
        return net_t(embedding_features=embedding_features, _plugins=(*_plugins, ("cfg", embedding_max_length)),
                     **kwargs)
    return _wrap(net_t, "ClassifierFreeGuidancePlugin", Net)
