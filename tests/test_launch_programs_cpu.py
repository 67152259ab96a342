"""The launch programs of the inference, sampling, conditioning and training plans, recorded on
the CPU and compared with tests/golden/launch_programs.json.gz.

Every launch function that unet.py and training.py call through `ops` is replaced by a recorder,
so plans build and run here without a GPU.  Each call is bound to the real function's signature
(defaults applied, so passing a default explicitly changes nothing) and every tensor argument is
recorded as (storage index by first use in the program, byte offset, shape, stride, dtype).  For
fp64 tensors (GroupNorm statistics slots, the loss accumulator) the offset is replaced by its
first-use index within the storage: which slot a value lands in has no meaning, only which
launches share it.  The program is therefore fixed up to allocation order, and a change to how
plans are built that alters any launch, argument, buffer aliasing or gradient-arena layout fails
here.

    python tests/test_launch_programs_cpu.py --write     # re-record the fixture
"""
import gzip
import inspect
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from audio_diffusion_pytorch_b200 import _lib, ops, training  # noqa: E402
from audio_diffusion_pytorch_b200.unet import UNetV0  # noqa: E402

FIXTURE = os.path.join(ROOT, "tests", "golden", "launch_programs.json.gz")

LAUNCHES = ("conv_gemm", "gn_silu", "gn_stats", "ln_film", "attention", "skinny_linear", "time_features",
            "silu_bf16", "stem_in", "stem_out", "narrow_conv", "step_select", "step_advance", "wgrad",
            "gn_silu_bwd", "gn_bwd_apply", "ln_film_bwd", "colsum", "skip_gate", "skip_gate_bwd",
            "cond_bwd", "narrow_conv_bwd", "stem_out_bwd", "stem_in_bwd", "attention_bwd", "ln_fold_bwd")

TINY = dict(in_channels=2, channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 2, 2],
            attentions=[0, 0, 1], attention_heads=2, attention_features=64)
TINY_TEXT = dict(TINY, cross_attentions=[0, 1, 1], use_embedding_cfg=True,
                 embedding_max_length=8, embedding_features=32)
README = dict(in_channels=2, channels=[8, 32, 64, 128, 256, 512, 512, 1024, 1024],
              factors=[1, 4, 4, 4, 2, 2, 2, 2, 2], items=[1, 2, 2, 2, 2, 2, 2, 4, 4],
              attentions=[0, 0, 0, 0, 0, 1, 1, 1, 1], attention_heads=8, attention_features=64)

# name -> (net kwargs, net attributes, B, T, M, inference modes, training (mode, want_dxin) pairs)
TRAIN_ALL = (("loss", True), ("loss", False), ("v", True), ("v", False))
NETS = {
    "tiny": (TINY, {}, 2, 4096, 0, ("v", "sample"), TRAIN_ALL),
    "tiny_unfused_thin": (TINY, {"fuse_thin_levels": False}, 2, 4096, 0, ("v", "sample"), ()),
    # the A-transform fusion applies to the unfused C >= 32 ConvBlocks only
    "tiny_fuse_groupnorm": (TINY, {"fuse_groupnorm": True, "fuse_thin_levels": False}, 2, 4096, 0,
                            ("v", "sample"), ()),
    "tiny_fp32": (TINY, {"verify_fp32": True}, 2, 4096, 0, ("v", "sample"), ()),
    "text_cfg": (TINY_TEXT, {}, 2, 4096, 8, ("v", "v_cfg", "sample_cfg"), (("loss", False), ("v", True))),
    "skipcat_adapter": (dict(in_channels=3, out_channels=2, channels=[8, 32, 64], factors=[1, 4, 4],
                             items=[1, 2, 2], use_modulation=False, use_time_conditioning=False),
                        {}, 2, 4096, 0, ("v",), (("v", True), ("loss", False))),
    "inject": (dict(TINY, context_channels=[0, 0, 4]), {}, 2, 4096, 0, ("v", "sample"),
               (("loss", False), ("v", True))),
    "append": (dict(TINY, in_channels=3, append_channels=1, out_channels=2), {}, 2, 4096, 0, ("v", "sample"),
               (("loss", True), ("v", True))),
    "att_narrow": (dict(TINY, attentions=[1, 0, 1]), {}, 2, 4096, 0, ("v", "sample"), (("loss", False),)),
    "head32_g4": (dict(TINY_TEXT, attention_heads=3, attention_features=32, resnet_groups=4), {}, 2, 4096, 8,
                  ("v", "sample_cfg"), (("loss", False),)),
    "head128_g4": (dict(TINY_TEXT, attention_heads=1, attention_features=128, resnet_groups=4), {}, 2, 4096,
                   8, ("v", "sample_cfg"), (("loss", False),)),
    "factor1_c128": (dict(TINY, channels=[8, 32, 128], factors=[1, 4, 1]), {}, 2, 4096, 0, ("v", "sample"),
                     (("loss", False),)),
    "readme": (README, {}, 1, 2 ** 13, 0, ("v", "sample"), (("loss", False),)),
}


def _val(v, rec):
    if isinstance(v, torch.Tensor):
        return rec.tensor(v)
    if isinstance(v, (tuple, list)):
        return [_val(x, rec) for x in v]
    if v is None or isinstance(v, (bool, int, float, str)):
        return v
    raise TypeError(f"unrecorded argument type {type(v)}")


class Recorder:
    """Stands in for the launch functions of `ops`; one list of launches per program."""

    def __init__(self):
        self.launches, self.storages, self.slots, self.keep = [], {}, {}, []

    def tensor(self, t):
        self.keep.append(t)                     # no storage address is reused while recording
        st = t.untyped_storage()
        key = (st.data_ptr(), st.nbytes())
        sidx = self.storages.setdefault(key, len(self.storages))
        off = t.storage_offset() * t.element_size()
        if t.dtype == torch.float64:
            off = self.slots.setdefault((sidx, off), sum(1 for k in self.slots if k[0] == sidx))
        return ["T", sidx, off, list(t.shape), list(t.stride()), str(t.dtype).replace("torch.", "")]

    def make(self, name, real):
        sig = inspect.signature(real)

        def record(*args, **kwargs):
            b = sig.bind(*args, **kwargs)
            b.apply_defaults()
            self.launches.append([name] + [[k, _val(v, self)] for k, v in b.arguments.items()])
        return record

    def take(self):
        out, self.launches = self.launches, []
        return out


@pytest.fixture(scope="module")
def recorder():
    mp = pytest.MonkeyPatch()
    rec = install(mp)
    yield rec
    mp.undo()


def install(mp):
    rec = Recorder()
    for name in LAUNCHES:
        mp.setattr(ops, name, rec.make(name, getattr(ops, name)))
    mp.setattr(ops, "device_check", lambda: None)

    def no_library():
        raise AssertionError("a launch reached the CUDA library")
    mp.setattr(_lib, "lib", no_library)
    return rec


def build_net(kw, attrs):
    torch.manual_seed(0)
    net = UNetV0(dim=1, **kw)
    for k, v in attrs.items():
        setattr(net, k, v)
    return net


def record_case(name, rec):
    kw, attrs, B, T, M, modes, trains = NETS[name]
    net = build_net(kw, attrs)
    names = {id(p): n for n, p in net.named_parameters()}
    out = {}
    for m in modes:
        cfg = m.endswith("_cfg")
        mode = m[:-4] if cfg else m
        Bh = 2 * B if cfg else B
        plan = net._plan(B, T, Bh, M, mode, (5.0 if cfg else None, False))
        plan.cfg_scale = 5.0 if cfg else None
        rec.storages, rec.slots, rec.keep = {}, {}, []
        for fn in getattr(plan, "pre", []):
            fn()
        pre = rec.take()
        plan.run_eager()
        out["infer_" + m] = {"pre": pre, "prog": rec.take(), "workspace_bytes": plan.workspace_bytes}
    if "sample" in modes and net.use_modulation:
        rec.storages, rec.slots, rec.keep = {}, {}, []
        net._cond_table(torch.zeros(6), None)
        out["cond_6"] = {"prog": rec.take()}
    for mode, want_dxin in trains:
        plan = training.build_train_plan(net, B, T, M, mode, want_dxin)
        rec.storages, rec.slots, rec.keep = {}, {}, []
        for fn in plan.fwd:
            fn()
        fwd = rec.take()
        marks = []
        plan.on_mark = lambda iv: marks.append(list(iv))
        plan.backward_program()
        plan.on_mark = None
        out[f"train_{mode}_{int(want_dxin)}"] = {
            "fwd": fwd, "bwd": rec.take(), "marks": marks, "flat": plan.flat.numel(),
            "specs": {names[k]: [v[0], v[1], list(v[2]), None if v[3] is None else list(v[3])]
                      for k, v in plan.specs.items()},
            "grads": {names[k]: list(v) for k, v in plan.grads.items()}}
    return out


def first_difference(got, want, where=""):
    if isinstance(want, dict) and isinstance(got, dict):
        for k in sorted(set(want) | set(got)):
            if k not in got or k not in want:
                return f"{where}/{k}: {'missing' if k not in got else 'unexpected'}"
            d = first_difference(got[k], want[k], f"{where}/{k}")
            if d:
                return d
        return None
    if isinstance(want, list) and isinstance(got, list) and where.rsplit("/", 1)[-1] in (
            "pre", "prog", "fwd", "bwd"):
        for i, (g, w) in enumerate(zip(got, want)):
            if g != w:
                return f"{where}[{i}]:\n  got  {json.dumps(g)}\n  want {json.dumps(w)}"
        if len(got) != len(want):
            return f"{where}: {len(got)} launches, fixture has {len(want)}"
        return None
    return None if got == want else f"{where}: got {json.dumps(got)}, want {json.dumps(want)}"


@pytest.fixture(scope="module")
def fixture():
    with gzip.open(FIXTURE, "rt") as f:
        return json.load(f)


@pytest.mark.parametrize("name", sorted(NETS))
def test_launch_program(name, recorder, fixture):
    got = json.loads(json.dumps(record_case(name, recorder)))
    d = first_difference(got, fixture[name], name)
    assert d is None, "launch program differs from the fixture at " + d


def test_fixture_covers_every_case(fixture):
    assert sorted(fixture) == sorted(NETS)


if __name__ == "__main__" and "--write" in sys.argv:
    mp = pytest.MonkeyPatch()
    rec = install(mp)
    data = {name: record_case(name, rec) for name in sorted(NETS)}
    mp.undo()
    with gzip.GzipFile(FIXTURE, "wb", mtime=0) as f:
        f.write(json.dumps(data, separators=(",", ":"), sort_keys=True).encode())
    for name, cases in data.items():
        print(name, {k: {p: len(v[p]) for p in ("pre", "prog", "fwd", "bwd") if p in v} for k, v in cases.items()})
    print(f"wrote {FIXTURE} ({os.path.getsize(FIXTURE)} bytes)")
