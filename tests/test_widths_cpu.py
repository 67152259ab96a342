"""Level, attention and embedding widths on the CPU.

  * the constructor accepts level widths of 8 or a multiple of 16 up to B200UNet.MAX_WIDTH (level 0
    up to MAX_C0), attention widths heads * D and embedding widths up to MAX_WIDTH, and refuses
    everything else with a message that names the limit;
  * tiny nets at the new widths run their inference, sampling and guidance programs on the CPU
    with fake kernels that write the launch checker's fp64 restatements (tests/launch_check.py),
    against the CPU oracle built with the same arguments: this pins the host plans (weight packs,
    LayerNorm folds, arena layout) at those widths without a GPU.
"""
import pytest
import torch

import launch_check as lc
from audio_diffusion_pytorch_b200 import _lib, ops
from audio_diffusion_pytorch_b200.diffusion import VSampler
from audio_diffusion_pytorch_b200.models import DiffusionModel
from audio_diffusion_pytorch_b200.unet import B200UNet, UNetV0
from test_launch_check_cpu import rel_l2

V_TOL, BRANCH_TOL = 1e-4, 1.2e-2


def _net(c0=8, c=64, **kw):
    return dict(in_channels=2, channels=[c0, 32, c], factors=[1, 2, 2], items=[1, 1, 1], **kw)


def _att(mid_heads, D, **kw):
    return _net(attentions=[0, 0, 1], attention_heads=mid_heads, attention_features=D, **kw)


def _text(E):
    return _net(attentions=[0, 0, 1], cross_attentions=[0, 0, 1], attention_heads=2, attention_features=32,
                use_embedding_cfg=True, embedding_max_length=4, embedding_features=E)


# accepted by the constructor; also run once each on the GPU (tests/test_widths_gpu.py)
ACCEPTED = {
    **{f"level_{c}": _net(c=c) for c in (16, 48, 96, 192, 320, 1536, 2048)},
    **{f"level0_{c}": _net(c0=c) for c in (16, 48, 96)},
    **{f"embedding_{e}": _text(e) for e in (1536, 2048)},
    "attention_1024": _att(8, 128), "attention_2048": _att(16, 128),
}
REFUSED = [
    *[(f"level_{c}", _net(c=c), rf"channels\[2\]={c}: ") for c in (24, 40)],
    ("level_2064", _net(c=2064), rf"channels\[2\]=2064: .*at most {B200UNet.MAX_WIDTH} wide"),
    *[(f"level0_{c}", _net(c0=c), rf"channels\[0\]={c}: levels are 8 channels wide or a multiple of 16")
      for c in (24, 40)],
    ("level0_2064", _net(c0=2064), rf"channels\[0\]=2064: .*at most {B200UNet.MAX_C0} wide"),
    ("level0_272", _net(c0=272), rf"channels\[0\]=272: .*at most {B200UNet.MAX_C0} wide"),
    ("embedding_2056", _text(2056), rf"embedding_features=2056: .*up to {B200UNet.MAX_WIDTH}"),
    ("attention_2304", _att(18, 128), rf"= 2304: .*at most {B200UNet.MAX_WIDTH}"),
]


@pytest.mark.parametrize("name", sorted(ACCEPTED))
def test_accepted_widths_construct(name):
    UNetV0(dim=1, **ACCEPTED[name])


@pytest.mark.parametrize("name,kw,msg", REFUSED, ids=[r[0] for r in REFUSED])
def test_refused_widths_name_their_limit(name, kw, msg):
    with pytest.raises(AssertionError, match=msg):
        UNetV0(dim=1, **kw)


def test_fuse_groupnorm_keeps_wide_levels_unfused(monkeypatch):
    """The conv GEMM's GroupNorm A transform holds MAX_FUSED_GN_C input channels: wider levels run
    gn_silu -> conv_gemm under fuse_groupnorm."""
    from test_launch_programs_cpu import install
    rec = install(monkeypatch)
    torch.manual_seed(0)
    net = UNetV0(dim=1, **_net(c=2048))
    net.fuse_groupnorm, net.fuse_thin_levels = True, False
    plan = net._plan(1, 256, 1, 0, "v", (None, False))
    plan.run_eager()
    launches = [(k[0], dict(k[1:])) for k in rec.take()]
    fused = {a["c_in"] for n, a in launches if n == "conv_gemm" and a["gn"] is not None}
    unfused = {a["c_in"] for n, a in launches if n == "conv_gemm" and a["gn"] is None}
    assert fused and max(fused) <= B200UNet.MAX_FUSED_GN_C
    assert 2048 in unfused and any(n == "gn_silu" and a["x"][3][-1] == 2048 for n, a in launches)


# ------------------------------------------------------------------------------ programs
NETS = {
    # level widths 48 / 96 / 192 with group sizes 2, 6, 12 and 24, attention at the last two levels
    "thin_odd": dict(in_channels=2, channels=[16, 48, 96, 192], factors=[1, 2, 2, 2], items=[1, 1, 1, 1],
                     attentions=[0, 0, 1, 1], attention_heads=2, attention_features=32),
    # levels beyond 1024, 16 heads x 64, cross-attention on a 2048-wide embedding
    "wide_text": dict(in_channels=2, channels=[8, 64, 384, 1536], factors=[1, 4, 4, 2], items=[1, 1, 1, 1],
                      attentions=[0, 0, 0, 1], cross_attentions=[0, 0, 0, 1], attention_heads=16,
                      attention_features=64, use_embedding_cfg=True, embedding_max_length=4,
                      embedding_features=2048),
}


@pytest.fixture
def cpu_launches(monkeypatch):
    monkeypatch.setattr(ops, "device_check", lambda: None)
    monkeypatch.setattr(ops, "require_cuda", lambda x: None)

    def no_library():
        raise AssertionError("a launch reached the CUDA library")
    monkeypatch.setattr(_lib, "lib", no_library)


def _pair(oracle_port, cfg):
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**cfg)
    model = DiffusionModel(net_t=UNetV0, **cfg)
    model.net.load_reference_parameters(ref.net)
    model.net.use_cuda_graph = False           # every call runs the plan's launches eagerly
    return ref, model.net


@pytest.mark.parametrize("name", sorted(NETS))
def test_program_vs_oracle(cpu_launches, oracle_port, name):
    cfg = NETS[name]
    ref, net = _pair(oracle_port, cfg)
    g = torch.Generator().manual_seed(3)
    x, sigma = torch.randn(2, 2, 1024, generator=g), torch.rand(2, generator=g)
    emb = torch.randn(2, 4, cfg["embedding_features"], generator=g) if "embedding_features" in cfg else None
    kw = dict(embedding=emb) if emb is not None else {}
    with torch.no_grad():
        cases = [(1.0, V_TOL, BRANCH_TOL)] + ([(5.0, 3e-4, 2.5 * BRANCH_TOL)] if emb is not None else [])
        for scale, v_tol, b_tol in cases:
            want = ref.net(x, sigma, embedding_scale=scale, **kw) if emb is not None else ref.net(x, sigma)
            with lc.Shadow(fake=True) as sh:
                v = net(x, sigma, embedding=emb, embedding_scale=scale)
            assert sh.n_checked == sh.n_launch > 0
            e_v, e_b = rel_l2(v, want), rel_l2(v - x, want - x)
            print(f"{name} scale {scale}: rel-L2(v) {e_v:.3e} rel-L2(branch) {e_b:.3e}")
            assert e_v <= v_tol and e_b <= b_tol


def test_sampling_program_vs_oracle(cpu_launches, oracle_port):
    ref, net = _pair(oracle_port, NETS["thin_odd"])
    noise = torch.randn(2, 2, 1024, generator=torch.Generator().manual_seed(4))
    with torch.no_grad():
        want = ref.sample(noise, num_steps=3)
        with lc.Shadow(fake=True) as sh:
            s = VSampler(net=net)(noise, num_steps=3)
    assert sh.n_checked == sh.n_launch > 0
    e = rel_l2(s, want)
    print(f"thin_odd 3-step sample: rel-L2 {e:.3e}")
    assert e <= 5e-3
