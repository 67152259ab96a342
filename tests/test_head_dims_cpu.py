"""Attention head dims other than 64 on the CPU: UNetV0(attention_features=D) constructs for
D in {32, 64, 128} and refuses anything else, reference weights and checkpoints built at D = 32
and 128 load tensor for tensor, and the head-dim entry points of the C ABI are declared,
exported and refuse an unsupported head dim before touching the device."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = dict(in_channels=2, channels=[8, 32, 64], factors=[1, 4, 4], items=[1, 2, 2])
HD_SYMBOLS = ("adp_attention_hd", "adp_attention_bwd_hd", "adp_f32_attention_hd")


def _att(heads, features, **extra):
    return dict(TINY, attentions=[0, 0, 1], attention_heads=heads, attention_features=features, **extra)


def _text(heads, features):
    return _att(heads, features, cross_attentions=[0, 1, 1], use_embedding_cfg=True,
                embedding_max_length=8, embedding_features=32)


@pytest.mark.parametrize("features", [32, 64, 128])
def test_supported_head_dims_construct(features):
    import audio_diffusion_pytorch_b200 as adp
    net = adp.UNetV0(dim=1, **_att(2, features))
    assert net.head_features == features
    adp.UNetV0(dim=1, **_text(2, features))


@pytest.mark.parametrize("features", [16, 48, 96, 256])
def test_unsupported_head_dims_are_refused(features):
    import audio_diffusion_pytorch_b200 as adp
    with pytest.raises(AssertionError, match=r"head dims 32, 64, 128"):
        adp.UNetV0(dim=1, **_att(2, features))
    with pytest.raises(AssertionError, match=r"head dims 32, 64, 128"):
        adp.UNetV0(dim=1, **_text(2, features))


@pytest.mark.parametrize("heads,features", [(4, 32), (1, 128), (3, 32)])
def test_reference_parameters_load_at_other_head_dims(oracle_port, heads, features):
    import audio_diffusion_pytorch_b200 as adp
    for cfg in (_att(heads, features), _text(heads, features)):
        torch.manual_seed(0)
        ref = oracle_port.DiffusionModelPort(**cfg)
        ours = adp.DiffusionModel(net_t=adp.UNetV0, **cfg)
        assert [tuple(p.shape) for p in ours.net.parameters()] == \
            [tuple(p.shape) for p in ref.net.parameters()]
        ours.net.load_reference_parameters(ref.net)
        for a, b in zip(ours.net.parameters(), ref.net.parameters()):
            assert torch.equal(a, b)


@pytest.mark.parametrize("features", [32, 128])
def test_reference_checkpoints_load_at_other_head_dims(oracle_port, tmp_path, features):
    import audio_diffusion_pytorch_b200 as adp
    cfg = _text(2, features)
    torch.manual_seed(0)
    ref = oracle_port.DiffusionModelPort(**cfg)
    ours = adp.DiffusionModel(net_t=adp.UNetV0, **cfg)
    path = tmp_path / f"ref_d{features}.pt"
    torch.save(ref.state_dict(), path)
    ours.load_reference_state_dict(torch.load(path))
    for a, b in zip(ours.net.parameters(), ref.net.parameters()):
        assert torch.equal(a, b)
    # a checkpoint saved at another head dim has other projection shapes: refused
    other = oracle_port.DiffusionModelPort(**_text(2, 64))
    with pytest.raises(AssertionError):
        ours.load_reference_state_dict(other.state_dict())


def test_head_dim_entry_points_declared_and_exported():
    from audio_diffusion_pytorch_b200 import _build, _lib
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "adp_b200.h")).read(), flags=re.S)
    lib = ctypes.CDLL(_build.build())
    for name in HD_SYMBOLS:
        assert re.search(r"\b%s\s*\(" % name, text), f"{name} not declared"
        assert hasattr(lib, name), f"{name} not exported"
        assert name in _lib.EXPORTS


@pytest.mark.parametrize("head_dim", [0, 16, 48, 96, 256])
def test_unsupported_head_dim_is_an_abi_error(head_dim):
    """The head-dim check comes first, so these calls return an error without a device."""
    from audio_diffusion_pytorch_b200 import _build, _lib
    _build.build()
    L = _lib.lib()
    rc = L.adp_attention_hd(None, None, None, None, 1, 1, head_dim, 1, 1, 512, 512, 512, 512,
                            0.125, None, None)
    assert rc != 0 and b"head_dim" in L.adp_last_error()
    rc = L.adp_attention_bwd_hd(None, head_dim, None)
    assert rc != 0 and b"head_dim" in L.adp_last_error()
    rc = L.adp_f32_attention_hd(None, None, None, None, 1, 1, head_dim, 1, 1, 512, 512, 512, 512,
                                0.125, None)
    assert rc != 0 and b"head_dim" in L.adp_last_error()
