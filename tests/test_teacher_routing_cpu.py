"""Routing of VisionTransformer.forward / forward_features between the module path and the frozen fused path
(vit_ops.frozen_path_ok), checked without a GPU: CPU and fp32 calls run the module path, unchanged."""
import warnings

import pytest
import torch

from imagefolder_b200 import vit_ops
from imagefolder_b200.dino_enc import vision_transformer as vt


def _frozen(name="vit_small_patch14_dinov2.lvd142m", **kw):
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = vt.create_model(name, pretrained=False, img_size=64, patch_size=16, drop_path_rate=0.0, **kw)
    m.eval()
    for p in m.parameters():
        p.requires_grad = False
    return m


def _module_forward_features(m, x):
    x = m.patch_embed(x)
    x = m._pos_embed(x)
    x = m.norm_pre(m.patch_drop(x))
    return m.norm(m.blocks(x))


@pytest.mark.parametrize("name", ["vit_small_patch14_dinov2.lvd142m", "vit_base_patch16_clip_224.openai",
                                  "vit_small_patch14_reg4_dinov2.lvd142m"])
def test_cpu_calls_run_the_module_path(name, monkeypatch):
    m = _frozen(name, depth=2)
    x = torch.rand(2, 3, 64, 64) * 2 - 1

    def boom(*a, **k):
        raise AssertionError("the frozen fused path ran for a CPU call")
    monkeypatch.setattr(vt, "frozen_forward", boom)
    assert not vit_ops.frozen_path_ok(m, x)
    with torch.no_grad():
        ref = _module_forward_features(m, x)
        assert torch.equal(m.forward_features(x), ref)
        assert torch.equal(m(x), ref[:, 0])
        with torch.autocast("cpu", dtype=torch.bfloat16):
            ref16 = _module_forward_features(m, x)
            assert torch.equal(m.forward_features(x), ref16)


def test_routing_rule_on_a_cpu_tensor_stays_false():
    m = _frozen(depth=1)
    x = torch.rand(1, 3, 64, 64)
    assert not vit_ops.frozen_path_ok(m, x)
    assert not vit_ops.frozen_path_ok(m, x.double())


def test_unfrozen_teacher_trains_on_the_module_path():
    m = _frozen(depth=1)
    m.blocks[0].attn.qkv.weight.requires_grad_(True)
    x = torch.rand(2, 3, 64, 64)
    (m(x) * torch.randn(2, 384)).sum().backward()          # a plain sum of a LayerNorm output has no gradient
    g = m.blocks[0].attn.qkv.weight.grad
    assert g is not None and bool(g.abs().sum() > 0)


def test_teacher_state_dict_keys_unchanged():
    """the routing adds no parameter, buffer or state_dict key"""
    m = _frozen("vit_base_patch16_clip_224.openai", depth=2)
    keys = set(m.state_dict())
    assert "norm_pre.weight" in keys and "blocks.1.mlp.fc2.bias" in keys
    assert not any("frozen" in k or "_assemble" in k for k in keys)
