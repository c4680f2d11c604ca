"""The giant (ViT-g/14, SwiGLU MLP) and four-register DINOv2 backbones on the CPU: registry and constructor arguments, timm
checkpoint keys, local-checkpoint loading, the reg4 + abs_pos_embed refusal, the SwiGLU C-ABI refusals, and parity with
goldens from the reference's own modules (tests/golden/make_vit_giant_golden.py) at the 1e-3 bar of test_vit_golden.py.
The giant goldens keep the full width (D = 1536, fc1 1536 -> 8192, fc2 4096 -> 1536) with the depth cut to two blocks."""
import ast
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

from imagefolder_b200 import config as xcfg
from imagefolder_b200.dino_enc import dinov2, vision_transformer as vt

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from vit_det_init import apply_det_init, golden_inputs  # noqa: E402

GIANT = "vit_giant_patch14_dinov2.lvd142m"
REG4 = ["vit_small_patch14_reg4_dinov2.lvd142m", "vit_base_patch14_reg4_dinov2.lvd142m",
        "vit_large_patch14_reg4_dinov2.lvd142m", "vit_giant_patch14_reg4_dinov2.lvd142m"]
NEW = [GIANT] + REG4
# (embed_dim, depth, heads, fc1 width, fc2 input width) -- timm's vision_transformer.py:2925-2995
SHAPES = {GIANT: (1536, 40, 24, 8192, 4096), REG4[0]: (384, 12, 6, 1536, 1536), REG4[1]: (768, 12, 12, 3072, 3072),
          REG4[2]: (1024, 24, 16, 4096, 4096), REG4[3]: (1536, 40, 24, 8192, 4096)}


def timm_keys(name, depth):
    """the state_dict keys of timm's VisionTransformer for these entries (num_classes = 0: no head parameters)"""
    keys = ["cls_token", "pos_embed", "patch_embed.proj.weight", "patch_embed.proj.bias"]
    if "_reg4_" in name:
        keys.append("reg_token")
    for i in range(depth):
        for k in ("norm1.weight", "norm1.bias", "attn.qkv.weight", "attn.qkv.bias", "attn.proj.weight", "attn.proj.bias",
                  "ls1.gamma", "norm2.weight", "norm2.bias", "mlp.fc1.weight", "mlp.fc1.bias", "mlp.fc2.weight",
                  "mlp.fc2.bias", "ls2.gamma"):
            keys.append(f"blocks.{i}.{k}")
    return sorted(keys + ["norm.weight", "norm.bias"])


@pytest.mark.parametrize("name", NEW)
def test_registry_arguments_and_checkpoint_keys(name):
    D, depth, heads, n1, n2 = SHAPES[name]
    m = vt.create_model(name, img_size=28, patch_size=14, depth=2)          # depth cut: the keys repeat per block
    assert m.embed_dim == D and len(m.blocks) == 2 and m.blocks[0].attn.num_heads == heads and vt._ARCH[name]["depth"] == depth
    assert m.blocks[0].attn.head_dim == 64
    assert sorted(m.state_dict().keys()) == timm_keys(name, 2)
    mlp = m.blocks[0].mlp
    assert tuple(mlp.fc1.weight.shape) == (n1, D) and tuple(mlp.fc2.weight.shape) == (D, n2)
    if "giant" in name:
        assert isinstance(mlp, vt.GluMlp) and isinstance(mlp.act, nn.SiLU) and isinstance(mlp.norm, nn.Identity)
    else:
        assert type(mlp) is vt.Mlp and isinstance(mlp.act, nn.GELU)
    if "_reg4_" in name:
        assert m.num_prefix_tokens == 5 and m.no_embed_class and tuple(m.pos_embed.shape) == (1, 4, D)
        assert tuple(m.reg_token.shape) == (1, 4, D)
    else:
        assert m.num_prefix_tokens == 1 and tuple(m.pos_embed.shape) == (1, 5, D)
    assert name in dinov2._NAMES


def test_glu_mlp_is_silu_gate_times_up():
    torch.manual_seed(0)
    mlp = vt.GluMlp(16, hidden_features=32)
    x = torch.randn(3, 16)
    h = mlp.fc1(x)
    want = mlp.fc2(torch.nn.functional.silu(h[:, :16]) * h[:, 16:])
    torch.testing.assert_close(mlp(x), want, rtol=0, atol=0)


@pytest.mark.parametrize("name", [GIANT, REG4[0]])
def test_local_timm_checkpoint_loads(name, tmp_path, monkeypatch):
    """a timm-format checkpoint at the 518 px / patch-14 geometry loads, resampled to 256 px / patch 16"""
    src = vt.create_model(name, depth=2)                                     # timm's geometry: 37 x 37 patches of 14
    state = {k: torch.randn_like(v) for k, v in src.state_dict().items()}
    path = tmp_path / "ckpt.pth"
    torch.save(state, path)
    monkeypatch.setenv("XQ_TIMM_CKPT_" + name.replace(".", "_").upper(), str(path))
    m = vt.create_model(name, pretrained=True, img_size=256, patch_size=16, depth=2)
    assert m.pretrained_loaded
    torch.testing.assert_close(m.blocks[1].mlp.fc1.weight, state["blocks.1.mlp.fc1.weight"])
    if "_reg4_" in name:
        torch.testing.assert_close(m.reg_token, state["reg_token"])
        assert tuple(m.pos_embed.shape) == (1, 256, m.embed_dim)             # no_embed_class: patch positions only


def test_reg4_with_abs_pos_embed_is_refused_at_construction():
    g = np.load(os.path.join(HERE, "golden", "vit_reg4_abs.npz"))
    # what the reference does with this configuration: both forwards fail on the level-embedding shape
    assert "must match" in str(g["encode_error"]) and "must match" in str(g["decode_error"])
    kw = dict(model_kwargs={'img_size': 28, 'patch_size': 14, 'drop_path_rate': 0.0}, pretrained=False, tuning_method='full',
              num_latent_tokens=4)
    for cls in (dinov2.DINOv2Encoder, dinov2.DINOv2Decoder):
        with pytest.raises(ValueError, match="abs_pos_embed"):
            cls(model_name=REG4[0], abs_pos_embed=True, **kw)
        cls(model_name=REG4[0], abs_pos_embed=False, **kw)                   # the reg4 backbones work without it
    dinov2.DINOv2Encoder(model_name=GIANT.replace("giant", "small"), abs_pos_embed=True, **kw)


def test_swiglu_entry_points_refuse_bad_arguments_without_writing():
    """every refusal comes before a launch (the pointers below are never dereferenced)"""
    from imagefolder_b200 import _capi
    L = _capi.lib()
    f = ctypes.cast(ctypes.c_void_p(4096), ctypes.POINTER(ctypes.c_float))
    for sfx in ("", "_f16"):
        fwd, bwd = getattr(L, "xq_vit_swiglu_fwd" + sfx), getattr(L, "xq_vit_swiglu_bwd" + sfx)
        assert fwd(None, f, 4096, 4, 64, None) == -1
        assert fwd(4096, f, 4096, 4, 60, None) == -1                        # H % 8 != 0
        assert fwd(4096, f, 4096, 0, 64, None) == -1
        assert bwd(4096, f, None, 4096, f, 4, 64, None) == -1
        assert bwd(4096, f, 4096, 4096, f, 4, 12, None) == -1
    assert L.xq_vit_residual_ln_fwd(None, None, None, None, None, 1, None, None, 1e-6, 4, 1536, None, None, None, None,
                                    None) == -1


def test_swiglu_dispatch_conditions():
    from imagefolder_b200 import _capi, vit_ops
    assert 1536 in vit_ops._SUPPORTED_D
    # the giant MLP has no fused SwiGLU GEMMs: an export of one means a stale object file in the library
    L = _capi.lib()
    for name in ("xq_vit_fc1_swiglu_fwd", "xq_vit_fc2_dswiglu_bwd"):
        assert not hasattr(L, name) and not hasattr(L, name + "_f16"), name


# ---- goldens from the reference's own modules ---------------------------------------------------------------------
CASES = ["vit_giant_vq", "vit_giant_relpos", "vit_reg4_relpos"]


def load_case(name):
    g = np.load(os.path.join(HERE, "golden", name + ".npz"))
    return g, ast.literal_eval(str(g["cfg_json"]))


def build_ours(cfg, depth, monkeypatch):
    """the product's VQModel for a golden's configuration, giant entries cut to the golden's depth"""
    for name in (GIANT, REG4[3]):
        monkeypatch.setitem(vt._ARCH, name, dict(vt._ARCH[name], depth=depth))
    args = xcfg.parse_args([])
    for k, v in cfg.items():
        setattr(args, k, v)
    torch.manual_seed(0)
    model = xcfg.build_vq_model(args).eval()
    apply_det_init(model)
    return model


def check(g, tok, h, dec, rtol, atol):
    st = int(g["token_stride"])
    np.testing.assert_allclose(tok[:, ::st], g["tok_sub"], rtol=rtol, atol=atol)
    assert tuple(h.shape) == tuple(g["h_shape"])
    np.testing.assert_allclose(h.reshape(h.shape[0], h.shape[1], -1)[:, :, ::4], g["h_sub"], rtol=rtol, atol=atol)
    np.testing.assert_allclose(dec[:, :, ::4, ::4], g["dec_sub"], rtol=rtol, atol=atol)
    assert abs(float(tok.astype(np.float64).sum()) - float(g["tok_sum"])) <= atol * tok.size * 0.05 + rtol * float(g["tok_abs"])
    assert abs(float(dec.astype(np.float64).sum()) - float(g["dec_sum"])) <= atol * dec.size * 0.05 + rtol * float(g["dec_abs"])


@pytest.mark.parametrize("name", CASES)
def test_product_matches_reference_golden_cpu(name, monkeypatch):
    g, cfg = load_case(name)
    model = build_ours(cfg, int(g["giant_depth"]), monkeypatch)
    x, q = golden_inputs(int(g["q_shape"][1]), int(g["q_shape"][2]))
    with torch.no_grad():
        tok, h, dec = model.encoder(x), model.encode(x), model.decode(q)
    check(g, tok.numpy(), h.numpy(), dec.numpy(), rtol=1e-3, atol=1e-4)
    assert int(g["enc_S"]) == {"vit_giant_vq": 513, "vit_giant_relpos": 513, "vit_reg4_relpos": 517}[name]
