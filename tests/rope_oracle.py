"""Functional restatement of the RoPE decoder (DINOv2Decoder(use_rope=True), dino_enc/dinov2.py:313-365 with RoPEAttention,
dino_enc/vision_transformer.py:238-270) over a state_dict, in whatever precision the tensors carry (fp64 in the tests).
Test infrastructure only: the tight gradient reference of the RoPE path, pinned to the reference by the vit_rope_*.npz
goldens.  Reuses the LayerNorm of oracle/vit_ref.py; everything else is written out here."""
import math
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.vit_ref import _ln  # noqa: E402

IMG = 256


def rotate(t, c):
    """t [..., T, 64] as 32 complex pairs times c (broadcast over [T, 32] or [H, T, 32])"""
    tc = torch.view_as_complex(t.reshape(*t.shape[:-1], -1, 2).contiguous())
    return torch.view_as_real(tc * c).flatten(-2)


def rope_cis(freqs, num_heads, dtype):
    """polar(1, t_x fx + t_y fy) [H, 256, 32] for the 16 x 16 image grid"""
    i = torch.arange(IMG, dtype=dtype, device=freqs.device)
    tx, ty = (i % 16)[None, :, None], torch.div(i, 16, rounding_mode="floor")[None, :, None]
    fr = freqs.view(2, num_heads, 1, -1)
    theta = tx * fr[0] + ty * fr[1]
    return torch.polar(torch.ones_like(theta), theta)


def rope_attention(x, sd, prefix, num_heads, P, L):
    B, N, C = x.shape
    qkv = F.linear(x, sd[prefix + ".qkv.weight"], sd[prefix + ".qkv.bias"])
    qkv = qkv.reshape(B, N, 3, num_heads, C // num_heads).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    c_img, c_lat = rope_cis(sd[prefix + ".freqs"], num_heads, x.dtype), sd[prefix + ".freqs_1d"]
    q = torch.cat([q[:, :, :P], rotate(q[:, :, P:N - L], c_img), rotate(q[:, :, N - L:], c_lat)], dim=2)
    k = torch.cat([k[:, :, :P], rotate(k[:, :, P:N - L], c_img), rotate(k[:, :, N - L:], c_lat)], dim=2)
    att = ((q * (C // num_heads) ** -0.5) @ k.transpose(-2, -1)).softmax(dim=-1)
    y = (att @ v).transpose(1, 2).reshape(B, N, C)
    return F.linear(y, sd[prefix + ".proj.weight"], sd[prefix + ".proj.bias"])


def rope_block(x, sd, prefix, num_heads, P, L):
    x = x + rope_attention(_ln(x, sd, prefix + ".norm1"), sd, prefix + ".attn", num_heads, P, L) * sd[prefix + ".ls1.gamma"]
    h = F.gelu(F.linear(_ln(x, sd, prefix + ".norm2"), sd[prefix + ".mlp.fc1.weight"], sd[prefix + ".mlp.fc1.bias"]))
    return x + F.linear(h, sd[prefix + ".mlp.fc2.weight"], sd[prefix + ".mlp.fc2.bias"]) * sd[prefix + ".ls2.gamma"]


def rope_decoder_forward(sd, z, num_heads: int, patch=16):
    """z [B, L, D] -> image [B, 3, 16 patch, 16 patch]; sd = DINOv2Decoder(use_rope=True).state_dict() (tuning 'full')"""
    B, L, _ = z.shape
    prefix = [sd["model.cls_token"]] + ([sd["model.reg_token"]] if "model.reg_token" in sd else [])
    prefix = [t.expand(B, -1, -1) for t in prefix]
    P = sum(t.shape[1] for t in prefix)
    t = torch.cat(prefix + [sd["mask_token"].expand(B, IMG, -1), z], dim=1)
    depth = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("model.blocks."))
    for i in range(depth):
        t = rope_block(t, sd, f"model.blocks.{i}", num_heads, P, L)
    t = _ln(t, sd, "model.norm")[:, P:P + IMG]
    t = F.linear(t, sd["to_pixel.model.weight"], sd["to_pixel.model.bias"])
    h = int(math.sqrt(IMG))
    t = t.reshape(B, h, h, patch, patch, 3)
    return torch.einsum("nhwpqc->nchpwq", t).reshape(B, 3, h * patch, h * patch)


def fp64_state(module, requires_grad=True):
    """the module's parameters and buffers in fp64 / complex128, as leaves"""
    sd = {}
    for k, v in module.state_dict().items():
        v = v.detach().to(torch.complex128 if v.is_complex() else torch.float64).clone()
        sd[k] = v.requires_grad_(requires_grad) if v.is_floating_point() or v.is_complex() else v
    return sd
