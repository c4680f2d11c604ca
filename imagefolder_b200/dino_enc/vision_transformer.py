"""ViT backbone used by the tokenizer encoder/decoder.

Restates the subset of timm==1.0.9's VisionTransformer that the reference instantiates through
its vendored copy (tokenizer/tokenizer_image/dino_enc/vision_transformer.py): `Attention` (:145),
`RoPEAttention` (:200, helpers :58-142), `LayerScale` (:280), `Block` (:295), `VisionTransformer` (:587, `_pos_embed` :814-848), and the
model-name registry entries the reference's DINOv2 encoder / decoder accept (`vit_{small,base,large,giant}_patch14_dinov2
.lvd142m` and their `_reg4_` variants, :2893-2995).
timm itself is not vendored in the reference nor installed here, so `PatchEmbed`, `Mlp`, `DropPath`
and `resample_abs_pos_embed` follow timm 1.0.9's published behaviour (SURVEY.md section 8c:
this boundary is "parity unpinned" by the reference); so does `GluMlp` (timm's SwiGLUPacked) of the giant backbones.

Parameter names (= checkpoint keys) are identical to timm's: patch_embed.proj, cls_token,
pos_embed, blocks.{i}.{norm1,attn.qkv,attn.proj,ls1.gamma,norm2,mlp.fc1,mlp.fc2,ls2.gamma}, norm.

GEMMs run on cuBLAS and attention on the fused SDPA library kernel (plain library calls); the
elementwise / normalisation glue is what imagefolder_b200.vit_ops replaces with sm_90a kernels.  A frozen model (every
parameter requires_grad=False: the semantic / detail guide teachers) called on a CUDA fp32 image that needs no gradient under
bf16 / fp16 autocast runs `forward` / `forward_features` on those kernels too (vit_ops.frozen_forward); everything else
runs the module path below.
"""
from __future__ import annotations

import math
from functools import partial

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..vit_ops import frozen_forward, frozen_path_ok


def trunc_normal_(t, std=0.02):
    return nn.init.trunc_normal_(t, mean=0.0, std=std, a=-2.0, b=2.0)  # timm trunc_normal_: absolute cut-offs


class PatchEmbed(nn.Module):
    """timm.layers.PatchEmbed: Conv2d(k = s = patch) -> flatten -> NLC (norm = Identity)."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768, bias=True, **_):
        super().__init__()
        self.img_size = (img_size, img_size)
        self.patch_size = (patch_size, patch_size)
        self.grid_size = (img_size // patch_size, img_size // patch_size)
        self.num_patches = self.grid_size[0] * self.grid_size[1]
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size, bias=bias)
        self.norm = nn.Identity()

    def forward(self, x):
        x = self.proj(x)
        return x.flatten(2).transpose(1, 2)


class Mlp(nn.Module):
    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.0, **_):
        super().__init__()
        out_features = out_features or in_features
        hidden_features = hidden_features or in_features
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.act = act_layer()
        self.fc2 = nn.Linear(hidden_features, out_features)

    def forward(self, x):
        return self.fc2(self.act(self.fc1(x)))


class GluMlp(nn.Module):
    """timm.layers.GluMlp with gate_last=False, as timm's SwiGLUPacked builds it for the giant backbones
    (vision_transformer.py:2925-2937: mlp_layer=SwiGLUPacked, act_layer=nn.SiLU, norm Identity): fc1 -> [gate | up] halves ->
    act(gate) * up -> fc2.  Attribute and checkpoint key names are timm's (mlp.fc1 / mlp.fc2)."""

    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.SiLU, drop=0.0, **_):
        super().__init__()
        out_features = out_features or in_features
        hidden_features = hidden_features or in_features
        assert hidden_features % 2 == 0
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.act = act_layer()
        self.norm = nn.Identity()
        self.fc2 = nn.Linear(hidden_features // 2, out_features)

    def forward(self, x):
        x1, x2 = self.fc1(x).chunk(2, dim=-1)
        return self.fc2(self.norm(self.act(x1) * x2))


class DropPath(nn.Module):
    """timm.layers.DropPath (stochastic depth per sample, scale_by_keep=True)."""

    def __init__(self, drop_prob: float = 0.0, scale_by_keep: bool = True):
        super().__init__()
        self.drop_prob = drop_prob
        self.scale_by_keep = scale_by_keep

    def forward(self, x):
        if self.drop_prob == 0.0 or not self.training:
            return x
        keep_prob = 1 - self.drop_prob
        shape = (x.shape[0],) + (1,) * (x.ndim - 1)
        random_tensor = x.new_empty(shape).bernoulli_(keep_prob)
        if keep_prob > 0.0 and self.scale_by_keep:
            random_tensor.div_(keep_prob)
        return x * random_tensor


def resample_abs_pos_embed(posemb, new_size, old_size=None, num_prefix_tokens=1, interpolation='bicubic',
                           antialias=True):
    """timm.layers.resample_abs_pos_embed (1.0.9)."""
    num_pos_tokens = posemb.shape[1]
    num_new_tokens = new_size[0] * new_size[1] + num_prefix_tokens
    if num_new_tokens == num_pos_tokens and new_size[0] == new_size[1]:
        return posemb
    if old_size is None:
        hw = int(math.sqrt(num_pos_tokens - num_prefix_tokens))
        old_size = hw, hw
    if num_prefix_tokens:
        posemb_prefix, posemb = posemb[:, :num_prefix_tokens], posemb[:, num_prefix_tokens:]
    else:
        posemb_prefix = None
    embed_dim = posemb.shape[-1]
    orig_dtype = posemb.dtype
    posemb = posemb.float()
    posemb = posemb.reshape(1, old_size[0], old_size[1], -1).permute(0, 3, 1, 2)
    posemb = F.interpolate(posemb, size=new_size, mode=interpolation, antialias=antialias)
    posemb = posemb.permute(0, 2, 3, 1).reshape(1, -1, embed_dim).to(orig_dtype)
    if posemb_prefix is not None:
        posemb = torch.cat([posemb_prefix, posemb], dim=1)
    return posemb


class Attention(nn.Module):
    """vision_transformer.py:145-197 (fused SDPA branch; qk_norm unused by the shipped configs)."""

    def __init__(self, dim, num_heads=8, qkv_bias=False, qk_norm=False, attn_drop=0.0, proj_drop=0.0,
                 norm_layer=nn.LayerNorm, **kwargs):
        super().__init__()
        assert dim % num_heads == 0, 'dim should be divisible by num_heads'
        self.num_heads = num_heads
        self.head_dim = dim // num_heads
        self.scale = self.head_dim ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.q_norm = norm_layer(self.head_dim) if qk_norm else nn.Identity()
        self.k_norm = norm_layer(self.head_dim) if qk_norm else nn.Identity()
        self.attn_drop = nn.Dropout(attn_drop)
        self.proj = nn.Linear(dim, dim)
        self.proj_drop = nn.Dropout(proj_drop)

    def forward(self, x, attn_mask=None):
        B, N, C = x.shape
        qkv = self.qkv(x).reshape(B, N, 3, self.num_heads, self.head_dim).permute(2, 0, 3, 1, 4)
        q, k, v = qkv.unbind(0)
        q, k = self.q_norm(q), self.k_norm(k)
        x = F.scaled_dot_product_attention(q, k, v, dropout_p=self.attn_drop.p if self.training else 0.0,
                                           attn_mask=attn_mask)
        x = x.transpose(1, 2).reshape(B, N, C)
        return self.proj_drop(self.proj(x))


def init_1d_freqs(dim: int, end: int, theta: float = 10000.0):
    """vision_transformer.py:58-79: complex64 [end, dim/2], polar(1, t * theta^(-2k/dim))."""
    freqs = 1.0 / (theta ** (torch.arange(0, dim, 2)[: (dim // 2)].float() / dim))
    t = torch.arange(end, device=freqs.device)
    freqs = torch.outer(t, freqs).float()
    return torch.polar(torch.ones_like(freqs), freqs)


def init_2d_freqs(dim: int, num_heads: int, theta: float = 10.0, rotate: bool = True):
    """vision_transformer.py:82-95: [2, H, dim/2] (fx, fy); one torch.rand(1) angle per head, in head order."""
    freqs_x, freqs_y = [], []
    mag = 1 / (theta ** (torch.arange(0, dim, 4)[: (dim // 4)].float() / dim))
    for _ in range(num_heads):
        angles = torch.rand(1) * 2 * torch.pi if rotate else torch.zeros(1)
        freqs_x.append(torch.cat([mag * torch.cos(angles), mag * torch.cos(torch.pi / 2 + angles)], dim=-1))
        freqs_y.append(torch.cat([mag * torch.sin(angles), mag * torch.sin(torch.pi / 2 + angles)], dim=-1))
    return torch.stack([torch.stack(freqs_x, dim=0), torch.stack(freqs_y, dim=0)], dim=0)


def init_t_xy(end_x: int, end_y: int):
    """vision_transformer.py:98-102: t_x = n mod end_x, t_y = n div end_x (fp32)."""
    t = torch.arange(end_x * end_y, dtype=torch.float32)
    return (t % end_x).float(), torch.div(t, end_x, rounding_mode='floor').float()


def compute_mixed_cis(freqs, t_x, t_y, num_heads: int):
    """vision_transformer.py:105-112: polar(1, t_x fx + t_y fy) -> complex64 [H, N, dim/2], with autocast off."""
    N = t_x.shape[0]
    with torch.autocast(device_type=freqs.device.type, enabled=False):
        freqs_x = (t_x.unsqueeze(-1) @ freqs[0].unsqueeze(-2)).view(N, num_heads, -1).permute(1, 0, 2)
        freqs_y = (t_y.unsqueeze(-1) @ freqs[1].unsqueeze(-2)).view(N, num_heads, -1).permute(1, 0, 2)
        return torch.polar(torch.ones_like(freqs_x), freqs_x + freqs_y)


def apply_rotary_emb(xq, xk, freqs_cis):
    """vision_transformer.py:134-142: q / k [..., T, dim] as dim/2 complex pairs times freqs_cis ([T, dim/2] or
    [H, T, dim/2]) in fp32, returned in the input dtype."""
    xq_ = torch.view_as_complex(xq.float().reshape(*xq.shape[:-1], -1, 2))
    xk_ = torch.view_as_complex(xk.float().reshape(*xk.shape[:-1], -1, 2))
    shape = [1] * (xq_.ndim - freqs_cis.ndim) + list(freqs_cis.shape)
    freqs_cis = freqs_cis.view(*shape)
    return (torch.view_as_real(xq_ * freqs_cis).flatten(3).type_as(xq),
            torch.view_as_real(xk_ * freqs_cis).flatten(3).type_as(xk))


class RoPEAttention(Attention):
    """vision_transformer.py:200-270: Attention with rotary position embeddings on q and k -- 2-D mixed frequencies
    (`freqs`, learnable fp32 [2, H*dim/2]) for the image tokens, a learnable complex64 table (`freqs_1d`, [L, dim/2]) for the
    latent tokens, prefix tokens untouched.  Token order [prefix | image | latent].

    The forward here is the module path (CPU, fp32, autocast dtypes the fused kernels do not cover); vit_ops runs the
    bf16 / fp16 CUDA path on csrc/rope_kernel.cu.  It writes the rotated slices into new tensors instead of into the qkv view
    in place, so its fp32 backward works; the reference's fails there (DESIGN.md section 8).  rope_mixed=False (the axial
    branch) is not reachable from DINOv2Decoder and is refused."""

    def __init__(self, *args, num_prefix_tokens=1, num_latent_tokens=32, num_image_tokens=256, rope_theta=10.0,
                 rope_mixed=True, **kwargs):
        super().__init__(*args, **kwargs)
        if not rope_mixed:
            raise NotImplementedError("RoPEAttention(rope_mixed=False) (axial frequencies) is not reachable from "
                                      "DINOv2Decoder; not built")
        self.rope_mixed = rope_mixed
        self.num_prefix_tokens = num_prefix_tokens
        self.num_latent_tokens = num_latent_tokens
        self.num_image_tokens = num_image_tokens
        self.num_axis_tokens = int(num_image_tokens ** 0.5)
        freqs = init_2d_freqs(dim=self.head_dim, num_heads=self.num_heads, theta=rope_theta, rotate=True).view(2, -1)
        self.freqs = nn.Parameter(freqs, requires_grad=True)
        t_x, t_y = init_t_xy(end_x=self.num_axis_tokens, end_y=self.num_axis_tokens)
        self.register_buffer('freqs_t_x', t_x)
        self.register_buffer('freqs_t_y', t_y)
        self.freqs_1d = nn.Parameter(init_1d_freqs(dim=self.head_dim, end=self.num_latent_tokens), requires_grad=True)

    def forward(self, x, attn_mask=None):
        B, N, C = x.shape
        P, L = self.num_prefix_tokens, self.num_latent_tokens
        qkv = self.qkv(x).reshape(B, N, 3, self.num_heads, C // self.num_heads).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0], qkv[1], qkv[2]
        t_x, t_y = self.freqs_t_x, self.freqs_t_y
        if t_x.shape[0] != N - P - L:                     # :237-240
            side = math.sqrt(N - 1)
            t_x, t_y = init_t_xy(end_x=side, end_y=side)
            t_x, t_y = t_x.to(x.device), t_y.to(x.device)
        freqs_cis = compute_mixed_cis(self.freqs, t_x, t_y, self.num_heads)
        dtype = x.dtype
        with torch.autocast(device_type=x.device.type, enabled=False):
            qi, ki = apply_rotary_emb(q[:, :, P:N - L], k[:, :, P:N - L], freqs_cis)
            ql, kl = apply_rotary_emb(q[:, :, N - L:], k[:, :, N - L:], self.freqs_1d)
            q = torch.cat([q[:, :, :P], qi, ql], dim=2)
            k = torch.cat([k[:, :, :P], ki, kl], dim=2)
        q, k = q.to(dtype), k.to(dtype)
        attn = (q * self.scale) @ k.transpose(-2, -1)          # attn_mask is ignored, as in the reference
        attn = self.attn_drop(attn.softmax(dim=-1))
        x = (attn @ v).transpose(1, 2).reshape(B, N, C)
        return self.proj_drop(self.proj(x))


class LayerScale(nn.Module):
    def __init__(self, dim, init_values=1e-5, inplace=False):
        super().__init__()
        self.inplace = inplace
        self.gamma = nn.Parameter(init_values * torch.ones(dim))

    def forward(self, x):
        return x.mul_(self.gamma) if self.inplace else x * self.gamma


class Block(nn.Module):
    """vision_transformer.py:295-339: pre-LN block with LayerScale + DropPath."""

    def __init__(self, dim, num_heads, mlp_ratio=4.0, qkv_bias=False, qk_norm=False, proj_drop=0.0, attn_drop=0.0,
                 init_values=None, drop_path=0.0, act_layer=nn.GELU, norm_layer=nn.LayerNorm, mlp_layer=Mlp,
                 attn_layer=Attention):
        super().__init__()
        self.norm1 = norm_layer(dim)
        self.attn = attn_layer(dim, num_heads=num_heads, qkv_bias=qkv_bias, qk_norm=qk_norm, attn_drop=attn_drop,
                               proj_drop=proj_drop, norm_layer=norm_layer)
        self.ls1 = LayerScale(dim, init_values=init_values) if init_values else nn.Identity()
        self.drop_path1 = DropPath(drop_path) if drop_path > 0.0 else nn.Identity()
        self.norm2 = norm_layer(dim)
        self.mlp = mlp_layer(in_features=dim, hidden_features=int(dim * mlp_ratio), act_layer=act_layer, drop=proj_drop)
        self.ls2 = LayerScale(dim, init_values=init_values) if init_values else nn.Identity()
        self.drop_path2 = DropPath(drop_path) if drop_path > 0.0 else nn.Identity()

    def forward(self, x, attn_mask=None):
        x = x + self.drop_path1(self.ls1(self.attn(self.norm1(x), attn_mask)))
        x = x + self.drop_path2(self.ls2(self.mlp(self.norm2(x))))
        return x


class VisionTransformer(nn.Module):
    """vision_transformer.py:587-756 restricted to what DINOv2Encoder/Decoder touch."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, num_classes=0, embed_dim=768, depth=12, num_heads=12,
                 mlp_ratio=4.0, qkv_bias=True, init_values=None, class_token=True, no_embed_class=False, reg_tokens=0,
                 pre_norm=False, drop_path_rate=0.0, attn_layer=Attention, num_latent_tokens=32, global_pool='token',
                 norm_eps=1e-6, mlp_layer=Mlp, act_layer=nn.GELU, **unused):
        super().__init__()
        norm_layer = partial(nn.LayerNorm, eps=norm_eps)     # timm: 1e-6 for the DINOv2 / plain ViTs, 1e-5 for the CLIP variants
        self.num_classes = num_classes
        self.global_pool = global_pool
        self.num_features = self.embed_dim = embed_dim
        self.num_prefix_tokens = (1 if class_token else 0) + reg_tokens
        self.num_reg_tokens = reg_tokens
        self.has_class_token = class_token
        self.no_embed_class = no_embed_class
        self.dynamic_img_size = False
        self.patch_embed = PatchEmbed(img_size=img_size, patch_size=patch_size, in_chans=in_chans, embed_dim=embed_dim,
                                      bias=not pre_norm)
        num_patches = self.patch_embed.num_patches
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim)) if class_token else None
        self.reg_token = nn.Parameter(torch.zeros(1, reg_tokens, embed_dim)) if reg_tokens else None
        embed_len = num_patches if no_embed_class else num_patches + self.num_prefix_tokens
        self.pos_embed = nn.Parameter(torch.randn(1, embed_len, embed_dim) * .02)
        self.pos_drop = nn.Dropout(p=0.0)
        self.patch_drop = nn.Identity()
        self.norm_pre = norm_layer(embed_dim) if pre_norm else nn.Identity()
        dpr = [x.item() for x in torch.linspace(0, drop_path_rate, depth)]
        self.blocks = nn.Sequential(*[
            Block(dim=embed_dim, num_heads=num_heads, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias, init_values=init_values,
                  drop_path=dpr[i], norm_layer=norm_layer, mlp_layer=mlp_layer, act_layer=act_layer,
                  attn_layer=partial(attn_layer, num_prefix_tokens=self.num_prefix_tokens,        # :728-731
                                     num_latent_tokens=num_latent_tokens, patch_size=patch_size))
            for i in range(depth)])
        self.norm = norm_layer(embed_dim)
        self.fc_norm = nn.Identity()
        self.head_drop = nn.Dropout(0.0)
        self.head = nn.Linear(embed_dim, num_classes) if num_classes > 0 else nn.Identity()
        self.init_weights()

    def init_weights(self):
        trunc_normal_(self.pos_embed, std=.02)
        if self.cls_token is not None:
            nn.init.normal_(self.cls_token, std=1e-6)
        for m in self.modules():
            if isinstance(m, nn.Linear):
                trunc_normal_(m.weight, std=.02)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)

    def no_weight_decay(self):
        return {'pos_embed', 'cls_token', 'dist_token'}

    def _pos_embed(self, x):
        """vision_transformer.py:814-848."""
        if len(x.shape) == 4:
            B, H, W, C = x.shape
            pos_embed = resample_abs_pos_embed(self.pos_embed, (H, W),
                                               num_prefix_tokens=0 if self.no_embed_class else self.num_prefix_tokens)
            x = x.view(B, -1, C)
        else:
            pos_embed = self.pos_embed
        to_cat = []
        if self.cls_token is not None:
            to_cat.append(self.cls_token.expand(x.shape[0], -1, -1))
        if self.reg_token is not None:
            to_cat.append(self.reg_token.expand(x.shape[0], -1, -1))
        if self.no_embed_class:
            x = x + pos_embed
            if to_cat:
                x = torch.cat(to_cat + [x], dim=1)
        else:
            if to_cat:
                x = torch.cat(to_cat + [x], dim=1)
            x = x + pos_embed
        return self.pos_drop(x)

    def forward_features(self, x):
        if frozen_path_ok(self, x):
            return frozen_forward(self, x)      # a frozen teacher under bf16 / fp16 autocast: the fused kernels
        x = self.patch_embed(x)
        x = self._pos_embed(x)
        x = self.patch_drop(x)
        x = self.norm_pre(x)
        x = self.blocks(x)
        return self.norm(x)

    def forward_head(self, x, pre_logits: bool = False):
        if self.global_pool == 'token':
            x = x[:, 0]
        elif self.global_pool == 'avg':
            x = x[:, self.num_prefix_tokens:].mean(dim=1)
        x = self.fc_norm(x)
        x = self.head_drop(x)
        return x if pre_logits else self.head(x)

    def forward(self, x):
        if self.global_pool == 'token' and frozen_path_ok(self, x):
            # only row 0 of the final norm is read: the last block runs its attention, proj and MLP on the class rows
            return self.head(self.head_drop(self.fc_norm(frozen_forward(self, x, cls_only=True))))
        return self.forward_head(self.forward_features(x))


# name -> architecture (vision_transformer.py:2893-2935 and the CLIP entry used by `detail_guide`)
_ARCH = {
    'vit_small_patch14_dinov2.lvd142m': dict(patch_size=14, embed_dim=384, depth=12, num_heads=6, init_values=1e-5, img_size=518),
    'vit_base_patch14_dinov2.lvd142m': dict(patch_size=14, embed_dim=768, depth=12, num_heads=12, init_values=1e-5, img_size=518),
    'vit_large_patch14_dinov2.lvd142m': dict(patch_size=14, embed_dim=1024, depth=24, num_heads=16, init_values=1e-5, img_size=518),
    # hidden_features = int(1536 * 5.33334) = 8192: the packed [gate | up] width of fc1 (fc2 takes 4096)
    'vit_giant_patch14_dinov2.lvd142m': dict(patch_size=14, embed_dim=1536, depth=40, num_heads=24, init_values=1e-5,
                                             mlp_ratio=2.66667 * 2, mlp_layer=GluMlp, act_layer=nn.SiLU, img_size=518),
    # four register tokens; pos_embed covers the patch tokens only (:2942-2995)
    'vit_small_patch14_reg4_dinov2.lvd142m': dict(patch_size=14, embed_dim=384, depth=12, num_heads=6, init_values=1e-5,
                                                  reg_tokens=4, no_embed_class=True, img_size=518),
    'vit_base_patch14_reg4_dinov2.lvd142m': dict(patch_size=14, embed_dim=768, depth=12, num_heads=12, init_values=1e-5,
                                                 reg_tokens=4, no_embed_class=True, img_size=518),
    'vit_large_patch14_reg4_dinov2.lvd142m': dict(patch_size=14, embed_dim=1024, depth=24, num_heads=16, init_values=1e-5,
                                                  reg_tokens=4, no_embed_class=True, img_size=518),
    'vit_giant_patch14_reg4_dinov2.lvd142m': dict(patch_size=14, embed_dim=1536, depth=40, num_heads=24, init_values=1e-5,
                                                  mlp_ratio=2.66667 * 2, mlp_layer=GluMlp, act_layer=nn.SiLU, reg_tokens=4,
                                                  no_embed_class=True, img_size=518),
    'vit_base_patch16_clip_224.openai': dict(patch_size=16, embed_dim=768, depth=12, num_heads=12, pre_norm=True, img_size=224),
}


# timm builds its CLIP variants with norm_layer=nn.LayerNorm (eps 1e-5); the DINOv2 ones with eps 1e-6
_NORM_EPS = {'vit_base_patch16_clip_224.openai': 1e-5}


def _resample_checkpoint(state, model):
    """timm's checkpoint_filter_fn for the two tensors whose shape depends on (img_size, patch_size):
    pos_embed (bicubic, antialias, prefix tokens kept) and patch_embed.proj.weight (bicubic resize of the kernel)."""
    out = dict(state)
    pe = out.get('pos_embed')
    if pe is not None and pe.shape != model.pos_embed.shape:
        npt = 0 if model.no_embed_class else model.num_prefix_tokens
        out['pos_embed'] = resample_abs_pos_embed(pe, model.patch_embed.grid_size, num_prefix_tokens=npt)
    w = out.get('patch_embed.proj.weight')
    if w is not None and w.shape != model.patch_embed.proj.weight.shape:
        out['patch_embed.proj.weight'] = F.interpolate(w.float(), size=model.patch_embed.proj.weight.shape[-2:],
                                                       mode='bicubic', antialias=True, align_corners=False).to(w.dtype)
    return out


def create_model(model_name: str, pretrained: bool = False, **kwargs) -> VisionTransformer:
    """stand-in for timm.models.create_model for the names the reference uses.  There is no network here:
    `pretrained=True` loads a LOCAL timm-format checkpoint named by the environment variable
    XQ_TIMM_CKPT_<NAME> (NAME = model name upper-cased, non-alphanumerics -> '_'; e.g.
    XQ_TIMM_CKPT_VIT_BASE_PATCH14_DINOV2_LVD142M), resampling pos_embed / patch_embed to the requested geometry the way
    timm's checkpoint filter does (37x37 -> 16x16, patch 14 -> 16 for the reference's 256px / patch-16 models).  Without
    that file the weights stay at their random initialisation and this is said LOUDLY (warning, or an exception with
    XQ_REQUIRE_PRETRAINED=1): a frozen `semantic_guide` / `detail_guide` teacher on random weights regresses noise --
    configure those guides as 'none' unless their checkpoints are present."""
    import os
    import re
    import warnings
    if model_name not in _ARCH:
        raise RuntimeError(f"Unknown model ({model_name})")
    args = dict(_ARCH[model_name])
    args.update(kwargs)
    if model_name in _NORM_EPS:
        args.setdefault('norm_eps', _NORM_EPS[model_name])
    model = VisionTransformer(**args)
    model.pretrained_requested = bool(pretrained)
    model.pretrained_loaded = False
    if pretrained:
        env = "XQ_TIMM_CKPT_" + re.sub(r"[^A-Za-z0-9]", "_", model_name).upper()
        path = os.environ.get(env, "")
        if path and os.path.exists(path):
            state = torch.load(path, map_location="cpu")
            state = state.get("state_dict", state.get("model", state))
            res = model.load_state_dict(_resample_checkpoint(state, model), strict=False)
            bad = [k for k in res.missing_keys if not k.startswith('head')]
            if bad:
                raise RuntimeError(f"{path}: not a timm checkpoint of {model_name} (missing {bad[:4]})")
            model.pretrained_loaded = True
        else:
            msg = (f"create_model({model_name!r}, pretrained=True): no local checkpoint ({env} is unset or missing); "
                   "the model keeps its RANDOM initialisation")
            if os.environ.get("XQ_REQUIRE_PRETRAINED", "0") == "1":
                raise RuntimeError(msg)
            warnings.warn(msg)
    return model
