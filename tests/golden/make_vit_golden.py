"""ViT encoder / decoder goldens from the REFERENCE'S OWN modules (CPU, fp32).

    python tests/golden/make_vit_golden.py        # writes tests/golden/vit_*.npz   (build container only)

What runs is the reference's code: tokenizer/tokenizer_image/xqgan_model.py (VQModel.encode / decode :241-261),
dino_enc/dinov2.py (DINOv2Encoder :18-198, DINOv2Decoder :201-365) and the VENDORED
dino_enc/vision_transformer.py (Attention :145, LayerScale :280, Block :295, VisionTransformer :587, _pos_embed :814,
the vit_*_patch14_dinov2 entry points :2895+).  Only the pieces that live in the un-vendored timm==1.0.9
(environment.yml:102, not installed here) are functional stand-ins written below from timm's published semantics:
    timm.layers.PatchEmbed, Mlp, DropPath, resample_abs_pos_embed, trunc_normal_, get_norm_layer/get_act_layer,
    timm.models.create_model / registry / build_model_with_cfg (construct the class, no pretrained weights)
so parity of the ViT stacks is pinned to the reference except for those four layers.

Weights: tests/golden/vit_det_init.py (seeded per parameter NAME; identical on both sides).  Outputs are stored
subsampled (every 4th token / pixel) plus full-tensor sums, which keeps each file ~150 KB.
"""
import math
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from vit_det_init import apply_det_init, golden_inputs  # noqa: E402

REF = os.environ.get("XQ_REFERENCE", "")    # a checkout of lxa9867/ImageFolder (the reference)


# ---- functional stand-ins for timm (test infrastructure) -----------------------------------------------------------
class PatchEmbed(nn.Module):
    """timm.layers.PatchEmbed: Conv2d(kernel = stride = patch) -> flatten(2).transpose(1, 2) -> norm."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768, norm_layer=None, flatten=True,
                 output_fmt=None, bias=True, strict_img_size=True, dynamic_img_pad=False):
        super().__init__()
        self.patch_size = (patch_size, patch_size) if isinstance(patch_size, int) else tuple(patch_size)
        self.img_size = (img_size, img_size) if isinstance(img_size, int) else tuple(img_size)
        self.grid_size = tuple(s // p for s, p in zip(self.img_size, self.patch_size))
        self.num_patches = self.grid_size[0] * self.grid_size[1]
        self.flatten = flatten
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=self.patch_size, stride=self.patch_size, bias=bias)
        self.norm = norm_layer(embed_dim) if norm_layer else nn.Identity()

    def forward(self, x):
        x = self.proj(x)
        if self.flatten:
            x = x.flatten(2).transpose(1, 2)
        return self.norm(x)


class Mlp(nn.Module):
    """timm.layers.Mlp: fc1 -> act -> drop1 -> norm -> fc2 -> drop2."""

    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, norm_layer=None, bias=True,
                 drop=0.0, use_conv=False):
        super().__init__()
        out_features = out_features or in_features
        hidden_features = hidden_features or in_features
        self.fc1 = nn.Linear(in_features, hidden_features, bias=bias)
        self.act = act_layer()
        self.drop1 = nn.Dropout(drop)
        self.norm = norm_layer(hidden_features) if norm_layer is not None else nn.Identity()
        self.fc2 = nn.Linear(hidden_features, out_features, bias=bias)
        self.drop2 = nn.Dropout(drop)

    def forward(self, x):
        return self.drop2(self.fc2(self.norm(self.drop1(self.act(self.fc1(x))))))


class DropPath(nn.Module):
    def __init__(self, drop_prob=0.0, scale_by_keep=True):
        super().__init__()
        self.drop_prob, self.scale_by_keep = drop_prob, scale_by_keep

    def forward(self, x):
        if self.drop_prob == 0.0 or not self.training:
            return x
        keep = 1 - self.drop_prob
        mask = x.new_empty((x.shape[0],) + (1,) * (x.ndim - 1)).bernoulli_(keep)
        if keep > 0.0 and self.scale_by_keep:
            mask.div_(keep)
        return x * mask


def resample_abs_pos_embed(posemb, new_size, old_size=None, num_prefix_tokens=1, interpolation="bicubic", antialias=True,
                           verbose=False):
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
        posemb_prefix, posemb = None, posemb
    embed_dim = posemb.shape[-1]
    orig_dtype = posemb.dtype
    posemb = posemb.float().reshape(1, old_size[0], old_size[1], -1).permute(0, 3, 1, 2)
    posemb = F.interpolate(posemb, size=new_size, mode=interpolation, antialias=antialias)
    posemb = posemb.permute(0, 2, 3, 1).reshape(1, -1, embed_dim).to(orig_dtype)
    if posemb_prefix is not None:
        posemb = torch.cat([posemb_prefix, posemb], dim=1)
    return posemb


def named_apply(fn, module, name="", depth_first=True, include_root=False):
    if not depth_first and include_root:
        fn(module=module, name=name)
    for child_name, child in module.named_children():
        child_name = ".".join((name, child_name)) if name else child_name
        named_apply(fn=fn, module=child, name=child_name, depth_first=depth_first, include_root=True)
    if depth_first and include_root:
        fn(module=module, name=name)
    return module


_REGISTRY = {}


def register_model(fn):
    _REGISTRY[fn.__name__] = fn
    return fn


def create_model(model_name, pretrained=False, **kwargs):
    return _REGISTRY[model_name.split(".")[0]](pretrained=False, **kwargs)


def build_model_with_cfg(model_cls, variant, pretrained, **kwargs):
    for k in ("pretrained_filter_fn", "pretrained_strict", "feature_cfg", "pretrained_cfg", "pretrained_cfg_overlay"):
        kwargs.pop(k, None)
    return model_cls(**kwargs)


def install_stand_ins():
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    const = (0.5, 0.5, 0.5)
    ident = lambda *a, **k: None   # noqa: E731
    mod("timm")
    mod("timm.data", IMAGENET_DEFAULT_MEAN=const, IMAGENET_DEFAULT_STD=const, IMAGENET_INCEPTION_MEAN=const,
        IMAGENET_INCEPTION_STD=const, OPENAI_CLIP_MEAN=const, OPENAI_CLIP_STD=const)
    mod("timm.layers", PatchEmbed=PatchEmbed, Mlp=Mlp, DropPath=DropPath, AttentionPoolLatent=None, RmsNorm=None,
        PatchDropout=None, SwiGLUPacked=None, trunc_normal_=nn.init.trunc_normal_, lecun_normal_=ident,
        resample_patch_embed=ident, resample_abs_pos_embed=resample_abs_pos_embed, use_fused_attn=lambda *a, **k: True,
        get_act_layer=lambda x: x, get_norm_layer=lambda x: x, LayerType=object)
    mod("timm.models", create_model=create_model, safe_model_name=lambda s: s)
    mod("timm.models._builder", build_model_with_cfg=build_model_with_cfg)
    mod("timm.models._features", feature_take_indices=ident)
    mod("timm.models._manipulate", named_apply=named_apply, checkpoint_seq=ident, adapt_input_conv=ident)
    mod("timm.models._registry", generate_default_cfgs=lambda d: d, register_model=register_model,
        register_model_deprecations=ident)
    mod("peft")
    mod("webdataset")


def build_reference(cfg):
    sys.path.insert(0, REF)
    install_stand_ins()
    import torch.distributed as tdist
    if not tdist.is_initialized():
        tdist.init_process_group("gloo", init_method="tcp://127.0.0.1:29541", rank=0, world_size=1)
    from tokenizer.tokenizer_image.xqgan_model import ModelArgs, VQModel
    args = ModelArgs(**cfg)
    torch.manual_seed(0)
    model = VQModel(args).eval()
    apply_det_init(model)
    return model


# the shipped configs (configs/*.yaml; num_latent_tokens is PER product-quant branch) at ViT-S width; sequence lengths: encoder / decoder
CASES = {
    "vit_vq": dict(codebook_size=8192, codebook_embed_dim=32, v_patch_nums=[16], num_latent_tokens=256, abs_pos_embed=True,
                   product_quant=1),                                                   # S = 513 / 514
    "vit_vp2": dict(codebook_size=16384, codebook_embed_dim=32, v_patch_nums=[16], num_latent_tokens=256, abs_pos_embed=True,
                    product_quant=2),                                                  # S = 769 / 514
    "vit_ms": dict(codebook_size=4096, codebook_embed_dim=32, v_patch_nums=[1, 1, 2, 3, 3, 4, 5, 6, 8, 11],
                   num_latent_tokens=121, abs_pos_embed=True, product_quant=2, codebook_drop=0.1),   # S = 499 / 379
    "vit_relpos": dict(codebook_size=4096, codebook_embed_dim=32, v_patch_nums=[16], num_latent_tokens=256,
                       abs_pos_embed=False, product_quant=1),                          # latent_pos_embed path, S = 513 / 513
}
COMMON = dict(enc_type="dinov2", dec_type="dinov2", semantic_guide="none", detail_guide="none",
              encoder_model="vit_small_patch14_dinov2.lvd142m", decoder_model="vit_small_patch14_dinov2.lvd142m")


def main():
    for name, c in CASES.items():
        cfg = dict(COMMON, **c)
        model = build_reference(cfg)
        pq = cfg["product_quant"]
        side = int(math.sqrt(model.config.num_latent_tokens // pq))   # VQModel.__init__ scales num_latent_tokens by PQ (:85)
        x, q = golden_inputs(cfg["codebook_embed_dim"] * pq, side)
        with torch.no_grad():
            tok = model.encoder(x)               # [1, L, D]   dinov2.py:146-198
            h = model.encode(x)                  # quant_conv on top  xqgan_model.py:241-254
            dec = model.decode(q)                # post_quant_conv -> DINOv2Decoder -> ToPixel   :256-261
        np.savez_compressed(os.path.join(HERE, name + ".npz"), cfg_json=np.array(repr(cfg)),
                            x_sum=np.float64(x.double().sum()), q_sum=np.float64(q.double().sum()), q_shape=np.array(q.shape),
                            tok_sub=tok[:, ::4].numpy(), tok_sum=np.float64(tok.double().sum()), tok_abs=np.float64(tok.double().abs().sum()),
                            h_sub=h.flatten(2)[:, :, ::4].numpy(), h_shape=np.array(h.shape), h_sum=np.float64(h.double().sum()),
                            dec_sub=dec[:, :, ::4, ::4].numpy(), dec_sum=np.float64(dec.double().sum()),
                            dec_abs=np.float64(dec.double().abs().sum()),
                            enc_S=model.encoder.num_img_tokens + model.encoder.num_prefix_tokens + model.encoder.num_latent_tokens)
        print(name, "tokens", tuple(tok.shape), "h", tuple(h.shape), "dec", tuple(dec.shape), "tok |mean|",
              float(tok.abs().mean()), "dec |mean|", float(dec.abs().mean()))


if __name__ == "__main__":
    main()
