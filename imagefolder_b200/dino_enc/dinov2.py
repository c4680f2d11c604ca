"""DINOv2Encoder / DINOv2Decoder -- drop-in for tokenizer/tokenizer_image/dino_enc/dinov2.py
(:18 and :201): ViT backbone + learnable latent tokens, level embedding, mask tokens, ToPixel.

DINOv2Decoder(use_rope=True) builds its blocks with RoPEAttention (rotary q / k, no latent positional embedding).
tuning_method 'full', 'frozen', 'lora' and 'lora_unfreeze_patch_embed' are built, in the constructors and in `finetine`; the
LoRA ones wrap the ViT with lora.py, a restatement of the peft 0.13.0 calls the reference makes.  'lat_lora' is not built.
Sub-module / parameter names match the reference so released checkpoints load unchanged.

Both classes split their forward into (1) the token ASSEMBLY -- everything between the batch-dependent rows (patch
tokens / quantised latents) and the first transformer block: prefix tokens, positional embeddings, latent or mask
tokens, level embedding -- and (2) the blocks.  (1) is affine in the batch-dependent rows, so under bf16 autocast it
runs as `table[t] + src[b, t - t0]` in one fused pass (vit_ops.assemble_tokens, which checks that property once per
module); (2) runs on the fused ViT glue (vit_ops.run_blocks).
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from ..vit_ops import assemble_tokens, patch_embed, run_blocks
from .lora import LoraConfig, get_peft_model
from .to_pixel import ToPixel
from .vision_transformer import Attention, RoPEAttention, create_model, trunc_normal_

_NAMES = ['vit_small_patch14_dinov2.lvd142m', 'vit_base_patch14_dinov2.lvd142m', 'vit_large_patch14_dinov2.lvd142m',
          'vit_giant_patch14_dinov2.lvd142m', 'vit_small_patch14_reg4_dinov2.lvd142m', 'vit_base_patch14_reg4_dinov2.lvd142m',
          'vit_large_patch14_reg4_dinov2.lvd142m', 'vit_giant_patch14_reg4_dinov2.lvd142m']
# modules_to_save of the reference's two LoRA methods (dinov2.py:57, 63); both adapt exactly the MLP Linears
_LORA_SAVE = {'lora': ['norm'], 'lora_unfreeze_patch_embed': ['patch_embed.proj', 'patch_embed.norm', 'norm']}
_LORA_TARGETS = r".*\.mlp\.fc\d"
_LAT_LORA_MSG = ("tuning_method='lat_lora' needs models.peft_models.lora.LatentLoRALinear, which the reference imports "
                 "(dinov2.py:69, 132) but does not contain; not built")


def _autocast_off(x):
    return torch.autocast(device_type=x.device.type, enabled=False)


def _main_dtype(x):
    temp = x.new_ones(8, 8)
    return torch.matmul(temp, temp).dtype


def _freeze(module):
    for param in module.parameters():
        param.requires_grad = False


def _tuned(model, tuning_method, tuning_kwargs):
    """the backbone for `tuning_method` (dinov2.py:51-80 / 114-142 / 241-253 / 291-304): `model` itself for 'full', with
    frozen parameters for 'frozen', wrapped with rank-r adapters on every mlp.fc1 / mlp.fc2 for the LoRA methods"""
    if tuning_method == 'full':
        return model
    if tuning_method == 'frozen':
        _freeze(model)
        return model
    if tuning_method in _LORA_SAVE:
        peft_model = get_peft_model(model, LoraConfig(target_modules=_LORA_TARGETS, modules_to_save=_LORA_SAVE[tuning_method],
                                                      **tuning_kwargs))
        peft_model.print_trainable_parameters()
        return peft_model
    if tuning_method == 'lat_lora':
        raise NotImplementedError(_LAT_LORA_MSG)
    raise NotImplementedError(f"tuning_method={tuning_method!r} is not one of the reference's; not built")


def _adopt_backbone(owner, model, tuning_method, tuning_kwargs):
    """`self.model` = the backbone tuned by `tuning_method` (dinov2.py:51-80 / 241-253)."""
    owner.model = _tuned(model, tuning_method, tuning_kwargs)
    owner.embed_dim = model.embed_dim
    owner.num_img_tokens = model.patch_embed.num_patches
    owner.num_prefix_tokens = model.num_prefix_tokens


def _check_prefix(model_name, abs_pos_embed):
    """abs_pos_embed sizes the level-embedding index row for ONE prefix token (dinov2.py:91, 98, 266); the reference's
    forward then fails on a shape mismatch for the four-register backbones (five prefix tokens).  Refused here, at
    construction, with the reason (DESIGN.md section 8)."""
    if abs_pos_embed and '_reg4_' in model_name:
        raise ValueError(f"{model_name} has 5 prefix tokens (cls + 4 registers), but abs_pos_embed=True sizes the level "
                         "embedding for 1 (the reference's lvl1LC, dinov2.py:91/266) and fails in its forward; use "
                         "abs_pos_embed=False with the reg4 backbones")


def _level_embedding(owner, n_levels, dim, segment_lengths):
    """`lvl_embed` (trunc-normal, std sqrt(1/3D)) + the `lvl1LC` index row: segment i of the sequence gets level i."""
    owner.lvl_embed = nn.Embedding(n_levels, dim)
    nn.init.trunc_normal_(owner.lvl_embed.weight.data, mean=0, std=math.sqrt(1 / dim / 3))
    idx = torch.cat([torch.full((n,), lvl) for lvl, n in enumerate(segment_lengths)])
    owner.register_buffer('lvl1LC', idx.view(1, -1))


def _square_side(n):
    side = int(math.sqrt(n))
    assert side * side == n
    return side


def _static_sequence(vit, training):
    """nothing stochastic between the batch-dependent rows and the first block (patch_drop / pos_drop inactive)"""
    return (isinstance(vit.patch_drop, nn.Identity) and not vit.no_embed_class
            and (not training or getattr(vit.pos_drop, "p", 0.0) == 0.0))


class _Tunable:
    def finetine(self, tuning_method, tuning_kwargs={'r': 8}):            # (sic) the reference's spelling
        self.model = _tuned(self.model, tuning_method, tuning_kwargs)


class DINOv2Encoder(_Tunable, nn.Module):
    def __init__(self, in_channels=3, num_latent_tokens=32, use_attn_mask=False,
                 model_name='vit_small_patch14_dinov2.lvd142m',
                 model_kwargs={'img_size': 224, 'patch_size': 14, 'drop_path_rate': 0.0, },
                 pretrained=True, tuning_method='lora', tuning_kwargs={'r': 8}, abs_pos_embed=False, product_quant=1):
        super().__init__()
        assert model_name in _NAMES, f"{model_name} not found"
        _check_prefix(model_name, abs_pos_embed and bool(num_latent_tokens))
        self.num_latent_tokens, self.use_attn_mask = num_latent_tokens, use_attn_mask
        self.product_quant, self.abs_pos_embed = product_quant, abs_pos_embed
        _adopt_backbone(self, create_model(model_name, pretrained=pretrained, **model_kwargs), tuning_method, tuning_kwargs)
        if not num_latent_tokens:
            return
        D, L = self.embed_dim, num_latent_tokens
        self.latent_tokens = nn.Parameter(torch.zeros(1, L, D))
        nn.init.normal_(self.latent_tokens, std=1e-6)
        if abs_pos_embed:
            # level 0 = [cls | image tokens] -- the reference sizes it as patch_size^2 + 1 (dinov2.py:72,80), i.e. it assumes
            # a 16 x 16 token grid for patch 16 -- then one level per product-quantisation branch
            n_img = model_kwargs['patch_size'] ** 2 + 1
            _level_embedding(self, 1 + product_quant, D, [n_img] + [L // product_quant] * product_quant)
        else:
            self.latent_pos_embed = nn.Parameter(torch.zeros(1, L, D))
            trunc_normal_(self.latent_pos_embed, std=.02)
        if use_attn_mask:                        # image tokens must not look at the latent tokens (dinov2.py:95-101)
            n_front = self.num_prefix_tokens + self.num_img_tokens
            mask = torch.zeros(n_front + L, n_front + L)
            mask[:n_front, -L:] = -torch.inf
            self.register_buffer('attn_mask', mask[None, None])

    def no_weight_decay(self):
        return ['model.pos_embed', 'model.cls_token', 'model.dist_token', 'latent_tokens', 'latent_pos_embed']

    def _latent_rows(self, batch):
        """the latent tokens with their positional term: 2-D pos-embed resampled to each branch's grid when abs_pos_embed
        (the cls row that _pos_embed prepends is dropped, dinov2.py:160-166), else the learned latent_pos_embed"""
        z = self.latent_tokens.expand(batch, -1, -1)
        if not self.abs_pos_embed:
            return [z + self.latent_pos_embed]
        side = _square_side(self.num_latent_tokens // self.product_quant)
        grids = z.view(batch, self.product_quant * side, side, -1).chunk(chunks=self.product_quant, dim=1)
        return [self.model._pos_embed(g)[:, 1:] for g in grids]

    def _assemble(self, x):
        """dinov2.py:151-170.  x: patch tokens [B, N, D] -> fp32 [B, prefix + N + L, D]."""
        with _autocast_off(x):
            x = self.model.patch_drop(self.model._pos_embed(x))
            if self.num_latent_tokens:
                x = torch.cat([x] + self._latent_rows(x.size(0)), dim=1)
                if self.abs_pos_embed:
                    x += self.lvl_embed(self.lvl1LC.expand(x.size(0), -1))
        return x

    def forward(self, x, masks=None):
        """dinov2.py:146-198 -> [B, num_latent_tokens, D]"""
        x = patch_embed(self.model.patch_embed, x)
        if _static_sequence(self.model, self.training):
            x = assemble_tokens(self, self._assemble, x, self.num_prefix_tokens)
        else:
            x = self._assemble(x)
        # norm_pre -> blocks -> norm (dinov2.py:176-190); fused CUDA glue under bf16 autocast
        x = run_blocks(self.model, x, self.attn_mask if self.use_attn_mask else None)
        return x[:, -self.num_latent_tokens:] if self.num_latent_tokens else x[:, self.num_prefix_tokens:]


class DINOv2Decoder(_Tunable, nn.Module):
    def __init__(self, in_channels=3, model_name='vit_small_patch14_dinov2.lvd142m',
                 model_kwargs={'img_size': 224, 'patch_size': 14, 'drop_path_rate': 0.0}, pretrained=True,
                 tuning_method='lora', tuning_kwargs={'r': 8}, num_latent_tokens=32, to_pixel='linear', use_rope=False,
                 cond_latent=False, abs_pos_embed=False):
        super().__init__()
        assert model_name in _NAMES
        if use_rope and abs_pos_embed:
            # the reference builds no level embedding with use_rope (dinov2.py:264) but its forward still adds one (:342)
            raise ValueError("use_rope=True with abs_pos_embed=True: the reference's forward adds lvl_embed[lvl1LC], which "
                             "it does not create for use_rope, and fails; use abs_pos_embed=False with use_rope")
        _check_prefix(model_name, abs_pos_embed)
        if cond_latent:
            raise NotImplementedError("cond_latent=True is not selected by any shipped config; not built")
        self.use_rope, self.cond_latent = use_rope, cond_latent
        self.num_latent_tokens, self.abs_pos_embed = num_latent_tokens, abs_pos_embed
        vit_kwargs = dict(model_kwargs, num_latent_tokens=num_latent_tokens,
                          attn_layer=RoPEAttention if use_rope else Attention)
        model = create_model(model_name, pretrained=pretrained, **vit_kwargs)
        # the decoder never embeds pixels: drop the unused projection so that it is neither trained nor checkpointed (before
        # any LoRA wrapping, so that a saved copy of patch_embed.proj holds no parameters either)
        del model.patch_embed.proj.bias
        del model.patch_embed.proj.weight
        _adopt_backbone(self, model, tuning_method, tuning_kwargs)
        D = self.embed_dim
        self.mask_token = nn.Parameter(torch.zeros(1, 1, D))
        nn.init.normal_(self.mask_token, std=1e-6)
        if use_rope:
            pass                                 # positions enter through the rotary embedding only (dinov2.py:264)
        elif abs_pos_embed:
            # level 0 = [cls | mask tokens], level 1 = the latents WITH the cls slot _pos_embed gives them (dinov2.py:266-272)
            _level_embedding(self, 2, D, [model_kwargs['patch_size'] ** 2 + 1, num_latent_tokens + 1])
        else:
            self.latent_pos_embed = nn.Parameter(torch.zeros(1, num_latent_tokens, D))
            trunc_normal_(self.latent_pos_embed, std=.02)
        self.to_pixel = ToPixel(to_pixel=to_pixel, img_size=model_kwargs['img_size'], in_channels=in_channels, in_dim=D,
                                patch_size=model_kwargs['patch_size'])

    def no_weight_decay(self):
        return ['model.pos_embed', 'model.cls_token', 'model.dist_token', 'mask_token', 'latent_pos_embed']

    @property
    def last_layer(self):
        return self.to_pixel.model.weight

    def _assemble(self, z):
        """dinov2.py:318-344.  z: latents [B, L, D] -> fp32 [B, prefix + N_img + (prefix if abs_pos_embed) + L, D]."""
        masks = self.mask_token.expand(z.size(0), self.num_img_tokens, -1)
        if self.use_rope:                        # prefix tokens, mask tokens and latents, no positional terms (:336-344)
            with _autocast_off(masks):
                vit = self.model
                prefix = [t.expand(z.size(0), -1, -1) for t in (vit.cls_token, vit.reg_token) if t is not None]
                return torch.cat([vit.patch_drop(torch.cat(prefix + [masks], dim=1)), z.float()], dim=1)
        with _autocast_off(masks):
            front = self.model._pos_embed(masks)
            if self.abs_pos_embed:
                side = _square_side(self.num_latent_tokens)
                back = self.model._pos_embed(z.view(z.size(0), side, side, -1))   # keeps its cls slot (L + 1 rows), :330
            else:
                back = z + self.latent_pos_embed
            x = torch.cat([self.model.patch_drop(front), back], dim=1)
            if self.abs_pos_embed:
                x += self.lvl_embed(self.lvl1LC.expand(x.size(0), -1))
        return x

    def forward(self, z):
        """dinov2.py:313-365: z [B, L, D] -> image [B, 3, H, W]"""
        if _static_sequence(self.model, self.training):
            n_front = self.num_prefix_tokens + self.num_img_tokens
            t0 = n_front + (self.num_prefix_tokens if self.abs_pos_embed else 0)      # where the latent rows start
            x = assemble_tokens(self, self._assemble, z, t0)
        else:
            x = self._assemble(z)
        x = run_blocks(self.model, x)
        return self.to_pixel(x[:, self.num_prefix_tokens:self.num_prefix_tokens + self.num_img_tokens])
