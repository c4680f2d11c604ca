"""CPU ORACLE for the encode -> quantize -> decode path (TEST INFRASTRUCTURE ONLY).

A plain-PyTorch fp32 restatement (floating-point kernels keep a torch fp32 reference) of
  DINOv2Encoder.forward   tokenizer/tokenizer_image/dino_enc/dinov2.py:146-198
  DINOv2Decoder.forward   dinov2.py:313-365
  Block / Attention       dino_enc/vision_transformer.py:145-197, 295-339   (explicit softmax(QK^T)V)
  _pos_embed              vision_transformer.py:814-848
  ToPixel                 dino_enc/to_pixel.py:70-86
  VQModel.encode/decode/forward   tokenizer/tokenizer_image/xqgan_model.py:241-301
written functionally over a state_dict (the weights are an INPUT to parity), with the quantizer
stage delegated to the C/numpy oracle (oracle/xq_oracle.py) through CPU autograd Functions.

PARITY: pinned by tests/golden/vit_*.npz, which tests/golden/make_vit_golden.py produces by running the
reference's own dinov2.py + vendored vision_transformer.py + VQModel.encode/decode (tests/test_vit_golden.py,
1e-3).  Only timm's PatchEmbed / Mlp / DropPath / resample_abs_pos_embed (timm==1.0.9, environment.yml:102, not
vendored, not installed here) are stand-ins in that generator: those four layers remain parity-unpinned.

Only tests/, __graft_entry__.smoke() and bench.py (cpu_baseline / --impl reference) import it.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

from . import xq_oracle as xo


# ----------------------------------------------------------------------------------------------
# ViT pieces
# ----------------------------------------------------------------------------------------------
def _ln(x, sd, prefix, eps=1e-6):
    return F.layer_norm(x, (x.shape[-1],), sd[prefix + ".weight"], sd[prefix + ".bias"], eps)


def _attention(x, sd, prefix, num_heads):
    B, N, C = x.shape
    hd = C // num_heads
    qkv = F.linear(x, sd[prefix + ".qkv.weight"], sd[prefix + ".qkv.bias"])
    qkv = qkv.reshape(B, N, 3, num_heads, hd).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    att = (q * hd ** -0.5) @ k.transpose(-2, -1)
    att = att.softmax(dim=-1)
    y = (att @ v).transpose(1, 2).reshape(B, N, C)
    return F.linear(y, sd[prefix + ".proj.weight"], sd[prefix + ".proj.bias"])


def _block(x, sd, prefix, num_heads, keep: Optional[List[torch.Tensor]] = None):
    """pre-LN block with LayerScale; `keep` = optional per-sample DropPath multipliers (2 tensors)."""
    a = _attention(_ln(x, sd, prefix + ".norm1"), sd, prefix + ".attn", num_heads) * sd[prefix + ".ls1.gamma"]
    if keep is not None:
        a = a * keep[0]
    x = x + a
    h = _ln(x, sd, prefix + ".norm2")
    h = F.linear(h, sd[prefix + ".mlp.fc1.weight"], sd[prefix + ".mlp.fc1.bias"])
    h = F.gelu(h)
    h = F.linear(h, sd[prefix + ".mlp.fc2.weight"], sd[prefix + ".mlp.fc2.bias"]) * sd[prefix + ".ls2.gamma"]
    if keep is not None:
        h = h * keep[1]
    return x + h


def _resample_pos(posemb, new_hw, num_prefix=1):
    """timm.layers.resample_abs_pos_embed (bicubic, antialias=True)."""
    n = posemb.shape[1]
    if new_hw[0] * new_hw[1] + num_prefix == n and new_hw[0] == new_hw[1]:
        return posemb
    old = int(math.sqrt(n - num_prefix))
    pre, grid = posemb[:, :num_prefix], posemb[:, num_prefix:]
    D = grid.shape[-1]
    grid = grid.reshape(1, old, old, D).permute(0, 3, 1, 2)
    grid = F.interpolate(grid, size=new_hw, mode="bicubic", antialias=True)
    grid = grid.permute(0, 2, 3, 1).reshape(1, -1, D)
    return torch.cat([pre, grid], dim=1)


def _pos_embed(x, sd, prefix):
    """x: [B,N,D] or [B,H,W,D] -> cls + x + pos  (vision_transformer.py:814-848, no_embed_class=False)."""
    pos = sd[prefix + ".pos_embed"]
    if x.dim() == 4:
        B, H, W, D = x.shape
        pos = _resample_pos(pos, (H, W))
        x = x.reshape(B, -1, D)
    cls = sd[prefix + ".cls_token"].expand(x.shape[0], -1, -1)
    return torch.cat([cls, x], dim=1) + pos


def _depth(sd, prefix):
    return 1 + max(int(k[len(prefix) + 8:].split(".")[0]) for k in sd if k.startswith(prefix + ".blocks."))


def _blocks(t, sd, prefix, num_heads, keep):
    """the transformer blocks; keep[i] = None or the (attention, MLP) DropPath multipliers of block i, each [B] or None"""
    for i in range(_depth(sd, prefix)):
        k = keep[i] if keep is not None else None
        if k is not None:
            k = [torch.ones((), dtype=t.dtype, device=t.device) if m is None else m.to(t).view(-1, 1, 1) for m in k]
        t = _block(t, sd, f"{prefix}.blocks.{i}", num_heads, k)
    return t


def encoder_forward(sd: Dict[str, torch.Tensor], x, num_heads: int, num_latent: int, product_quant: int,
                    prefix="encoder", patch=16, keep=None):
    w, b = sd[prefix + ".model.patch_embed.proj.weight"], sd[prefix + ".model.patch_embed.proj.bias"]
    t = F.conv2d(x, w, b, stride=patch).flatten(2).transpose(1, 2)
    t = _pos_embed(t, sd, prefix + ".model")
    z = sd[prefix + ".latent_tokens"].expand(t.shape[0], -1, -1)
    D = z.shape[-1]
    if prefix + ".lvl_embed.weight" in sd:          # abs_pos_embed=True (dinov2.py:155-169)
        s = int(math.sqrt(num_latent // product_quant))
        zs = z.reshape(t.shape[0], product_quant * s, s, D).chunk(product_quant, dim=1)
        zs = [_pos_embed(zi, sd, prefix + ".model")[:, 1:] for zi in zs]
        t = torch.cat([t] + zs, dim=1)
        t = t + sd[prefix + ".lvl_embed.weight"][sd[prefix + ".lvl1LC"].long()].expand(t.shape[0], -1, -1)
    else:                                           # learned latent positions (dinov2.py:170-171)
        t = torch.cat([t, z + sd[prefix + ".latent_pos_embed"]], dim=1)
    t = _blocks(t, sd, prefix + ".model", num_heads, keep)
    t = _ln(t, sd, prefix + ".model.norm")
    return t[:, -num_latent:]


def decoder_forward(sd, z, num_heads: int, num_latent: int, num_img_tokens=256, prefix="decoder", patch=16, keep=None):
    B = z.shape[0]
    x = sd[prefix + ".mask_token"].expand(B, num_img_tokens, -1)
    x = _pos_embed(x, sd, prefix + ".model")
    if prefix + ".lvl_embed.weight" in sd:          # abs_pos_embed=True
        s = int(math.sqrt(num_latent))
        zz = _pos_embed(z.reshape(B, s, s, -1), sd, prefix + ".model")  # keeps the cls slot (dinov2.py:330)
        t = torch.cat([x, zz], dim=1)
        t = t + sd[prefix + ".lvl_embed.weight"][sd[prefix + ".lvl1LC"].long()].expand(B, -1, -1)
    else:                                           # dinov2.py:332-333
        t = torch.cat([x, z + sd[prefix + ".latent_pos_embed"]], dim=1)
    t = _blocks(t, sd, prefix + ".model", num_heads, keep)
    t = _ln(t, sd, prefix + ".model.norm")
    t = t[:, 1:1 + num_img_tokens]
    t = F.linear(t, sd[prefix + ".to_pixel.model.weight"], sd[prefix + ".to_pixel.model.bias"])
    h = int(math.sqrt(num_img_tokens))
    t = t.reshape(B, h, h, patch, patch, 3)
    return torch.einsum("nhwpqc->nchpwq", t).reshape(B, 3, h * patch, h * patch)


# ----------------------------------------------------------------------------------------------
# quantizer stage as CPU autograd Functions over the C/numpy oracle
# ----------------------------------------------------------------------------------------------
class _VQ(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z, E, beta, codebook_norm):
        fwd = xo.vq_forward(z.detach().numpy(), E.detach().numpy(), beta, codebook_norm)
        ctx.fwd, ctx.E, ctx.beta, ctx.cn = fwd, E.detach().numpy(), beta, codebook_norm
        idx = torch.from_numpy(fwd["idx"])
        ctx.mark_non_differentiable(idx)
        return (torch.from_numpy(fwd["out"]), torch.tensor(fwd["vq"], dtype=torch.float32),
                torch.tensor(fwd["commit"], dtype=torch.float32), idx)

    @staticmethod
    def backward(ctx, g_out, g_vq, g_commit, _):
        gz, gE = xo.vq_backward(ctx.fwd, ctx.E, g_out.numpy(), float(g_vq), float(g_commit), ctx.beta, ctx.cn)
        return torch.from_numpy(gz.astype(np.float32)), torch.from_numpy(gE.astype(np.float32)), None, None


class _VQ2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, f, E, phi_w, phi_b, patch_nums, znorm, beta, codebook_drop, dropout):
        fn, En, wn, bn = f.detach().numpy(), E.detach().numpy(), phi_w.detach().numpy(), phi_b.detach().numpy()
        fwd = xo.vq2_forward(fn, En, wn, bn, patch_nums, using_znorm=znorm, beta=beta, codebook_drop=codebook_drop,
                             dropout=dropout)
        ctx.pack = (fwd, fn, En, wn, bn, patch_nums, beta)
        return (torch.from_numpy(fwd["out"]), torch.tensor(fwd["vq"], dtype=torch.float32),
                torch.tensor(fwd["commit"], dtype=torch.float32))

    @staticmethod
    def backward(ctx, g_out, g_vq, g_commit):
        fwd, fn, En, wn, bn, pn, beta = ctx.pack
        gf, gE, gw, gb = xo.vq2_backward(fwd, fn, En, wn, bn, pn, g_out.numpy(), float(g_vq), float(g_commit), beta)
        t = lambda a: torch.from_numpy(a.astype(np.float32))
        return t(gf), t(gE), t(gw), t(gb), None, None, None, None, None


class _LFQ(torch.autograd.Function):
    @staticmethod
    def forward(ctx, f, phi_w, phi_b, patch_nums, znorm, beta, codebook_drop, dropout, scaler, entropy_weight):
        fn, wn, bn = f.detach().numpy(), phi_w.detach().numpy(), phi_b.detach().numpy()
        fwd = xo.lfq_forward(fn, wn, bn, patch_nums, using_znorm=znorm, beta=beta, codebook_drop=codebook_drop,
                             dropout=dropout, entropy_weight=entropy_weight, scaler=scaler)
        ctx.pack = (fwd, fn, wn, bn, patch_nums, znorm, beta, entropy_weight)
        return (torch.from_numpy(fwd["out"]), torch.tensor(fwd["vq"], dtype=torch.float32),
                torch.tensor(fwd["commit"], dtype=torch.float32), torch.tensor(fwd["entropy"], dtype=torch.float32))

    @staticmethod
    def backward(ctx, g_out, g_vq, g_commit, g_ent):
        fwd, fn, wn, bn, pn, znorm, beta, ew = ctx.pack
        gf, gw, gb = xo.lfq_backward(fwd, fn, wn, bn, pn, g_out.numpy(), float(g_vq), float(g_commit), float(g_ent),
                                     using_znorm=znorm, beta=beta, entropy_weight=ew)
        t = lambda a: torch.from_numpy(a.astype(np.float32))
        return t(gf), t(gw), t(gb), None, None, None, None, None, None, None


# ----------------------------------------------------------------------------------------------
# the whole path
# ----------------------------------------------------------------------------------------------
class RefTokenizer:
    """encode -> quantize -> decode from a VQModel state_dict, in fp32 on the CPU unless `dtype` / `device` say otherwise
    (fp64 on a GPU is what the gradient tests use).  The quantizer stage always runs the fp32 C/numpy oracle on the CPU.

    cfg keys: codebook_size, codebook_embed_dim, product_quant, v_patch_nums, num_latent_tokens (per branch),
    lfq, num_heads, codebook_drop, beta, entropy_weight, codebook_l2_norm
    `keep` (encode / decode / forward): per-block DropPath multipliers of that ViT, see `_blocks`.
    """

    def __init__(self, state_dict: Dict[str, torch.Tensor], cfg: Dict, requires_grad: bool = False,
                 dtype: torch.dtype = torch.float32, device="cpu"):
        self.cfg = dict(cfg)
        self.sd = {}
        for k, v in state_dict.items():
            v = v.detach().to(device)
            v = v.to(dtype).clone() if v.is_floating_point() else v.clone()
            if requires_grad and v.is_floating_point() and "ema_vocab_hit" not in k and "scaler" not in k:
                v.requires_grad_(True)
            self.sd[k] = v

    def parameters(self):
        return [v for v in self.sd.values() if v.requires_grad]

    def _qprefix(self, i):
        return f"quantizes.{i}" if self.cfg["product_quant"] > 1 else "quantize"

    def encode(self, x, keep=None):
        c = self.cfg
        PQ = c["product_quant"]
        h = encoder_forward(self.sd, x, c["num_heads"], c["num_latent_tokens"] * PQ, PQ, keep=keep)
        b, l, d = h.shape
        if PQ > 1:
            h = h.reshape(b, l, 1, d).permute(0, 3, 1, 2)
        else:
            s = int(math.sqrt(l))
            h = h.reshape(b, s, s, d).permute(0, 3, 1, 2)
        return F.conv2d(h, self.sd["quant_conv.weight"], self.sd["quant_conv.bias"])

    def _branches(self, h):
        PQ = self.cfg["product_quant"]
        if PQ == 1:
            return [h]
        b, c, l, _ = h.shape
        s = int(math.sqrt(l // PQ))
        return [t.reshape(b, c, s, s) for t in h.chunk(PQ, dim=2)]

    def _phi(self, q):
        ks = sorted({int(k.split(".")[-2]) for k in self.sd if k.startswith(q + ".quant_resi.qresi_ls.")})
        w = torch.stack([self.sd[f"{q}.quant_resi.qresi_ls.{i}.weight"] for i in ks])
        b = torch.stack([self.sd[f"{q}.quant_resi.qresi_ls.{i}.bias"] for i in ks])
        return w, b

    def quantize(self, h, dropout=None):
        """-> quant [B, PQ*C, s, s], (vq, commit, entropy) in h's dtype and device"""
        c = self.cfg
        pn = list(c["v_patch_nums"])
        o = lambda t: t.float().cpu()           # the oracle's operands: fp32 on the CPU (no-ops for the fp32 CPU tokenizer)
        outs, vqs, cms, ens = [], [], [], []
        for i, hi in enumerate(self._branches(h)):
            q = self._qprefix(i)
            hi = o(hi.contiguous())
            if len(pn) == 1:
                out, vq, cm, _ = _VQ.apply(hi, o(self.sd[q + ".embedding.weight"]), c.get("beta", 0.25),
                                           c.get("codebook_l2_norm", True))
                en = torch.zeros(())
            elif not c.get("lfq", False):
                w, b = self._phi(q)
                out, vq, cm = _VQ2.apply(hi, o(self.sd[q + ".embedding.weight"]), o(w), o(b), pn, True,
                                         c.get("beta", 0.25), c.get("codebook_drop", 0.0), dropout)
                en = torch.zeros(())
            else:
                w, b = self._phi(q)
                out, vq, cm, en = _LFQ.apply(hi, o(w), o(b), pn, c.get("codebook_l2_norm", True), c.get("beta", 0.25),
                                             c.get("codebook_drop", 0.0), dropout, o(self.sd[q + ".scaler"]).numpy(),
                                             c.get("entropy_weight", 0.0))
            outs.append(out.to(h)), vqs.append(vq.to(h)), cms.append(cm.to(h)), ens.append(en.to(h))
        n = len(outs)
        return torch.cat(outs, dim=1), (sum(vqs) / n, sum(cms) / n, sum(ens) / n)

    def decode(self, quant, keep=None):
        c = self.cfg
        t = F.conv2d(quant, self.sd["post_quant_conv.weight"], self.sd["post_quant_conv.bias"])
        t = t.flatten(2).permute(0, 2, 1)
        return decoder_forward(self.sd, t, c["num_heads"], c["num_latent_tokens"], keep=keep)

    def forward(self, x, dropout=None, enc_keep=None, dec_keep=None):
        h = self.encode(x, enc_keep)
        quant, losses = self.quantize(h, dropout)
        return self.decode(quant, dec_keep), losses, h

    def train_step(self, x, opt, dropout=None):
        """the in-scope generator step: fwd + bwd of (MSE rec + vq + commit + entropy) + optimizer."""
        dec, (vq, cm, en), _ = self.forward(x, dropout)
        loss = F.mse_loss(dec, x) + vq + cm + en
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        return float(loss)


def cfg_from_model_args(args, num_heads=12) -> Dict:
    """args: the ModelArgs the product VQModel was built from (after its PQ scaling of num_latent_tokens)."""
    return dict(codebook_size=args.codebook_size, codebook_embed_dim=args.codebook_embed_dim,
                product_quant=args.product_quant, v_patch_nums=list(args.v_patch_nums),
                num_latent_tokens=args.num_latent_tokens // args.product_quant, lfq=args.lfq, num_heads=num_heads,
                codebook_drop=args.codebook_drop, beta=args.commit_loss_beta, entropy_weight=args.entropy_loss_ratio,
                codebook_l2_norm=args.codebook_l2_norm)
