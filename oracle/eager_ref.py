"""Plain-PyTorch restatement of the reference's quantizer forward passes (TEST INFRASTRUCTURE / BASELINE ONLY).

Device-agnostic eager code that does what the reference modules do, op for op in behaviour (materialised
N x V distance matrix, per-scale Python loop, bincount + usage .item() syncs), so that
  * tests can check it against the same golden vectors as the C oracle (a second, independent restatement), and
  * bench.py --impl eager can time "the reference's way of computing this path" on the SAME GPU, which is the
    denominator of the north star's ">= 6x reference PyTorch-eager" target.
It borrows the PARAMETERS of the product modules (embedding, Phi convs, buffers) and never calls libxqb200.

Follows: VectorQuantizer.forward            tokenizer/tokenizer_image/xqgan_model.py:745-801
         add_perturbation                   tokenizer/tokenizer_image/latent_perturbation.py:4-35
         VectorQuantizer2.forward           tokenizer/tokenizer_image/quant.py:64-144
         LFQ.forward / soft_entropy_loss    tokenizer/tokenizer_image/lookup_free_quantize.py:149-250, 283-300
"""
from __future__ import annotations

import weakref

import torch
import torch.nn.functional as F

# module -> the restatement's own `record_hit`.  The product modules keep theirs on the device, where reading it costs a host
# sync the reference does not make: it is read once per module, at the module's first update, and counted here from then on
# (the module's own counter does not advance).
_record_hit = weakref.WeakKeyDictionary()


def _sync_usage(ema, margin):
    return (ema >= margin).float().mean().item() * 100       # the reference's host sync


def _next_record_hit(mod):
    """the reference's `record_hit` for this update, then `record_hit += 1`."""
    rh = _record_hit.get(mod)
    if rh is None:
        rh = mod.record_hit
    _record_hit[mod] = rh + 1
    return rh


def _ema_(ema_row, hit, record_hit):
    if record_hit == 0:
        ema_row.copy_(hit)
    elif record_hit < 100:
        ema_row.mul_(0.9).add_(hit.mul(0.1))
    else:
        ema_row.mul_(0.99).add_(hit.mul(0.01))


def vq_forward(mod, z):
    """mod: a module with embedding / beta / codebook_norm / ema_vocab_hit_SV / record_hit / vocab_size."""
    zt = z.permute(0, 2, 3, 1).contiguous()
    flat = zt.reshape(-1, zt.shape[-1])
    if mod.codebook_norm:
        zt = F.normalize(zt, p=2, dim=-1)
        flat = F.normalize(flat, p=2, dim=-1)
        emb = F.normalize(mod.embedding.weight, p=2, dim=-1)
    else:
        emb = mod.embedding.weight
    d = flat.pow(2).sum(1, keepdim=True) + emb.pow(2).sum(1) - 2 * flat @ emb.t()     # N x V, materialised
    idx = d.argmin(dim=1)
    zq = mod.embedding(idx).view(zt.shape)
    if mod.codebook_norm:
        zq = F.normalize(zq, p=2, dim=-1)
    usage = None
    if mod.training:
        hit = idx.bincount(minlength=mod.vocab_size).float()
        _ema_(mod.ema_vocab_hit_SV, hit, _next_record_hit(mod))
        usage = _sync_usage(mod.ema_vocab_hit_SV, flat.shape[0] / mod.vocab_size * 0.08)
    commit = mod.beta * (zq.detach() - zt).pow(2).mean()
    vq = (zq - zt.detach()).pow(2).mean()
    zq = zt + (zq - zt).detach()
    return zq.permute(0, 3, 1, 2), [usage], vq, commit, idx


def perturb(z, z_q, mod, alpha, beta, delta):
    zt = z.permute(0, 2, 3, 1).contiguous()
    flat = zt.reshape(-1, zt.shape[-1])
    if mod.codebook_norm:
        zt = F.normalize(zt, p=2, dim=-1)
        flat = F.normalize(flat, p=2, dim=-1)
        emb = F.normalize(mod.embedding.weight, p=2, dim=-1)
    else:
        emb = mod.embedding.weight
    d = flat.pow(2).sum(1, keepdim=True) + emb.pow(2).sum(1) - 2 * flat @ emb.t()
    cand = d.topk(delta, dim=1, largest=False).indices
    u = torch.rand(cand.shape[0], device=d.device)
    j = torch.randint(0, delta, u.shape, device=d.device)
    j = torch.where(u > alpha, 0, j)
    sel = cand[torch.arange(cand.shape[0], device=d.device), j]
    p = mod.embedding(sel).view(zt.shape)
    if mod.codebook_norm:
        p = F.normalize(p, p=2, dim=-1)
    p = (zt + (p - zt).detach()).permute(0, 3, 1, 2)
    mask = (torch.arange(z.shape[0], device=z.device) < int(z.shape[0] * beta))[:, None, None, None]
    return torch.where(mask, p, z_q)


def _phi(mod, si, SN, h):
    m = mod.quant_resi[0] if SN == 1 else mod.quant_resi[si / (SN - 1)]
    return m(h)


def _n_quantizers(mod, B, dropout, device):
    SN = len(mod.v_patch_nums)
    nq = torch.ones((B,)) * (SN + 1)
    if mod.training and dropout is not None:
        nd = int(B * mod.codebook_drop)
        nq[:nd] = dropout[:nd]
    return nq.to(device)


def vq2_forward(mod, f, dropout=None):
    f = f.float()
    B, C, H, W = f.shape
    f_ng = f.detach()
    rest = f_ng.clone()
    fhat = torch.zeros_like(rest)
    SN = len(mod.v_patch_nums)
    nq = _n_quantizers(mod, B, dropout, f.device)
    vq = commit = 0.0
    with torch.autocast(device_type=f.device.type, enabled=False):
        for si, pn in enumerate(mod.v_patch_nums):
            rows = (F.interpolate(rest, size=(pn, pn), mode="area") if si != SN - 1 else rest)
            rows = rows.permute(0, 2, 3, 1).reshape(-1, C)
            if mod.using_znorm:
                idx = (F.normalize(rows, dim=-1) @ F.normalize(mod.embedding.weight.data.t(), dim=0)).argmax(1)
            else:
                d = rows.square().sum(1, keepdim=True) + mod.embedding.weight.data.square().sum(1)
                d.addmm_(rows, mod.embedding.weight.data.t(), alpha=-2, beta=1)
                idx = d.argmin(1)
            hit = idx.bincount(minlength=mod.vocab_size).float()
            h = mod.embedding(idx.view(B, pn, pn)).permute(0, 3, 1, 2)
            h = F.interpolate(h, size=(H, W), mode="bicubic").contiguous() if si != SN - 1 else h.contiguous()
            h = _phi(mod, si, SN, h)
            mask = (torch.full((B,), si, device=f.device) < nq)[:, None, None, None].int()
            fhat = fhat + h * mask
            rest = rest - h
            if mod.training:
                _ema_(mod.ema_vocab_hit_SV[si], hit, _next_record_hit(mod))
            ratio = mask.sum() / B
            vq = vq + F.mse_loss(fhat, f_ng, reduction="none").mul(mask).mean() / ratio
            commit = commit + F.mse_loss(fhat.detach(), f, reduction="none").mul(mask).mul(mod.beta / ratio).mean()
        vq = vq / SN
        out = (fhat.detach() - f_ng) + f
    margin = (f.numel() / C) / mod.vocab_size * 0.08
    usages = [_sync_usage(mod.ema_vocab_hit_SV[si], margin) for si in range(SN)]
    return out, usages, vq, commit, 0


def lfq_forward(mod, f, dropout):
    f = f.float()
    B, C, H, W = f.shape
    if mod.using_znorm:
        f = F.normalize(f, dim=1)
    f_ng = f.detach()
    rest = f_ng.clone()
    fhat = torch.zeros_like(rest)
    SN = len(mod.v_patch_nums)
    nq = _n_quantizers(mod, B, dropout, f.device)
    bitw = 2 ** torch.arange(C, device=f.device, dtype=torch.long)
    vq = commit = ent = 0.0

    def h2(p):
        return -(p * torch.log(p + 1e-8))

    with torch.autocast(device_type=f.device.type, enabled=False):
        for si, pn in enumerate(mod.v_patch_nums):
            s = mod.scaler[si].float()
            rows = (F.interpolate(rest, size=(pn, pn), mode="area") if si != SN - 1 else rest)
            rows = rows.permute(0, 2, 3, 1).reshape(-1, C)
            bits = rows > 0
            idx = (bits * bitw).sum(-1)
            hit = idx.bincount(minlength=mod.vocab_size).float()
            h = torch.where(bits, s, -s).view(B, pn, pn, C).permute(0, 3, 1, 2)
            h = F.interpolate(h, size=(H, W), mode="bicubic").contiguous() if si != SN - 1 else h.contiguous()
            h = _phi(mod, si, SN, h)
            x = (f - fhat.detach()).flatten(2).transpose(1, 2)             # b (hw) d
            mask = (torch.full((B,), si, device=f.device) < nq)[:, None, None, None].int()
            fhat = fhat + h * mask
            rest = rest - h
            if mod.training:
                _ema_(mod.ema_vocab_hit_SV[si], hit, _next_record_hit(mod))
            ratio = mask.sum() / B
            zsel = x[mask.view(B)]                                         # INT-mask gather of batch rows 0 / 1
            p = torch.sigmoid(-4 * zsel * s)
            prob = torch.stack([p, 1 - p], dim=-1)
            per_sample = h2(prob).sum(-1).sum(-1).mean()
            avg = prob.mean(dim=(0, 1))
            code_ent = h2(avg).sum()
            aux = mod.sample_minimization_weight * per_sample - mod.batch_maximization_weight * code_ent
            vq = vq + F.mse_loss(fhat, f_ng, reduction="none").mul(mask).mean() / ratio
            commit = commit + F.mse_loss(fhat.detach(), f, reduction="none").mul(mask).mul(mod.beta / ratio).mean()
            ent = ent + aux * (mod.entropy_weight / ratio)
        vq, commit, ent = vq / SN, commit / SN, ent / SN
        out = (fhat.detach() - f_ng) + f
    margin = (f.numel() / C) / mod.vocab_size * 0.08
    usages = [_sync_usage(mod.ema_vocab_hit_SV[si], margin) for si in range(SN)]
    return out, usages, vq, commit, ent


class EagerTokenizer(torch.nn.Module):
    """The product VQModel's parameters driven the reference's way: unfused ViT module path + the eager
    quantizers above (forward = xqgan_model.py:268-301 restricted to the in-scope path)."""

    def __init__(self, model):
        super().__init__()
        self.m = model

    def forward(self, x, epoch, alpha, beta, delta):
        from imagefolder_b200 import vit_ops
        m = self.m
        saved, saved_pe = vit_ops.fused_path_ok, vit_ops.patch_embed_ok
        vit_ops.fused_path_ok = vit_ops.patch_embed_ok = lambda *a, **k: False
        saved_as, vit_ops.ASSEMBLE_ENABLED[0] = vit_ops.ASSEMBLE_ENABLED[0], False
        try:
            h = m.encode(x)
            b, c, l, _ = h.shape
            SN = len(m.v_patch_nums)
            dropout = None if SN == 1 else torch.randint(m.start_drop, SN + 1, (b,))
            if m.product_quant > 1:
                outs, us, vqs, cms, ens = [], [], [], [], []
                for q, hi in zip(m.quantizes, m._split_branches(h)):
                    if SN == 1:
                        o, u, v, cm, _ = vq_forward(q, hi)
                        e = 0.0
                    elif type(q).__name__ == "LFQ":
                        o, u, v, cm, e = lfq_forward(q, hi, dropout)
                    else:
                        o, u, v, cm, e = vq2_forward(q, hi, dropout)
                    outs.append(o), us.append(u), vqs.append(v), cms.append(cm), ens.append(e)
                n = len(outs)
                quant = torch.cat(outs, dim=1)
                vq, cm, en = sum(vqs) / n, sum(cms) / n, sum(ens) / n
                usages = [sum(t) / n for t in zip(*us)]
            else:
                quant, usages, vq, cm, _ = vq_forward(m.quantize, h)
                quant = perturb(h, quant, m.quantize, alpha, beta, delta)     # runs even for alpha = beta = 0
                en = 0.0
            dec = m.decode(quant)
        finally:
            vit_ops.fused_path_ok, vit_ops.patch_embed_ok = saved, saved_pe
            vit_ops.ASSEMBLE_ENABLED[0] = saved_as
        return dec, (vq, cm, en, usages), None, None, 0.0
