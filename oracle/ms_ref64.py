"""fp64 restatement of the multi-scale residual quantizers, differentiated by autograd (TEST INFRASTRUCTURE ONLY).

    VectorQuantizer2.forward   tokenizer/tokenizer_image/quant.py:64-144          (training mode)
    LFQ.forward                tokenizer/tokenizer_image/lookup_free_quantize.py:149-250   (training, soft entropy)
    LFQ.soft_entropy_loss      lookup_free_quantize.py:283-308
    Phi / PhiShared / PhiPartiallyShared / PhiNonShared   quant.py:261-302

written in torch float64 on whatever device its inputs live on.  The discrete choices are INPUTS: the token indices
come from the product, so no argmin or sign decision enters a float comparison.  What the fp64 residual says about
those choices is returned as `idx_gap` (VQ: how far the chosen code's score is from the fp64 best; LFQ: the largest
|pooled residual| whose sign disagrees with the given bit), so a caller can check that the product's choices are the
fp64 ones up to near-ties.

Gradients are whatever torch.autograd makes of this forward: nothing here shares a derivation with the closed forms
of oracle/xq_oracle.py or with the backward kernels.  Pinned to the reference's own outputs by
tests/test_ms_ref64_golden_cpu.py.

`mutant` builds one plausible bug into the fp64 side (for tests that must show a bug of that kind is caught):
    phi_r_twice / phi_r_dropped   the Phi ratio r applied twice / not at all in the gradient to the Phi input
    share_map_shift               scale si uses Phi module k+1 (mod K) instead of k
    nq_plus_one                   every sample keeps one scale more than n_quantizers allows
    ent_row1_to_row0              LFQ: the soft-entropy gradient of batch row 1 is delivered to row 0
    bicubic_T_align_corners       the bicubic upsample's transpose uses align_corners=True
    area_floor                    area pooling with floor instead of ceil end bounds
    swap_vq_commit                (losses_and_grads) the vq and commit loss weights are exchanged
share_map_shift and nq_plus_one also change the forward values; area_floor changes only `idx_gap` (the indices are
inputs); the others change gradients only.

Only tests/ import this module; the product never does.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

MUTANTS = ("phi_r_twice", "phi_r_dropped", "share_map_shift", "nq_plus_one", "ent_row1_to_row0",
           "bicubic_T_align_corners", "area_floor", "swap_vq_commit")


def phi_map(SN: int, K: int) -> List[int]:
    """scale -> Phi module (quant.py:110-113 with PhiShared :271, PhiPartiallyShared :279-288, PhiNonShared :294)."""
    if K == 1 or SN == 1:
        return [0] * SN
    ticks = np.linspace(1 / 3 / K, 1 - 1 / 3 / K, K) if K == 4 else np.linspace(1 / 2 / K, 1 - 1 / 2 / K, K)
    return [int(np.argmin(np.abs(ticks - si / (SN - 1)))) for si in range(SN)]


def n_quantizers(B: int, SN: int, codebook_drop: float, dropout) -> torch.Tensor:
    """quant.py:79-86 / lookup_free_quantize.py:167-173: the first int(B * codebook_drop) samples keep dropout[b]
    scales, every other sample all of them."""
    nq = torch.full((B,), float(SN + 1), dtype=torch.float64)
    if dropout is not None:
        nd = int(B * codebook_drop)
        nq[:nd] = torch.as_tensor(np.asarray(dropout)[:nd], dtype=torch.float64)
    return nq


def _area_floor(x: torch.Tensor, P: int) -> torch.Tensor:
    """area pooling whose cell i spans [floor(i H / P), floor((i+1) H / P)) -- the `area_floor` mutant."""
    H = x.shape[-1]
    A = torch.zeros(P, H, dtype=x.dtype, device=x.device)
    for i in range(P):
        lo, hi = (i * H) // P, ((i + 1) * H) // P
        A[i, lo:hi] = 1.0 / (hi - lo)
    return torch.einsum("ph,bchw,qw->bcpq", A, x, A)


def _value_as_grad_of(value: torch.Tensor, grad_path: torch.Tensor) -> torch.Tensor:
    """`value` in the forward, `grad_path`'s gradient in the backward."""
    return grad_path + (value - grad_path).detach()


def forward(f: torch.Tensor, idx: Sequence[torch.Tensor], patch_nums: Sequence[int], *, lfq: bool,
            E: Optional[torch.Tensor] = None, phi_w: Optional[torch.Tensor] = None,
            phi_b: Optional[torch.Tensor] = None, nq: Optional[torch.Tensor] = None, using_znorm: bool = True,
            beta: float = 0.25, resi_ratio: float = 0.5, scaler: Optional[Sequence[float]] = None,
            entropy_weight: float = 0.1, w_sample: float = 1.0, w_batch: float = 1.0,
            mutant: Optional[str] = None) -> Dict:
    """One training-mode forward in float64.

    f [B,C,H,W] float64 (set requires_grad on it, E, phi_w, phi_b to differentiate); idx: per scale [B, pn*pn] token
    indices (for LFQ bit c of the index is the sign of channel c); nq: n_quantizers [B] (None: every sample keeps every
    scale).  -> dict(out, vq, commit, entropy, fhat (unmasked cumulative f_hat after every scale, as
    f_to_idxBl_or_fhat(to_fhat=True) returns it), idx_gap)."""
    assert mutant is None or mutant in MUTANTS, mutant
    B, C, H, W = f.shape
    SN = len(patch_nums)
    dev, dt = f.device, f.dtype
    K = 0 if phi_w is None else phi_w.shape[0]
    pmap = phi_map(SN, K) if K else [-1] * SN
    if mutant == "share_map_shift":
        pmap = [(k + 1) % K for k in pmap]
    r = float(resi_ratio)
    nq = torch.full((B,), float(SN + 1), dtype=dt, device=dev) if nq is None else nq.to(dev, dt)
    if mutant == "nq_plus_one":
        nq = nq + 1

    if lfq and using_znorm:
        f = F.normalize(f, dim=1)                              # lookup_free_quantize.py:153
    f_ng = f.detach()
    rest = f_ng.clone()
    fhat = torch.zeros_like(f_ng)                              # masked, differentiable (quant.py:116)
    fhat_acc = torch.zeros_like(f_ng)                          # unmasked (f_to_idxBl_or_fhat)
    fhat_list = []
    vq = commit = ent = torch.zeros((), dtype=dt, device=dev)
    idx_gap = 0.0
    if lfq:
        bitw = torch.arange(C, device=dev)
    for si, pn in enumerate(patch_nums):
        # ---- the residual the search looked at (quant.py:91-97, lookup_free_quantize.py:179-180)
        if si == SN - 1:
            rest_p = rest
        elif mutant == "area_floor":
            rest_p = _area_floor(rest, pn)
        else:
            rest_p = F.interpolate(rest, size=(pn, pn), mode="area")
        ix = idx[si].to(dev).reshape(B, pn, pn).long()
        if lfq:
            s = float(scaler[si])
            bits = ((ix[..., None] >> bitw) & 1).bool()                      # [B,pn,pn,C]
            code = (bits.to(dt) * 2 - 1) * s                                 # indices_to_bits(idx, si)  :270-281
            x = rest_p.permute(0, 2, 3, 1)
            wrong = (x > 0) != bits                                          # :182-183 (torch.where(z > 0, v, -v))
            if wrong.any():
                idx_gap = max(idx_gap, float(x.abs()[wrong].max()))
        else:
            code = E[ix]                                                     # self.embedding(idx)  quant.py:107
            idx_gap = max(idx_gap, _vq_gap(rest_p.permute(0, 2, 3, 1).reshape(-1, C), E.detach(), ix.reshape(-1),
                                           using_znorm))
        code = code.permute(0, 3, 1, 2)
        # ---- bicubic up to H x W; the last scale is not interpolated (quant.py:107-109)
        if si == SN - 1:
            u = code
        elif mutant == "bicubic_T_align_corners":
            u = _value_as_grad_of(F.interpolate(code, size=(H, W), mode="bicubic"),
                                  F.interpolate(code, size=(H, W), mode="bicubic", align_corners=True))
        else:
            u = F.interpolate(code, size=(H, W), mode="bicubic")
        # ---- Phi: h (1 - r) + conv3x3(h) r   (quant.py:261-268)
        k = pmap[si]
        if k >= 0:
            uc = u
            if mutant == "phi_r_twice":
                uc = _value_as_grad_of(u, u * r)
            elif mutant == "phi_r_dropped":
                uc = _value_as_grad_of(u, u / r)
            h = u * (1 - r) + F.conv2d(uc, phi_w[k], phi_b[k], padding=1) * r
        else:
            h = u
        # ---- LFQ soft entropy on x = f - f_hat before this scale (lookup_free_quantize.py:197, 217-219, 283-308)
        m_int = (si < nq).long()
        m = m_int.to(dt)[:, None, None, None]
        ratio = m.sum() / B
        if lfq:
            xr = (f - fhat.detach()).permute(0, 2, 3, 1).reshape(B, H * W, 1, C)
            if mutant == "ent_row1_to_row0":
                xr = torch.cat([xr[:1], _value_as_grad_of(xr[1:2], xr[:1]), xr[2:]])
            z = xr[m_int]                                                    # the int mask gathers rows 0 / 1  :285
            p = torch.sigmoid(-4 * z * s)
            prob = torch.stack([p, 1 - p], dim=-1)
            per_sample = (-(prob * torch.log(prob + 1e-8)).sum(-1)).sum(-1).mean()
            avg = prob.reshape(-1, C, 2).mean(0)
            codebook_ent = (-(avg * torch.log(avg + 1e-8)).sum(-1)).sum()
            ent = ent + (w_sample * per_sample - w_batch * codebook_ent) * (entropy_weight / ratio)
        # ---- masked accumulation, residual update, losses (quant.py:115-132)
        fhat = fhat + h * m
        fhat_acc = fhat_acc + h.detach()
        fhat_list.append(fhat_acc)
        rest = rest - h.detach()
        vq = vq + F.mse_loss(fhat, f_ng, reduction="none").mul(m).mean() / ratio
        commit = commit + F.mse_loss(fhat.detach(), f, reduction="none").mul(m).mul(beta / ratio).mean()
    vq = vq / SN                                                             # quant.py:134
    if lfq:                                                                  # lookup_free_quantize.py:238-240
        commit = commit / SN
        ent = ent / SN
    out = (fhat.detach() - f_ng) + f                                         # straight-through  quant.py:135
    return dict(out=out, vq=vq, commit=commit, entropy=ent, fhat=fhat_list, idx_gap=idx_gap)


def _vq_gap(rows: torch.Tensor, E: torch.Tensor, idx: torch.Tensor, using_znorm: bool, chunk: int = 4096) -> float:
    """largest amount by which the chosen code's fp64 score falls short of the fp64 best (quant.py:90-101):
    cosine for znorm, squared distance relative to max(1, |r|^2 + |e|^2) for L2."""
    gap = 0.0
    En = F.normalize(E, dim=1) if using_znorm else E
    ee = (E * E).sum(1)
    for i in range(0, rows.shape[0], chunk):
        r = rows[i:i + chunk]
        j = idx[i:i + chunk]
        if using_znorm:
            s = F.normalize(r, dim=1) @ En.T
            g = s.max(1).values - s.gather(1, j[:, None])[:, 0]
        else:
            rr = (r * r).sum(1, keepdim=True)
            d = rr + ee[None] - 2 * r @ E.T
            g = (d.gather(1, j[:, None])[:, 0] - d.min(1).values) / torch.clamp(rr[:, 0] + ee[j], min=1.0)
        gap = max(gap, float(g.max()))
    return gap


def losses_and_grads(fwd: Dict, wrt: Dict[str, torch.Tensor], g_out: torch.Tensor, w_vq: float, w_commit: float,
                     w_ent: float = 0.0, mutant: Optional[str] = None) -> Dict[str, torch.Tensor]:
    """autograd gradients of  sum(out * g_out) + w_vq vq + w_commit commit + w_ent entropy  with respect to every
    tensor in `wrt` (name -> leaf).  A leaf the loss does not reach gets a zero gradient."""
    if mutant == "swap_vq_commit":
        w_vq, w_commit = w_commit, w_vq
    loss = (fwd["out"] * g_out).sum() + w_vq * fwd["vq"] + w_commit * fwd["commit"] + w_ent * fwd["entropy"]
    names = list(wrt)
    gs = torch.autograd.grad(loss, [wrt[n] for n in names], allow_unused=True)
    return {n: (torch.zeros_like(wrt[n]) if g is None else g) for n, g in zip(names, gs)}
