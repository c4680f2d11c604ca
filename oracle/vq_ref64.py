"""fp64 restatement of the single-scale quantizer and the latent perturbation, differentiated by autograd (TEST
INFRASTRUCTURE ONLY).

    VectorQuantizer.forward    tokenizer/tokenizer_image/xqgan_model.py:745-801   (training mode)
    f_to_idxBl_or_fhat         xqgan_model.py:803-833                             (to_fhat=True)
    add_perturbation           tokenizer/tokenizer_image/latent_perturbation.py:4-35

written in torch float64 on whatever device its inputs live on.  The discrete choices are INPUTS: the quantizer's
indices and the perturbation's selected codes come from the product, so no argmin or top-k enters a float comparison.
What the fp64 distances say about those choices is returned: `idx_gap`, how far the chosen code's squared distance
lies above the fp64 best, and `rank_gap`, how far the selected code's squared distance lies from the fp64 j-th order
statistic of the row (j the rank the row drew), so that a caller can check the product's choices are the fp64 ones up
to near-ties.

Gradients are whatever torch.autograd makes of this forward: nothing here shares a derivation with the closed forms of
oracle/xq_oracle.py or with the backward kernels.  Pinned to the reference's own outputs by
tests/test_vq_ref64_golden_cpu.py.

`mutant` builds one plausible bug into the fp64 side (for tests that must show a bug of that kind is caught):
    no_norm_jacobian_z     the gradient to z skips F.normalize's projection (divides by |z| only), wherever z is
                           normalised: the quantizer and the perturbation
    no_norm_jacobian_E     the same for the codebook rows
    swap_vq_commit         (losses_and_grads) the vq and commit loss weights are exchanged
    mean_over_rows         vq and commit are averaged over the N rows instead of the N * C elements
    perturb_mask_plus_one  int(B * beta) + 1 samples are perturbed
    perturb_grad_dropped   the perturbed samples pass no gradient to z
    rank_plus_one          the selection is judged against order statistic j + 1 (a rank select one off)
mean_over_rows and perturb_mask_plus_one also change forward values; rank_plus_one changes only `rank_gap` (the
selections are inputs); the others change gradients only.

Not a mutant, because it changes no value of a training step: routing the perturbed samples' gradient through z_q
instead of z (or an unperturbed sample's through z instead of z_q).  The quantizer's output is itself straight-through
on the normalised z, so either route gives the same dz; only the perturbation's own gradients, with z and z_q
separate leaves, tell the routes apart.

Only tests/ import this module; the product never does.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn.functional as F

MUTANTS = ("no_norm_jacobian_z", "no_norm_jacobian_E", "swap_vq_commit", "mean_over_rows", "perturb_mask_plus_one",
           "perturb_grad_dropped", "rank_plus_one")

EPS = 1e-12                                                    # F.normalize's default eps


def _value_as_grad_of(value: torch.Tensor, grad_path: torch.Tensor) -> torch.Tensor:
    """`value` in the forward, `grad_path`'s gradient in the backward."""
    return grad_path + (value - grad_path).detach()


def _normalize(x: torch.Tensor, no_jacobian: bool) -> torch.Tensor:
    """F.normalize(x, p=2, dim=-1); with no_jacobian the backward divides by max(|x|, eps) and skips the projection."""
    y = F.normalize(x, p=2, dim=-1)
    if no_jacobian:
        y = _value_as_grad_of(y, x / x.norm(dim=-1, keepdim=True).clamp_min(EPS).detach())
    return y


def _rows(z: torch.Tensor) -> torch.Tensor:
    """[B,C,H,W] -> [B*H*W, C]   (einsum 'b c h w -> b h w c' and view(-1, C), xqgan_model.py:750-751)"""
    return z.permute(0, 2, 3, 1).reshape(-1, z.shape[1])


def _nchw(rows: torch.Tensor, shape) -> torch.Tensor:
    B, C, H, W = shape
    return rows.reshape(B, H, W, C).permute(0, 3, 1, 2)


def _sq_dist(zn: torch.Tensor, En: torch.Tensor) -> torch.Tensor:
    """|zn|^2 + |e|^2 - 2 zn.e for every code (xqgan_model.py:760-763, latent_perturbation.py:16-18)"""
    return (zn * zn).sum(1, keepdim=True) + (En * En).sum(1)[None] - 2 * zn @ En.T


def _row_chunk(V: int) -> int:
    return max(1, (1 << 25) // V)                              # a [chunk, V] fp64 block stays at 256 MiB


def forward(z: torch.Tensor, E: torch.Tensor, idx: torch.Tensor, *, beta: float = 0.25, codebook_norm: bool = True,
            mutant: Optional[str] = None) -> Dict:
    """One training-mode VectorQuantizer.forward in float64.

    z [B,C,H,W], E [V,C] float64 (set requires_grad to differentiate); idx [B*H*W] the chosen codes.
    -> dict(out (straight-through, NCHW), vq, commit, fhat (the normalised codes in NCHW, as
    f_to_idxBl_or_fhat(to_fhat=True) returns them), y (E[idx], the per-row codebook rows: a differentiable
    intermediate whose gradient is each row's contribution to E.grad), idx_gap)."""
    assert mutant is None or mutant in MUTANTS, mutant
    C = z.shape[1]
    idx = idx.to(z.device).reshape(-1).long()
    rows = _rows(z)
    if codebook_norm:                                                        # xqgan_model.py:753-756
        zn = _normalize(rows, mutant == "no_norm_jacobian_z")
    else:
        zn = rows
    y = E[idx]                                                               # self.embedding(idx)  :769
    q = _normalize(y, mutant == "no_norm_jacobian_E") if codebook_norm else y   # :770-771
    n = rows.shape[0] if mutant == "mean_over_rows" else rows.numel()
    commit = beta * ((q.detach() - zn) ** 2).sum() / n                       # :792
    vq = ((q - zn.detach()) ** 2).sum() / n                                  # :793
    out = zn + (q - zn).detach()                                             # straight-through  :796
    with torch.no_grad():
        En = F.normalize(E, p=2, dim=-1) if codebook_norm else E
        gap = 0.0
        ch = _row_chunk(E.shape[0])
        for s in range(0, rows.shape[0], ch):
            d = _sq_dist(zn[s:s + ch], En)
            g = d.gather(1, idx[s:s + ch, None])[:, 0] - d.min(1).values
            gap = max(gap, float(g.max()))
    return dict(out=_nchw(out, z.shape), vq=vq, commit=commit, fhat=_nchw(q.detach(), z.shape), y=y, idx_gap=gap)


def add_perturbation(z: torch.Tensor, z_q: torch.Tensor, E: torch.Tensor, sel: torch.Tensor, rand_u: torch.Tensor,
                     rand_j: torch.Tensor, *, alpha: float, beta: float, delta: int, codebook_norm: bool = True,
                     mutant: Optional[str] = None) -> Dict:
    """add_perturbation in float64.

    z, z_q [B,C,H,W] float64 (z_q: the quantizer's output); E [V,C]; sel: the selected code of every row the mask
    takes (rows in NHW order; at least int(B * beta) * H * W of them); rand_u, rand_j: the two random draws
    (latent_perturbation.py:21-22).  -> dict(out, rank [rows the mask takes], rank_gaps (per such row), rank_gap)."""
    assert mutant is None or mutant in MUTANTS, mutant
    B, C, H, W = z.shape
    HW = H * W
    nb = int(B * beta)                                                       # latent_perturbation.py:32
    if mutant == "perturb_mask_plus_one":
        nb = min(B, nb + 1)
    rows = _rows(z)
    zn = _normalize(rows, mutant == "no_norm_jacobian_z") if codebook_norm else rows      # :9-12
    nr = nb * HW
    sel = sel.to(z.device).reshape(-1).long()
    assert sel.numel() >= nr, "a selection is needed for every row the mask takes"
    rank = torch.where(rand_u.to(z.device).reshape(-1)[:nr].float() > alpha, 0,
                       rand_j.to(z.device).reshape(-1)[:nr].long())          # :23, the fp32 draw against alpha
    if mutant == "rank_plus_one":
        rank = rank + 1
    # the perturbed rows: straight-through on the normalised z  (:26-29)
    sel = sel[:nr]
    Ed = E.detach()
    p = Ed[sel]
    if codebook_norm:
        p = F.normalize(p, p=2, dim=-1)
    zp = zn[:nr]
    pz = zp + (p - zp).detach()
    if mutant == "perturb_grad_dropped":
        pz = pz.detach()
    # torch.where over the first nb samples  (:32-35)
    out = torch.cat([_nchw(pz, (nb, C, H, W)), z_q[nb:]]) if nb > 0 else z_q
    with torch.no_grad():
        En = F.normalize(Ed, p=2, dim=-1) if codebook_norm else Ed
        gaps = torch.zeros(nr, dtype=z.dtype, device=z.device)
        ch = _row_chunk(E.shape[0])
        for s in range(0, nr, ch):
            d = _sq_dist(zp[s:s + ch], En)
            r = rank[s:s + ch].clamp(max=E.shape[0] - 1)
            kth = torch.topk(d, int(r.max()) + 1, dim=1, largest=False).values.gather(1, r[:, None])[:, 0]
            gaps[s:s + ch] = (d.gather(1, sel[s:s + ch, None])[:, 0] - kth).abs()
    return dict(out=out, rank=rank, rank_gaps=gaps, rank_gap=float(gaps.max()) if nr else 0.0)


def losses_and_grads(out: torch.Tensor, vq: torch.Tensor, commit: torch.Tensor, wrt: Dict[str, torch.Tensor],
                     g_out: torch.Tensor, w_vq: float, w_commit: float,
                     mutant: Optional[str] = None) -> Dict[str, torch.Tensor]:
    """autograd gradients of  sum(out * g_out) + w_vq vq + w_commit commit  with respect to every tensor in `wrt`
    (name -> leaf or intermediate).  A tensor the loss does not reach gets a zero gradient."""
    if mutant == "swap_vq_commit":
        w_vq, w_commit = w_commit, w_vq
    loss = (out * g_out).sum() + w_vq * vq + w_commit * commit
    names = list(wrt)
    gs = torch.autograd.grad(loss, [wrt[n] for n in names], allow_unused=True)
    return {n: (torch.zeros_like(wrt[n]) if g is None else g) for n, g in zip(names, gs)}
