"""fp64 closed form of LFQ's full-softmax entropy loss, LFQ(soft_entropy=False) (TEST INFRASTRUCTURE ONLY).

The reference builds logits = 2 x.code_j over all 2^C codes code_j = +-s and calls entropy_loss at temperature 0.01
(lookup_free_quantize.py:41-79, 220-229).  With logits linear in the code's signs the softmax factorises over the bits,
P(bit k = 1 | row) = q_k = sigmoid(400 s x_k), so

  sample entropy    S  = mean over masked rows of sum_k H_b(q_k)
  codebook entropy  Hc = -sum_j a_j log(a_j + 1e-5),   a_j = mean over masked rows of prod_k q_k(bit k of j)

with a = A^T Bm / (n1 HW), A over the low C // 2 bits and Bm over the rest.  Everything else of LFQ.forward (indices,
f_hat, vq / commit losses and their gradients) is the soft path's oracle, oracle/xq_oracle.lfq_forward / lfq_backward.
"""
from __future__ import annotations

from typing import Dict

import numpy as np
from scipy.special import expit as _sig       # logistic sigmoid, accurate in both tails

from oracle import xq_oracle as xo

T_INV2 = 400.0      # 2 / temperature(0.01) * 2: the logit gap between a bit's two values is 2 * 2 s x / 0.01


def _bit_products(fp, fm):
    """[R, n] factors for bit = 1 / bit = 0 -> [R, 2^n] products, column j = prod_k (bit k of j ? fp : fm)."""
    P = np.ones((fp.shape[0], 1))
    for k in range(fp.shape[1]):
        P = np.concatenate([P * fm[:, k:k + 1], P * fp[:, k:k + 1]], axis=1)
    return P


def _bit_grad(gP, qp, qm):
    """d/dq_k of sum_j gP[r, j] prod_k' f_k'(j) for every k: the product with factor k replaced by (-1, +1)."""
    R, n = qp.shape
    out = np.empty((R, n))
    for k in range(n):
        fp, fm = qp.copy(), qm.copy()
        fp[:, k], fm[:, k] = 1.0, -1.0
        out[:, k] = np.sum(gP * _bit_products(fp, fm), axis=1)
    return out


def hard_entropy_scale(x, s, mask, w_sample=1.0, w_batch=1.0):
    """One scale of entropy_loss on logits 2 x.code (codes +-s), masked mean over images with mask[b] != 0.
    x [B,C,H,W] fp64.  Returns (sample_entropy, codebook_entropy, loss, d loss / d x [B,C,H,W], a [2^lo, 2^hi])."""
    x = np.asarray(x, np.float64)
    B, C, H, W = x.shape
    sel = np.asarray(mask) != 0
    n1 = int(sel.sum())
    rows = x[sel].transpose(0, 2, 3, 1).reshape(-1, C)                 # [n1*HW, C]
    N = rows.shape[0]
    z = T_INV2 * s * rows
    qp, qm = _sig(z), _sig(-z)
    az = np.abs(z)
    Hb = np.logaddexp(0.0, -az) + az * _sig(-az)
    S = Hb.sum() / N
    lo = C // 2
    A, Bm = _bit_products(qp[:, :lo], qm[:, :lo]), _bit_products(qp[:, lo:], qm[:, lo:])
    a = A.T @ Bm / N
    Hc = float(-(a * np.log(a + 1e-5)).sum())
    loss = w_sample * S - w_batch * Hc
    G = -np.log(a + 1e-5) - a / (a + 1e-5)
    dq = np.concatenate([_bit_grad(Bm @ G.T, qp[:, :lo], qm[:, :lo]), _bit_grad(A @ G, qp[:, lo:], qm[:, lo:])], axis=1)
    pq = qp * qm
    dz = (w_sample * (-z * pq) - w_batch * dq * pq) / N
    gx = np.zeros_like(x)
    gx[sel] = (dz * T_INV2 * s).reshape(n1, H, W, C).transpose(0, 3, 1, 2)
    return float(S), Hc, float(loss), gx, a


def lfq_hard_forward(f, phi_w, phi_b, patch_nums, using_znorm=False, beta=0.25, resi_ratio=0.5, codebook_drop=0.0,
                     dropout=None, scale=1.0, entropy_weight=0.1, w_sample=1.0, w_batch=1.0, scaler=None) -> Dict:
    """LFQ.forward (lookup_free_quantize.py:149-250), training mode, soft_entropy=False."""
    fwd = xo.lfq_forward(f, phi_w, phi_b, patch_nums, using_znorm=using_znorm, beta=beta, resi_ratio=resi_ratio,
                         codebook_drop=codebook_drop, dropout=dropout, scale=scale, entropy_weight=entropy_weight,
                         w_sample=w_sample, w_batch=w_batch, scaler=scaler)
    fn64 = fwd["fn"].astype(np.float64)
    SN = len(patch_nums)
    ent, gx_scales, parts = 0.0, [], []
    for si in range(SN):
        Fprev = np.zeros_like(fn64) if si == 0 else fwd["F"][si - 1].astype(np.float64)
        S, Hc, loss, gx, a = hard_entropy_scale(fn64 - Fprev, float(fwd["scaler"][si]), fwd["masks"][si], w_sample, w_batch)
        ent += loss * entropy_weight / fwd["ratios"][si]
        gx_scales.append(gx * entropy_weight / fwd["ratios"][si])
        parts.append(dict(S=S, Hc=Hc, loss=loss, a=a))
    fwd["entropy"] = ent / SN
    fwd["hard_gx"] = gx_scales
    fwd["hard_parts"] = parts
    return fwd


def lfq_hard_backward(fwd: Dict, f, phi_w, phi_b, patch_nums, g_out, g_vq, g_commit, g_ent, using_znorm=False,
                      beta=0.25, resi_ratio=0.5, entropy_weight=0.1, w_sample=1.0, w_batch=1.0):
    """Gradients wrt f, phi_w, phi_b.  The entropy term reaches f through fn only (x = fn - detached f_hat)."""
    gf, gw, gb = xo.lfq_backward(fwd, f, phi_w, phi_b, patch_nums, g_out, g_vq, g_commit, 0.0, using_znorm=using_znorm,
                                 beta=beta, resi_ratio=resi_ratio, entropy_weight=entropy_weight, w_sample=w_sample,
                                 w_batch=w_batch)
    SN = len(patch_nums)
    gfn = g_ent * sum(fwd["hard_gx"]) / SN
    B, C = gfn.shape[:2]
    if using_znorm:
        g_rows = gfn.reshape(B, C, -1).transpose(0, 2, 1).reshape(-1, C)
        g_rows = xo._norm_jvp_T(g_rows, fwd["fn_rows"], fwd["fden"])
        gfn = g_rows.reshape(B, -1, C).transpose(0, 2, 1).reshape(gfn.shape)
    return gf + gfn, gw, gb
