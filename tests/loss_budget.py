"""fp64 references, per-element error budgets, a rounding model, seeded input families and named mutants for the loss
stack kernels (imagefolder_b200/csrc/loss_kernels.cu) (TEST INFRASTRUCTURE ONLY).

References, written fresh in torch float64 and differentiated by autograd (no hand-derived gradient):
  LPIPS stage (lpips.py:83-86): channel-normalise both maps with torch.linalg.vector_norm + eps, subtract, square, the
    1x1 lin weights, spatial mean.  vector_norm's gradient is 0 at an all-zero pixel, which is the kernel's convention
    (the reference module's sqrt(sum x^2) gives NaN there).
  DiffAug (diffaug.py, translation / colour / cutout): a gather through a 1-pixel zero border, brightness, the channel
    mean for saturation, the image mean for contrast, the clamped cutout index grid.  The integer and float parameters
    come from oracle.loss_oracle.diffaug_params (the reference's float32 ops).

Budgets.  u = 2^-24 (fp32), u16 = 2^-8 (bf16 storage).  Each bound is the first-order worst case of the rounding points
read off the kernels; the asserted budget is K = 2 times it, so that the rounding model (`lpips_model`, `diffaug_model`)
sits at <= 1/2 of it.
  LPIPS forward, one per image.  Each 8-channel fp32 FMA chunk sum (w a rounded, then 8 fused adds) carries at most
    9u sum_chunk |w| a^2 (resp. |w b^2|, |w a b|); the fp64 fold adds nothing visible.  After the fp64 combine
    Swaa/na^2 + Swbb/nb^2 - 2 Swab/(na nb) that is an ABSOLUTE floor per pixel
        9u sum_c |w_c| (a^_c^2 + b^_c^2 + 2|a^_c b^_c|),
    independent of the distance itself: for near-identical maps the relative error of the value grows as delta^-2.
    The norms: saa is one fp32 FMA chain over C channels, then sqrtf and + eps (float eps), so na has relative error
    rho = (C/2 + 3)u; val moves by 2 rho |sum_c w_c a^_c (a^_c - b^_c)| per norm.  Then the fp64 spatial sum and one
    fp32 rounding of the mean.
  LPIPS gradient (of f1; f0 swaps the maps), one per element.  Tsum = 2 (Swbb/nb - Swab/na) inherits the chunk-sum
    floor and rho; kb = Tsum / (nb nb nb0) three fp32 roundings and the norms' rho; ra, rb one rounding each;
    d = b rb - a ra, o = gs (2w d rb - b kb) a few roundings each (4u on both terms covers any contraction order).
    bf16 adds the storage rounding u16 |o|.
  DiffAug output, one per element.  Without colour every output is a copy of an input (or 0): exact.  With colour the
    fp32 chain v = x + br, m = sum_c v / C, t = (v - m) sat + m, M = sums/(C HW) + br, y = (t - M) con + M, and in the
    backward gbar = sum(mask g)/(C HW), v = con g + (1 - con) gbar, gx = sat v + (1 - sat) mean_c v, each rounding
    bounded by u times the magnitude of its operands.

Mutants are one-line changes to the rounding model (`mutant=` argument); each must exceed the budget on the family built
for it (LP_MUTANT_CASE; DiffAug: the `edges` family under the flags of AUG_MUTANT_FLAGS).  `control` (the fp64 values
rounded once to the output type) must not.  Dropping a cutout's out-of-range cells instead of clamping them onto the
edge is not a mutant: for every offset the reference can draw it zeroes the same cells (test_loss_budget_cpu.py checks
this), so the cutout mutant moves a hanging rectangle back inside the image instead.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle import loss_oracle as lo

U = 2.0 ** -24
U16 = 2.0 ** -8
K = 2.0
EPS = 1e-10
EPS32 = np.float32(EPS)
LP_CHUNK = 8
LP_THREADS = 256
CHUNK_SUM = LP_CHUNK + 1          # rounding of w a, then LP_CHUNK fused adds
CUTOUT = 0.2

LP_FAMILIES = ("indep", "sparse", "near1e-1", "near1e-2", "near1e-3", "prop", "zero", "tiny", "lin")
LP_OUTS = ("val", "g0", "g1")
LP_MUTANTS = ("last_block", "partial_chunk", "no_kb", "kb_na", "eps_in_sqrt", "g0_all", "pair_swap")
# mutant -> (family it is built to be caught on, dtype, shape (B, C, H, W) where the bug is visible)
LP_MUTANT_CASE = {"last_block": ("indep", torch.float32, (2, 64, 20, 29)),        # HW = 580 > 256: 3 blocks
                  "partial_chunk": ("lin", torch.float32, (2, 130, 9, 9)),      # C % 8 = 2
                  "no_kb": ("indep", torch.float32, (2, 64, 12, 12)),
                  "kb_na": ("indep", torch.float32, (2, 64, 12, 12)),
                  "eps_in_sqrt": ("tiny", torch.float32, (2, 64, 12, 12)),
                  "g0_all": ("indep", torch.float32, (3, 64, 12, 12)),
                  "pair_swap": ("indep", torch.bfloat16, (2, 64, 12, 12))}

AUG_MUTANTS = ("trans_sign", "cut_shifted", "contrast_untranslated", "contrast_no_br", "gbar_unmasked", "unread_nonzero")
# the flag set each DiffAug mutant needs to be visible (1 translation, 2 colour, 4 cutout)
AUG_MUTANT_FLAGS = {"trans_sign": 1, "cut_shifted": 4, "contrast_untranslated": 3, "contrast_no_br": 2,
                    "gbar_unmasked": 6, "unread_nonzero": 1}


def ratio(val, ref, bud):
    """max |val - ref| / bud, 0 where the error is 0, inf where it is not finite or the budget is 0"""
    err = (val.double() - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bud)
    return float(r.nan_to_num(nan=math.inf, posinf=math.inf).max()) if r.numel() else 0.0


# ======================================================================================================================
# LPIPS stage
# ======================================================================================================================
def lpips_inputs(family, B, C, H, W, dtype, seed, device="cpu", chunk=16):
    """(f0, f1 [B,C,H,W] in `dtype`, lin weights [C] fp32, upstream gradient [B] fp32), generated from `seed`.
    The maps are built `chunk` samples at a time, so the training shapes need little more than the maps themselves.
      indep     VGG-like ReLU maps, per-channel scales log-uniform over 1e-2 .. 1e2, f0 and f1 independent
      sparse    ~70 % zeros, like stage 5
      near<d>   f1 = relu(f0 + d n) on unit ReLU maps; in bf16 a copy of f0 with a fraction d of its non-zero elements
                moved by one ulp
      prop      f1 = s f0, s = 2 on even samples and 0.7 on odd ones: the true distance is ~0
      zero      pixels all-zero in f0, in f1, in both; pixels with a single non-zero channel in f0, in f1, in both
      tiny      pixel norms log-uniform over 1e-11 .. 1e-9, where eps matters
      lin       unit ReLU maps; the even channels' lin weights zero, the last channel's ~100x the others (for C % 8 != 0
                it sits in the partial last chunk)"""
    g = torch.Generator(device=device).manual_seed(seed)
    scale = 10.0 ** (torch.rand(C, generator=g, device=device) * 4 - 2)
    w = torch.rand(C, generator=g, device=device) * 0.1
    if family == "lin":
        w[0::2] = 0
        w[C - 1] = 100.0 * float(w.max()) + 1.0
    gout = torch.randn(B, generator=g, device=device)
    f0 = torch.empty(B, C, H, W, dtype=dtype, device=device)
    f1 = torch.empty_like(f0)
    for s in range(0, B, chunk):
        n = min(chunk, B - s)
        gc = torch.Generator(device=device).manual_seed(seed * 1009 + s + 1)

        def rn():
            return torch.randn(n, C, H, W, generator=gc, device=device)
        sc = scale.view(1, C, 1, 1)
        if family in ("indep", "zero"):
            a, b = torch.relu(rn()) * sc, torch.relu(rn()) * sc
        elif family == "lin":
            a, b = torch.relu(rn()), torch.relu(rn())
        elif family == "sparse":
            a, b = torch.relu(rn() - 0.5244) * sc, torch.relu(rn() - 0.5244) * sc
        elif family.startswith("near"):
            delta = float(family[4:])
            a = torch.relu(rn())
            b = torch.relu(a + delta * rn())
        elif family == "prop":
            a = torch.relu(rn()) * sc
            fac = torch.where(torch.arange(s, s + n, device=device) % 2 == 0, 2.0, 0.7).view(n, 1, 1, 1)
            b = a.to(dtype).float() * fac
        elif family == "tiny":
            a, b = rn().abs(), rn().abs()
            for t in (a, b):
                nrm = 10.0 ** (torch.rand(n, 1, H, W, generator=gc, device=device) * 2 - 11)
                t.mul_(nrm / torch.linalg.vector_norm(t, dim=1, keepdim=True))
        else:
            raise ValueError(family)
        if family == "zero":
            p = torch.arange(H * W, device=device).view(1, 1, H, W) % 8
            one = torch.arange(C, device=device).view(1, C, 1, 1) == (torch.arange(H * W, device=device).view(1, 1, H, W) % C)
            a = torch.where((p == 0) | (p == 2), 0.0, a)
            b = torch.where((p == 1) | (p == 2), 0.0, b)
            a = torch.where(((p == 3) | (p == 5)) & ~one, 0.0, a)
            b = torch.where(((p == 4) | (p == 5)) & ~one, 0.0, b)
        f0[s:s + n] = a
        f1[s:s + n] = b
        if family.startswith("near") and dtype == torch.bfloat16:
            delta = float(family[4:])
            a16 = f0[s:s + n]
            move = (torch.rand(a16.shape, generator=gc, device=device) < delta) & (a16 != 0)
            step = torch.where(torch.rand(a16.shape, generator=gc, device=device) < 0.5, 1, -1).to(torch.int16)
            bits = a16.view(torch.int16) + torch.where(move, step, torch.zeros_like(step))
            f1[s:s + n] = bits.view(torch.bfloat16)
    return f0, f1, w, gout


def lpips_reference(f0, f1, w, g):
    """fp64 value [B] and both map gradients of  sum_b g_b val_b"""
    a = f0.double().requires_grad_(True)
    b = f1.double().requires_grad_(True)
    na = torch.linalg.vector_norm(a, dim=1, keepdim=True) + EPS
    nb = torch.linalg.vector_norm(b, dim=1, keepdim=True) + EPS
    val = (w.double().view(1, -1, 1, 1) * (a / na - b / nb) ** 2).sum(1).mean((1, 2))
    ga, gb = torch.autograd.grad(val, (a, b), g.double())
    return {"val": val.detach(), "g0": ga, "g1": gb}


def _rho(C):
    return (C / 2 + 3) * U


def lpips_value_budget(f0, f1, w):
    """per image"""
    a, b = f0.double(), f1.double()
    C, HW = a.shape[1], a.shape[2] * a.shape[3]
    aw = w.double().abs().view(1, -1, 1, 1)
    ah = a / (torch.linalg.vector_norm(a, dim=1, keepdim=True) + EPS)
    bh = b / (torch.linalg.vector_norm(b, dim=1, keepdim=True) + EPS)
    d = (ah - bh).abs()
    floor = CHUNK_SUM * U * (aw * (ah * ah + bh * bh + 2 * (ah * bh).abs())).sum(1)
    rho = _rho(C)
    norms = 2 * rho * (aw * (ah.abs() + bh.abs()) * d).sum(1) + 3 * rho * rho * (aw * (ah * ah + bh * bh)).sum(1)
    val = (aw * d * d).sum(1).mean((1, 2))
    pix = (floor + norms).mean((1, 2))
    return K * (pix + U * val + 2.0 ** -50 * (aw * (ah * ah + bh * bh)).sum(1).mean((1, 2)) + 1e-45)


def lpips_grad_budget(f0, f1, w, g, bf16):
    """per element, for the gradient of the SECOND map (call with the maps swapped for the first)"""
    a, b = f0.double(), f1.double()
    C, HW = a.shape[1], a.shape[2] * a.shape[3]
    w64 = w.double().view(1, -1, 1, 1)
    aw = w64.abs()
    rho, rho0 = _rho(C), (C / 2 + 1) * U
    na0 = torch.linalg.vector_norm(a, dim=1, keepdim=True)
    nb0 = torch.linalg.vector_norm(b, dim=1, keepdim=True)
    na, nb = na0 + EPS, nb0 + EPS
    ah, bh = a / na, b / nb
    d = bh - ah
    T = (2 * w64 * d * b).sum(1, keepdim=True)
    sb = (aw * b * b).sum(1, keepdim=True) / nb
    sab = (aw * (a * b).abs()).sum(1, keepdim=True) / na
    eT = 2 * (CHUNK_SUM * U * (sb + sab) + rho * sb + rho * sab) + U * T.abs()
    den = nb * nb * nb0
    live = nb0 > 0
    k = torch.where(live, T / torch.where(live, den, 1.0), 0.0)
    ek = torch.where(live, (eT + (3 * U + 2 * rho + rho0) * T.abs()) / torch.where(live, den, 1.0), 0.0)
    ed = (rho + 2 * U) * (ah.abs() + bh.abs()) + U * d.abs()
    t1 = 2 * aw * d.abs() / nb
    e1 = 2 * aw / nb * (ed + (rho + U) * d.abs())
    t2 = b.abs() * k.abs()
    e2 = b.abs() * ek
    gs = (g.double() / HW).abs().view(-1, 1, 1, 1)
    bound = gs * (e1 + e2 + 4 * U * (t1 + t2))
    if bf16:
        o = gs * (2 * w64 * d / nb - b * k).abs()
        bound = bound + U16 * (o + bound)
    return K * bound


def lpips_evaluate(f0, f1, w, g, candidates, chunk_elems=2 ** 25, report=None):
    """max |candidate - reference| / budget per output ("val", "g0", "g1") for every candidate: name -> {output: tensor
    over the whole batch (any device)} or a callable (sample slice, reference dict) -> such a dict.  The samples go in
    chunks of <= chunk_elems map elements, so the fp64 intermediates of the training shapes stay a few GB.
    report: a dict that receives the relative error of each candidate's value (|err| / |ref|, max over images)."""
    B = f0.shape[0]
    per = f0[0].numel()
    step = max(1, chunk_elems // per)
    bf16 = f0.dtype == torch.bfloat16
    res = {name: {} for name in candidates}
    for s in range(0, B, step):
        sl = slice(s, min(B, s + step))
        a, b, gg = f0[sl], f1[sl], g[sl]
        ref = lpips_reference(a, b, w, gg)
        bud = {"val": lpips_value_budget(a, b, w), "g1": lpips_grad_budget(a, b, w, gg, bf16),
               "g0": lpips_grad_budget(b, a, w, gg, bf16)}
        for name, c in candidates.items():
            outs = c(sl, ref) if callable(c) else {k: v[sl] for k, v in c.items()}
            for key, v in outs.items():
                v = v.to(ref[key].device)
                res[name][key] = max(res[name].get(key, 0.0), ratio(v, ref[key], bud[key]))
                if report is not None and key == "val":
                    rel = float(((v.double() - ref["val"]).abs() / ref["val"].abs()).max())
                    report[name] = max(report.get(name, 0.0), rel)
        del ref, bud
    return res


def lpips_control(sl, ref, bf16):
    """the exact fp64 values rounded once to the output types"""
    gt = torch.bfloat16 if bf16 else torch.float32
    return {"val": ref["val"].float(), "g0": ref["g0"].to(gt), "g1": ref["g1"].to(gt)}


# ---- numpy model of the kernels' rounding points ---------------------------------------------------------------------
def _fma(x, y, z):
    """fp32 fused multiply-add (the product is exact in fp64; the sum is rounded to fp64, then to fp32)"""
    return (x.astype(np.float64) * y + z).astype(np.float32)


def _norm(s, mutant):
    if mutant == "eps_in_sqrt":
        return np.sqrt(s + EPS32)
    return np.sqrt(s) + EPS32


def _lp_sums(a, b, w, mutant):
    """pixel_sums: fp32 saa / sbb over all channels, fp32 chunk sums of LP_CHUNK channels folded into fp64"""
    B, C, P = a.shape
    saa, sbb = np.zeros((B, P), np.float32), np.zeros((B, P), np.float32)
    S = [np.zeros((B, P)) for _ in range(3)]
    last = (C - 1) // LP_CHUNK * LP_CHUNK
    for c0 in range(0, C, LP_CHUNK):
        if mutant == "partial_chunk" and C % LP_CHUNK and c0 == last:
            break
        ch = [np.zeros((B, P), np.float32) for _ in range(3)]
        for c in range(c0, min(C, c0 + LP_CHUNK)):
            ac, bc = a[:, c], b[:, c]
            wa, wb = w[c] * ac, w[c] * bc
            saa, sbb = _fma(ac, ac, saa), _fma(bc, bc, sbb)
            ch = [_fma(wa, ac, ch[0]), _fma(wb, bc, ch[1]), _fma(wa, bc, ch[2])]
        S = [S[i] + ch[i] for i in range(3)]
    return saa, sbb, S


def _lp_value(a, b, w, bf16, mutant):
    saa, sbb, (waa, wbb, wab) = _lp_sums(a, b, w, mutant)
    na, nb = _norm(saa, mutant).astype(np.float64), _norm(sbb, mutant).astype(np.float64)
    pix = waa / (na * na) + wbb / (nb * nb) - 2.0 * wab / (na * nb)
    P = a.shape[2]
    if mutant == "last_block":                     # the reduce stops one block short
        blk = LP_THREADS * (2 if bf16 else 1)
        pix[:, (P - 1) // blk * blk:] = 0
    return (pix.sum(1) / P).astype(np.float32)


def _lp_grad(a, b, w, g, bf16, mutant):
    """gradient of the second map"""
    B, C, P = a.shape
    saa, sbb, (waa, wbb, wab) = _lp_sums(a, b, w, None)
    nb0 = np.sqrt(sbb)
    na, nb = _norm(saa, mutant), _norm(sbb, mutant)
    tsum = (2.0 * (wbb / nb.astype(np.float64) - wab / na.astype(np.float64))).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        den = (na * na * nb0) if mutant == "kb_na" else (nb * nb * nb0)
        kb = np.where(nb0 > 0, tsum / den, np.float32(0)).astype(np.float32)
    if mutant == "no_kb":
        kb = np.zeros_like(kb)
    ra, rb = np.float32(1) / na, np.float32(1) / nb
    gsrc = np.full_like(g, g[0]) if mutant == "g0_all" else g
    gs = (gsrc / np.float32(P)).astype(np.float32)[:, None]
    out = np.empty_like(a)
    for c in range(C):
        ac, bc = a[:, c], b[:, c]
        d = _fma(bc, rb, -(ac * ra))
        t1 = (np.float32(2) * w[c] * d) * rb
        out[:, c] = gs * (t1 - bc * kb)
    if bf16:
        out = torch.from_numpy(out).to(torch.bfloat16).float().numpy()
        if mutant == "pair_swap":
            out = out.reshape(B, C, P // 2, 2)[..., ::-1].reshape(B, C, P)
    return out


def lpips_model(f0, f1, w, g, mutant=None):
    """the forward / backward kernels' rounding points on the given maps (torch, any device) -> {val, g0, g1} on CPU.
    bf16 maps of odd HW take the fp32 kernel, as the wrapper does."""
    B, C, H, W = f0.shape
    bf16 = f0.dtype == torch.bfloat16 and (H * W) % 2 == 0
    a = f0.float().cpu().numpy().reshape(B, C, H * W)
    b = f1.float().cpu().numpy().reshape(B, C, H * W)
    wn, gn = w.float().cpu().numpy(), g.float().cpu().numpy()
    out = {"val": _lp_value(a, b, wn, bf16, mutant),
           "g0": _lp_grad(b, a, wn, gn, bf16, mutant).reshape(B, C, H, W),
           "g1": _lp_grad(a, b, wn, gn, bf16, mutant).reshape(B, C, H, W)}
    return {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in out.items()}


# ======================================================================================================================
# DiffAug
# ======================================================================================================================
def flags3(flags):
    return (flags & 1, (flags >> 1) & 1, (flags >> 2) & 1)


def cut_size(H, W):
    return round(H * CUTOUT), round(W * CUTOUT)


def aug_params(rand01, flags, H, W, device="cpu"):
    """diffaug_params as torch tensors: th, tw, oh, ow (int64 [B]), br, sat, con (fp64 [B], the float32 values)"""
    th, tw, br, sat, con, oh, ow, ch, cw = lo.diffaug_params(np.asarray(rand01, np.float32), flags3(flags), H, W, CUTOUT)
    t = {k: torch.from_numpy(np.asarray(v)).to(device) for k, v in
         dict(th=th, tw=tw, oh=oh, ow=ow, br=br.astype(np.float64), sat=sat.astype(np.float64),
              con=con.astype(np.float64)).items()}
    t["ch"], t["cw"] = ch, cw
    return t


def translate(x, th, tw):
    """x[b, :, h + th_b, w + tw_b], zero outside: the reference's gather through a 1-pixel zero border"""
    B, C, H, W = x.shape
    pad = torch.nn.functional.pad(x, [1, 1, 1, 1])
    gh = (torch.arange(H, device=x.device)[None] + th[:, None] + 1).clamp(0, H + 1)
    gw = (torch.arange(W, device=x.device)[None] + tw[:, None] + 1).clamp(0, W + 1)
    bi = torch.arange(B, device=x.device).view(B, 1, 1, 1)
    ci = torch.arange(C, device=x.device).view(1, C, 1, 1)
    return pad[bi, ci, gh.view(B, 1, H, 1), gw.view(B, 1, 1, W)]


def cut_mask(p, H, W, device):
    """[B, 1, H, W] fp64: 0 on the cutout cells of the reference's clamped index grid, 1 elsewhere"""
    B = p["oh"].shape[0]
    ch, cw = p["ch"], p["cw"]
    gh = (torch.arange(ch, device=device)[None] + p["oh"][:, None] - ch // 2).clamp(0, H - 1)
    gw = (torch.arange(cw, device=device)[None] + p["ow"][:, None] - cw // 2).clamp(0, W - 1)
    m = torch.ones(B, H, W, dtype=torch.float64, device=device)
    m[torch.arange(B, device=device).view(B, 1, 1), gh.view(B, ch, 1), gw.view(B, 1, cw)] = 0
    return m[:, None]


def diffaug_reference(x, g, rand01, flags):
    """fp64 forward and its autograd backward -> (y, gx)"""
    B, C, H, W = x.shape
    p = aug_params(rand01, flags, H, W, x.device)
    xr = x.double().requires_grad_(True)
    t = translate(xr, p["th"], p["tw"]) if flags & 1 else xr
    if flags & 2:
        t = t + p["br"].view(B, 1, 1, 1)
        m = t.mean(1, keepdim=True)
        t = (t - m) * p["sat"].view(B, 1, 1, 1) + m
        M = t.mean((1, 2, 3), keepdim=True)
        t = (t - M) * p["con"].view(B, 1, 1, 1) + M
    if flags & 4:
        t = t * cut_mask(p, H, W, x.device)
    (gx,) = torch.autograd.grad(t, xr, g.double())
    return t.detach(), gx


def diffaug_budget(x, g, rand01, flags):
    """per-element budgets (y, gx); zero where the kernel must be exact (no colour, and the cut cells)"""
    B, C, H, W = x.shape
    p = aug_params(rand01, flags, H, W, x.device)
    if not flags & 2:
        return torch.zeros(x.shape, dtype=torch.float64, device=x.device), torch.zeros(x.shape, dtype=torch.float64, device=x.device)
    br, sat, con = (p[k].view(B, 1, 1, 1) for k in ("br", "sat", "con"))
    mask = cut_mask(p, H, W, x.device) if flags & 4 else torch.ones(B, 1, H, W, dtype=torch.float64, device=x.device)
    xt = translate(x.double(), p["th"], p["tw"]) if flags & 1 else x.double()
    # forward
    v = xt + br
    ev = U * v.abs()
    m = v.mean(1, keepdim=True)
    mv = v.abs().mean(1, keepdim=True)
    em = ev.mean(1, keepdim=True) + (C + 1) * U * mv
    t = (v - m) * sat + m
    et = sat.abs() * (ev + em + U * (v - m).abs()) + em + U * t.abs()
    S = xt.mean((1, 2, 3), keepdim=True)
    M = S + br
    eM = 3 * U * (S.abs() + M.abs()) + 2.0 ** -50 * xt.abs().mean((1, 2, 3), keepdim=True)
    y = (t - M) * con + M
    ey = con.abs() * (et + eM + U * (t - M).abs()) + eM + U * y.abs()
    # backward (output grid, then the translation's transpose = the opposite translation)
    gm = g.double() * mask
    gbar = gm.mean((1, 2, 3), keepdim=True)
    egb = 2 * U * gbar.abs() + 2.0 ** -50 * gm.abs().mean((1, 2, 3), keepdim=True)
    vb = con * gm + (1 - con) * gbar
    evb = U * (2 * (con * gm).abs() + 3 * ((1 - con) * gbar).abs() + vb.abs()) + (1 - con).abs() * egb
    mb = vb.mean(1, keepdim=True)
    emb = evb.mean(1, keepdim=True) + (C + 1) * U * vb.abs().mean(1, keepdim=True)
    gxs = sat * vb + (1 - sat) * mb
    eg = sat.abs() * evb + (1 - sat).abs() * emb + U * (2 * (sat * vb).abs() + 3 * ((1 - sat) * mb).abs() + gxs.abs())
    if flags & 1:
        eg = translate(eg, -p["th"], -p["tw"])
    return K * ey * mask, K * eg


def diffaug_model(x, g, rand01, flags, mutant=None):
    """diffaug_sum_kernel / diffaug_fwd_kernel / diffaug_bwd_kernel's fp32 rounding points -> (y, gx) fp32 CPU tensors"""
    x = x.float().cpu().numpy()
    g = g.float().cpu().numpy()
    B, C, H, W = x.shape
    th, tw, br, sat, con, oh, ow, ch, cw = lo.diffaug_params(np.asarray(rand01, np.float32), flags3(flags), H, W, CUTOUT)
    y, gx = np.zeros_like(x), np.zeros_like(g)
    hh, ww = np.arange(H)[:, None], np.arange(W)[None, :]
    CHW = np.float32(C * H * W)
    for b in range(B):
        sg = -1 if mutant == "trans_sign" else 1
        hs, ws = hh + sg * th[b], ww + sg * tw[b]
        inside = (hs >= 0) & (hs < H) & (ws >= 0) & (ws < W)
        xt = np.where(inside[None], x[b][:, hs.clip(0, H - 1), ws.clip(0, W - 1)], np.float32(0))
        h0, w0 = oh[b] - ch // 2, ow[b] - cw // 2
        if mutant == "cut_shifted":                # the hanging rectangle moved back inside instead of its cells clamped
            h0, w0 = min(max(h0, 0), H - ch), min(max(w0, 0), W - cw)
        a_h, b_h = min(max(h0, 0), H - 1), min(max(h0 + ch - 1, 0), H - 1)
        a_w, b_w = min(max(w0, 0), W - 1), min(max(w0 + cw - 1, 0), W - 1)
        cut = bool(flags & 4) & (hh >= a_h) & (hh <= b_h) & (ww >= a_w) & (ww <= b_w)
        # forward
        v = xt + br[b]
        if flags & 2:
            src = x[b] if mutant == "contrast_untranslated" else xt
            M = np.float32(np.float32(src.astype(np.float64).sum()) / CHW)
            if mutant != "contrast_no_br":
                M = M + br[b]
            m = np.zeros((H, W), np.float32)
            for c in range(C):
                m = m + v[c]
            m = m / np.float32(C)
            t = _fma(v - m, sat[b], m)
            v = _fma(t - M, con[b], M)
        y[b] = np.where(cut[None], np.float32(0), v)
        # backward: one thread per source pixel (hs, ws) reads the output pixel (hs - th, ws - tw)
        g3 = np.where(cut[None], np.float32(0), g[b])
        if flags & 2:
            gsum = g[b] if mutant == "gbar_unmasked" else g3
            gbar = np.float32(np.float32(gsum.astype(np.float64).sum()) / CHW)
            vb = _fma(con[b], g3, (np.float32(1) - con[b]) * gbar)
            mb = np.zeros((H, W), np.float32)
            for c in range(C):
                mb = mb + vb[c]
            mb = mb / np.float32(C)
            go = _fma(sat[b], vb, (np.float32(1) - sat[b]) * mb)
        else:
            go = g3
        oh_, ow_ = hh - sg * th[b], ww - sg * tw[b]
        read = (oh_ >= 0) & (oh_ < H) & (ow_ >= 0) & (ow_ < W)
        gather = go[:, oh_.clip(0, H - 1), ow_.clip(0, W - 1)]
        gx[b] = gather if mutant == "unread_nonzero" else np.where(read[None], gather, np.float32(0))
    return torch.from_numpy(y), torch.from_numpy(gx)


def edges_rand01(B, H, W, seed):
    """rand01 [7, B] float32 chosen per sample so that the batch covers th, tw in {-dh, -1, 0, 1, dh}; cutouts over
    each edge, each corner and fully inside; sat = 0 and ~2, con = 0.5 and ~1.5, br = -0.5 and ~+0.5 (and random)"""
    rng = np.random.default_rng(seed)
    r = rng.random((7, B)).astype(np.float64)
    dh, dw = round(H * 0.125), round(W * 0.125)
    ch, cw = cut_size(H, W)
    nh, nw = H + 1 - ch % 2, W + 1 - cw % 2

    def at(k, n):                                  # the middle of bin k of n
        return (k + 0.5) / n
    for i in range(B):
        tsel = (-dh, -1, 0, 1, dh)
        tsel_w = (-dw, -1, 0, 1, dw)
        r[0, i] = at(tsel[i % 5] + dh, 2 * dh + 1)
        r[1, i] = at(tsel_w[(i // 5) % 5] + dw, 2 * dw + 1)
        vh, vw = (0, H // 2, nh - 1), (0, W // 2, nw - 1)            # over the first edge, inside, over the last edge
        r[5, i] = at(vh[i % 3], nh)
        r[6, i] = at(vw[(i // 3) % 3], nw)
        r[2, i] = (0.0, 0.99995, r[2, i])[(i // 9) % 3]
        r[3, i] = (0.0, 0.9995, r[3, i])[i % 3]
        r[4, i] = (0.0, 0.9995, r[4, i])[(i // 3) % 3]
    return r.astype(np.float32)


def boundary_r(n, ulps=4):
    """every float32 r in [0, 1) within `ulps` ulps of a bin boundary k/n (k = 1 .. n-1) of floor(r * n)"""
    out = []
    for k in range(1, n):
        r = np.float32(k / n)
        lo_, hi_ = r, r
        cand = [r]
        for _ in range(ulps):
            lo_, hi_ = np.nextafter(lo_, np.float32(0)), np.nextafter(hi_, np.float32(1))
            cand += [lo_, hi_]
        out += [c for c in cand if 0 <= c < 1]
    return np.unique(np.asarray(out, np.float32))
