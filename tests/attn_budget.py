"""fp64 reference, per-element error budgets, constructed inputs and named mutants for the wgmma attention kernels
(imagefolder_b200/csrc/attn_kernel.cu) (TEST INFRASTRUCTURE ONLY).

Reference: the op of the 16-bit inputs exactly as given, in fp64 (natural-log scores, scale = 0.125):
    S = q k^T scale,  P = softmax(S),  O = P v,  L2 = log2 sum exp2(S / ln 2)
    dP = dO v^T,  delta = rowsum(O o dO),  dS = P o (dP - delta),  dQ = scale dS k,  dK = scale dS^T q,  dV = P^T dO

Budgets.  Each bound below is the first-order worst case of the rounding points the kernels have, read off the code;
the asserted budget is K = 2 times it, so that an exact model of those rounding points (`emulate`) sits at <= 1/2 of it.
u is the unit roundoff of the 16-bit type (2^-8 bf16, 2^-11 f16).
  forward (attn_fwd_kernel): P is rounded to 16 bits relative to the running maximum of its 128-key block, l sums the
    unrounded fp32 p, O = o / l is rounded once:   |O_kernel - O| <= (u + rho + gam) (P|v| + |O|)
  lse: fp32 scores, the fp32 sum of N terms, the block rescales and log2f: no 16-bit rounding at all.
  backward (attn_bwd_kernel): P is recomputed from the kernel's L2 (within its budget) and rounded; delta comes from the
    kernel's rounded O (prep kernel), so the forward budget enters as sum_d budget(O)|dO|; dS = round(P (dP - delta));
    dK / dV are fp32 MMA sums rounded once, dQ goes through fp32 atomics and is rounded in attn_dq_convert_kernel.  The
    error matrix of dS propagates to dQ / dK through |k| / |q|, the one of P to dV through |dO|, as fp64 matmuls.
  trailing keys (attn_bwd_prep_kernel<E, 1..4>: N mod 128 in 1..4, N > 128): p and dS stay fp32, inside the same budget.
rho (per query row) is the relative error of an fp32 exponential: the score error of a 64-term fp32 dot product
(|q| |k| 2^-17, the sum may truncate), the fp32 rounding of the exponent argument, of m c / L2 and of c, and ex2.approx.
gam = (N + 2 nK + 64) 2^-23 is an fp32 sum over the keys (or queries) with its per-block rescales.
f16 adds an absolute floor for subnormal P and dS (spacing 2^-24 below 2^-14); bf16's floor is the ftz of ex2.approx.

Mutants are named, plausible kernel bugs written as fp64 functions of the same inputs; each must exceed the budget on
the input family built for it.  `control` (delta from the fp64 O instead of the kernel's rounded O) must not: it shows
the budget is not an identity check on one rounding sequence.
"""
from __future__ import annotations

import math

import torch

SCALE = 0.125
LN2 = math.log(2.0)
C2 = SCALE / LN2                        # c = scale log2(e): natural scores -> base-2 exponents
BK = 128                                # keys per block of attn_fwd_kernel / attn_bwd_kernel
KTAIL_MAX = 4                           # trailing keys attn_bwd_prep_kernel handles on CUDA cores
K_HEADROOM = 2.0
SUM64 = 2.0 ** -17                      # a 64-term fp32 dot product: 64 x 2^-23
U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
# (absolute error of one rounding at the bottom of the range, magnitude below which it can occur)
FLOOR = {torch.bfloat16: (2.0 ** -126, 2.0 ** -125), torch.float16: (2.0 ** -25, 2.0 ** -13)}
OUTS = ("O", "L2", "dQ", "dK", "dV")
FAMILIES = ("gauss1", "gauss2.5", "neg", "max_last", "max_first", "tail", "onehot")


def ktail(N: int) -> int:
    """keys attn_bwd_prep_kernel takes instead of a tensor-core key block (0 = none)"""
    r = N % BK
    return r if (N > BK and 0 < r <= KTAIL_MAX) else 0


# ---- layouts ---------------------------------------------------------------------------------------------------------
def pairs(qkv, H):
    """packed projection [B, N, 3*H*64] -> q, k, v as [B*H, N, 64]"""
    B, N, _ = qkv.shape
    x = qkv.reshape(B, N, 3, H, 64).permute(2, 0, 3, 1, 4).reshape(3, B * H, N, 64)
    return x[0], x[1], x[2]


def heads(t, H):
    """[B, N, H*64] -> [B*H, N, 64]"""
    B, N, _ = t.shape
    return t.reshape(B, N, H, 64).transpose(1, 2).reshape(B * H, N, 64)


def kernel_outputs(out, lse2, dqkv, H):
    """the kernels' results in the reference's [B*H, N, ...] layout"""
    B, N, _ = out.shape
    dq, dk, dv = pairs(dqkv, H)
    return {"O": heads(out, H), "L2": lse2.reshape(B * H, N), "dQ": dq, "dK": dk, "dV": dv}


# ---- inputs ------------------------------------------------------------------------------------------------------------
def make_inputs(family, B, N, H, dtype, seed, device="cpu"):
    """(qkv [B, N, 3*H*64], dO [B, N, H*64]) in `dtype`, generated from `seed`:
      gauss1 / gauss2.5  i.i.d. Gaussian q, k, v at that amplitude
      neg        every real score <= -12 (q ~ +a d, k ~ -a d): a zero-filled key past N would carry >= 99 % of the weight
      max_last   each row's maximum is a key of the last (partial) key block, 20+ above the rest: every earlier block
                 is rescaled by alpha ~ 0
      max_first  the mirror: the maximum in block 0
      tail       the trailing min(4, N) keys (the prep kernel's keys when N mod 128 is 1..4) take most of the weight of
                 every even-numbered query, so the prep kernel's dK / dV rows and the dQ fold carry O(1) of the gradient
      onehot     near one-hot rows: each query is a multiple of one key, ~10 above the rest"""
    g = torch.Generator(device=device).manual_seed(seed)

    def rn(*s):
        return torch.randn(*s, generator=g, device=device, dtype=torch.float64)

    def unit(n):
        d = rn(n, 64)
        return d / d.norm(dim=-1, keepdim=True)

    BH = B * H
    dO = rn(BH, N, 64)
    v = rn(BH, N, 64)
    if family in ("gauss1", "gauss2.5"):
        amp = 1.0 if family == "gauss1" else 2.5
        q, k, v = rn(BH, N, 64) * amp, rn(BH, N, 64) * amp, v * amp
    elif family == "neg":
        d = unit(BH)[:, None]
        q = 12.0 * d + 0.25 * rn(BH, N, 64)
        k = -12.0 * d + 0.25 * rn(BH, N, 64)
    elif family in ("max_last", "max_first"):
        d = unit(BH)[:, None]
        q = 8.0 * d + 0.3 * rn(BH, N, 64)
        k = 0.5 * rn(BH, N, 64)
        lo = (N - 1) // BK * BK if family == "max_last" else 0
        hi = N if family == "max_last" else min(N, BK)
        j = torch.randint(lo, hi, (BH,), generator=g, device=device)
        k[torch.arange(BH, device=device), j] = 26.0 * d[:, 0]
    elif family == "tail":
        nt = ktail(N) or min(KTAIL_MAX, N)
        d = unit(BH * nt).reshape(BH, nt, 64)
        q, k = rn(BH, N, 64), rn(BH, N, 64)
        k[:, N - nt:] = 2.0 * (math.log(N) + 1.0) * d + 0.1 * rn(BH, nt, 64)
        t = torch.randint(0, nt, (BH, N), generator=g, device=device)
        cap = (torch.arange(N, device=device) % 2 == 0).expand(BH, N)          # every other query is captured
        dq = torch.gather(d, 1, t[..., None].expand(BH, N, 64))
        q = torch.where(cap[..., None], 4.0 * dq + 0.5 * rn(BH, N, 64), q)
    elif family == "onehot":
        k = rn(BH, N, 64)
        j = torch.randint(0, N, (BH, N), generator=g, device=device)
        q = 1.25 * torch.gather(k, 1, j[..., None].expand(BH, N, 64)) + 0.2 * rn(BH, N, 64)
    else:
        raise ValueError(family)
    q, k, v, dO = (t.to(dtype) for t in (q, k, v, dO))
    qkv = torch.stack([t.reshape(B, H, N, 64) for t in (q, k, v)], 0).permute(1, 3, 0, 2, 4).reshape(B, N, 3 * H * 64)
    g_out = dO.reshape(B, H, N, 64).transpose(1, 2).reshape(B, N, H * 64)
    return qkv.contiguous(), g_out.contiguous()


# ---- fp64 reference ----------------------------------------------------------------------------------------------------
def reference(q, k, v, dO):
    """fp64 [n, N, 64] tensors -> the op and its analytic backward (plus the intermediates the budget needs)"""
    S = (q @ k.mT) * SCALE
    m = S.amax(-1, keepdim=True)
    E = torch.exp(S - m)
    l = E.sum(-1, keepdim=True)
    P = E / l
    O = P @ v
    dP = dO @ v.mT
    delta = (O * dO).sum(-1, keepdim=True)
    dS = P * (dP - delta)
    return {"S": S, "P": P, "dP": dP, "delta": delta, "dS": dS, "O": O, "L2": ((m + torch.log(l)) / LN2)[..., 0],
            "dQ": SCALE * (dS @ k), "dK": SCALE * (dS.mT @ q), "dV": P.mT @ dO}


def budget(r, q, k, v, dO, dtype):
    """per-element budgets of O, L2, dQ, dK, dV (see the module docstring)"""
    N = q.shape[1]
    u = U[dtype]
    f, thr = FLOOR[dtype]
    nK = (N + BK - 1) // BK
    gam = (N + 2 * nK + 64) * 2.0 ** -23
    P, S, O, L2 = r["P"], r["S"], r["O"], r["L2"]
    av, adO = v.abs(), dO.abs()
    # relative error of one fp32 exp2, per query row
    kmax = k.norm(dim=-1).amax(-1, keepdim=True)
    smax = S.abs().amax(-1)
    rho = SUM64 * SCALE * q.norm(dim=-1) * kmax + 2.0 ** -22 * (2 * C2 * smax + L2.abs() + 1)
    M = (P < thr).to(P.dtype)
    small = dtype == torch.float16                       # bf16: M <= 1 is bound enough for an ftz floor of 2^-126
    Pv = P @ av
    Mv = (M @ av) if small else av.sum(-2, keepdim=True)
    bO = (u + rho + gam)[..., None] * (Pv + O.abs()) + f * Mv + f
    bL = (rho + gam + nK * 2.0 ** -21 * (1 + 2 * C2 * smax)) / LN2 + 2.0 ** -22 * (L2.abs() + math.log2(N) + 2)
    BO, BL = K_HEADROOM * bO, K_HEADROOM * bL
    # backward: P from the kernel's L2 (within BL), delta from the kernel's O (within BO)
    rho_b = rho + LN2 * BL
    e_delta = (BO * adO).sum(-1) + SUM64 * ((O.abs() + BO) * adO).sum(-1)
    x = (r["dP"] - r["delta"]).abs()
    e1 = SUM64 * dO.norm(dim=-1)[..., None] * v.norm(dim=-1)[:, None, :] + e_delta[..., None]
    E = (2 * u + rho_b)[..., None] * P * x + (1 + 3 * u) * P * e1 + f * (M * (x + e1) + 1)
    G = E + gam * (r["dS"].abs() + E)
    w = (u + rho_b + gam)[..., None] * adO
    Mdo = (M.mT @ adO) if small else adO.sum(-2, keepdim=True)
    bV = P.mT @ w + f * Mdo + u * r["dV"].abs() + f
    bK = SCALE * (G.mT @ q.abs()) + u * r["dK"].abs() + f
    bQ = SCALE * (G @ k.abs()) + u * r["dQ"].abs() + f
    return {"O": BO, "L2": BL, "dQ": K_HEADROOM * bQ, "dK": K_HEADROOM * bK, "dV": K_HEADROOM * bV}


# ---- CPU model of the kernels' rounding sequence ----------------------------------------------------------------------
def _r32(x):
    return x.float().double()


C32 = float(torch.tensor(1.4426950408889634, dtype=torch.float32)) * SCALE      # the kernels' fp32 c


def emulate(q, k, v, dO, dtype, delta_from=None):
    """attn_fwd_kernel / attn_bwd_prep_kernel / attn_bwd_kernel / attn_dq_convert_kernel with every 16-bit and fp32
    rounding point named in the module docstring; sums in fp64.  delta_from: an O to take delta from instead of the
    rounded one (the control mutant)."""
    def r16(t):
        return t.to(dtype).double()

    N = k.shape[1]
    s = _r32(q @ k.mT)                                   # fp32 scores (unscaled)
    m = torch.full(s.shape[:-1] + (1,), -math.inf, dtype=s.dtype, device=s.device)
    l = torch.zeros_like(m)
    o = torch.zeros_like(q)
    for j in range(0, N, BK):
        sb = s[..., j:j + BK]
        mn = torch.maximum(m, sb.amax(-1, keepdim=True))
        alpha = _r32(torch.exp2(_r32((m - mn) * C32)))
        p = _r32(torch.exp2(_r32(sb * C32 - _r32(mn * C32))))
        l = l * alpha + p.sum(-1, keepdim=True)          # unrounded p
        o = o * alpha + r16(p) @ v[:, j:j + BK]          # P rounded to 16 bits for P V
        m = mn
    O = r16(o / l)
    L2 = _r32(m * C32 + torch.log2(l))
    delta = _r32(((O if delta_from is None else delta_from) * dO).sum(-1, keepdim=True))
    P = _r32(torch.exp2(_r32(s * C32 - L2)))
    nt = ktail(N)
    Pr = r16(P)
    dS = _r32(Pr * (_r32(dO @ v.mT) - delta))
    dSr = r16(dS)
    if nt:                                               # prep kernel: p and dS stay fp32
        Pr[..., N - nt:] = P[..., N - nt:]
        dSr[..., N - nt:] = dS[..., N - nt:]
    return {"O": O, "L2": L2[..., 0], "dQ": r16(SCALE * (dSr @ k)), "dK": r16(SCALE * (dSr.mT @ q)), "dV": r16(Pr.mT @ dO)}


def emulated(c):
    """emulate() as an evaluate() candidate"""
    return emulate(c.q, c.k, c.v, c.dO, c.dtype)


# ---- mutants -----------------------------------------------------------------------------------------------------------
def mut_leaked_key(c):
    """one zero-filled key past N let into the softmax"""
    z = torch.zeros_like(c.k[:, :1])
    r = reference(c.q, torch.cat([c.k, z], 1), torch.cat([c.v, z], 1), c.dO)
    return {"O": r["O"], "L2": r["L2"], "dQ": r["dQ"], "dK": r["dK"][:, :-1], "dV": r["dV"][:, :-1]}


def mut_dropped_key(c):
    """the last key masked out"""
    N = c.k.shape[1]
    if N < 2:
        return None
    r = reference(c.q, c.k[:, :-1], c.v[:, :-1], c.dO)
    z = torch.zeros_like(c.k[:, :1])
    return {"O": r["O"], "L2": r["L2"], "dQ": r["dQ"], "dK": torch.cat([r["dK"], z], 1), "dV": torch.cat([r["dV"], z], 1)}


def mut_no_l_rescale(c):
    """online softmax without `l *= alpha` when a later key block raises the row maximum"""
    S = (c.q @ c.k.mT) * SCALE
    N = S.shape[-1]
    m = torch.full(S.shape[:-1] + (1,), -math.inf, dtype=S.dtype, device=S.device)
    l = torch.zeros_like(m)
    o = torch.zeros_like(c.q)
    for j in range(0, N, BK):
        mn = torch.maximum(m, S[..., j:j + BK].amax(-1, keepdim=True))
        p = torch.exp(S[..., j:j + BK] - mn)
        l = l + p.sum(-1, keepdim=True)
        o = o * torch.exp(m - mn) + p @ c.v[:, j:j + BK]
        m = mn
    return {"O": o / l, "L2": ((m + torch.log(l)) / LN2)[..., 0]}


def mut_no_tail_dq_fold(c):
    """attn_dq_convert_kernel without dQ += sum_t dS[q][t] k_t for the prep kernel's trailing keys"""
    N = c.k.shape[1]
    nt = ktail(N)
    if not nt:
        return None
    return {"dQ": c.ref["dQ"] - SCALE * (c.ref["dS"][..., N - nt:] @ c.k[:, N - nt:])}


def mut_tail_dk_unscaled(c):
    """the prep kernel's dK rows written without `scale`"""
    N = c.k.shape[1]
    nt = ktail(N)
    if not nt:
        return None
    dK = c.ref["dK"].clone()
    dK[:, N - nt:] /= SCALE
    return {"dK": dK}


def control(c):
    """the kernels' rounding sequence with delta from the fp64 O instead of the rounded O: must stay inside the budget"""
    return emulate(c.q, c.k, c.v, c.dO, c.dtype, delta_from=c.ref["O"])


MUTANTS = {"leaked_key": mut_leaked_key, "dropped_key": mut_dropped_key, "no_l_rescale": mut_no_l_rescale,
           "no_tail_dq_fold": mut_no_tail_dq_fold, "tail_dk_unscaled": mut_tail_dk_unscaled}
# the family each mutant is built to be caught on, and the lengths where the bug exists
MUTANT_FAMILY = {"leaked_key": ("neg", lambda N: True), "dropped_key": ("tail", lambda N: N >= 2),
                 "no_l_rescale": ("max_last", lambda N: N > BK), "no_tail_dq_fold": ("tail", lambda N: ktail(N) > 0),
                 "tail_dk_unscaled": ("tail", lambda N: ktail(N) > 0)}


# ---- evaluation --------------------------------------------------------------------------------------------------------
class Ctx:
    def __init__(self, sl, q, k, v, dO, ref, dtype):
        self.sl, self.q, self.k, self.v, self.dO, self.ref, self.dtype = sl, q, k, v, dO, ref, dtype


def evaluate(qkv, g, H, candidates, chunk_elems=2 ** 24, colsums=False):
    """max |candidate - reference| / budget per output, for every candidate: name -> fn(Ctx) -> {output: fp64 tensor}
    (or None: not applicable).  The (batch, head) pairs go in chunks of <= chunk_elems score elements, so that the
    training shapes fit in a few GB.  Ratios are inf where a candidate is not finite.
    colsums: also return the reference's and the budget's column sums over (batch, token) of dQ / dK / dV ([3, H, 64]),
    for the qkv-bias gradient."""
    dtype = qkv.dtype
    q, k, v = pairs(qkv, H)
    dO = heads(g, H)
    BH, N = q.shape[:2]
    step = max(1, chunk_elems // (N * N))
    res = {name: {} for name in candidates}
    cs_ref = torch.zeros(3, BH, 64, dtype=torch.float64, device=qkv.device)
    cs_bud = torch.zeros_like(cs_ref)
    for s in range(0, BH, step):
        sl = slice(s, min(BH, s + step))
        c = [t[sl].double() for t in (q, k, v, dO)]
        ref = reference(*c)
        bud = budget(ref, *c, dtype)
        ctx = Ctx(sl, *c, ref, dtype)
        for name, fn in candidates.items():
            outs = fn(ctx)
            if outs is None:
                continue
            for key, val in outs.items():
                ratio = ((val.double() - ref[key]).abs() / bud[key]).nan_to_num(nan=math.inf).max().item()
                res[name][key] = max(res[name].get(key, 0.0), ratio)
        if colsums:
            for i, key in enumerate(("dQ", "dK", "dV")):
                cs_ref[i, sl] = ref[key].sum(1)
                cs_bud[i, sl] = bud[key].sum(1)
        del ref, bud, ctx, c
    if colsums:
        B = BH // H
        return res, cs_ref.reshape(3, B, H, 64).sum(1), cs_bud.reshape(3, B, H, 64).sum(1)
    return res
