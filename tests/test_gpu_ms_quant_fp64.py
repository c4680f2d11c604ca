"""The multi-scale residual quantizers (csrc/ms_kernels.cu) against fp64 at the training shape.

Every case runs one training step of `VectorQuantizer2` or `LFQ` (soft entropy) at B = 128, v_patch_nums =
[1,1,2,3,3,4,5,6,8,11], with random Phi weights and biases, an explicit `dropout` in which every scale count from 1 to 10
occurs, and the loss  sum(out * g_out) + 1.3 vq + 0.7 commit (+ 1.1 entropy).  g_out is scaled by 1 / numel so that the
straight-through term does not drown the loss terms' share of f.grad: a term sent to the wrong place shows.

  indices    every scale of all 128 images equal, bit for bit, to the fp32 C oracle's (oracle/xq_oracle.py).  Inputs are
             screened image by image, as the goldens' seeds are, so that no top-2 margin of the oracle's search (VQ) and
             no |pooled residual| (LFQ signs) is below 1e-5; an image that has one is redrawn.
  values     out, every f_to_idxBl_or_fhat(to_fhat=True) entry, vq, commit and entropy against oracle/ms_ref64.py, the
             fp64 restatement fed the product's own indices.  ms_ref64 also checks those indices against its fp64
             residual: every VQ code is the fp64 best and every LFQ bit the fp64 sign, up to 1e-5.
  gradients  f.grad, embedding.weight.grad and every Phi weight.grad / bias.grad against torch.autograd of ms_ref64.
  batch      images 0..127 as one batch and as 64 batches of 2 with the same per-image n_quantizers: out, every scale's
             indices and every f_to_idxBl_or_fhat(to_fhat=True) entry are bitwise equal.

Bars, fixed before anything was measured: per tensor, normwise |x - x64| / |x64| <= 2e-5 and elementwise
|x - x64| <= 1e-4 max|x64|.  `pytest -s` prints, per case and tensor, both errors as a share of their bar.  Mutants
(fp64 gradients or forwards with one plausible bug, oracle/ms_ref64.MUTANTS) must exceed a bar or contradict the
product's indices; the printed margin is the largest share of a bar they reach.

Measured on an H100 80GB HBM3 (700 W power limit): the largest share of a bar over every tensor of every case is 0.19
(LFQ's entropy at C = 12, normwise 3.9e-6); every other tensor stays below 0.07, and the fp64 index gap is 0 in every
case.  Every gradient mutant exceeds a bar at least 2,600x (the transposed bicubic with align_corners=True, msvr_l2
being the closest); area_floor moves no value past its bar but contradicts the product's indices, its fp64 index gap
being at least 7e4 times the 1e-5 tie.  The file takes about 35 s and at most 1.3 GiB of extra device memory.

The shape ladder at the end measured: at C = 32 training runs up to a 13 x 13 last scale and the forward refuses 14 x 14
and 16 x 16, whose forward fits in shared memory (192 KB / 216 KB) but whose backward does not (239 KB / 288 KB).
"""
import functools
import time

import numpy as np
import pytest
import torch

from oracle import ms_ref64, xq_oracle as xo

pytestmark = pytest.mark.gpu

PN = [1, 1, 2, 3, 3, 4, 5, 6, 8, 11]
SN = len(PN)
B = 128
HW = PN[-1]
NORM_BAR, ELEM_BAR = 2e-5, 1e-4
TIE = 1e-5
W_VQ, W_COMMIT, W_ENT = 1.3, 0.7, 1.1

CASES = {
    "msvr4096": dict(lfq=False, C=32, V=4096, znorm=True, share=4, drop=0.1, seed=41),
    "msvr16384": dict(lfq=False, C=32, V=16384, znorm=True, share=4, drop=0.5, seed=42),
    "msvr_l2": dict(lfq=False, C=32, V=4096, znorm=False, share=1, drop=0.1, seed=43),
    "msbr4096": dict(lfq=True, C=12, V=4096, znorm=True, share=4, drop=0.1, seed=44),
    "msbr16384": dict(lfq=True, C=14, V=16384, znorm=True, share=4, drop=0.5, seed=45),
}
# LFQ codes are constants, so nothing flows back through its Phi input or bicubic upsample; with one Phi module the
# share map has nothing to shift
_VQ_MUTANTS = ["phi_r_twice", "phi_r_dropped", "share_map_shift", "nq_plus_one", "swap_vq_commit",
               "bicubic_T_align_corners", "area_floor"]
MUTANTS = {
    "msvr4096": _VQ_MUTANTS,
    "msvr16384": _VQ_MUTANTS,
    "msvr_l2": [m for m in _VQ_MUTANTS if m != "share_map_shift"],
    "msbr4096": ["share_map_shift", "nq_plus_one", "swap_vq_commit", "ent_row1_to_row0", "area_floor"],
    "msbr16384": ["share_map_shift", "nq_plus_one", "swap_vq_commit", "ent_row1_to_row0", "area_floor"],
}


def npy(t):
    return t.detach().cpu().numpy()


def _module(cfg, gen):
    from imagefolder_b200 import LFQ, VectorQuantizer2
    C = cfg["C"]
    kw = dict(v_patch_nums=PN, num_latent_tokens=HW * HW, share_quant_resi=cfg["share"], codebook_drop=cfg["drop"])
    if cfg["lfq"]:
        q = LFQ(cfg["V"], C, using_znorm=cfg["znorm"], entropy_weight=0.1, **kw)
    else:
        q = VectorQuantizer2(cfg["V"], C, using_znorm=cfg["znorm"], **kw)
    with torch.no_grad():
        if not cfg["lfq"]:
            q.embedding.weight.copy_(torch.randn(cfg["V"], C, generator=gen) * 0.5)
        for m in q.quant_resi.modules_list():
            m.weight.copy_(torch.randn(m.weight.shape, generator=gen) * 0.06)
            m.bias.copy_(torch.randn(C, generator=gen) * 0.1)
    return q.cuda().train()


def _oracle(cfg, q, f):
    """fp32 C oracle on f[n]: (per-scale indices, per-image smallest margin)."""
    mods = q.quant_resi.modules_list()
    w, b = np.stack([npy(m.weight) for m in mods]), np.stack([npy(m.bias) for m in mods])
    n = f.shape[0]
    if not cfg["lfq"]:
        fw = xo.vq2_forward(f, npy(q.embedding.weight), w, b, PN, using_znorm=cfg["znorm"])
        margin = np.min([fw["margins"][si].min(axis=1) for si in range(SN)], axis=0)
        return fw["idx"], margin
    fw = xo.lfq_forward(f, w, b, PN, using_znorm=cfg["znorm"], scaler=npy(q.scaler))
    rest = fw["fn"].astype(np.float32).copy()
    margin = np.full(n, np.inf)
    for si, p in enumerate(PN):
        rows = np.abs(xo.area_pool_rows(rest, p)).reshape(n, -1)
        margin = np.minimum(margin, rows.min(axis=1))
        rest = (rest - fw["h"][si]).astype(np.float32)
    return fw["idx"], margin


def _screened_input(cfg, q, gen):
    """f [B,C,H,W] whose every image is clear of oracle near-ties (an image that has one is redrawn)."""
    C = cfg["C"]
    f = torch.randn(B, C, HW, HW, generator=gen).numpy()
    idx = [np.empty((B, p * p), np.int64) for p in PN]
    todo = np.arange(B)
    for _ in range(50):
        ix, margin = _oracle(cfg, q, f[todo])
        for si in range(SN):
            idx[si][todo] = ix[si]
        todo = todo[margin <= TIE]
        if len(todo) == 0:
            return f, idx
        f[todo] = torch.randn(len(todo), C, HW, HW, generator=gen).numpy()
    raise AssertionError("could not draw images clear of near-ties")


@functools.lru_cache(maxsize=None)
def _case(name):
    """the product's training step on the case's inputs, and everything the checks need"""
    cfg = CASES[name]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mem0 = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    gen = torch.Generator().manual_seed(cfg["seed"])
    q = _module(cfg, gen)
    f, idx_oracle = _screened_input(cfg, q, gen)
    nd = int(B * cfg["drop"])
    dropout = torch.randint(1, SN + 1, (B,), generator=gen)
    dropout[:SN] = torch.randperm(SN, generator=gen) + 1          # every scale count 1..10 among the dropped samples
    assert nd >= SN
    g_out = torch.randn(B, cfg["C"], HW, HW, generator=gen) / f.size
    ft = torch.from_numpy(f).cuda().requires_grad_(True)
    out, _, vq, commit, ent = q(ft, dropout=dropout)
    idx = [t.clone() for t in q.last_idx_Bl]
    loss = (out * g_out.cuda()).sum() + W_VQ * vq + W_COMMIT * commit + (W_ENT * ent if cfg["lfq"] else 0.0)
    loss.backward()
    mods = q.quant_resi.modules_list()
    prod = dict(out=out.detach(), vq=vq.detach(), commit=commit.detach(), f=ft.grad.clone(),
                phi_w=[m.weight.grad.clone() for m in mods], phi_b=[m.bias.grad.clone() for m in mods],
                fhat=q.f_to_idxBl_or_fhat(ft.detach(), to_fhat=True), idx=idx)
    if cfg["lfq"]:
        prod["entropy"] = ent.detach()
    else:
        prod["E"] = q.embedding.weight.grad.clone()
    nq = ms_ref64.n_quantizers(B, SN, cfg["drop"], dropout.numpy())
    return dict(cfg=cfg, q=q, f=f, idx_oracle=idx_oracle, nq=nq, g_out=g_out, prod=prod,
                setup_s=time.perf_counter() - t0, mem0=mem0)


def _ref64(c, mutant=None):
    cfg, q = c["cfg"], c["q"]
    mods = q.quant_resi.modules_list()
    leaf = lambda t: t.detach().double().requires_grad_(True)
    wrt = dict(f=leaf(torch.from_numpy(c["f"]).cuda()), phi_w=leaf(torch.stack([m.weight for m in mods])),
               phi_b=leaf(torch.stack([m.bias for m in mods])))
    kw = dict(phi_w=wrt["phi_w"], phi_b=wrt["phi_b"], nq=c["nq"], using_znorm=cfg["znorm"], mutant=mutant)
    if cfg["lfq"]:
        kw.update(scaler=[float(s) for s in q.scaler.tolist()], entropy_weight=0.1)
    else:
        kw["E"] = wrt["E"] = leaf(q.embedding.weight)
    fwd = ms_ref64.forward(wrt["f"], c["prod"]["idx"], PN, lfq=cfg["lfq"], **kw)
    gr = ms_ref64.losses_and_grads(fwd, wrt, c["g_out"].cuda().double(), W_VQ, W_COMMIT,
                                   W_ENT if cfg["lfq"] else 0.0, mutant=mutant)
    return fwd, gr


def _shares(x, x64):
    """(normwise error / its bar, elementwise error / its bar)"""
    x, x64 = x.detach().double(), x64.detach().double()
    d = (x - x64).abs()
    ref = float(x64.abs().max())
    if ref == 0:                          # a Phi module no scale uses: its gradient must be exactly zero
        return (0.0, 0.0) if float(d.max()) == 0 else (float("inf"), float("inf"))
    return float((x - x64).norm() / x64.norm()) / NORM_BAR, float(d.max()) / (ELEM_BAR * ref)


def _compare(c, fwd, gr):
    """[(tensor name, normwise share, elementwise share)] for every value and gradient the quantizer owns"""
    p, rows = c["prod"], []
    names = ["out", "vq", "commit"] + (["entropy"] if c["cfg"]["lfq"] else [])
    for n in names:
        rows.append((n,) + _shares(p[n], fwd[n]))
    for si in range(SN):
        rows.append((f"fhat[{si}]",) + _shares(p["fhat"][si], fwd["fhat"][si]))
    rows.append(("f.grad",) + _shares(p["f"], gr["f"]))
    if not c["cfg"]["lfq"]:
        rows.append(("embedding.grad",) + _shares(p["E"], gr["E"]))
    for k in range(len(p["phi_w"])):
        rows.append((f"phi[{k}].weight.grad",) + _shares(p["phi_w"][k], gr["phi_w"][k]))
        rows.append((f"phi[{k}].bias.grad",) + _shares(p["phi_b"][k], gr["phi_b"][k]))
    return rows


@pytest.mark.parametrize("name", list(CASES))
def test_indices_of_every_image_match_the_oracle(name):
    c = _case(name)
    for si in range(SN):
        np.testing.assert_array_equal(npy(c["prod"]["idx"][si]), c["idx_oracle"][si], err_msg=f"scale {si}")


@pytest.mark.parametrize("name", list(CASES))
def test_values_and_gradients_against_fp64(name):
    c = _case(name)
    t0 = time.perf_counter()
    fwd, gr = _ref64(c)
    rows = _compare(c, fwd, gr)
    print(f"\n{name}: setup {c['setup_s']:.1f} s, fp64 {time.perf_counter() - t0:.1f} s, index gap {fwd['idx_gap']:.1e}, "
          f"peak extra {(torch.cuda.max_memory_allocated() - c['mem0']) / 2 ** 30:.2f} GiB")
    for n, a, e in rows:
        print(f"  {n:22s} normwise {a * NORM_BAR:.2e} ({a:.3f} of bar)   elementwise {e * ELEM_BAR:.2e} ({e:.3f})")
    worst = max(max(a, e) for _, a, e in rows)
    print(f"  worst share of a bar: {worst:.3f}")
    assert fwd["idx_gap"] <= TIE, f"product index is not the fp64 choice (gap {fwd['idx_gap']:.2e})"
    bad = [(n, a, e) for n, a, e in rows if a > 1 or e > 1]
    assert not bad, bad


@pytest.mark.parametrize("name", list(CASES))
def test_mutants_fail_the_bar(name):
    c = _case(name)
    print()
    for mut in MUTANTS[name]:
        fwd, gr = _ref64(c, mut)
        rows = _compare(c, fwd, gr)
        n, a, e = max(rows, key=lambda r: max(r[1], r[2]))
        gap = fwd["idx_gap"] / TIE
        print(f"  {name} {mut:24s} largest share of a bar {max(a, e):10.1f} ({n}), index gap / tie {gap:.1f}")
        assert max(a, e, gap) > 1, f"mutant {mut} passes"


@pytest.mark.parametrize("name", list(CASES))
def test_batch_of_128_equals_64_batches_of_2(name):
    c = _case(name)
    q, p = c["q"], c["prod"]
    f = torch.from_numpy(c["f"]).cuda()
    drop = q.codebook_drop
    q.codebook_drop = 1.0                 # every sample of a pair takes its n_quantizers from `dropout`
    try:
        with torch.no_grad():
            for i in range(0, B, 2):
                out, _, _, _, _ = q(f[i:i + 2], dropout=c["nq"][i:i + 2])
                assert torch.equal(out, p["out"][i:i + 2]), f"out of images {i}, {i + 1}"
                for si in range(SN):
                    assert torch.equal(q.last_idx_Bl[si], p["idx"][si][i:i + 2]), f"images {i}, {i + 1} scale {si}"
                fh = q.f_to_idxBl_or_fhat(f[i:i + 2], to_fhat=True)
                for si in range(SN):
                    assert torch.equal(fh[si], p["fhat"][si][i:i + 2]), f"f_hat of images {i}, {i + 1} scale {si}"
    finally:
        q.codebook_drop = drop


# ------------------------------------------------------------------------------------------------------------------
# forward and backward accept the same shapes
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,last", [(32, 12), (32, 13), (32, 14), (32, 16), (24, 16), (48, 11)])
def test_training_forward_never_outruns_its_backward(C, last):
    """Around the shared-memory limit of one image's CTA: the train-mode forward either refuses up front, naming the
    shape, or forward and backward both run and match the oracle (indices bit for bit) and fp64 (values, gradients).
    A forward that succeeds and a backward that then refuses is the failure this guards against."""
    from imagefolder_b200 import VectorQuantizer2
    from imagefolder_b200._capi import XqError
    pn = [1, 2, 3, last]
    V, Bs = 512, 2
    gen = torch.Generator().manual_seed(100 * C + last)
    q = VectorQuantizer2(V, C, v_patch_nums=pn, num_latent_tokens=last * last, share_quant_resi=4)
    with torch.no_grad():
        q.embedding.weight.copy_(torch.randn(V, C, generator=gen) * 0.5)
        for m in q.quant_resi.modules_list():
            m.weight.copy_(torch.randn(m.weight.shape, generator=gen) * 0.06)
            m.bias.copy_(torch.randn(C, generator=gen) * 0.1)
    q = q.cuda().train()
    ft = torch.randn(Bs, C, last, last, generator=gen).cuda().requires_grad_(True)
    try:
        out, _, vq, commit, _ = q(ft)
    except XqError as e:
        print(f"\nC = {C}, {last} x {last}: refused: {e}")
        assert "unsupported" in str(e) and f"C = {C}" in str(e) and f"{last} x {last}" in str(e), str(e)
        return
    g_out = torch.randn(out.shape, generator=gen).cuda() / out.numel()
    ((out * g_out).sum() + W_VQ * vq + W_COMMIT * commit).backward()   # must not refuse
    print(f"\nC = {C}, {last} x {last}: forward and backward run")
    mods = q.quant_resi.modules_list()
    w = np.stack([npy(m.weight) for m in mods])
    b = np.stack([npy(m.bias) for m in mods])
    fw = xo.vq2_forward(npy(ft), npy(q.embedding.weight), w, b, pn)
    margin = min(float(m.min()) for m in fw["margins"])
    if margin > TIE:                      # index equality is only defined away from near-ties
        for si in range(len(pn)):
            np.testing.assert_array_equal(npy(q.last_idx_Bl[si]), fw["idx"][si])
    leaf = lambda t: t.detach().double().requires_grad_(True)
    wrt = dict(f=leaf(ft), E=leaf(q.embedding.weight), phi_w=leaf(torch.stack([m.weight for m in mods])),
               phi_b=leaf(torch.stack([m.bias for m in mods])))
    r = ms_ref64.forward(wrt["f"], q.last_idx_Bl, pn, lfq=False, E=wrt["E"], phi_w=wrt["phi_w"], phi_b=wrt["phi_b"])
    gr = ms_ref64.losses_and_grads(r, wrt, g_out.double(), W_VQ, W_COMMIT)
    assert r["idx_gap"] <= TIE
    for x, x64 in [(out, r["out"]), (vq, r["vq"]), (commit, r["commit"]), (ft.grad, gr["f"]),
                   (q.embedding.weight.grad, gr["E"])] + \
            [(m.weight.grad, gr["phi_w"][k]) for k, m in enumerate(mods)] + \
            [(m.bias.grad, gr["phi_b"][k]) for k, m in enumerate(mods)]:
        a, e = _shares(x, x64)
        assert a <= 1 and e <= 1, (a, e)
