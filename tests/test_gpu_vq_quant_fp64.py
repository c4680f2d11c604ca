"""The single-scale quantizer (csrc/vq_kernels.cu, the tensor-core search of csrc/vq_tc_kernel.cu) and RobustTok's
latent perturbation against fp64 at the training batch.

Every case runs one training step at B = 128 with 16 x 16 latents (N = 32768 rows) and the loss
sum(out * g_out) + 1.3 vq + 0.7 commit, g_out scaled by 1 / numel so that the straight-through term does not drown the
loss terms' share of dz.  The codebook is drawn the reference way (uniform +-1/V, normalised), except in vq4096_l2,
whose codes are 0.5 randn: un-normalised codes of size 1/V would leave the straight-through output z + (q - z) with an
fp32 cancellation error of |z| / 2^24, the reference's own rounding, larger than the bar relative to |q|.

  vq8192            C = 32, V = 8192: VQ-8192, the benchmarked workload; tensor-core search
  vq4096_c64        C = 64, V = 4096: VQ-4096; tensor-core search at C = 64
  vq16384_c8        C = 8, V = 16384: the trainer's defaults; exact CUDA-core search
  vq4096_l2         C = 32, V = 4096, codebook_norm=False: the un-normalised branches of search and backward
  hot_codes         C = 32, V = 8192: 16 codes near the data's mean direction take most rows (thousands of gE atomics
                    on each)
  vp2_16384         two VectorQuantizers (V = 16384 each) fed by VQModel._split_branches of a [128, 32, 512, 1] latent,
                    losses averaged as in VQModel.forward
  robusttok         C = 64, V = 4096, then add_perturbation(alpha 1.0, beta 0.1, delta 100) as in VQModel.forward
  robusttok_anneal  the same past the anneal (config.perturbation_schedule: alpha 0.5, delta 50), so about half the
                    perturbed rows draw rank 0

  indices       every row's code lies within the fp32 rounding bound of the fp64 best (_fp64_check of
                test_gpu_vq_search_adversarial.py); for 8 whole images indices and out equal xq_oracle.vq_forward.
  perturbation  the selections (xq_perturb_forward's sel buffer) equal xq_oracle.rank_select, lie within the same
                rounding bound of the fp64 j-th order statistic, and a row that drew rank 0 selects the quantizer's
                own code and has its out row, bit for bit.  With z and z_q separate leaves, the perturbed samples'
                dz matches fp64 and every other sample's gradient goes to z_q untouched (in a whole step both routes
                give the same dz, so only this sees a sample sent the wrong way).
  values       out, vq, commit, dz (through the perturbation too), embedding.weight.grad and
                f_to_idxBl_or_fhat(to_fhat=True) against oracle/vq_ref64.py, the fp64 autograd restatement fed the
                product's own indices and selections.
  determinism   the same step twice: idx, out, vq, commit, hist and dz bitwise equal, gE within its bar.
  batch         images 0..127 as one batch and as 64 batches of 2: out, idx, f_to_idxBl_or_fhat and the perturbed
                output bitwise equal.
  usage EMA     three training forwards at record_hit 0, 99 and 100 against xq_oracle.ema_update of the bincount.

Bars, fixed before anything was measured: per tensor, normwise |x - x64| / |x64| <= 2e-5 and elementwise
|x - x64| <= 1e-4 max|x64| (the multi-scale test's).  hot_codes' gE is judged instead against the a-priori summation
bound (m_v + 2C) 2^-24 sum|contribution| per code v (m_v rows chose v; the contributions are the fp64 per-row
gradients of the code row).  Mutants (oracle/vq_ref64.MUTANTS) must exceed a bar or an index / rank gap of 1e-5;
`pytest -s` prints each tensor's error as a share of its bar and each mutant's margin.

Measured on an H100 80GB HBM3 (700 W power limit): the largest share of a bar over every tensor of every case is 0.014
(embedding.weight.grad normwise at C = 64, in vq4096_c64 and both RobustTok cases); every other tensor stays below
0.01, hot_codes' gE reaches 0.003 of its summation bound, and the fp64 index gap is 0 in every case (the largest rank
gap is 1e-7, in robusttok_anneal).  Every mutant exceeds a bar at least 5,200x (no_norm_jacobian_E on hot_codes,
against the summation bound, is the closest); rank_plus_one moves no value but its rank gap is at least 1.8e4 times
the 1e-5 tie.  The hot_codes fixture puts 32765 of the 32768 rows on its 16 codes, 611 to 3680 on each.  The file
takes about 15 s and at most 3.3 GiB of extra device memory.
"""
import functools
import time
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import vq_ref64, xq_oracle as xo
from test_gpu_vq_search_adversarial import _fp64_check

pytestmark = pytest.mark.gpu

B, S = 128, 16
HW = S * S
N = B * HW
NORM_BAR, ELEM_BAR = 2e-5, 1e-4
TIE = 1e-5
U = 2.0 ** -24
W_VQ, W_COMMIT = 1.3, 0.7
BETA = 0.25                      # commit_loss_beta
ORACLE_IMAGES = 8

CASES = {
    "vq8192": dict(C=32, V=8192, seed=61),
    "vq4096_c64": dict(C=64, V=4096, seed=62),
    "vq16384_c8": dict(C=8, V=16384, seed=63),
    "vq4096_l2": dict(C=32, V=4096, cn=False, seed=64),
    "hot_codes": dict(C=32, V=8192, hot=16, seed=65),
    "vp2_16384": dict(C=32, V=16384, branches=2, seed=66),
    "robusttok": dict(C=64, V=4096, epoch="start", seed=67),
    "robusttok_anneal": dict(C=64, V=4096, epoch="after_anneal", seed=68),
}
_BASE = ["swap_vq_commit", "mean_over_rows"]
_NORM = ["no_norm_jacobian_z", "no_norm_jacobian_E"]
_PERT = ["perturb_mask_plus_one", "perturb_grad_dropped", "rank_plus_one"]
MUTANTS = {n: (_NORM if c.get("cn", True) else []) + _BASE + (_PERT if "epoch" in c else []) for n, c in CASES.items()}
PERTURBED = [n for n, c in CASES.items() if "epoch" in c]


def npy(t):
    return t.detach().cpu().numpy()


@pytest.fixture(scope="module", autouse=True)
def _report_cost():
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield
    torch.cuda.synchronize()
    print(f"\n[vq fp64] {time.time() - t0:.1f} s, peak extra device memory "
          f"{(torch.cuda.max_memory_allocated() - base) / 2 ** 30:.2f} GiB")


def _schedule(epoch):
    """RobustTok's (alpha, beta, delta) at the start of training or after its anneal (config.perturbation_schedule)"""
    from imagefolder_b200 import config
    p = config.make_parser()
    p.set_defaults(**config.SHIPPED_CONFIGS["RobustTok"])
    args, _ = p.parse_known_args([])
    return config.perturbation_schedule(args, 0 if epoch == "start" else args.anneal_end + 1)


# ------------------------------------------------------------------------------------------------------------------
# fixtures
# ------------------------------------------------------------------------------------------------------------------
def _codebook(cfg, gen):
    V, C = cfg["V"], cfg["C"]
    if not cfg.get("cn", True):
        return torch.randn(V, C, generator=gen) * 0.5
    E = (torch.rand(V, C, generator=gen) * 2 - 1) / V           # uniform_(-1/V, 1/V), then F.normalize (vq.py:32-34)
    return F.normalize(E, p=2, dim=-1)


def _latent(cfg, gen, E):
    C = cfg["C"]
    if cfg.get("branches", 1) > 1:
        return torch.randn(B, C, cfg["branches"] * HW, 1, generator=gen)
    if "hot" not in cfg:
        return torch.randn(B, C, S, S, generator=gen)
    mu = F.normalize(torch.randn(C, generator=gen), dim=0)
    hot = (torch.arange(cfg["hot"]) * 509 + 7) % cfg["V"]
    E[hot] = F.normalize(mu[None] + 0.05 * torch.randn(cfg["hot"], C, generator=gen), dim=1)
    return mu[None, :, None, None] + 0.1 * torch.randn(B, C, S, S, generator=gen)


def _branches(cfg, x):
    """the latent each quantizer sees: VQModel._split_branches for product quantization, else x itself"""
    if cfg.get("branches", 1) == 1:
        return [x]
    from imagefolder_b200.xqgan_model import VQModel
    return VQModel._split_branches(types.SimpleNamespace(product_quant=cfg["branches"]), x)


def _quantizers(cfg, Es):
    from imagefolder_b200 import VectorQuantizer
    qs = []
    for E in Es:
        q = VectorQuantizer(cfg["V"], cfg["C"], BETA, cfg.get("cn", True))
        q.embedding.weight.data.copy_(E)
        qs.append(q.cuda().train())
    return qs


def _step(c):
    """one training step of fresh quantizers (and the perturbation) on the case's inputs"""
    from imagefolder_b200 import add_perturbation
    cfg = c["cfg"]
    qs = _quantizers(cfg, c["E"])
    x = c["x"].cuda().requires_grad_(True)
    outs, vqs, commits, idx = [], [], [], []
    for q, z in zip(qs, _branches(cfg, x)):
        o, _, v, cm, _ = q(z)
        outs.append(o)
        vqs.append(v)
        commits.append(cm)
        idx.append(q.last_idx.clone())
    vq, commit = sum(vqs) / len(qs), sum(commits) / len(qs)           # xqgan_model.py VQModel.forward
    if c["pert"]:
        alpha, beta, delta = c["pert"]
        out = add_perturbation(x, outs[0], cfg["C"], qs[0].codebook_norm, qs[0].embedding, alpha, beta, delta,
                               rand_u=c["ru"].cuda(), rand_j=c["rj"].cuda())
    else:
        out = torch.cat(outs, dim=1)
    ((out * c["g_out"].cuda()).sum() + W_VQ * vq + W_COMMIT * commit).backward()
    with torch.no_grad():
        fhat = [q.f_to_idxBl_or_fhat(z, to_fhat=True)[0] for q, z in zip(qs, _branches(cfg, x.detach()))]
    return dict(qs=qs, out=out.detach(), out_q=[o.detach() for o in outs], vq=vq.detach(), commit=commit.detach(),
                idx=idx, gx=x.grad.clone(), gE=[q.embedding.weight.grad.clone() for q in qs], fhat=fhat,
                hist=[q.ema_vocab_hit_SV.clone() for q in qs])           # record_hit 0: the EMA is the histogram


def _perturb_abi(z, zq, E, ru, rj, cn, alpha, n_perturb, delta):
    """xq_perturb_forward through the C ABI with a sel buffer (-1 where the kernel writes nothing)"""
    from imagefolder_b200 import _capi as Cc
    Bz, C = z.shape[:2]
    V = E.shape[0]
    out = torch.empty_like(z)
    sel = torch.full((Bz * HW,), -1, dtype=torch.int64, device=z.device)
    L = Cc.lib()
    ws = Cc.workspace(L.xq_perturb_workspace_bytes(Bz, C, HW, V), z.device)
    nk = (1 if n_perturb < Bz else 0) + (2 if n_perturb > 0 else 0)
    Cc.call("xq_perturb_forward", nk, L.xq_perturb_forward, Cc.ptr(z), Cc.ptr(zq), Cc.ptr(E), Cc.ptr(ru), Cc.ptr(rj),
            Bz, C, HW, V, int(cn), float(alpha), int(n_perturb), int(delta), Cc.ptr(out), Cc.ptr(sel), Cc.ptr(ws),
            ws.numel(), Cc.stream_ptr(z.device))
    return out, sel


@functools.lru_cache(maxsize=None)
def _case(name):
    cfg = CASES[name]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mem0 = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    gen = torch.Generator().manual_seed(cfg["seed"])
    Es = [_codebook(cfg, gen) for _ in range(cfg.get("branches", 1))]
    x = _latent(cfg, gen, Es[0])
    c = dict(cfg=cfg, E=Es, x=x, pert=None, ru=None, rj=None)
    if "epoch" in cfg:
        alpha, beta, delta = _schedule(cfg["epoch"])
        c.update(pert=(alpha, beta, delta), nb=int(B * beta), ru=torch.rand(N, generator=gen),
                 rj=torch.randint(0, delta, (N,), generator=gen))
    c["g_out"] = torch.randn(B, cfg["C"] * len(Es), S, S, generator=gen) / (B * cfg["C"] * len(Es) * HW)
    c["prod"] = _step(c)
    if c["pert"]:
        # the product's selection for every row (n_perturb = B): the perturbation mutants need the rows of one image
        # more than the step perturbs
        alpha, _, delta = c["pert"]
        z = x.cuda()
        _, c["sel_all"] = _perturb_abi(z, c["prod"]["out_q"][0], c["E"][0].cuda(), c["ru"].cuda(), c["rj"].cuda(),
                                       cfg.get("cn", True), alpha, B, delta)
    c.update(setup_s=time.perf_counter() - t0, mem0=mem0)
    return c


# ------------------------------------------------------------------------------------------------------------------
# fp64 restatement and comparison
# ------------------------------------------------------------------------------------------------------------------
def _ref64(c, mutant=None):
    cfg, p = c["cfg"], c["prod"]
    cn = cfg.get("cn", True)
    leaf = lambda t: t.detach().cuda().double().requires_grad_(True)
    x = leaf(c["x"])
    Es = [leaf(E) for E in c["E"]]
    fq = [vq_ref64.forward(z, E, ix, beta=BETA, codebook_norm=cn, mutant=mutant)
          for z, E, ix in zip(_branches(cfg, x), Es, p["idx"])]
    vq, commit = sum(f["vq"] for f in fq) / len(fq), sum(f["commit"] for f in fq) / len(fq)
    rank_gap = 0.0
    if c["pert"]:
        alpha, beta, delta = c["pert"]
        fp = vq_ref64.add_perturbation(x, fq[0]["out"], Es[0], c["sel_all"], c["ru"], c["rj"], alpha=alpha, beta=beta,
                                       delta=delta, codebook_norm=cn, mutant=mutant)
        out, rank_gap = fp["out"], fp["rank_gap"]
    else:
        out = torch.cat([f["out"] for f in fq], dim=1)
    wrt = dict(x=x, **{f"E{i}": E for i, E in enumerate(Es)})
    if "hot" in cfg:
        wrt["y0"] = fq[0]["y"]                   # per-row contributions to gE, for the summation bound
    gr = vq_ref64.losses_and_grads(out, vq, commit, wrt, c["g_out"].cuda().double(), W_VQ, W_COMMIT, mutant=mutant)
    return dict(out=out, vq=vq, commit=commit, fhat=[f["fhat"] for f in fq], gr=gr, rank_gap=rank_gap,
                idx_gap=max(f["idx_gap"] for f in fq))


def _shares(x, x64):
    """(normwise error / its bar, elementwise error / its bar)"""
    x, x64 = x.detach().double(), x64.detach().double()
    d = (x - x64).abs()
    return float(d.norm() / x64.norm()) / NORM_BAR, float(d.max()) / (ELEM_BAR * float(x64.abs().max()))


def _sum_bound_share(c, gE, gE64, gy):
    """largest |gE - gE64| / ((m_v + 2C) u sum_rows |contribution|) over the codes (a code no row chose: exactly 0)"""
    C, V = c["cfg"]["C"], c["cfg"]["V"]
    idx = c["prod"]["idx"][0]
    m = torch.bincount(idx, minlength=V).double()
    a = torch.zeros(V, dtype=torch.float64, device=gy.device).index_add_(0, idx, gy.abs().sum(1))
    bound = ((m + 2 * C) * U * a)[:, None]
    d = (gE.double() - gE64.double()).abs()
    if bool((d[bound[:, 0] == 0] != 0).any()):
        return float("inf")
    return float((d / bound.clamp_min(1e-300)).max())


def _compare(c, r):
    """[(tensor name, normwise share, elementwise share)] for every value and gradient the step owns"""
    p, rows = c["prod"], []
    for n in ("out", "vq", "commit"):
        rows.append((n,) + _shares(p[n], r[n]))
    for i, fh in enumerate(p["fhat"]):
        rows.append((f"fhat[{i}]",) + _shares(fh, r["fhat"][i]))
    rows.append(("dz",) + _shares(p["gx"], r["gr"]["x"]))
    for i, gE in enumerate(p["gE"]):
        if "hot" in c["cfg"]:
            s = _sum_bound_share(c, gE, r["gr"][f"E{i}"], r["gr"]["y0"])
            rows.append((f"embedding[{i}].grad (sum bound)", s, s))
        else:
            rows.append((f"embedding[{i}].grad",) + _shares(gE, r["gr"][f"E{i}"]))
    return rows


# ------------------------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_indices_within_rounding_of_fp64_and_equal_to_the_oracle(name):
    c = _case(name)
    cfg, p = c["cfg"], c["prod"]
    cn = cfg.get("cn", True)
    for i, z in enumerate(_branches(cfg, c["x"])):
        z = z.contiguous()
        E = npy(c["E"][i])
        _fp64_check(npy(z.permute(0, 2, 3, 1).reshape(-1, cfg["C"])), E, p["idx"][i], cn)
        fw = xo.vq_forward(npy(z[:ORACLE_IMAGES]), E, BETA, cn)
        np.testing.assert_array_equal(npy(p["idx"][i][:ORACLE_IMAGES * HW]), fw["idx"], err_msg=f"branch {i}")
        np.testing.assert_array_equal(npy(p["out_q"][i][:ORACLE_IMAGES]), fw["out"], err_msg=f"branch {i}")
    if "hot" in cfg:
        m = torch.bincount(p["idx"][0], minlength=cfg["V"])
        top = m.topk(cfg["hot"]).values
        print(f"\nhot_codes: the {cfg['hot']} busiest codes take {int(top.sum())} of {N} rows, "
              f"{int(top.min())} to {int(top.max())} each")
        assert int(top.sum()) > 0.9 * N and int(top.min()) >= 500


def _rank_bound_check(zn, En, sel, rank):
    """every selection's fp64 squared distance within tau of the fp64 order statistic of its rank; zn, En the fp32
    normalised vectors and tau the bound of _fp64_check (test_gpu_vq_search_adversarial.py), which holds for order
    statistics as for the minimum: |d32 - d| <= delta on every code moves every order statistic by at most delta"""
    C = zn.shape[1]
    Ed = torch.from_numpy(En).cuda().double()
    ee = (Ed * Ed).sum(1)
    cmax, eemax = float(ee.max().sqrt()), float(ee.max())
    chunk = max(1, (1 << 27) // En.shape[0])
    worst = 0.0
    for s in range(0, zn.shape[0], chunk):
        zd = torch.from_numpy(zn[s:s + chunk]).cuda().double()
        zz = (zd * zd).sum(1)
        d = zz[:, None] + ee[None, :] - 2.0 * (zd @ Ed.T)
        r = rank[s:s + chunk, None]
        kth = torch.topk(d, int(r.max()) + 1, dim=1, largest=False).values.gather(1, r)[:, 0]
        gap = (d.gather(1, sel[s:s + chunk, None])[:, 0] - kth).abs()
        zl = zz.sqrt()
        tau = 2.0 * U * (2 * C * zl * cmax + (C + 1) * (zz + eemax) + (zl + cmax) ** 2)
        bad = gap > tau
        assert not bool(bad.any()), f"rows {(s + torch.nonzero(bad)[:8, 0]).tolist()} selected beyond the rounding bound"
        worst = max(worst, float((gap / tau).max()))
    return worst


@pytest.mark.parametrize("name", PERTURBED)
def test_perturbation_selections(name):
    c = _case(name)
    cfg, p = c["cfg"], c["prod"]
    alpha, beta, delta = c["pert"]
    nb = c["nb"]
    nr = nb * HW
    assert nb == 12
    z, E = c["x"].cuda(), c["E"][0].cuda()
    out, sel = _perturb_abi(z, p["out_q"][0], E, c["ru"].cuda(), c["rj"].cuda(), True, alpha, nb, delta)
    assert torch.equal(out, p["out"]), "the C ABI's output differs from the autograd path's"
    assert bool((sel[nr:] == -1).all()), "a selection written past the perturbed rows"
    assert torch.equal(sel[:nr], c["sel_all"][:nr]), "the selections depend on n_perturb"
    rank = torch.where(c["ru"] > alpha, 0, c["rj"])[:nr]
    zn = xo.l2norm_rows(npy(z[:nb].permute(0, 2, 3, 1).reshape(-1, cfg["C"])))[0]
    En = xo.l2norm_rows(npy(E))[0]
    np.testing.assert_array_equal(npy(sel[:nr]), xo.rank_select(zn, En, npy(rank), delta))
    worst = _rank_bound_check(zn, En, sel[:nr], rank.cuda())
    r0 = (rank == 0).cuda()
    n0 = int(r0.sum())
    print(f"\n{name}: alpha {alpha}, delta {delta}: {n0} of {nr} perturbed rows drew rank 0; "
          f"largest rank gap / rounding bound {worst:.2e}")
    assert n0 > 0
    assert torch.equal(sel[:nr][r0], p["idx"][0][:nr][r0]), "a rank-0 selection is not the quantizer's code"
    rows = lambda t: t[:nb].permute(0, 2, 3, 1).reshape(-1, cfg["C"])
    assert torch.equal(rows(p["out"])[r0], rows(p["out_q"][0])[r0]), "a rank-0 row's output is not the quantizer's"
    if name == "robusttok_anneal":
        assert 0.4 * nr < n0 < 0.6 * nr


@pytest.mark.parametrize("name", PERTURBED)
def test_perturbation_gradients_to_z_and_zq(name):
    """the perturbation alone, z and z_q separate leaves: the perturbed samples' gradient goes to z through the
    normalisation, every other sample's to z_q untouched.  In a training step both routes end in the same dz (the
    quantizer's output is straight-through on the normalised z), so only this check sees a sample sent the wrong way."""
    from imagefolder_b200 import add_perturbation
    c = _case(name)
    cfg, p = c["cfg"], c["prod"]
    alpha, beta, delta = c["pert"]
    nb = c["nb"]
    x = c["x"].cuda().requires_grad_(True)
    zq = p["out_q"][0].clone().requires_grad_(True)
    emb = torch.nn.Embedding.from_pretrained(c["E"][0].cuda())
    g = c["g_out"].cuda()
    out = add_perturbation(x, zq, cfg["C"], True, emb, alpha, beta, delta, rand_u=c["ru"].cuda(), rand_j=c["rj"].cuda())
    (out * g).sum().backward()
    leaf = lambda t: t.detach().double().requires_grad_(True)
    x64, zq64 = leaf(x), leaf(zq)
    fp = vq_ref64.add_perturbation(x64, zq64, emb.weight.double(), c["sel_all"], c["ru"], c["rj"], alpha=alpha,
                                   beta=beta, delta=delta)
    zero = torch.zeros((), dtype=torch.float64, device=x.device)
    gr = vq_ref64.losses_and_grads(fp["out"], zero, zero, dict(z=x64, zq=zq64), g.double(), 0.0, 0.0)
    a, e = _shares(x.grad[:nb], gr["z"][:nb])
    print(f"\n{name}: perturbed samples' dz normwise ({a:.3f} of bar)   elementwise ({e:.3f})")
    assert a <= 1 and e <= 1
    assert torch.equal(out[:nb], p["out"][:nb]) and torch.equal(out[nb:], zq[nb:])
    assert bool((x.grad[nb:] == 0).all()), "an unperturbed sample passes gradient to z"
    assert bool((zq.grad[:nb] == 0).all()), "a perturbed sample passes gradient to z_q"
    assert torch.equal(zq.grad[nb:], g[nb:]), "an unperturbed sample's gradient to z_q is not g"


@pytest.mark.parametrize("name", list(CASES))
def test_values_and_gradients_against_fp64(name):
    c = _case(name)
    t0 = time.perf_counter()
    r = _ref64(c)
    rows = _compare(c, r)
    print(f"\n{name}: setup {c['setup_s']:.1f} s, fp64 {time.perf_counter() - t0:.1f} s, index gap {r['idx_gap']:.1e}, "
          f"rank gap {r['rank_gap']:.1e}, peak extra {(torch.cuda.max_memory_allocated() - c['mem0']) / 2 ** 30:.2f} GiB")
    for n, a, e in rows:
        print(f"  {n:30s} normwise ({a:.3f} of bar)   elementwise ({e:.3f})")
    print(f"  worst share of a bar: {max(max(a, e) for _, a, e in rows):.3f}")
    assert r["idx_gap"] <= TIE, f"a product index is not the fp64 choice (gap {r['idx_gap']:.2e})"
    assert r["rank_gap"] <= TIE, f"a product selection is not the fp64 order statistic (gap {r['rank_gap']:.2e})"
    bad = [(n, a, e) for n, a, e in rows if a > 1 or e > 1]
    assert not bad, bad


@pytest.mark.parametrize("name", list(CASES))
def test_mutants_fail_the_bar(name):
    c = _case(name)
    print()
    for mut in MUTANTS[name]:
        r = _ref64(c, mut)
        n, a, e = max(_compare(c, r), key=lambda t: max(t[1], t[2]))
        gap = max(r["idx_gap"], r["rank_gap"]) / TIE
        print(f"  {name} {mut:22s} largest share of a bar {max(a, e):12.1f} ({n}), index / rank gap / tie {gap:.1f}")
        assert max(a, e, gap) > 1, f"mutant {mut} passes"


@pytest.mark.parametrize("name", list(CASES))
def test_same_step_twice_is_bitwise_equal(name):
    c = _case(name)
    p, p2 = c["prod"], _step(c)
    for k in ("out", "vq", "commit", "gx"):
        assert torch.equal(p[k], p2[k]), k
    for k in ("out_q", "idx", "fhat", "hist"):
        for i in range(len(p[k])):
            assert torch.equal(p[k][i], p2[k][i]), f"{k}[{i}]"
    for i in range(len(p["gE"])):
        assert torch.equal(p["hist"][i], torch.bincount(p["idx"][i], minlength=c["cfg"]["V"]).float())
        r = _ref64(c)
        gE64 = r["gr"][f"E{i}"]
        if "hot" in c["cfg"]:
            assert _sum_bound_share(c, p2["gE"][i], gE64, r["gr"]["y0"]) <= 1
        else:
            assert max(_shares(p2["gE"][i], gE64)) <= 1


@pytest.mark.parametrize("name", list(CASES))
def test_batch_of_128_equals_64_batches_of_2(name):
    from imagefolder_b200 import ops
    c = _case(name)
    cfg, p = c["cfg"], c["prod"]
    qs = _quantizers(cfg, c["E"])
    x = c["x"].cuda()
    with torch.no_grad():
        for i in range(0, B, 2):
            rs = slice(i * HW, (i + 2) * HW)
            for k, (q, z) in enumerate(zip(qs, _branches(cfg, x[i:i + 2]))):
                o, _, _, _, _ = q(z, ret_usages=False)
                assert torch.equal(o, p["out_q"][k][i:i + 2]), f"out of images {i}, {i + 1} (branch {k})"
                assert torch.equal(q.last_idx, p["idx"][k][rs]), f"idx of images {i}, {i + 1} (branch {k})"
                fh = q.f_to_idxBl_or_fhat(z, to_fhat=True)[0]
                assert torch.equal(fh, p["fhat"][k][i:i + 2]), f"f_hat of images {i}, {i + 1} (branch {k})"
                if c["pert"]:
                    alpha, _, delta = c["pert"]
                    npair = min(2, max(0, c["nb"] - i))
                    po = ops.perturb(z, o, q.embedding.weight, c["ru"][rs].cuda(), c["rj"][rs].cuda(),
                                     q.codebook_norm, alpha, npair, delta)
                    assert torch.equal(po, p["out"][i:i + 2]), f"perturbed out of images {i}, {i + 1}"


@pytest.mark.parametrize("name", ["vq8192", "vq16384_c8"])
def test_usage_ema_at_the_training_batch(name):
    """three training forwards at record_hit 0, 99 and 100 (xqgan_model.py:773-788): the EMA equals the oracle's
    update of the exact bincount bit for bit, usage is (ema >= margin).float().mean() * 100 with the reference's
    margin, and record_hit advances by one per step"""
    c = _case(name)
    cfg = c["cfg"]
    V = cfg["V"]
    (q,) = _quantizers(cfg, c["E"])
    margin = N / V * 0.08                         # world size 1 * (z.numel() / C) / V * 0.08
    x = c["x"]
    ema = np.zeros(V, np.float32)
    for step, (rh, z) in enumerate(zip([0, 99, 100], [x, -x, x.roll(1, dims=1)])):
        if step < 2:
            q.record_hit = rh                     # the third step starts at 100 by itself
        assert q.record_hit == rh
        with torch.no_grad():
            _, usage, _, _, _ = q(z.cuda())
        hit = np.bincount(npy(q.last_idx), minlength=V).astype(np.float32)
        ema = xo.ema_update(ema, hit, rh)
        np.testing.assert_array_equal(npy(q.ema_vocab_hit_SV), ema, err_msg=f"record_hit {rh}")
        want = (q.ema_vocab_hit_SV >= margin).float().mean() * 100
        assert float(usage[0]) == float(want), (rh, float(usage[0]), float(want))
        assert q.record_hit == rh + 1
