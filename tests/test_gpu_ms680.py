"""The multi-scale quantizers at VAR's default 680-token pyramid, v_patch_nums = [1,2,3,4,5,6,8,10,13,16], on the GPU.

A 16 x 16 last scale at C = 32 is the largest shape one image's CTA holds: the backward's shared memory is laid out by
buffer lifetime (csrc/ms_kernels.cu, ms_bwd_layout), 217.3 KiB at this shape.

  goldens     the reference's own VectorQuantizer2 (tests/golden/make_ms680_golden.py, inputs regenerated from the
              stored seed by tests/ms680_inputs.py): indices equal to the golden
              and the fp32 C oracle, out and every f_to_idxBl_or_fhat entry bitwise equal to the oracle; losses, usage
              EMA and gradients within the goldens' tolerances; idxBl_to_var_input, embed_to_fhat and the
              get_next_autoregressive_input chain against the goldens and bitwise against the oracle.
  fp64        one training step at the training batch against oracle/ms_ref64.py with the bars and mutants of
              tests/test_gpu_ms_quant_fp64.py: V = 4096 at B = 128, V = 16384 at B = 32, znorm and L2 metric, LFQ at
              C = 12 / 14; an explicit `dropout` in which every scale count from 1 to 10 occurs.
  batch       each fp64 case's images as one batch and as batches of 2: out, indices and f_hat bitwise equal.
  ladder      C in {8, 16, 24, 32} x last scale in {12, 13, 14, 16} train and match the oracle and fp64; C = 40 at
              16 x 16 and C = 48 at 11 x 11 refuse up front with the shape named.
  LFQ         the full-softmax entropy (soft_entropy=False) at C = 12 / 14 against tests/lfq_hard_oracle.py.
  model       a PQ-2 MSVR VQModel with num_latent_tokens = 256 on this pyramid: one bf16-autocast training step, and
              2 x 680 tokens per image from img_to_idxBl and pretokenize, equal to the oracle on the model's latent.
"""
import functools
import time

import numpy as np
import pytest
import torch

from conftest import load_golden
from ms680_inputs import FHAT_SUB, VAR_SUB, load680
from oracle import ms_ref64, xq_oracle as xo
from test_gpu_ms_quant_fp64 import ELEM_BAR, NORM_BAR, TIE, W_COMMIT, W_ENT, W_VQ, _VQ_MUTANTS, _shares
from test_gpu_quantizers import close, dev, make_vq2

pytestmark = pytest.mark.gpu

PN = [1, 2, 3, 4, 5, 6, 8, 10, 13, 16]
SN = len(PN)
HW = PN[-1]

CASES = {
    "msvr680_4096": dict(lfq=False, C=32, V=4096, B=128, znorm=True, share=4, drop=0.1, seed=51),
    "msvr680_16384": dict(lfq=False, C=32, V=16384, B=32, znorm=True, share=4, drop=0.5, seed=52),
    "msvr680_l2": dict(lfq=False, C=32, V=4096, B=128, znorm=False, share=4, drop=0.1, seed=53),
    "msbr680_4096": dict(lfq=True, C=12, V=4096, B=128, znorm=True, share=4, drop=0.1, seed=54),
    "msbr680_16384": dict(lfq=True, C=14, V=16384, B=32, znorm=True, share=4, drop=0.5, seed=55),
}
_LFQ_MUTANTS = ["share_map_shift", "nq_plus_one", "swap_vq_commit", "ent_row1_to_row0", "area_floor"]
MUTANTS = {n: (_LFQ_MUTANTS if c["lfq"] else _VQ_MUTANTS) for n, c in CASES.items()}


def npy(t):
    return t.detach().cpu().numpy()


def _phi_np(q):
    mods = q.quant_resi.modules_list()
    return np.stack([npy(m.weight) for m in mods]), np.stack([npy(m.bias) for m in mods])


# ------------------------------------------------------------------------------------------------------------------
# reference goldens
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["msvr680_znorm", "msvr680_l2"])
def test_680_token_golden(name):
    g = load680(name)
    pn = [int(p) for p in g["patch_nums"]]
    assert pn == PN
    zn = bool(g["using_znorm"])
    V, C = g["E"].shape
    cd = float(g["codebook_drop"])
    q = make_vq2(g, V, C, pn, zn, int(g["share"]), cd)
    f = dev(g["f"], grad=True)
    out, usages, vq, commit, _ = q(f, ret_usages=True, dropout=torch.tensor(g["dropout"]))
    fwd = xo.vq2_forward(g["f"], g["E"], g["phi_w"], g["phi_b"], pn, using_znorm=zn, codebook_drop=cd,
                         dropout=g["dropout"])
    for si in range(SN):
        np.testing.assert_array_equal(npy(q.last_idx_Bl[si]), fwd["idx"][si])
        np.testing.assert_array_equal(npy(q.last_idx_Bl[si]), g[f"idx{si}"])
    np.testing.assert_array_equal(npy(out), fwd["out"])
    close(out, g["out"])
    close(vq, g["vq"])
    close(commit, g["commit"])
    close(torch.stack(usages), g["usages"], rtol=1e-5, atol=1e-3)
    close(q.ema_vocab_hit_SV, g["ema"], rtol=1e-6)
    g_out = g["g_out"]
    (out * dev(g_out)).sum().add(float(g["w_vq"]) * vq).add(float(g["w_commit"]) * commit).backward()
    close(f.grad, g["gf"])
    close(q.embedding.weight.grad, g["gE"])
    gf, gE, gw, gb = xo.vq2_backward(fwd, g["f"], g["E"], g["phi_w"], g["phi_b"], pn, g_out, float(g["w_vq"]),
                                     float(g["w_commit"]))
    close(f.grad, gf, rtol=1e-4)
    close(q.embedding.weight.grad, gE, rtol=1e-4)
    for i, m in enumerate(q.quant_resi.modules_list()):
        close(m.weight.grad, g["gphi_w"][i], atol=2e-4 * float(np.abs(g["gphi_w"]).max()))
        close(m.bias.grad, g["gphi_b"][i], atol=2e-4 * float(np.abs(g["gphi_b"]).max()))
        close(m.weight.grad, gw[i], atol=1e-4 * float(np.abs(gw).max()))
        close(m.bias.grad, gb[i], atol=1e-4 * float(np.abs(gb).max()))
    # inference surfaces: f_to_idxBl_or_fhat, token decode, idxBl_to_var_input
    idx_list = q.f_to_idxBl_or_fhat(f.detach(), to_fhat=False, v_patch_nums=pn)
    fh_list = q.f_to_idxBl_or_fhat(f.detach(), to_fhat=True, v_patch_nums=pn)
    fh_oracle = xo.vq2_f_to_idxBl_or_fhat(g["f"], g["E"], g["phi_w"], g["phi_b"], pn, using_znorm=zn, to_fhat=True)
    for si in range(SN):
        np.testing.assert_array_equal(npy(idx_list[si]), g[f"idx{si}"])
        np.testing.assert_array_equal(npy(fh_list[si]), fh_oracle[si])
        close(fh_list[si][FHAT_SUB], g[f"fhat_sub{si}"])
    np.testing.assert_array_equal(npy(q.idx_to_fhat(idx_list)), npy(fh_list[-1]))
    var = q.idxBl_to_var_input([dev(g[f"idx{si}"], torch.int64) for si in range(SN)])
    assert tuple(var.shape) == (2, 680 - 1, C)
    close(var[VAR_SUB], g["var_input_sub"])
    want = np.concatenate([xo.area_pool_rows(fh_oracle[si], pn[si + 1]).reshape(2, -1, C) for si in range(SN - 1)],
                          axis=1)
    np.testing.assert_array_equal(npy(var), want)


def test_680_token_var_helpers_golden():
    from imagefolder_b200 import VectorQuantizer2
    g = load_golden("varhelp680")
    pn = [int(p) for p in g["patch_nums"]]
    C = g["h0"].shape[1]
    q = VectorQuantizer2(64, C, v_patch_nums=pn, num_latent_tokens=pn[-1] ** 2,
                         share_quant_resi=int(g["share"])).cuda().eval()
    for i, m in enumerate(q.quant_resi.modules_list()):
        m.weight.data.copy_(dev(g["phi_w"][i]))
        m.bias.data.copy_(dev(g["phi_b"][i]))
    hs = [dev(g[f"h{si}"]) for si in range(SN)]
    want = xo.embed_to_fhat([g[f"h{si}"] for si in range(SN)], g["phi_w"], g["phi_b"], pn)
    fl = q.embed_to_fhat(hs, all_to_max_scale=True, last_one=False)
    for si in range(SN):
        np.testing.assert_array_equal(npy(fl[si]), want[si])
        close(fl[si], g[f"fh{si}"])
    last = q.embed_to_fhat(hs, all_to_max_scale=True, last_one=True)
    np.testing.assert_array_equal(npy(last), want[-1])
    close(last, g["fh_last"])
    f_hat = torch.zeros_like(last)
    Fo = np.zeros_like(want[-1])
    for si in range(SN):
        _, nxt = q.get_next_autoregressive_input(si, SN, f_hat, hs[si])
        Fo, no = xo.get_next_autoregressive_input(si, Fo, g[f"h{si}"], g["phi_w"], g["phi_b"], pn)
        np.testing.assert_array_equal(npy(f_hat), Fo)
        np.testing.assert_array_equal(npy(nxt), no)
        close(nxt, g[f"next{si}"])
    close(f_hat, g["ar_f_hat"])


# ------------------------------------------------------------------------------------------------------------------
# one training step at the training batch against fp64
# ------------------------------------------------------------------------------------------------------------------
def _module(cfg, gen, pn=PN):
    from imagefolder_b200 import LFQ, VectorQuantizer2
    C = cfg["C"]
    kw = dict(v_patch_nums=pn, num_latent_tokens=pn[-1] ** 2, share_quant_resi=cfg["share"], codebook_drop=cfg["drop"])
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
    """fp32 C oracle on f: (per-scale indices, per-image smallest margin)"""
    w, b = _phi_np(q)
    n = f.shape[0]
    if not cfg["lfq"]:
        fw = xo.vq2_forward(f, npy(q.embedding.weight), w, b, PN, using_znorm=cfg["znorm"])
        return fw["idx"], np.min([fw["margins"][si].min(axis=1) for si in range(SN)], axis=0)
    fw = xo.lfq_forward(f, w, b, PN, using_znorm=cfg["znorm"], scaler=npy(q.scaler))
    rest = fw["fn"].astype(np.float32).copy()
    margin = np.full(n, np.inf)
    for si, p in enumerate(PN):
        margin = np.minimum(margin, np.abs(xo.area_pool_rows(rest, p)).reshape(n, -1).min(axis=1))
        rest = (rest - fw["h"][si]).astype(np.float32)
    return fw["idx"], margin


def _screened_input(cfg, q, gen):
    """f [B,C,H,W] whose every image is clear of oracle near-ties (an image that has one is redrawn)"""
    B, C = cfg["B"], cfg["C"]
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
    cfg = CASES[name]
    B = cfg["B"]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    gen = torch.Generator().manual_seed(cfg["seed"])
    q = _module(cfg, gen)
    f, idx_oracle = _screened_input(cfg, q, gen)
    assert int(B * cfg["drop"]) >= SN
    dropout = torch.randint(1, SN + 1, (B,), generator=gen)
    dropout[:SN] = torch.randperm(SN, generator=gen) + 1          # every scale count 1..10 among the dropped samples
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
                setup_s=time.perf_counter() - t0)


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


def _compare(c, fwd, gr):
    p, rows = c["prod"], []
    for n in ["out", "vq", "commit"] + (["entropy"] if c["cfg"]["lfq"] else []):
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
def test_680_indices_of_every_image_match_the_oracle(name):
    c = _case(name)
    for si in range(SN):
        np.testing.assert_array_equal(npy(c["prod"]["idx"][si]), c["idx_oracle"][si], err_msg=f"scale {si}")


@pytest.mark.parametrize("name", list(CASES))
def test_680_values_and_gradients_against_fp64(name):
    c = _case(name)
    t0 = time.perf_counter()
    fwd, gr = _ref64(c)
    rows = _compare(c, fwd, gr)
    print(f"\n{name}: setup {c['setup_s']:.1f} s, fp64 {time.perf_counter() - t0:.1f} s, index gap {fwd['idx_gap']:.1e}")
    for n, a, e in rows:
        print(f"  {n:22s} normwise {a * NORM_BAR:.2e} ({a:.3f} of bar)   elementwise {e * ELEM_BAR:.2e} ({e:.3f})")
    print(f"  worst share of a bar: {max(max(a, e) for _, a, e in rows):.3f}")
    assert fwd["idx_gap"] <= TIE, f"product index is not the fp64 choice (gap {fwd['idx_gap']:.2e})"
    bad = [(n, a, e) for n, a, e in rows if a > 1 or e > 1]
    assert not bad, bad


@pytest.mark.parametrize("name", list(CASES))
def test_680_mutants_fail_the_bar(name):
    c = _case(name)
    print()
    for mut in MUTANTS[name]:
        fwd, gr = _ref64(c, mut)
        n, a, e = max(_compare(c, fwd, gr), key=lambda r: max(r[1], r[2]))
        gap = fwd["idx_gap"] / TIE
        print(f"  {name} {mut:24s} largest share of a bar {max(a, e):10.1f} ({n}), index gap / tie {gap:.1f}")
        assert max(a, e, gap) > 1, f"mutant {mut} passes"


@pytest.mark.parametrize("name", list(CASES))
def test_680_batch_equals_batches_of_2(name):
    c = _case(name)
    q, p, B = c["q"], c["prod"], c["cfg"]["B"]
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
# shape ladder around the shared-memory limit
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("last", [12, 13, 14, 16])
@pytest.mark.parametrize("C", [8, 16, 24, 32])
def test_shape_ladder_trains(C, last):
    """a 6-scale pyramid ending at `last`: five bicubic scales (whose transposed upsample borrows the padded dh planes)
    before the full-resolution one, both metrics"""
    from imagefolder_b200 import VectorQuantizer2
    pn = [1, 2, 3, 5, 8, last]
    V, Bs = 512, 2
    for zn in (True, False):
        gen = torch.Generator().manual_seed(1000 * C + 10 * last + zn)
        q = VectorQuantizer2(V, C, using_znorm=zn, v_patch_nums=pn, num_latent_tokens=last * last,
                             share_quant_resi=4, codebook_drop=0.5)
        with torch.no_grad():
            q.embedding.weight.copy_(torch.randn(V, C, generator=gen) * 0.5)
            for m in q.quant_resi.modules_list():
                m.weight.copy_(torch.randn(m.weight.shape, generator=gen) * 0.06)
                m.bias.copy_(torch.randn(C, generator=gen) * 0.1)
        q = q.cuda().train()
        f = torch.randn(Bs, C, last, last, generator=gen)
        dropout = torch.tensor([3, len(pn) + 1])
        ft = f.cuda().requires_grad_(True)
        out, _, vq, commit, _ = q(ft, dropout=dropout)
        g_out = torch.randn(out.shape, generator=gen) / out.numel()
        ((out * g_out.cuda()).sum() + W_VQ * vq + W_COMMIT * commit).backward()
        mods = q.quant_resi.modules_list()
        w, b = _phi_np(q)
        fw = xo.vq2_forward(f.numpy(), npy(q.embedding.weight), w, b, pn, using_znorm=zn, codebook_drop=0.5,
                            dropout=dropout.numpy())
        for si in range(len(pn)):           # same canonical fp32 arithmetic: equal even at near-ties
            np.testing.assert_array_equal(npy(q.last_idx_Bl[si]), fw["idx"][si])
        np.testing.assert_array_equal(npy(out), fw["out"])
        gf, gE, gw, gb = xo.vq2_backward(fw, f.numpy(), npy(q.embedding.weight), w, b, pn, npy(g_out), W_VQ, W_COMMIT)
        close(ft.grad, gf, rtol=1e-4)
        close(q.embedding.weight.grad, gE, rtol=1e-4)
        leaf = lambda t: t.detach().double().requires_grad_(True)
        wrt = dict(f=leaf(ft), E=leaf(q.embedding.weight), phi_w=leaf(torch.stack([m.weight for m in mods])),
                   phi_b=leaf(torch.stack([m.bias for m in mods])))
        nq = ms_ref64.n_quantizers(Bs, len(pn), 0.5, dropout.numpy())
        r = ms_ref64.forward(wrt["f"], q.last_idx_Bl, pn, lfq=False, E=wrt["E"], phi_w=wrt["phi_w"],
                             phi_b=wrt["phi_b"], nq=nq, using_znorm=zn)
        gr = ms_ref64.losses_and_grads(r, wrt, g_out.cuda().double(), W_VQ, W_COMMIT)
        if min(float(m.min()) for m in fw["margins"]) > TIE:
            assert r["idx_gap"] <= TIE
        for nm, x, x64 in [("out", out, r["out"]), ("vq", vq, r["vq"]), ("commit", commit, r["commit"]),
                           ("f.grad", ft.grad, gr["f"]), ("E.grad", q.embedding.weight.grad, gr["E"])] + \
                [(f"phi[{k}].w", m.weight.grad, gr["phi_w"][k]) for k, m in enumerate(mods)] + \
                [(f"phi[{k}].b", m.bias.grad, gr["phi_b"][k]) for k, m in enumerate(mods)]:
            a, e = _shares(x, x64)
            assert a <= 1 and e <= 1, (zn, nm, a, e)


@pytest.mark.parametrize("C,last", [(40, 16), (48, 11)])
def test_shape_ladder_refuses_beyond_the_limit(C, last):
    from imagefolder_b200 import VectorQuantizer2
    from imagefolder_b200._capi import XqError
    q = VectorQuantizer2(512, C, v_patch_nums=[1, 2, 3, last], num_latent_tokens=last * last).cuda().train()
    ft = torch.randn(2, C, last, last, device="cuda", requires_grad=True)
    with pytest.raises(XqError) as e:
        q(ft)
    msg = str(e.value)
    assert "unsupported" in msg and f"C = {C}" in msg and f"{last} x {last}" in msg, msg


# ------------------------------------------------------------------------------------------------------------------
# LFQ with the full-softmax entropy at this pyramid
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [12, 14])
def test_680_lfq_full_softmax_entropy_against_oracle(C):
    import lfq_hard_oracle as lho
    from imagefolder_b200 import LFQ
    B = 4
    torch.manual_seed(C)
    q = LFQ(2 ** C, C, using_znorm=True, v_patch_nums=PN, num_latent_tokens=HW * HW, codebook_drop=0.5,
            entropy_weight=0.1, soft_entropy=False).cuda().train()
    for m in q.quant_resi.modules_list():
        m.weight.data.normal_(0, 0.1)
        m.bias.data.normal_(0, 0.05)
    gen = torch.Generator().manual_seed(C + 1)
    f = torch.randn(B, C, HW, HW, generator=gen)
    dr = torch.tensor([4, 7, SN + 1, SN + 1])
    fg = f.cuda().requires_grad_(True)
    out, _, vq, commit, ent = q(fg, dropout=dr)
    ent.backward()
    pw, pb = _phi_np(q)
    fwd = lho.lfq_hard_forward(f.numpy(), pw, pb, PN, using_znorm=True, codebook_drop=0.5, dropout=dr.numpy(),
                               entropy_weight=0.1, scaler=npy(q.scaler))
    for si in range(SN):
        np.testing.assert_array_equal(npy(q.last_idx_Bl[si]), fwd["idx"][si])
    np.testing.assert_array_equal(npy(out), fwd["out"])
    np.testing.assert_allclose(float(vq), fwd["vq"], rtol=1e-5)
    np.testing.assert_allclose(float(commit), fwd["commit"], rtol=1e-5)
    np.testing.assert_allclose(float(ent.detach()), fwd["entropy"], rtol=1e-4)
    gf, _, _ = lho.lfq_hard_backward(fwd, f.numpy(), pw, pb, PN, np.zeros(f.shape), 0.0, 0.0, 1.0, using_znorm=True,
                                     entropy_weight=0.1)
    assert np.abs(gf).max() > 0
    # the entropy gradient is the remainder of a cancellation at C >= 12 (tests/test_gpu_lfq_hard_entropy.py)
    close(fg.grad, gf, rtol=0, atol=1e-3 * float(np.abs(gf).max()))


# ------------------------------------------------------------------------------------------------------------------
# model level: PQ-2 MSVR with 2 x 680 tokens per image
# ------------------------------------------------------------------------------------------------------------------
def _model680():
    from test_model_cpu import small_model
    model, _ = small_model("MSVR10P2-4096", num_latent_tokens=256, v_patch_nums=PN)
    return model.cuda()


def test_pq2_680_token_model_trains_bf16():
    model = _model680().train()
    assert model.product_quant == 2 and list(model.v_patch_nums) == PN
    x = (torch.rand(4, 3, 256, 256) * 2 - 1).cuda()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        dec, (vq, commit, ent, usages), _, _, _ = model(x, 0, 0.0, 0.0, 100)
        loss = torch.nn.functional.mse_loss(dec.float(), x) + vq + commit
    loss.backward()
    for v in (loss, vq, commit):
        assert torch.isfinite(v).all()
    missing = [n for n, p in model.named_parameters() if p.requires_grad and p.grad is None]
    assert not missing, missing
    bad = [n for n, p in model.named_parameters() if p.requires_grad and not torch.isfinite(p.grad).all()]
    assert not bad, bad
    for q in model._quantizers():
        assert float(q.embedding.weight.grad.abs().sum()) > 0


def test_pq2_680_token_model_tokens_match_the_oracle(tmp_path):
    from imagefolder_b200 import pretokenize as pt
    model = _model680().eval()
    x = torch.rand(2, 3, 256, 256) * 2 - 1
    with torch.no_grad():
        toks = model.img_to_idxBl(x.cuda())
        branches = model._latent_branches(x.cuda())
    assert len(toks) == 2
    for q, h, ls in zip(model._quantizers(), branches, toks):
        assert [t.shape[1] for t in ls] == [p * p for p in PN] and sum(t.shape[1] for t in ls) == 680
        w, b = _phi_np(q)
        ix = xo.vq2_f_to_idxBl_or_fhat(np.ascontiguousarray(npy(h.float())), npy(q.embedding.weight), w, b, PN,
                                       using_znorm=q.using_znorm)
        for si in range(SN):
            np.testing.assert_array_equal(npy(ls[si]), ix[si])
    path = str(tmp_path / "tokens.jsonl")
    n = pt.pretokenize(model, [(x, torch.tensor([3, 7]))], path, flip=False, autocast_dtype=None)
    assert n == 2
    recs = list(pt.read_tokens(path))
    got = torch.stack([t for _, t in recs])
    assert got.shape == (2, 2 * 680)
    want = torch.cat([torch.cat([t.cpu() for t in ls], dim=1) for ls in toks], dim=1)
    assert torch.equal(got.to(torch.int64), want)
