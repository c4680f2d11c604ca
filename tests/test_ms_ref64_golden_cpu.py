"""Pins the fp64 autograd restatement of the multi-scale quantizers (oracle/ms_ref64.py) to the reference: on every
multi-scale golden (tests/golden/make_golden.py runs the reference's own VectorQuantizer2 / LFQ), fed the golden's own
indices, its out / vq / commit / entropy and the gradients of  sum(out * g_out) + w_vq vq + w_commit commit
+ w_ent entropy  with respect to f, the codebook and every Phi weight and bias match the reference's, at the goldens'
tolerance (tests/test_oracle_golden.py).  The fp64 residual must also agree with the golden's indices: every VQ index
is the fp64 best code and every LFQ bit the sign of the fp64 pooled residual, up to near-ties below 1e-5."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import ms_ref64
from test_oracle_golden import close


def _run(g, lfq):
    pn = [int(p) for p in g["patch_nums"]]
    SN = len(pn)
    f = torch.from_numpy(g["f"]).double().requires_grad_(True)
    w = torch.from_numpy(g["phi_w"]).double().requires_grad_(True)
    b = torch.from_numpy(g["phi_b"]).double().requires_grad_(True)
    wrt = dict(f=f, phi_w=w, phi_b=b)
    kw = dict(phi_w=w, phi_b=b, using_znorm=bool(g["using_znorm"]),
              nq=ms_ref64.n_quantizers(f.shape[0], SN, float(g["codebook_drop"]), g["dropout"]))
    if lfq:
        kw.update(scaler=[float(s) for s in g["scaler"]], entropy_weight=float(g["entropy_weight"]))
    else:
        kw["E"] = wrt["E"] = torch.from_numpy(g["E"]).double().requires_grad_(True)
    idx = [torch.from_numpy(g[f"idx{si}"]) for si in range(SN)]
    fwd = ms_ref64.forward(f, idx, pn, lfq=lfq, **kw)
    grads = ms_ref64.losses_and_grads(fwd, wrt, torch.from_numpy(g["g_out"]).double(), float(g["w_vq"]),
                                      float(g["w_commit"]), float(g["w_ent"]) if lfq else 0.0)
    return fwd, grads


@pytest.mark.parametrize("name", ["msvr_small", "msvr_4096", "msvr_l2", "msvr_shared1"])
def test_vq2_ref64_vs_golden(name):
    g = load_golden(name)
    fwd, gr = _run(g, lfq=False)
    assert fwd["idx_gap"] < 1e-5, fwd["idx_gap"]
    close(fwd["out"].detach(), g["out"])
    close(float(fwd["vq"].detach()), g["vq"])
    close(float(fwd["commit"].detach()), g["commit"])
    close(gr["f"], g["gf"])
    close(gr["E"], g["gE"])
    close(gr["phi_w"], g["gphi_w"])
    close(gr["phi_b"], g["gphi_b"])
    SN = len(g["patch_nums"])
    close(fwd["fhat"][-1], g["fhat_last"])
    close(fwd["fhat"][SN // 2], g["fhat_mid"])


@pytest.mark.parametrize("name", ["msbr_small", "msbr_14", "lfq_nonorm"])
def test_lfq_ref64_vs_golden(name):
    g = load_golden(name)
    fwd, gr = _run(g, lfq=True)
    assert fwd["idx_gap"] < 1e-5, fwd["idx_gap"]
    close(fwd["out"].detach(), g["out"])
    close(float(fwd["vq"].detach()), g["vq"])
    close(float(fwd["commit"].detach()), g["commit"])
    close(float(fwd["entropy"].detach()), g["entropy"])
    close(gr["f"], g["gf"])
    close(gr["phi_w"], g["gphi_w"])
    close(gr["phi_b"], g["gphi_b"])
    close(fwd["fhat"][-1], g["fhat_last"])


@pytest.mark.parametrize("name,lfq", [("msvr_small", False), ("msbr_small", True)])
def test_ref64_mutants_disagree_with_golden(name, lfq):
    """each mutant that can show at the golden's shape moves a golden quantity beyond the tolerance the faithful
    restatement meets, or contradicts the golden's indices"""
    g = load_golden(name)
    muts = ["share_map_shift", "nq_plus_one", "swap_vq_commit", "area_floor"]
    # LFQ codes are constants: nothing flows back through the Phi input or the bicubic upsample.  (The entropy-row
    # mutant is not listed: next to the goldens' unit-sized g_out the entropy gradient is below their tolerance.)
    if not lfq:
        muts += ["phi_r_twice", "phi_r_dropped", "bicubic_T_align_corners"]
    for mut in muts:
        orig_fwd = ms_ref64.forward
        ms_ref64.forward = lambda *a, _m=mut, **k: orig_fwd(*a, mutant=_m, **k)
        orig_lg = ms_ref64.losses_and_grads
        ms_ref64.losses_and_grads = lambda *a, _m=mut, **k: orig_lg(*a, mutant=_m, **k)
        try:
            fwd, gr = _run(g, lfq)
        finally:
            ms_ref64.forward, ms_ref64.losses_and_grads = orig_fwd, orig_lg
        bad = fwd["idx_gap"] >= 1e-5
        pairs = [("f", "gf"), ("phi_w", "gphi_w"), ("phi_b", "gphi_b")] + ([] if lfq else [("E", "gE")])
        for mine, ref in pairs:
            try:
                close(gr[mine], g[ref])
            except AssertionError:
                bad = True
        assert bad, f"mutant {mut} agrees with {name}"
