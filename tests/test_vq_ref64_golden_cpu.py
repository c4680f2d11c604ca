"""Pins the fp64 autograd restatement of the single-scale quantizer and the latent perturbation (oracle/vq_ref64.py) to
the reference: on the single-scale goldens (tests/golden/make_golden.py runs the reference's own VectorQuantizer and
add_perturbation), fed the golden's own indices and selections, its out / vq / commit and the gradients of
sum(out * g_out) + w_vq vq + w_commit commit  with respect to z and the codebook (z and z_q for the perturbation) match
the reference's, at the goldens' tolerance (tests/test_oracle_golden.py).  The fp64 distances must also agree with the
golden's choices: every index is the fp64 nearest code and every selection the fp64 order statistic of its row's rank,
up to near-ties below 1e-5."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import vq_ref64, xq_oracle as xo
from test_oracle_golden import big_vq_inputs, close

TIE = 1e-5


def _vq_inputs(name):
    g = load_golden(name)
    if "z" in g:
        return g, g["z"], g["E"], g["g_out"], bool(g["codebook_norm"]), float(g["beta"])
    E, z, g_out = big_vq_inputs(g)
    return g, z, E, g_out, True, 0.25


def _vq_run(name, mutant=None):
    g, z, E, g_out, cn, beta = _vq_inputs(name)
    zt = torch.from_numpy(z).double().requires_grad_(True)
    Et = torch.from_numpy(E).double().requires_grad_(True)
    fwd = vq_ref64.forward(zt, Et, torch.from_numpy(g["idx"].astype(np.int64)), beta=beta, codebook_norm=cn,
                           mutant=mutant)
    gr = vq_ref64.losses_and_grads(fwd["out"], fwd["vq"], fwd["commit"], dict(z=zt, E=Et),
                                   torch.from_numpy(g_out).double(), float(g["w_vq"]), float(g["w_commit"]),
                                   mutant=mutant)
    gE_ref = np.zeros(E.shape, np.float32)
    gE_ref[g["gE_rows"]] = g["gE_vals"]
    return g, fwd, gr, gE_ref


def _vq_compare(g, fwd, gr, gE_ref):
    sub = "out_sub" in g
    pick = (lambda t: t[:, :, ::2, ::2]) if sub else (lambda t: t)
    close(pick(fwd["out"].detach()), g["out_sub" if sub else "out"])
    if not sub:
        close(fwd["fhat"], g["fhat"])
    close(float(fwd["vq"].detach()), g["vq"])
    close(float(fwd["commit"].detach()), g["commit"])
    close(pick(gr["z"]), g["gz_sub" if sub else "gz"])
    close(gr["E"], gE_ref)


@pytest.mark.parametrize("name", ["vq4096_b1", "vq300_nonorm", "vq8192_c32", "vq16384_c32"])
def test_vq_ref64_vs_golden(name):
    g, fwd, gr, gE_ref = _vq_run(name)
    assert fwd["idx_gap"] < TIE, fwd["idx_gap"]
    _vq_compare(g, fwd, gr, gE_ref)


def _perturb_run(name, mutant=None):
    g = load_golden(name)
    cn = bool(g["codebook_norm"])
    alpha, beta, delta = float(g["alpha"]), float(g["beta"]), int(g["delta"])
    sel = xo.add_perturbation(g["z"], g["zq"], g["E"], cn, alpha, beta, delta, g["rand_u"], g["rand_j"])["sel"]
    z = torch.from_numpy(g["z"]).double().requires_grad_(True)
    zq = torch.from_numpy(g["zq"]).double().requires_grad_(True)
    fwd = vq_ref64.add_perturbation(z, zq, torch.from_numpy(g["E"]).double(), torch.from_numpy(sel),
                                    torch.from_numpy(g["rand_u"]), torch.from_numpy(g["rand_j"]), alpha=alpha,
                                    beta=beta, delta=delta, codebook_norm=cn, mutant=mutant)
    zero = torch.zeros((), dtype=torch.float64)
    gr = vq_ref64.losses_and_grads(fwd["out"], zero, zero, dict(z=z, zq=zq), torch.from_numpy(g["g"]).double(),
                                   0.0, 0.0)
    return g, fwd, gr


def _perturb_compare(g, fwd, gr):
    close(fwd["out"].detach(), g["out"])
    close(gr["z"], g["gz"], atol=1e-6)                   # test_oracle_golden.test_add_perturbation's tolerances
    close(gr["zq"], g["gzq"])


@pytest.mark.parametrize("name", ["perturb_a07", "perturb_a0"])
def test_perturbation_ref64_vs_golden(name):
    g, fwd, gr = _perturb_run(name)
    assert fwd["rank_gap"] < TIE, fwd["rank_gap"]
    _perturb_compare(g, fwd, gr)


@pytest.mark.parametrize("name,mutants", [
    ("vq4096_b1", ["no_norm_jacobian_z", "no_norm_jacobian_E", "swap_vq_commit", "mean_over_rows"]),
    ("vq300_nonorm", ["swap_vq_commit", "mean_over_rows"]),
    ("perturb_a07", ["no_norm_jacobian_z", "perturb_mask_plus_one", "perturb_grad_dropped", "rank_plus_one"]),
])
def test_ref64_mutants_disagree_with_golden(name, mutants):
    """each mutant that can show at the golden's shape moves a golden quantity beyond the tolerance the faithful
    restatement meets, or contradicts the golden's choices (the normalisation mutants need codebook_norm; swap_vq_commit
    and mean_over_rows need a loss the perturbation golden does not have)"""
    for mut in mutants:
        if name.startswith("perturb"):
            g, fwd, gr = _perturb_run(name, mut)
            bad, run = fwd["rank_gap"] >= TIE, lambda: _perturb_compare(g, fwd, gr)
        else:
            g, fwd, gr, gE_ref = _vq_run(name, mut)
            bad, run = fwd["idx_gap"] >= TIE, lambda: _vq_compare(g, fwd, gr, gE_ref)
        try:
            run()
        except AssertionError:
            bad = True
        assert bad, f"mutant {mut} agrees with {name}"
