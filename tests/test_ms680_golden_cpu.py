"""Pins the CPU oracles to the reference at VAR's default 680-token pyramid, v_patch_nums = [1,2,3,4,5,6,8,10,13,16]
(tests/golden/make_ms680_golden.py runs the reference's own VectorQuantizer2 at C = 32, V = 4096, B = 2 on inputs drawn
by tests/ms680_inputs.py from the stored seed):

  msvr680_znorm  using_znorm, share_quant_resi = 4, codebook_drop = 0.5 (one of the two images dropped)
  msvr680_l2     the L2 metric, VAR's own quantizer
  varhelp680     embed_to_fhat and the get_next_autoregressive_input chain

The fp32 C oracle (oracle/xq_oracle.py) must reproduce indices, out, losses, usage EMA, every gradient and every
f_to_idxBl_or_fhat entry (on the stored stride-3 grid); the fp64 restatement (oracle/ms_ref64.py), fed the golden's indices, the values and gradients
and an index gap below the 1e-5 tie.  Tolerances are those of tests/test_oracle_golden.py."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import ms_ref64, xq_oracle as xo
from ms680_inputs import FHAT_SUB, PN680, VAR_SUB, load680
from test_oracle_golden import check_idx, close

NAMES = ["msvr680_znorm", "msvr680_l2"]


def var_input_from_fhat(fhats, pn):
    """idxBl_to_var_input (quant.py:226-244): scale si's cumulative f_hat area-pooled to the next scale, as
    [B, sum_{si>=1} pn^2, C] rows"""
    B, C = fhats[0].shape[:2]
    return np.concatenate([xo.area_pool_rows(fhats[si], pn[si + 1]).reshape(B, -1, C) for si in range(len(pn) - 1)],
                          axis=1)


@pytest.mark.parametrize("name", NAMES)
def test_golden_is_the_680_token_pyramid(name):
    g = load680(name)
    assert [int(p) for p in g["patch_nums"]] == PN680
    assert g["E"].shape == (4096, 32) and g["f"].shape == (2, 32, 16, 16)
    assert sum(g[f"idx{si}"].shape[1] for si in range(len(PN680))) == 680


@pytest.mark.parametrize("name", NAMES)
def test_oracle_reproduces_680_token_golden(name):
    g = load680(name)
    pn = [int(p) for p in g["patch_nums"]]
    zn = bool(g["using_znorm"])
    fwd = xo.vq2_forward(g["f"], g["E"], g["phi_w"], g["phi_b"], pn, using_znorm=zn,
                         codebook_drop=float(g["codebook_drop"]), dropout=g["dropout"])
    for si in range(len(pn)):
        assert check_idx(fwd["idx"][si], g[f"idx{si}"], fwd["margins"][si]) == 0
    close(fwd["out"], g["out"])
    close(fwd["vq"], g["vq"])
    close(fwd["commit"], g["commit"])
    gf, gE, gw, gb = xo.vq2_backward(fwd, g["f"], g["E"], g["phi_w"], g["phi_b"], pn, g["g_out"], float(g["w_vq"]),
                                     float(g["w_commit"]))
    close(gf, g["gf"])
    close(gE, g["gE"])
    close(gw, g["gphi_w"])
    close(gb, g["gphi_b"])
    fh = xo.vq2_f_to_idxBl_or_fhat(g["f"], g["E"], g["phi_w"], g["phi_b"], pn, using_znorm=zn, to_fhat=True)
    for si in range(len(pn)):
        close(fh[si][FHAT_SUB], g[f"fhat_sub{si}"])
    SN, V = len(pn), g["E"].shape[0]
    ema = np.zeros((SN, V), np.float32)
    for si in range(SN):                      # record_hit advances once per scale (quant.py:121-127)
        ema[si] = xo.ema_update(ema[si], fwd["hist"][si], si)
    close(ema, g["ema"], rtol=1e-6)
    N = g["f"].shape[0] * g["f"].shape[2] * g["f"].shape[3]
    close((ema >= N / V * 0.08).mean(axis=1) * 100, g["usages"], rtol=1e-5, atol=1e-3)
    close(var_input_from_fhat(fh, pn)[VAR_SUB], g["var_input_sub"])


@pytest.mark.parametrize("name", NAMES)
def test_ref64_reproduces_680_token_golden(name):
    g = load680(name)
    pn = [int(p) for p in g["patch_nums"]]
    SN = len(pn)
    leaf = lambda a: torch.from_numpy(a).double().requires_grad_(True)
    wrt = dict(f=leaf(g["f"]), E=leaf(g["E"]), phi_w=leaf(g["phi_w"]), phi_b=leaf(g["phi_b"]))
    nq = ms_ref64.n_quantizers(g["f"].shape[0], SN, float(g["codebook_drop"]), g["dropout"])
    idx = [torch.from_numpy(g[f"idx{si}"]) for si in range(SN)]
    fwd = ms_ref64.forward(wrt["f"], idx, pn, lfq=False, E=wrt["E"], phi_w=wrt["phi_w"], phi_b=wrt["phi_b"], nq=nq,
                           using_znorm=bool(g["using_znorm"]))
    gr = ms_ref64.losses_and_grads(fwd, wrt, torch.from_numpy(g["g_out"]).double(), float(g["w_vq"]),
                                   float(g["w_commit"]))
    assert fwd["idx_gap"] < 1e-5, fwd["idx_gap"]
    close(fwd["out"].detach(), g["out"])
    close(float(fwd["vq"].detach()), g["vq"])
    close(float(fwd["commit"].detach()), g["commit"])
    close(gr["f"], g["gf"])
    close(gr["E"], g["gE"])
    close(gr["phi_w"], g["gphi_w"])
    close(gr["phi_b"], g["gphi_b"])
    for si in range(SN):
        close(fwd["fhat"][si].detach()[FHAT_SUB], g[f"fhat_sub{si}"])


def test_oracle_reproduces_680_token_var_helpers():
    g = load_golden("varhelp680")
    pn = [int(p) for p in g["patch_nums"]]
    assert pn == PN680
    SN = len(pn)
    hs = [g[f"h{si}"] for si in range(SN)]
    fl = xo.embed_to_fhat(hs, g["phi_w"], g["phi_b"], pn)
    for si in range(SN):
        close(fl[si], g[f"fh{si}"])
    close(xo.embed_to_fhat(hs, g["phi_w"], g["phi_b"], pn, last_one=True), g["fh_last"])
    F = np.zeros_like(g["fh_last"])
    for si in range(SN):
        F, nxt = xo.get_next_autoregressive_input(si, F, hs[si], g["phi_w"], g["phi_b"], pn)
        assert nxt.shape == g[f"next{si}"].shape
        close(nxt, g[f"next{si}"])
    close(F, g["ar_f_hat"])
