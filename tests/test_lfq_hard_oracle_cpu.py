"""LFQ(soft_entropy=False): the fp64 closed form of the full-softmax entropy loss (tests/lfq_hard_oracle.py) against
  * a brute-force restatement of the reference's entropy_loss (explicit 2^C softmax, masked_mean, autograd), and
  * golden vectors made by the reference's own LFQ module (tests/golden/make_lfq_hard_golden.py)."""
import numpy as np
import pytest
import torch

import lfq_hard_oracle as lho
from conftest import load_golden

HARD_GOLDENS = ["lfq_hard_c4", "lfq_hard_c5_nonorm", "lfq_hard_c6", "lfq_hard_c8"]


def brute_entropy_loss(x, s, mask, w_sample, w_batch):
    """lookup_free_quantize.py:25-79 + :220-229 in fp64: logits over every code, masked_mean with the int mask."""
    B, C, H, W = x.shape
    idx = torch.arange(2 ** C)
    codebook = (((idx[:, None] >> torch.arange(C)) & 1) * 2.0 - 1.0).double() * s
    xr = x.permute(0, 2, 3, 1).reshape(B, H * W, 1, C)
    logits = 2 * torch.einsum("... i d, j d -> ... i j", xr, codebook)
    m = torch.as_tensor(mask, dtype=torch.int64)
    probs = torch.softmax(logits / 0.01, -1)
    log_probs = torch.log_softmax(logits / 0.01 + 1e-5, -1)

    def masked_mean(t, mm):
        t = t * mm.reshape(mm.shape + (1,) * (t.ndim - mm.ndim))
        return (t / mm.sum()).sum(tuple(range(mm.ndim)))

    avg_probs = masked_mean(probs, m).reshape(-1, 2 ** C).mean(0)
    avg_entropy = -torch.sum(avg_probs * torch.log(avg_probs + 1e-5))
    sample_entropy = masked_mean(-torch.sum(probs * log_probs, -1), m).mean()
    return sample_entropy, avg_entropy, w_sample * sample_entropy - w_batch * avg_entropy


@pytest.mark.parametrize("C", [1, 2, 3, 5, 8, 10])
# z = 400 s x stays below ~10 at these spreads: where a bit's probability saturates, the explicit softmax's autograd
# gradient cancels (p (g - sum p g) with p = 1 - tiny) and is itself no longer good to 1e-10
@pytest.mark.parametrize("spread", [0.005, 0.03])
def test_closed_form_matches_explicit_softmax(C, spread):
    rng = np.random.default_rng(100 + C)
    B, H, W = 3, 4, 3
    x = rng.standard_normal((B, C, H, W)) * spread
    s = 0.7 / np.sqrt(C)
    mask = np.array([1, 0, 1])
    w_s, w_b = 0.8, 1.3
    S, Hc, loss, gx, _ = lho.hard_entropy_scale(x, s, mask, w_s, w_b)
    xt = torch.tensor(x, requires_grad=True)
    S_t, Hc_t, loss_t = brute_entropy_loss(xt, s, mask, w_s, w_b)
    loss_t.backward()
    np.testing.assert_allclose([S, Hc, loss], [float(S_t.detach()), float(Hc_t.detach()), float(loss_t.detach())],
                               rtol=1e-10, atol=1e-13)
    g = xt.grad.numpy()
    np.testing.assert_allclose(gx, g, rtol=0, atol=1e-10 * np.abs(g).max())
    assert np.all(gx[1] == 0.0)          # the masked-out image gets no gradient


def close(a, b, rtol=2e-4):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    np.testing.assert_allclose(a, b, rtol=rtol, atol=rtol * max(1e-30, float(np.abs(b).max())))


def _oracle_args(g):
    return dict(using_znorm=bool(g["using_znorm"]), codebook_drop=float(g["codebook_drop"]), dropout=g["dropout"],
                entropy_weight=float(g["entropy_weight"]), w_sample=float(g["w_sample"]), w_batch=float(g["w_batch"]),
                scaler=g["scaler"])


@pytest.mark.parametrize("name", HARD_GOLDENS)
def test_oracle_matches_reference_golden(name):
    g = load_golden(name)
    pn = [int(p) for p in g["patch_nums"]]
    kw = _oracle_args(g)
    fwd = lho.lfq_hard_forward(g["f"], g["phi_w"], g["phi_b"], pn, **kw)
    for si in range(len(pn)):
        np.testing.assert_array_equal(fwd["idx"][si], g[f"idx{si}"])
    np.testing.assert_allclose(fwd["entropy"], float(g["entropy"]), rtol=1e-5)
    close(fwd["vq"], g["vq"])
    close(fwd["commit"], g["commit"])
    kb = {k: kw[k] for k in ("using_znorm", "entropy_weight", "w_sample", "w_batch")}
    gf, gw, gb = lho.lfq_hard_backward(fwd, g["f"], g["phi_w"], g["phi_b"], pn, g["g_out"], float(g["w_vq"]),
                                       float(g["w_commit"]), float(g["w_ent"]), **kb)
    close(gf, g["gf"])
    close(gw, g["gphi_w"])
    close(gb, g["gphi_b"])


def test_goldens_mask_images_at_late_scales():
    """every golden has an image that stops quantizing before the last scale, so the masked mean is exercised"""
    for name in HARD_GOLDENS:
        g = load_golden(name)
        nd = int(len(g["dropout"]) * float(g["codebook_drop"]))
        assert nd > 0 and int(g["dropout"][:nd].min()) < len(g["patch_nums"]), name


def test_reference_raises_at_batch_one():
    g = load_golden("lfq_hard_b1")
    assert str(g["error"]) == "EinopsError" and bool(g["is_runtime_error"])
