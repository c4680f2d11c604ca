"""LFQ(soft_entropy=False) on the GPU: the closed-form full-softmax entropy kernels (csrc/ms_kernels.cu, mode
XQ_MS_BSQ_HARD) against the reference's goldens and against the fp64 oracle (tests/lfq_hard_oracle.py).

Bar: token indices bit-exact; against the goldens everything as test_gpu_quantizers.test_lfq_golden; against the oracle
the entropy loss within 1e-4 relative and its gradient wrt f within 1e-4 of the gradient's largest magnitude."""
import ctypes

import numpy as np
import pytest
import torch

import lfq_hard_oracle as lho
from conftest import load_golden

pytestmark = pytest.mark.gpu

RTOL = 2e-4
MS = [1, 1, 2, 3, 3, 4, 5, 6, 8, 11]


def close(a, b, rtol=RTOL, atol=None):
    a = np.asarray(a.detach().cpu().numpy() if torch.is_tensor(a) else a, np.float64)
    b = np.asarray(b, np.float64)
    if atol is None:
        atol = rtol * max(1e-30, float(np.abs(b).max()))
    np.testing.assert_allclose(a, b, rtol=rtol, atol=atol)


def dev(a, dtype=torch.float32, grad=False):
    t = torch.tensor(np.asarray(a), dtype=dtype, device="cuda")
    return t.requires_grad_(True) if grad else t


def npy(t):
    return t.detach().cpu().numpy()


def make_lfq(C, pn, using_znorm=True, codebook_drop=0.0, scale=1.0, entropy_weight=0.1, w_sample=1.0, w_batch=1.0,
             seed=0):
    from imagefolder_b200 import LFQ
    torch.manual_seed(seed)
    q = LFQ(2 ** C, C, using_znorm=using_znorm, v_patch_nums=pn, num_latent_tokens=pn[-1] ** 2,
            codebook_drop=codebook_drop, scale=scale, entropy_weight=entropy_weight, sample_minimization_weight=w_sample,
            batch_maximization_weight=w_batch, soft_entropy=False).cuda().train()
    for m in q.quant_resi.modules_list():        # non-trivial Phi weights
        m.weight.data.normal_(0, 0.1)
        m.bias.data.normal_(0, 0.05)
    return q


def phi_params(q):
    mods = q.quant_resi.modules_list()
    return np.stack([npy(m.weight) for m in mods]), np.stack([npy(m.bias) for m in mods])


@pytest.mark.parametrize("name", ["lfq_hard_c4", "lfq_hard_c5_nonorm", "lfq_hard_c6", "lfq_hard_c8"])
def test_lfq_hard_golden(name):
    from imagefolder_b200 import LFQ
    g = load_golden(name)
    pn = [int(p) for p in g["patch_nums"]]
    zn = bool(g["using_znorm"])
    C = g["f"].shape[1]
    cd = float(g["codebook_drop"])
    ws, wb = float(g["w_sample"]), float(g["w_batch"])
    q = LFQ(2 ** C, C, using_znorm=zn, v_patch_nums=pn, num_latent_tokens=pn[-1] ** 2, codebook_drop=cd,
            scale=float(g["scale"]), entropy_weight=float(g["entropy_weight"]), sample_minimization_weight=ws,
            batch_maximization_weight=wb, soft_entropy=False).cuda().train()
    close(q.scaler, g["scaler"], rtol=1e-7)
    for i, m in enumerate(q.quant_resi.modules_list()):
        m.weight.data.copy_(dev(g["phi_w"][i]))
        m.bias.data.copy_(dev(g["phi_b"][i]))
    f = dev(g["f"], grad=True)
    out, usages, vq, commit, ent = q(f, ret_usages=True, dropout=torch.tensor(g["dropout"]))
    kw = dict(using_znorm=zn, codebook_drop=cd, dropout=g["dropout"], entropy_weight=float(g["entropy_weight"]),
              w_sample=ws, w_batch=wb, scaler=npy(q.scaler))
    fwd = lho.lfq_hard_forward(g["f"], g["phi_w"], g["phi_b"], pn, **kw)
    for si in range(len(pn)):
        np.testing.assert_array_equal(npy(q.last_idx_Bl[si]), fwd["idx"][si])
        np.testing.assert_array_equal(npy(q.last_idx_Bl[si]), g[f"idx{si}"])
    np.testing.assert_array_equal(npy(out), fwd["out"])
    close(out, g["out"])
    close(vq, g["vq"])
    close(commit, g["commit"])
    close(ent, g["entropy"])
    close(torch.stack(usages), g["usages"], rtol=1e-5, atol=1e-3)
    close(q.ema_vocab_hit_SV, g["ema"], rtol=1e-6)
    loss = (out * dev(g["g_out"])).sum() + float(g["w_vq"]) * vq + float(g["w_commit"]) * commit + float(g["w_ent"]) * ent
    loss.backward()
    close(f.grad, g["gf"])
    for i, m in enumerate(q.quant_resi.modules_list()):
        close(m.weight.grad, g["gphi_w"][i], atol=RTOL * float(np.abs(g["gphi_w"]).max()))
        close(m.bias.grad, g["gphi_b"][i], atol=RTOL * float(np.abs(g["gphi_b"]).max()))


# (C, B, patch_nums, using_znorm, codebook_drop, dropout (first int(B*codebook_drop) images), scale, w_sample, w_batch)
ORACLE_CASES = {
    "msbr16384_b128": (14, 128, MS, True, 0.1, "rand", 1.0, 1.0, 1.0),
    "msbr4096_b128": (12, 128, MS, True, 0.1, "rand", 1.0, 1.0, 1.0),
    "b2": (10, 2, [1, 2, 3, 5], True, 0.5, [3], 1.0, 1.0, 1.0),
    "b3_nonorm": (9, 3, [1, 2, 4], False, 0.0, None, 0.9, 1.0, 1.0),
    "one_image_left": (8, 3, [1, 2, 3, 5], True, 0.67, [1, 2], 1.0, 1.0, 1.0),
    "weights": (11, 4, [1, 2, 3, 5], True, 0.5, [2, 3], 1.1, 0.3, 2.5),
}
# C = 1 without using_znorm: normalising a single channel has a zero Jacobian, so no gradient would reach f
ORACLE_CASES.update({f"c{C}": (C, 3, [1, 2, 3], C > 1, 0.34, [2], 1.0, 1.0, 1.0) for C in range(1, 17)})
# With 27 rows and C >= 12 almost every row has codes of its own.  For such a row the sample-entropy and codebook-entropy
# gradients are equal and opposite up to the 1e-5 inside the log, so the gradient is the remainder of a cancellation.
# An fp32 restatement of the same arithmetic on the CPU is off by 2e-4 of the largest gradient at C = 14.
# These cases check the gradient to 1e-3 of its largest magnitude; the entropy value keeps the 1e-4 bound.
GRAD_TOL = {f"c{C}": 1e-3 for C in range(12, 17)}


def run_case(case, seed=0):
    C, B, pn, zn, cd, dropout, scale, ws, wb = ORACLE_CASES[case]
    q = make_lfq(C, pn, using_znorm=zn, codebook_drop=cd, scale=scale, w_sample=ws, w_batch=wb, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    f = torch.randn(B, C, pn[-1], pn[-1], generator=g)
    SN = len(pn)
    nd = int(B * cd)
    if dropout == "rand":
        dr = torch.randint(3, SN + 1, (B,), generator=g)
    else:
        dr = torch.full((B,), SN + 1, dtype=torch.int64)
        if dropout is not None:
            dr[:nd] = torch.tensor(dropout)[:nd]
    return q, f, dr


@pytest.mark.parametrize("case", list(ORACLE_CASES))
def test_lfq_hard_against_oracle(case):
    C, B, pn, zn, cd, _, scale, ws, wb = ORACLE_CASES[case]
    q, f, dr = run_case(case)
    fg = f.cuda().requires_grad_(True)
    out, _, vq, commit, ent = q(fg, dropout=dr)
    ent.backward()                                  # the entropy term's gradient alone
    pw, pb = phi_params(q)
    fwd = lho.lfq_hard_forward(f.numpy(), pw, pb, pn, using_znorm=zn, codebook_drop=cd, dropout=dr.numpy(),
                               entropy_weight=0.1, w_sample=ws, w_batch=wb, scaler=npy(q.scaler))
    for si in range(len(pn)):
        np.testing.assert_array_equal(npy(q.last_idx_Bl[si]), fwd["idx"][si])
    np.testing.assert_allclose(float(ent.detach()), fwd["entropy"], rtol=1e-4)
    gf, _, _ = lho.lfq_hard_backward(fwd, f.numpy(), pw, pb, pn, np.zeros(f.shape), 0.0, 0.0, 1.0, using_znorm=zn,
                                     entropy_weight=0.1, w_sample=ws, w_batch=wb)
    assert np.abs(gf).max() > 0
    close(fg.grad, gf, rtol=0, atol=GRAD_TOL.get(case, 1e-4) * float(np.abs(gf).max()))
    if case == "one_image_left":                    # scale 1 keeps images 1, 2; scales 2, 3 only image 2
        assert [int(m.sum()) for m in fwd["masks"]] == [3, 2, 1, 1]


def _entropy_and_grad(q, f, dr):
    fg = f.cuda().requires_grad_(True)
    out, _, vq, commit, ent = q(fg, dropout=dr)
    (out.sum() + vq + commit + ent).backward()
    return ent.detach().clone(), fg.grad.clone()


def test_lfq_hard_bitwise_repeatable():
    q, f, dr = run_case("msbr16384_b128")
    e1, g1 = _entropy_and_grad(q, f, dr)
    e2, g2 = _entropy_and_grad(q, f, dr)
    assert torch.equal(e1.view(torch.int32), e2.view(torch.int32))
    assert torch.equal(g1.view(torch.int32), g2.view(torch.int32))


def test_lfq_hard_side_stream():
    q, f, dr = run_case("msbr4096_b128")
    e0, g0 = _entropy_and_grad(q, f, dr)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        e1, g1 = _entropy_and_grad(q, f, dr)
    s.synchronize()
    assert torch.equal(e0.view(torch.int32), e1.view(torch.int32))
    assert torch.equal(g0.view(torch.int32), g1.view(torch.int32))


def test_lfq_hard_refuses_c17_and_writes_nothing():
    from imagefolder_b200 import _capi as C
    from imagefolder_b200 import LFQ
    L = C.lib()
    B, Cc, H = 2, 17, 3
    d = C.make_ms_desc(B, Cc, H, H, 2 ** Cc, 0, [1, 3], [-1, -1], C.XQ_MS_BSQ_HARD, scaler=[1.0, 1.0], loss_div_sn_all=True,
                       entropy_weight=0.1)
    assert L.xq_ms_workspace_bytes(ctypes.byref(d)) == 0 and L.xq_ms_saved_bytes(ctypes.byref(d)) == 0
    f = torch.randn(B, Cc, H, H, device="cuda")
    out = torch.full_like(f, 7.0)
    idx = torch.full((B * 10,), -5, dtype=torch.int64, device="cuda")
    loss = torch.full((3,), 7.0, device="cuda")
    buf = torch.full((1 << 20,), 3, dtype=torch.uint8, device="cuda")
    nq = torch.full((B,), 3.0, device="cuda")
    rc = L.xq_ms_forward(ctypes.byref(d), C.ptr(f), None, None, None, C.ptr(nq), 1, C.ptr(out), C.ptr(idx), None,
                         C.ptr(loss), None, C.ptr(buf[:1 << 19]), C.ptr(buf[1 << 19:]), 1 << 19, C.stream_ptr())
    torch.cuda.synchronize()
    assert rc == -4                                  # XQ_ERR_UNSUPPORTED
    assert bool((out == 7.0).all()) and bool((idx == -5).all()) and bool((loss == 7.0).all()) and bool((buf == 3).all())
    q = LFQ(2 ** 17, 17, v_patch_nums=[1, 3], num_latent_tokens=9, soft_entropy=False).cuda().train()
    with pytest.raises(NotImplementedError):
        q(f, dropout=torch.tensor([3, 3]))


def test_lfq_hard_batch_one_raises_like_reference():
    g = load_golden("lfq_hard_b1")
    assert bool(g["is_runtime_error"])
    q = make_lfq(4, [1, 2, 3], codebook_drop=0.5)
    with pytest.raises(RuntimeError):
        q(torch.randn(1, 4, 3, 3, device="cuda"), dropout=torch.tensor([2]))


def test_vq_model_pq2_hard_entropy_trains():
    """VQModel from ModelArgs(lfq=True, product_quant=2, soft_entropy=False) at ViT-S width: forward + backward."""
    from imagefolder_b200 import config as xcfg
    c = dict(xcfg.SHIPPED_CONFIGS["MSBR10P2-16384"])
    c.update(encoder_model="vit_small_patch14_dinov2.lvd142m", decoder_model="vit_small_patch14_dinov2.lvd142m",
             semantic_guide="none", detail_guide="none", guide_type_2="patch")
    args = xcfg.parse_args([])
    for k, v in c.items():
        setattr(args, k, v)
    torch.manual_seed(0)
    model = xcfg.build_vq_model(args, soft_entropy=False).cuda().train()
    assert model.config.lfq and model.config.product_quant == 2 and not model.config.soft_entropy
    assert all(not q.soft_entropy for q in model._quantizers())
    x = (torch.rand(2, 3, 256, 256) * 2 - 1).cuda()
    dec, (vq, commit, ent, usages), _, _, _ = model(x, 0, 0.0, 0.0, 100)
    loss = torch.nn.functional.mse_loss(dec.float(), x) + vq + commit + ent
    loss.backward()
    assert all(bool(torch.isfinite(t)) for t in (vq, commit, ent, loss))
    assert float(ent) != 0.0
    grads = [p.grad for p in model.parameters() if p.grad is not None]
    assert grads and all(bool(torch.isfinite(g).all()) for g in grads)
