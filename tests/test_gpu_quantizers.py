"""GPU parity tests proper: the CUDA path (through the C ABI) against the CPU oracle and against the
golden vectors made from the reference's own modules.

Bar: token indices and every index-bearing float (z_q / f_hat values) BIT-EXACT against the oracle
(canonical fp32 arithmetic); losses and gradients within 1e-4 relative (the north star allows
1e-3); against the reference goldens indices exact, floats within 2e-4.
"""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import xq_oracle as xo

pytestmark = pytest.mark.gpu

RTOL = 2e-4


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


# ------------------------------------------------------------------------------------------
# single-scale VQ
# ------------------------------------------------------------------------------------------
def make_vq(E, codebook_norm=True, beta=0.25):
    from imagefolder_b200 import VectorQuantizer
    V, C = E.shape
    q = VectorQuantizer(V, C, beta, codebook_norm).cuda().train()
    q.embedding.weight.data.copy_(dev(E))
    return q


@pytest.mark.parametrize("name", ["vq4096_b1", "vq512_randn", "vq300_nonorm"])
def test_vq_golden(name):
    g = load_golden(name)
    cn = bool(g["codebook_norm"])
    q = make_vq(g["E"], cn, float(g["beta"]))
    z = dev(g["z"], grad=True)
    for s in range(int(g["steps"])):
        out, usages, vq, commit, zero = q(z, ret_usages=True)
    assert zero == 0.0
    fwd = xo.vq_forward(g["z"], g["E"], float(g["beta"]), cn)
    np.testing.assert_array_equal(npy(q.last_idx), fwd["idx"])          # bit-exact vs oracle
    np.testing.assert_array_equal(npy(q.last_idx), g["idx"].reshape(-1))  # and vs the reference
    np.testing.assert_array_equal(npy(out), fwd["out"])
    close(out, g["out"])
    close(vq, g["vq"])
    close(commit, g["commit"])
    close(vq, fwd["vq"], rtol=1e-5)
    assert abs(float(usages[0]) - float(g["usage"])) < 1e-3
    close(q.ema_vocab_hit_SV, g["ema"], rtol=1e-6)
    (out * dev(g["g_out"])).sum().add(float(g["w_vq"]) * vq).add(float(g["w_commit"]) * commit).backward()
    close(z.grad, g["gz"])
    gE_ref = np.zeros_like(g["E"])
    gE_ref[g["gE_rows"]] = g["gE_vals"]
    close(q.embedding.weight.grad, gE_ref)
    # inference surface
    idx = q.f_to_idxBl_or_fhat(z.detach(), to_fhat=False, v_patch_nums=None)[0]
    fhat = q.f_to_idxBl_or_fhat(z.detach(), to_fhat=True, v_patch_nums=None)[0]
    assert idx.dtype == torch.int64
    np.testing.assert_array_equal(npy(idx), g["idx"].reshape(-1))
    np.testing.assert_array_equal(npy(fhat), fwd["q_nchw"])
    close(fhat, g["fhat"])


@pytest.mark.parametrize("B,C,hw,V,cn", [(1, 8, 1, 5, True), (3, 17, 7, 129, True), (2, 32, 16, 1000, True),
                                          (5, 64, 5, 4096, True), (2, 12, 9, 300, False), (7, 4, 3, 128, True)])
def test_vq_ragged_sizes(B, C, hw, V, cn):
    rng = np.random.default_rng(B * 1000 + V)
    z = rng.standard_normal((B, C, hw, hw)).astype(np.float32)
    E = (rng.standard_normal((V, C)) * 0.4).astype(np.float32)
    q = make_vq(E, cn)
    zt = dev(z, grad=True)
    out, usages, vq, commit, _ = q(zt)
    fwd = xo.vq_forward(z, E, 0.25, cn)
    np.testing.assert_array_equal(npy(q.last_idx), fwd["idx"])
    np.testing.assert_array_equal(npy(out), fwd["out"])
    close(vq, fwd["vq"], rtol=1e-5)
    g_out = rng.standard_normal(z.shape).astype(np.float32)
    (out * dev(g_out)).sum().add(1.3 * vq).add(0.6 * commit).backward()
    gz, gE = xo.vq_backward(fwd, E, g_out, 1.3, 0.6, 0.25, cn)
    close(zt.grad, gz, rtol=1e-4)
    close(q.embedding.weight.grad, gE, rtol=1e-4)
    hist = np.bincount(fwd["idx"], minlength=V)
    close(q.ema_vocab_hit_SV, hist, rtol=0, atol=0)


def test_vq_ties_first_index():
    """duplicated codebook rows: the lower index must win (torch.argmin semantics)."""
    rng = np.random.default_rng(7)
    E = (rng.standard_normal((64, 16))).astype(np.float32)
    E = np.concatenate([E, E, E], 0)  # rows v, v+64, v+128 are identical
    z = rng.standard_normal((2, 16, 6, 6)).astype(np.float32)
    q = make_vq(E, True)
    q(dev(z))
    idx = npy(q.last_idx)
    assert idx.max() < 64
    np.testing.assert_array_equal(idx, xo.vq_forward(z, E)["idx"])


def test_vq_full_size_properties():
    """BASELINE config #2 shape (VQ-8192, C=32, B=256 -> N=65536): size-independent properties +
    a bit-exact oracle check on a slice of the rows."""
    from imagefolder_b200 import VectorQuantizer
    torch.manual_seed(0)
    q = VectorQuantizer(8192, 32).cuda().train()
    z = torch.randn(256, 32, 16, 16, device="cuda")
    out, usages, vq, commit, _ = q(z)
    idx = q.last_idx.clone()
    assert idx.shape == (65536,) and int(idx.min()) >= 0 and int(idx.max()) < 8192
    assert float(q.ema_vocab_hit_SV.sum()) == 65536.0                       # histogram is a partition
    out2, _, vq2, _, _ = q(z)                                               # deterministic
    assert torch.equal(q.last_idx, idx) and torch.equal(out2, out) and float(vq2) == float(vq)
    # idempotence: a normalised code quantizes to itself
    zq, idx_q = q.f_to_idxBl_or_fhat(z, True)[0], None
    idx_again = q.f_to_idxBl_or_fhat(zq, False)[0]
    En = torch.nn.functional.normalize(q.embedding.weight.data, dim=-1)
    same_code = (En[idx_again] - En[idx]).abs().max(dim=-1).values == 0
    assert bool(same_code.all())
    assert abs(float(commit) - 0.25 * float(vq)) < 1e-7
    # oracle on the first 4 images (1024 rows)
    fwd = xo.vq_forward(npy(z[:4]), npy(q.embedding.weight))
    np.testing.assert_array_equal(npy(idx[:1024]), fwd["idx"])
    np.testing.assert_array_equal(npy(out[:4]), fwd["out"])


# ------------------------------------------------------------------------------------------
# perturbation
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["perturb_a07", "perturb_a0"])
def test_perturb_golden(name):
    from imagefolder_b200 import add_perturbation
    g = load_golden(name)
    cn = bool(g["codebook_norm"])
    emb = torch.nn.Embedding(*g["E"].shape).cuda()
    emb.weight.data.copy_(dev(g["E"]))
    z, zq = dev(g["z"], grad=True), dev(g["zq"], grad=True)
    out = add_perturbation(z, zq, g["z"].shape[1], cn, emb, float(g["alpha"]), float(g["beta"]), int(g["delta"]),
                           rand_u=dev(g["rand_u"]), rand_j=dev(g["rand_j"], torch.int64))
    ref = xo.add_perturbation(g["z"], g["zq"], g["E"], cn, float(g["alpha"]), float(g["beta"]), int(g["delta"]),
                              g["rand_u"], g["rand_j"])
    np.testing.assert_array_equal(npy(out), ref["out"])
    close(out, g["out"])
    (out * dev(g["g"])).sum().backward()
    close(z.grad, g["gz"], atol=1e-6)
    close(zq.grad, g["gzq"])


def test_perturb_rng_stream_matches_reference_calls():
    """without injected tensors the op must consume torch.rand(N) then torch.randint(0,delta,(N,))."""
    from imagefolder_b200 import add_perturbation
    rng = np.random.default_rng(3)
    E = (rng.standard_normal((300, 24)) * 0.3).astype(np.float32)
    z = rng.standard_normal((4, 24, 5, 5)).astype(np.float32)
    emb = torch.nn.Embedding(300, 24).cuda()
    emb.weight.data.copy_(dev(E))
    zt = dev(z)
    zq = torch.zeros_like(zt)
    torch.manual_seed(11)
    out = add_perturbation(zt, zq, 24, True, emb, 0.6, 0.75, 50)
    torch.manual_seed(11)
    u = torch.rand(100, device="cuda")
    j = torch.randint(0, 50, (100,), device="cuda")
    ref = xo.add_perturbation(z, npy(zq), E, True, 0.6, 0.75, 50, npy(u), npy(j))
    np.testing.assert_array_equal(npy(out), ref["out"])
    assert ref["nb"] == 3


def test_perturb_duplicate_codes_rank_order():
    """exact distance ties are ordered by index (canonical (d, idx) order)."""
    from imagefolder_b200 import add_perturbation
    rng = np.random.default_rng(5)
    E0 = (rng.standard_normal((40, 8))).astype(np.float32)
    E = np.concatenate([E0, E0], 0)
    z = rng.standard_normal((2, 8, 3, 3)).astype(np.float32)
    emb = torch.nn.Embedding(80, 8).cuda()
    emb.weight.data.copy_(dev(E))
    N = 18
    u = np.zeros(N, np.float32)
    j = (np.arange(N) % 10).astype(np.int64)
    out = add_perturbation(dev(z), torch.zeros(2, 8, 3, 3, device="cuda"), 8, True, emb, 1.0, 1.0, 10,
                           rand_u=dev(u), rand_j=dev(j, torch.int64))
    ref = xo.add_perturbation(z, np.zeros_like(z), E, True, 1.0, 1.0, 10, u, j)
    np.testing.assert_array_equal(npy(out), ref["out"])


# ------------------------------------------------------------------------------------------
# multi-scale VQ (MSVR)
# ------------------------------------------------------------------------------------------
def make_vq2(g, V, C, pn, zn, share, cd):
    from imagefolder_b200 import VectorQuantizer2
    q = VectorQuantizer2(V, C, using_znorm=zn, v_patch_nums=pn, num_latent_tokens=pn[-1] ** 2,
                         share_quant_resi=share, codebook_drop=cd).cuda().train()
    q.embedding.weight.data.copy_(dev(g["E"]))
    for i, m in enumerate(q.quant_resi.modules_list()):
        m.weight.data.copy_(dev(g["phi_w"][i]))
        m.bias.data.copy_(dev(g["phi_b"][i]))
    return q


@pytest.mark.parametrize("name", ["msvr_small", "msvr_4096", "msvr_l2", "msvr_shared1"])
def test_vq2_golden(name):
    g = load_golden(name)
    pn = [int(p) for p in g["patch_nums"]]
    zn = bool(g["using_znorm"])
    V, C = g["E"].shape
    cd = float(g["codebook_drop"])
    q = make_vq2(g, V, C, pn, zn, int(g["share"]), cd)
    f = dev(g["f"], grad=True)
    dropout = torch.tensor(g["dropout"])
    for _ in range(int(g["steps"])):
        out, usages, vq, commit, zero = q(f, ret_usages=True, dropout=dropout)
    assert zero == 0
    fwd = xo.vq2_forward(g["f"], g["E"], g["phi_w"], g["phi_b"], pn, using_znorm=zn, codebook_drop=cd,
                         dropout=g["dropout"])
    for si in range(len(pn)):
        np.testing.assert_array_equal(npy(q.last_idx_Bl[si]), fwd["idx"][si])
        np.testing.assert_array_equal(npy(q.last_idx_Bl[si]), g[f"idx{si}"])
    np.testing.assert_array_equal(npy(out), fwd["out"])
    close(out, g["out"])
    close(vq, g["vq"])
    close(commit, g["commit"])
    close(torch.stack(usages), g["usages"], rtol=1e-5, atol=1e-3)
    close(q.ema_vocab_hit_SV, g["ema"], rtol=1e-6)
    (out * dev(g["g_out"])).sum().add(float(g["w_vq"]) * vq).add(float(g["w_commit"]) * commit).backward()
    close(f.grad, g["gf"])
    close(q.embedding.weight.grad, g["gE"])
    mods = q.quant_resi.modules_list()
    for i, m in enumerate(mods):
        close(m.weight.grad, g["gphi_w"][i], atol=RTOL * float(np.abs(g["gphi_w"]).max()))
        close(m.bias.grad, g["gphi_b"][i], atol=RTOL * float(np.abs(g["gphi_b"]).max()))
    # inference surfaces
    idx_list = q.f_to_idxBl_or_fhat(f.detach(), to_fhat=False, v_patch_nums=pn)
    fh_list = q.f_to_idxBl_or_fhat(f.detach(), to_fhat=True, v_patch_nums=pn)
    for si in range(len(pn)):
        assert idx_list[si].shape == (g["f"].shape[0], pn[si] ** 2) and idx_list[si].dtype == torch.int64
        np.testing.assert_array_equal(npy(idx_list[si]), g[f"idx{si}"])
    close(fh_list[-1], g["fhat_last"])
    close(fh_list[len(pn) // 2], g["fhat_mid"])
    # decode from tokens reproduces the lookup's f_hat bit for bit; var input matches the reference
    np.testing.assert_array_equal(npy(q.idx_to_fhat(idx_list)), npy(fh_list[-1]))
    close(q.idxBl_to_var_input(idx_list), g["var_input"])


@pytest.mark.parametrize("B,C,V,pn,zn,share", [
    (3, 8, 64, [1, 2, 3], True, 4), (2, 32, 1000, [1, 1, 2, 3, 3, 4, 5, 6, 8, 11], True, 4),
    (5, 20, 130, [2, 4, 6], False, 0), (2, 16, 512, [1, 2, 4, 8, 16], True, 1), (1, 4, 32, [1, 5], True, 4),
    (2, 6, 40, [3], True, 4)])
def test_vq2_random_vs_oracle(B, C, V, pn, zn, share):
    from imagefolder_b200 import VectorQuantizer2
    rng = np.random.default_rng(B * 100 + V)
    H = pn[-1]
    torch.manual_seed(V)
    q = VectorQuantizer2(V, C, using_znorm=zn, v_patch_nums=pn, num_latent_tokens=H * H, share_quant_resi=share,
                         codebook_drop=0.5).cuda().train()
    E = (rng.standard_normal((V, C)) * 0.5).astype(np.float32)
    q.embedding.weight.data.copy_(dev(E))
    mods = q.quant_resi.modules_list()
    phi_w = np.stack([npy(m.weight) for m in mods])
    phi_b = np.stack([npy(m.bias) for m in mods])
    f = rng.standard_normal((B, C, H, H)).astype(np.float32)
    dropout = rng.integers(1, len(pn) + 1, B)
    ft = dev(f, grad=True)
    out, usages, vq, commit, _ = q(ft, ret_usages=True, dropout=torch.tensor(dropout))
    fwd = xo.vq2_forward(f, E, phi_w, phi_b, pn, using_znorm=zn, codebook_drop=0.5, dropout=dropout)
    assert fwd["pmap"] == q._phi_map(len(pn))
    for si in range(len(pn)):
        np.testing.assert_array_equal(npy(q.last_idx_Bl[si]), fwd["idx"][si])
    np.testing.assert_array_equal(npy(out), fwd["out"])
    close(vq, fwd["vq"], rtol=1e-5)
    close(commit, fwd["commit"], rtol=1e-5)
    g_out = rng.standard_normal(f.shape).astype(np.float32)
    (out * dev(g_out)).sum().add(1.1 * vq).add(0.9 * commit).backward()
    gf, gE, gw, gb = xo.vq2_backward(fwd, f, E, phi_w, phi_b, pn, g_out, 1.1, 0.9)
    close(ft.grad, gf, rtol=1e-4)
    close(q.embedding.weight.grad, gE, rtol=1e-4)
    for i, m in enumerate(mods):
        close(m.weight.grad, gw[i], atol=1e-4 * float(np.abs(gw).max()))
        close(m.bias.grad, gb[i], atol=1e-4 * float(np.abs(gb).max()))
    # record_hit is bumped once per scale (quant.py:121-127): only scale 0 copies, the rest blend 0.9/0.1
    ema = np.stack([xo.ema_update(np.zeros(V, np.float32), fwd["hist"][si], si) for si in range(len(pn))])
    close(q.ema_vocab_hit_SV, ema, rtol=1e-6)
    assert q.record_hit == len(pn)


def test_vq2_eval_and_no_dropout():
    """eval mode / dropout=None: every scale contributes for every sample."""
    from imagefolder_b200 import VectorQuantizer2
    rng = np.random.default_rng(1)
    pn = [1, 2, 3, 5]
    q = VectorQuantizer2(100, 8, v_patch_nums=pn, num_latent_tokens=25, codebook_drop=0.5).cuda().eval()
    f = rng.standard_normal((3, 8, 5, 5)).astype(np.float32)
    out, usages, vq, commit, _ = q(dev(f), ret_usages=True, dropout=torch.tensor([1, 1, 1]))
    mods = q.quant_resi.modules_list()
    fwd = xo.vq2_forward(f, npy(q.embedding.weight), np.stack([npy(m.weight) for m in mods]),
                         np.stack([npy(m.bias) for m in mods]), pn, codebook_drop=0.5, dropout=None)
    np.testing.assert_array_equal(npy(out), fwd["out"])
    close(vq, fwd["vq"], rtol=1e-5)
    assert float(q.ema_vocab_hit_SV.sum()) == 0.0 and q.record_hit == 0  # no EMA update in eval


def test_msvr_full_size_properties():
    """BASELINE config #4 branch shape: B=128, C=32, V=4096, 10 scales."""
    from imagefolder_b200 import VectorQuantizer2
    pn = [1, 1, 2, 3, 3, 4, 5, 6, 8, 11]
    torch.manual_seed(0)
    q = VectorQuantizer2(4096, 32, v_patch_nums=pn, num_latent_tokens=121, codebook_drop=0.1).cuda().train()
    q.embedding.weight.data.normal_(0, 0.5)
    f = torch.randn(128, 32, 11, 11, device="cuda")
    dropout = torch.randint(3, 11, (128,))
    out, usages, vq, commit, _ = q(f, ret_usages=True, dropout=dropout)
    out2, _, vq2, _, _ = q(f, ret_usages=True, dropout=dropout)
    assert torch.equal(out, out2) and float(vq) == float(vq2)              # deterministic
    for si, p in enumerate(pn):
        assert float(q.ema_vocab_hit_SV[si].sum()) > 0
    idx_list = q.f_to_idxBl_or_fhat(f, to_fhat=False, v_patch_nums=pn)
    fh = q.f_to_idxBl_or_fhat(f, to_fhat=True, v_patch_nums=pn)
    for si, p in enumerate(pn):
        assert torch.equal(idx_list[si], q.last_idx_Bl[si])                # dropout never changes indices
    assert torch.equal(q.idx_to_fhat(idx_list), fh[-1])                    # encode -> tokens -> decode round trip
    # residual energy decreases with scale
    errs = [float((fh[si] - f).pow(2).mean()) for si in range(len(pn))]
    assert errs[-1] < errs[0]
    # STE value equals the last cumulative f_hat up to fp32 rounding of (F - f) + f -- for the samples
    # without quantizer dropout (the first int(B*codebook_drop) samples lose their late scales)
    nd = int(128 * 0.1)
    assert float((out[nd:] - fh[-1][nd:]).abs().max()) < 1e-5
    assert float((out[:nd] - fh[-1][:nd]).abs().max()) > 1e-3
    # oracle on 2 images
    mods = q.quant_resi.modules_list()
    fwd = xo.vq2_f_to_idxBl_or_fhat(npy(f[:2]), npy(q.embedding.weight), np.stack([npy(m.weight) for m in mods]),
                                    np.stack([npy(m.bias) for m in mods]), pn, to_fhat=False)
    for si in range(len(pn)):
        np.testing.assert_array_equal(npy(idx_list[si][:2]), fwd[si])


# ------------------------------------------------------------------------------------------
# BSQ / LFQ (MSBR)
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["msbr_small", "msbr_14", "lfq_nonorm"])
def test_lfq_golden(name):
    from imagefolder_b200 import LFQ
    g = load_golden(name)
    pn = [int(p) for p in g["patch_nums"]]
    zn = bool(g["using_znorm"])
    C = g["f"].shape[1]
    cd = float(g["codebook_drop"])
    q = LFQ(2 ** C, C, using_znorm=zn, v_patch_nums=pn, num_latent_tokens=pn[-1] ** 2, codebook_drop=cd,
            scale=float(g["scale"]), entropy_weight=float(g["entropy_weight"])).cuda().train()
    close(q.scaler, g["scaler"], rtol=1e-7)
    for i, m in enumerate(q.quant_resi.modules_list()):
        m.weight.data.copy_(dev(g["phi_w"][i]))
        m.bias.data.copy_(dev(g["phi_b"][i]))
    f = dev(g["f"], grad=True)
    dropout = torch.tensor(g["dropout"])
    out, usages, vq, commit, ent = q(f, ret_usages=True, dropout=dropout)
    kw = dict(using_znorm=zn, codebook_drop=cd, dropout=g["dropout"], entropy_weight=float(g["entropy_weight"]),
              scaler=npy(q.scaler))
    fwd = xo.lfq_forward(g["f"], g["phi_w"], g["phi_b"], pn, **kw)
    for si in range(len(pn)):
        np.testing.assert_array_equal(npy(q.last_idx_Bl[si]), fwd["idx"][si])
        np.testing.assert_array_equal(npy(q.last_idx_Bl[si]), g[f"idx{si}"])
    np.testing.assert_array_equal(npy(out), fwd["out"])
    close(out, g["out"])
    close(vq, g["vq"])
    close(commit, g["commit"])
    close(ent, g["entropy"])
    close(torch.stack(usages), g["usages"], rtol=1e-5, atol=1e-3)
    if "ema" in g:
        close(q.ema_vocab_hit_SV, g["ema"], rtol=1e-6)
    loss = (out * dev(g["g_out"])).sum() + float(g["w_vq"]) * vq + float(g["w_commit"]) * commit + float(g["w_ent"]) * ent
    loss.backward()
    close(f.grad, g["gf"])
    for i, m in enumerate(q.quant_resi.modules_list()):
        close(m.weight.grad, g["gphi_w"][i], atol=RTOL * float(np.abs(g["gphi_w"]).max()))
        close(m.bias.grad, g["gphi_b"][i], atol=RTOL * float(np.abs(g["gphi_b"]).max()))
    idx_list = q.f_to_idxBl_or_fhat(f.detach(), to_fhat=False, v_patch_nums=pn)
    fh = q.f_to_idxBl_or_fhat(f.detach(), to_fhat=True, v_patch_nums=pn)
    for si in range(len(pn)):
        np.testing.assert_array_equal(npy(idx_list[si]), g[f"idx{si}"])
    close(fh[-1], g["fhat_last"])
    np.testing.assert_array_equal(npy(q.idx_to_fhat(idx_list)), npy(fh[-1]))
    # bit packing helpers (lookup_free_quantize.py:254-281)
    bits = q.indices_to_bits(idx_list[-1])
    assert torch.equal(q.bits_to_indices(bits), idx_list[-1])


def test_lfq_errors_like_reference():
    from imagefolder_b200 import LFQ
    q = LFQ(64, 6, v_patch_nums=[1, 2, 3], num_latent_tokens=9).cuda()
    f = torch.randn(2, 6, 3, 3, device="cuda")
    with pytest.raises(TypeError):
        q.eval()(f, dropout=torch.tensor([1, 1]))          # eval forward raises in the reference (:174)
    with pytest.raises(TypeError):
        q.train()(f, dropout=None)                         # None[:n] (:171)
    with pytest.raises(AssertionError):
        LFQ(100, 6, v_patch_nums=[1, 2])                   # codebook_size != 2**C (:95)
    with pytest.raises(IndexError):
        q.train()(f[:1], dropout=torch.tensor([1]))        # batch row 1 is indexed (:285) -> needs B >= 2


def test_msbr_full_size_properties():
    """BASELINE config #5 branch shape: B=128, C=14 (V=16384), 10 scales."""
    from imagefolder_b200 import LFQ
    pn = [1, 1, 2, 3, 3, 4, 5, 6, 8, 11]
    torch.manual_seed(0)
    q = LFQ(16384, 14, using_znorm=True, v_patch_nums=pn, num_latent_tokens=121, codebook_drop=0.1,
            entropy_weight=0.1).cuda().train()
    f = torch.randn(128, 14, 11, 11, device="cuda", requires_grad=True)
    dropout = torch.randint(3, 11, (128,))
    out, usages, vq, commit, ent = q(f, ret_usages=True, dropout=dropout)
    (out.sum() + vq + commit + ent).backward()
    assert torch.isfinite(f.grad).all()
    idx_list = q.f_to_idxBl_or_fhat(f.detach(), to_fhat=False, v_patch_nums=pn)
    for si, p in enumerate(pn):
        # histogram is a partition of the 128*p*p tokens; scale 0 copies it, later scales blend 0.9/0.1 (record_hit)
        expect = 128 * p * p * (1.0 if si == 0 else 0.1)
        assert abs(float(q.ema_vocab_hit_SV[si].sum()) - expect) < 1e-3 * expect
        assert int(idx_list[si].max()) < 16384 and int(idx_list[si].min()) >= 0
    fh = q.f_to_idxBl_or_fhat(f.detach(), to_fhat=True, v_patch_nums=pn)
    assert torch.equal(q.idx_to_fhat(idx_list), fh[-1])
    mods = q.quant_resi.modules_list()
    fwd = xo.lfq_forward(npy(f[:2]), np.stack([npy(m.weight) for m in mods]), np.stack([npy(m.bias) for m in mods]),
                         pn, using_znorm=True, dropout=np.array([11, 11]), scaler=npy(q.scaler))
    for si in range(len(pn)):
        np.testing.assert_array_equal(npy(idx_list[si][:2]), fwd["idx"][si])


# ------------------------------------------------------------------------------------------
# TF32 wgmma screening + exact rescoring == exact CUDA-core kernel == oracle (bit for bit)
# ------------------------------------------------------------------------------------------
def _run_vq_algo(algo, z, E):
    import os
    from imagefolder_b200 import ops
    old = os.environ.get("XQ_VQ_ALGO")
    os.environ["XQ_VQ_ALGO"] = algo
    try:
        out, vq, commit, idx, hist = ops.vq_forward(z, E, 0.25, True, True)
        q, idx2 = ops.vq_lookup(z, E, True)
        torch.cuda.synchronize()
    finally:
        if old is None:
            os.environ.pop("XQ_VQ_ALGO", None)
        else:
            os.environ["XQ_VQ_ALGO"] = old
    return out, vq, idx, hist, q, idx2


@pytest.mark.parametrize("B,C,hw,V,init", [(2, 32, 16, 1000, "randn"), (1, 32, 1, 5, "randn"), (5, 64, 5, 4096, "ref"),
                                           (3, 32, 7, 300, "dup"), (64, 32, 16, 8192, "ref"), (256, 32, 16, 8192, "randn"),
                                           (128, 64, 16, 4096, "randn"), (128, 32, 16, 16384, "ref")])
def test_vq_tcgen05_path_is_bit_identical(B, C, hw, V, init):
    """The tensor-core search (TF32 wgmma screening + exact rescoring; the name predates the sm_90a port) against the exact
    CUDA-core kernel and the oracle, bit for bit."""
    torch.manual_seed(B * 7 + V)
    z = torch.randn(B, C, hw, hw, device="cuda")
    if init == "ref":
        E = torch.empty(V, C, device="cuda").uniform_(-1.0 / V, 1.0 / V)
        E = torch.nn.functional.normalize(E, dim=-1)
    else:
        E = torch.randn(V, C, device="cuda") * 0.3
        if init == "dup":                      # exact ties: duplicated rows, lower index must win
            E = torch.cat([E[: V // 3]] * 3 + [E[: V - 3 * (V // 3)]], 0)
    o_e, vq_e, idx_e, hist_e, q_e, idx2_e = _run_vq_algo("exact", z, E)
    o_t, vq_t, idx_t, hist_t, q_t, idx2_t = _run_vq_algo("tc", z, E)
    assert torch.equal(idx_t, idx_e), f"{int((idx_t != idx_e).sum())} index mismatches"
    assert torch.equal(idx2_t, idx_e)
    assert torch.equal(o_t, o_e) and torch.equal(q_t, q_e) and torch.equal(hist_t, hist_e)
    assert abs(float(vq_t) - float(vq_e)) <= 1e-6 * float(vq_e)
    if init == "dup":
        assert int(idx_t.max()) < V // 3
    # and against the CPU oracle on a slice
    nb = min(B, 4)
    fwd = xo.vq_forward(npy(z[:nb]), npy(E))
    np.testing.assert_array_equal(npy(idx_t[: nb * hw * hw]), fwd["idx"])


def _make_varhelp(name):
    from imagefolder_b200 import VectorQuantizer2, LFQ
    g = load_golden(name)
    pn = [int(p) for p in g["patch_nums"]]
    C = g["h0"].shape[1]
    share = int(g["share"])
    if name.endswith("lfq"):
        q = LFQ(2 ** C, C, v_patch_nums=pn, num_latent_tokens=pn[-1] ** 2, share_quant_resi=share).cuda().eval()
    else:
        q = VectorQuantizer2(64, C, v_patch_nums=pn, num_latent_tokens=pn[-1] ** 2, share_quant_resi=share).cuda().eval()
    for i, m in enumerate(q.quant_resi.modules_list()):
        m.weight.data.copy_(dev(g["phi_w"][i]))
        m.bias.data.copy_(dev(g["phi_b"][i]))
    return q, g, pn


@pytest.mark.parametrize("name", ["varhelp_msvr", "varhelp_shared1", "varhelp_lfq"])
def test_var_feature_map_helpers_golden(name):
    """row f-3: embed_to_fhat / get_next_autoregressive_input through xq_ms_embed -- bit-exact vs the oracle,
    within tolerance of the reference modules' own outputs."""
    q, g, pn = _make_varhelp(name)
    SN = len(pn)
    hs = [dev(g[f"h{si}"]) for si in range(SN)]
    want = xo.embed_to_fhat([g[f"h{si}"] for si in range(SN)], g["phi_w"], g["phi_b"], pn)
    fl = q.embed_to_fhat(hs, all_to_max_scale=True, last_one=False)
    assert isinstance(fl, list) and len(fl) == SN
    for si in range(SN):
        np.testing.assert_array_equal(npy(fl[si]), want[si])
        close(fl[si], g[f"fh{si}"])
    last = q.embed_to_fhat(hs, all_to_max_scale=True, last_one=True)
    np.testing.assert_array_equal(npy(last), want[-1])
    close(last, g["fh_last"])
    # the AR loop of models/var.py:218-229: f_hat is updated in place and returned
    f_hat = torch.zeros_like(last)
    Fo = np.zeros_like(want[-1])
    for si in range(SN):
        ret, nxt = q.get_next_autoregressive_input(si, SN, f_hat, hs[si])
        assert ret is f_hat
        Fo, no = xo.get_next_autoregressive_input(si, Fo, g[f"h{si}"], g["phi_w"], g["phi_b"], pn)
        np.testing.assert_array_equal(npy(f_hat), Fo)
        if si != SN - 1:
            assert tuple(nxt.shape) == g[f"next{si}"].shape
            np.testing.assert_array_equal(npy(nxt), no)
            close(nxt, g[f"next{si}"])
        else:
            assert nxt is f_hat
    close(f_hat, g["ar_f_hat"])


def test_var_helpers_consistent_with_token_decode_and_errors():
    """embed_to_fhat on the gathered codes == idx_to_fhat on the tokens (same kernel, two entry forms);
    wrong shapes raise; unusual calls (SN mismatch) keep the reference op sequence."""
    from imagefolder_b200 import VectorQuantizer2
    torch.manual_seed(0)
    pn = [1, 2, 3, 5, 8]
    B, C, V = 5, 12, 96
    q = VectorQuantizer2(V, C, v_patch_nums=pn, num_latent_tokens=64).cuda().eval()
    q.embedding.weight.data.normal_()
    idx = [torch.randint(0, V, (B, p * p), device="cuda") for p in pn]
    hs = [q.embedding(i).transpose(1, 2).reshape(B, C, p, p).contiguous() for i, p in zip(idx, pn)]
    a = q.embed_to_fhat(hs, last_one=True)
    b = q.idx_to_fhat(idx)
    np.testing.assert_array_equal(npy(a), npy(b))
    var = q.idxBl_to_var_input(idx)                                 # [B, sum_{si>=1} pn^2, C]
    f_hat = torch.zeros(B, C, 8, 8, device="cuda")
    pos = 0
    for si in range(len(pn) - 1):
        _, nxt = q.get_next_autoregressive_input(si, len(pn), f_hat, hs[si])
        n = pn[si + 1] ** 2
        np.testing.assert_array_equal(npy(nxt.reshape(B, C, n).transpose(1, 2)), npy(var[:, pos:pos + n]))
        pos += n
    with pytest.raises(ValueError):
        q.embed_to_fhat(hs[:-1])
    with pytest.raises(ValueError):
        q.embed_to_fhat([h[:, :, :1] for h in hs])
    with pytest.raises(ValueError):
        q.get_next_autoregressive_input(1, len(pn), f_hat, hs[2])
    # unusual call (non-contiguous f_hat view): the reference's op sequence on library kernels, same values
    fv = torch.zeros(B, C, 8, 16, device="cuda")[:, :, :, ::2]
    f32 = torch.zeros(B, C, 8, 8, device="cuda")
    rv, nv = q.get_next_autoregressive_input(0, len(pn), fv, hs[0])
    r32, n32 = q.get_next_autoregressive_input(0, len(pn), f32, hs[0])
    assert rv is fv
    close(r32, npy(rv))
    close(n32, npy(nv))


# ------------------------------------------------------------------------------------------
# round 2: reference goldens at the BASELINE codebook sizes, and the unscreened multi-scale seed
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["vq8192_c32", "vq16384_c32"])
def test_vq_baseline_shaped_reference_goldens(name):
    """V = 8192 / 16384, C = 32 (BASELINE configs #2 / #3): indices bit-exact against the REFERENCE's own output
    (tests/golden/make_golden.py --round2-only), on both the tensor-core path and the exact CUDA-core path."""
    import os
    from test_oracle_golden import big_vq_inputs
    g = load_golden(name)
    E, z, g_out = big_vq_inputs(g)
    for algo in ("auto", "exact"):
        os.environ["XQ_VQ_ALGO"] = algo
        try:
            q = make_vq(E)
            zt = dev(z, grad=True)
            out, usage, vq, commit, _ = q(zt, ret_usages=True)
            np.testing.assert_array_equal(npy(q.last_idx).reshape(-1), g["idx"].reshape(-1).astype(np.int64))
            close(out[:, :, ::2, ::2], g["out_sub"])
            close(vq, g["vq"])
            close(commit, g["commit"])
            ((out * dev(g_out)).sum() + float(g["w_vq"]) * vq + float(g["w_commit"]) * commit).backward()
            close(zt.grad[:, :, ::2, ::2], g["gz_sub"])
            gE_ref = np.zeros(E.shape, np.float32)
            gE_ref[g["gE_rows"]] = g["gE_vals"]
            close(q.embedding.weight.grad, gE_ref)
        finally:
            os.environ.pop("XQ_VQ_ALGO", None)


def test_msvr_unscreened_seed_counts_mismatches_on_gpu():
    """The reference's indices on a seed that was NOT screened for near-ties: count the CUDA path's mismatches and
    require each first divergence to be a near-tie (top-2 margin < 1e-5, margins from the oracle on the same inputs)."""
    from imagefolder_b200 import VectorQuantizer2
    from test_oracle_golden import count_first_divergences, msvr_unscreened_inputs
    g = load_golden("msvr_unscreened")
    E, phi_w, phi_b, f, pn = msvr_unscreened_inputs(g)
    V, C = E.shape
    q = VectorQuantizer2(V, C, using_znorm=True, v_patch_nums=pn, num_latent_tokens=pn[-1] ** 2, share_quant_resi=4,
                         codebook_drop=0.0).cuda().eval()
    q.embedding.weight.data.copy_(dev(E))
    for i, m in enumerate(q.quant_resi.modules_list()):
        m.weight.data.copy_(dev(phi_w[i]))
        m.bias.data.copy_(dev(phi_b[i]))
    with torch.no_grad():
        idx = [npy(t) for t in q.f_to_idxBl_or_fhat(dev(f), to_fhat=False, v_patch_nums=pn)]
        fhat = q.f_to_idxBl_or_fhat(dev(f), to_fhat=True, v_patch_nums=pn)[-1]
    fw = xo.vq2_forward(f, E, phi_w, phi_b, pn, using_znorm=True)
    ref = [g[f"idx{si}"] for si in range(len(pn))]
    diverged, tokens = count_first_divergences(idx, ref, fw["margins"], f.shape[0])
    print("msvr_unscreened (GPU): samples diverged", diverged, "tokens", tokens)
    assert diverged <= 1
    if diverged == 0:
        close(fhat[:, :, ::2, ::2], g["fhat_sub"])


# ------------------------------------------------------------------------------------------
# torch.library registration (SURVEY.md section 8b): the usage-EMA step counter on the device, torch.compile(fullgraph=True)
# and CUDA-graph capture
# ------------------------------------------------------------------------------------------
def test_vq_library_ops_compile_fullgraph_and_cuda_graph():
    from imagefolder_b200 import VectorQuantizer
    rng = np.random.default_rng(5)
    V, C, B, hw = 512, 32, 4, 8
    E = (rng.standard_normal((V, C)) * 0.3).astype(np.float32)
    zs = [rng.standard_normal((B, C, hw, hw)).astype(np.float32) for _ in range(3)]

    def make():
        q = VectorQuantizer(V, C).cuda().train()
        q.embedding.weight.data.copy_(dev(E))
        return q

    # (1) three training steps against the oracle: indices and z_q bit for bit, gradients, the EMA schedule on the device counter
    qa = make()
    ema = np.zeros(V, np.float32)
    margin = B * hw * hw / V * 0.08
    for step, z in enumerate(zs):
        za = dev(z, grad=True)
        oa, ua, va, ca, _ = qa(za)
        (oa.sum() * 0.3 + va + ca).backward()
        fwd = xo.vq_forward(z, E)
        np.testing.assert_array_equal(npy(qa.last_idx), fwd["idx"])
        np.testing.assert_array_equal(npy(oa), fwd["out"])
        gz, gE = xo.vq_backward(fwd, E, np.full(z.shape, 0.3, np.float32), 1.0, 1.0, 0.25, True)
        close(za.grad, gz, rtol=1e-4)
        close(qa.embedding.weight.grad, gE, rtol=1e-4)
        qa.embedding.weight.grad = None
        ema = xo.ema_update(ema, np.bincount(fwd["idx"], minlength=V).astype(np.float32), step)
        np.testing.assert_array_equal(npy(qa.ema_vocab_hit_SV), ema)
        assert abs(float(ua[0]) - float((ema >= margin).mean() * 100)) < 1e-4
    assert qa.record_hit == 3

    # (2) torch.compile(fullgraph=True): no graph breaks, same numbers
    qc = make()
    fn = torch.compile(lambda zz: qc(zz)[0:4], fullgraph=True, backend="aot_eager")
    qd = make()
    for z in zs:
        oc, uc, vc, cc = fn(dev(z, grad=True))
        od, ud, vd, cd, _ = qd(dev(z, grad=True))
        assert torch.equal(oc, od) and float(vc) == float(vd) and float(uc[0]) == float(ud[0])
    assert torch.equal(qc.ema_vocab_hit_SV, qd.ema_vocab_hit_SV)

    # (3) CUDA-graph capture of forward + backward of the quantizer (static buffers; replay == eager)
    qg = make()
    z_static = dev(zs[0], grad=True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                      # warm-up on a side stream (allocations, lazy initialisation)
        o, u, v, c, _ = qg(z_static)
        (o.sum() * 0.3 + v + c).backward()
    torch.cuda.current_stream().wait_stream(s)
    qg2 = make()
    qg.load_state_dict(qg2.state_dict())
    qg._record_hit_dev.zero_()
    z_static.grad = None
    qg.embedding.weight.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        o, u, v, c, _ = qg(z_static)
        (o.sum() * 0.3 + v + c).backward()
    qe = make()
    for z in zs:
        z_static.data.copy_(dev(z))
        graph.replay()
        ze = dev(z, grad=True)
        oe, ue, ve, ce, _ = qe(ze)
        qe.embedding.weight.grad = None
        (oe.sum() * 0.3 + ve + ce).backward()
        torch.cuda.synchronize()
        assert torch.equal(o, oe) and float(v) == float(ve) and torch.equal(z_static.grad, ze.grad)
        assert torch.allclose(qg.embedding.weight.grad, qe.embedding.weight.grad, rtol=1e-5, atol=1e-8)
    assert torch.equal(qg.ema_vocab_hit_SV, qe.ema_vocab_hit_SV)


def test_multiscale_usage_counter_crosses_the_schedule_boundary():
    """one training forward of 4 scales from record_hit = 98: row i uses 98 + i, so rows 0-1 blend 0.9/0.1 and rows 2-3
    blend 0.99/0.01, and the device counter advances by SN"""
    from imagefolder_b200 import LFQ, VectorQuantizer2
    pn = [1, 2, 3, 4]
    B = 3
    torch.manual_seed(0)
    for q in (VectorQuantizer2(64, 8, v_patch_nums=pn, num_latent_tokens=16).cuda().train(),
              LFQ(64, 6, v_patch_nums=pn, num_latent_tokens=16).cuda().train()):
        V = q.vocab_size
        ema0 = (torch.rand(len(pn), V, device="cuda") * 50).round()
        q.ema_vocab_hit_SV.copy_(ema0)
        q.record_hit = 98
        q(torch.randn(B, q.Cvae, 4, 4, device="cuda"), ret_usages=True, dropout=torch.full((B,), len(pn) + 1))
        for si in range(len(pn)):
            hit = np.bincount(npy(q.last_idx_Bl[si]).reshape(-1), minlength=V).astype(np.float32)
            want = xo.ema_update(npy(ema0[si]), hit, 98 + si)
            np.testing.assert_array_equal(npy(q.ema_vocab_hit_SV[si]), want)
            w = 0.9 if si < 2 else 0.99
            close(q.ema_vocab_hit_SV[si], npy(ema0[si]) * w + hit * (1 - w), rtol=1e-6)
        assert q.record_hit == 102
