"""The VQ code searches on codebooks built to reach the branches random data never makes decisive: zero and tiny codes
(F1), collapsed clusters that overflow the tensor-core search's candidate list (F2), late winners that force compaction
(F3), in-group near ties whose order TF32 truncation reverses (F4), worst-case truncation (F5), the negative half-space
with ragged V (F6) and exact ties at group / tile boundaries (F7).  tests/vq_screen_model.py builds the inputs and
tests/test_vq_screen_model_cpu.py shows which branch each family reaches.

Bar: the tensor-core search (XQ_VQ_ALGO=tc), the exact CUDA-core search (exact), the default (auto) and the CPU oracle
agree bit for bit on indices, outputs, lookups and histograms; and on every row the chosen code is the fp64 argmin of
the real-number key up to the fp32 rounding of the canonical key (a check independent of the oracle)."""
import os

import numpy as np
import pytest
import torch

import vq_screen_model as m
from oracle import xq_oracle as xo

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                 # fp32 unit roundoff
ORACLE_MACS = 5e9              # rows x codes x channels the CPU oracle runs on in full


@pytest.fixture(scope="module", autouse=True)
def _report_cost():
    import time
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield
    torch.cuda.synchronize()
    print(f"\n[vq adversarial] {time.time() - t0:.1f} s, peak extra device memory "
          f"{(torch.cuda.max_memory_allocated() - base) / 2 ** 20:.0f} MiB")


def _npy(t):
    return t.detach().cpu().numpy()


def _run(algo, z, E, cn):
    from imagefolder_b200 import ops
    old = os.environ.get("XQ_VQ_ALGO")
    os.environ["XQ_VQ_ALGO"] = algo
    try:
        out, vq, _, idx, hist = ops.vq_forward(z, E, 0.25, cn, True)
        q, idx2 = ops.vq_lookup(z, E, cn)
        torch.cuda.synchronize()
    finally:
        if old is None:
            os.environ.pop("XQ_VQ_ALGO", None)
        else:
            os.environ["XQ_VQ_ALGO"] = old
    return dict(out=out, vq=float(vq), idx=idx, hist=hist, q=q, idx2=idx2)


def _fp64_check(z_rows, E, idx, cn):
    """d64 = zz + ee - 2 zn.c in fp64 from the fp32 normalised vectors (the canonical ones), on the GPU in row chunks.

    Bound: the canonical key is d32 = fl(fma(-2, dot32, fl(zz32 + ee32))), every term an fp32 fma chain over C
    channels.  With u = 2^-24: |dot32 - dot| <= C u sum|z_k c_k| <= C u |z||c|, |zz32 - zz| <= C u zz, |ee32 - ee| <= C u ee,
    the sum and the final fma add u (zz + ee) and u |d|.  So |d32 - d| <= delta = u (2 C |z||c| + (C + 1)(zz + ee) + |d|),
    with |d| <= (|z| + |c|)^2.  The chosen code minimises d32, so d(chosen) <= d32(chosen) + delta <= d32(best) + delta
    <= d(best) + 2 delta: tau = 2 delta, taken with the largest code norm.  fp64's own error (~1e-15) is far below it."""
    zn = m.normalise(z_rows) if cn else z_rows
    En = m.normalise(E) if cn else E
    C = zn.shape[1]
    Ed = torch.from_numpy(En).cuda().double()
    ee = (Ed * Ed).sum(1)
    cmax, eemax = float(ee.max().sqrt()), float(ee.max())
    idx = idx.view(-1, 1)
    chunk = max(1, (1 << 27) // max(1, En.shape[0]))
    for s in range(0, zn.shape[0], chunk):
        zd = torch.from_numpy(zn[s:s + chunk]).cuda().double()
        zz = (zd * zd).sum(1)
        d = zz[:, None] + ee[None, :] - 2.0 * (zd @ Ed.T)
        chosen = d.gather(1, idx[s:s + chunk]).squeeze(1)
        zl = zz.sqrt()
        tau = 2.0 * U * (2 * C * zl * cmax + (C + 1) * (zz + eemax) + (zl + cmax) ** 2)
        bad = chosen > d.min(1).values + tau
        assert not bool(bad.any()), f"rows {torch.nonzero(bad)[:8, 0].tolist()} chose a code beyond the fp32 rounding bound"


def _check_family(fam, V, C, B, hw, cn=True, algos=("tc", "exact", "auto")):
    N = B * hw * hw
    z_rows, E = m.FAMILIES[fam](V, C, N)
    z = torch.from_numpy(m.rows_to_nchw(z_rows, B, hw)).cuda()
    Et = torch.from_numpy(E).cuda()
    runs = {a: _run(a, z, Et, cn) for a in algos}
    ref = runs["exact"]
    for a, r in runs.items():
        bad = int((r["idx"] != ref["idx"]).sum())
        assert bad == 0, f"{fam} V={V} C={C}: {a} differs from exact on {bad} of {N} rows"
        assert torch.equal(r["idx2"], ref["idx"]), f"{a}: lookup indices"
        assert torch.equal(r["out"], ref["out"]) and torch.equal(r["q"], ref["q"]), f"{a}: outputs"
        assert torch.equal(r["hist"], ref["hist"]), f"{a}: histogram"
        assert abs(r["vq"] - ref["vq"]) <= 1e-6 * abs(ref["vq"]) + 1e-30, f"{a}: vq loss"
    # oracle on every row up to ORACLE_MACS, else on a slice of whole images
    nb = B if N * V * C <= ORACLE_MACS else max(1, int(ORACLE_MACS // (hw * hw * V * C)))
    fwd = xo.vq_forward(m.rows_to_nchw(z_rows[: nb * hw * hw], nb, hw), E, 0.25, cn)
    np.testing.assert_array_equal(_npy(ref["idx"][: nb * hw * hw]), fwd["idx"])
    np.testing.assert_array_equal(_npy(ref["out"][:nb]), fwd["out"])
    np.testing.assert_array_equal(_npy(ref["q"][:nb]), fwd["q_nchw"])
    _fp64_check(z_rows, E, ref["idx"], cn)
    return z_rows, E, ref


# (family, V, C, B, hw): both searches
BOTH = [("F1", 300, 32, 3, 7), ("F1", 1000, 32, 4, 16), ("F1", 4096, 64, 4, 16), ("F1", 8192, 32, 3, 7),
        ("F1", 16384, 32, 4, 16), ("F2", 1000, 32, 4, 16), ("F2", 4096, 64, 3, 7), ("F2", 16384, 32, 4, 16),
        ("F3", 4096, 32, 4, 16), ("F3", 8192, 64, 3, 7), ("F4", 300, 32, 4, 16), ("F4", 4096, 64, 3, 7),
        ("F5", 300, 64, 4, 16), ("F5", 4096, 32, 3, 7), ("F6", 5, 32, 3, 7), ("F6", 33, 32, 4, 16),
        ("F6", 129, 64, 4, 16), ("F6", 300, 32, 3, 7), ("F6", 1000, 64, 4, 16), ("F7", 33, 32, 3, 7),
        ("F7", 1000, 32, 4, 16), ("F7", 4096, 64, 4, 16), ("F7", 16384, 32, 3, 7)]


@pytest.mark.parametrize("fam,V,C,B,hw", BOTH)
def test_tc_exact_auto_and_oracle_agree(fam, V, C, B, hw):
    _check_family(fam, V, C, B, hw)


# the exact kernel alone: channel counts the tensor-core search does not take, and codebook_norm=False
@pytest.mark.parametrize("fam,V,C,cn", [("F1", 300, 8, True), ("F1", 1000, 17, False), ("F1", 4096, 48, True),
                                        ("F2", 1000, 48, False), ("F6", 33, 17, True), ("F6", 129, 8, False),
                                        ("F7", 1000, 17, True), ("F7", 33, 48, False), ("F4", 300, 48, True)])
def test_exact_search_other_channel_counts(fam, V, C, cn):
    _check_family(fam, V, C, 3, 7, cn=cn, algos=("exact", "auto"))


@pytest.mark.parametrize("fam", ["F1", "F2"])
def test_training_shape(fam):
    """N = 65536 (B = 256, 16 x 16), V = 8192, C = 32: the shape VQ-8192 trains at."""
    _check_family(fam, 8192, 32, 256, 16)


@pytest.mark.parametrize("algo", ["tc", "exact"])
@pytest.mark.parametrize("fam,V,C", [("F1", 300, 32), ("F2", 1000, 64), ("F6", 33, 32)])
def test_no_writes_past_n(algo, fam, V, C):
    """Ragged N = 147 (one partial 128-row CTA): idx, out, loss and hist are followed by sentinel tails that the
    C entry point must leave alone."""
    from imagefolder_b200 import _capi as Cc
    B, hw, G = 3, 7, 4096
    N, HW = B * hw * hw, hw * hw
    z_rows, E = m.FAMILIES[fam](V, C, N)
    z = torch.from_numpy(m.rows_to_nchw(z_rows, B, hw)).cuda()
    Et = torch.from_numpy(E).cuda()
    idx = torch.full((N + G,), -7, dtype=torch.int64, device="cuda")
    out = torch.full((N * C + G,), float("nan"), device="cuda")
    out[N * C:].view(torch.int32).fill_(0x7FC0DEAD)
    loss = torch.full((2 + G,), 3.5, device="cuda")
    hist = torch.zeros(V + G, device="cuda")
    hist[V:] = -1.0
    L = Cc.lib()
    ws = Cc.workspace(L.xq_vq_workspace_bytes(B, C, HW, V), z.device)
    old = os.environ.get("XQ_VQ_ALGO")
    os.environ["XQ_VQ_ALGO"] = algo
    try:
        Cc.call("xq_vq_forward", 3, L.xq_vq_forward, Cc.ptr(z), Cc.ptr(Et), B, C, HW, V, 1, 1, 0.25, Cc.ptr(idx),
                Cc.ptr(out), Cc.ptr(loss), Cc.ptr(hist), Cc.ptr(ws), ws.numel(), Cc.stream_ptr(z.device))
        torch.cuda.synchronize()
    finally:
        if old is None:
            os.environ.pop("XQ_VQ_ALGO", None)
        else:
            os.environ["XQ_VQ_ALGO"] = old
    assert bool((idx[N:] == -7).all()), "idx written past N"
    assert bool((out[N * C:].view(torch.int32) == 0x7FC0DEAD).all()), "out written past N"
    assert bool((loss[2:] == 3.5).all()), "loss written past its two values"
    assert bool((hist[V:] == -1.0).all()), "hist written past V"
    fwd = xo.vq_forward(m.rows_to_nchw(z_rows, B, hw), E)
    np.testing.assert_array_equal(_npy(idx[:N]), fwd["idx"])
    np.testing.assert_array_equal(_npy(out[:N * C]).reshape(fwd["out"].shape), fwd["out"])
    np.testing.assert_array_equal(_npy(hist[:V]), fwd["hist"])


# ------------------------------------------------------------------------------------------
# perturbation: rank select under exact ties (the > 256-way tie takes the serial fallback)
# ------------------------------------------------------------------------------------------
def _perturb(z_rows, E, B, hw, rand_j, delta):
    from imagefolder_b200 import _capi as Cc
    C, V, HW = E.shape[1], E.shape[0], hw * hw
    N = B * HW
    z = torch.from_numpy(m.rows_to_nchw(z_rows, B, hw)).cuda()
    zq = torch.zeros_like(z)
    Et = torch.from_numpy(E).cuda()
    ru = torch.zeros(N, device="cuda")                      # rand_u = 0 <= alpha: every row uses its rank
    rj = torch.from_numpy(rand_j).cuda()
    out = torch.empty_like(z)
    sel = torch.full((N,), -1, dtype=torch.int64, device="cuda")
    L = Cc.lib()
    ws = Cc.workspace(L.xq_perturb_workspace_bytes(B, C, HW, V), z.device)
    Cc.call("xq_perturb_forward", 3, L.xq_perturb_forward, Cc.ptr(z), Cc.ptr(zq), Cc.ptr(Et), Cc.ptr(ru), Cc.ptr(rj),
            B, C, HW, V, 1, 1.0, B, delta, Cc.ptr(out), Cc.ptr(sel), Cc.ptr(ws), ws.numel(), Cc.stream_ptr(z.device))
    torch.cuda.synchronize()
    ref = xo.add_perturbation(m.rows_to_nchw(z_rows, B, hw), np.zeros((B, C, hw, hw), np.float32), E, True, 1.0, 1.0,
                              delta, np.zeros(N, np.float32), rand_j)
    np.testing.assert_array_equal(_npy(sel), ref["sel"])
    np.testing.assert_array_equal(_npy(out), ref["out"])
    return _npy(sel)


def test_perturb_zero_and_tiny_codes():
    V, C, B, hw, delta = 16384, 32, 2, 8, 100
    z_rows, E = m.f1_zero_tiny(V, C, B * hw * hw)
    rj = np.random.default_rng(11).integers(0, delta, B * hw * hw).astype(np.int64)
    _perturb(z_rows, E, B, hw, rj, delta)


def test_perturb_300_way_tie_both_sides():
    """One row direction r; 50 codes nearer to r than a run of 300 identical codes, so the run holds ranks 50..349 and
    the ranks drawn from [0, 100) fall on both sides of its start; inside it the kernel's tie list (256 entries)
    overflows and it takes the serial scan.  Also 1-ulp neighbours and boundary duplicates (F7)."""
    V, C, B, hw, delta = 16384, 32, 2, 8, 100
    N = B * hw * hw
    z_rows, E = m.f7_exact_ties(V, C, N)
    rng = np.random.default_rng(12)
    r = m._unit(rng, 1, C)[0]
    run = m._with_dot(rng, r, 0.97)
    E[200:500] = run
    for j in range(50):
        E[5000 + 37 * j] = m._with_dot(rng, r, 0.99 + 1e-4 * j)
    z_rows = np.tile(r.astype(np.float32), (N, 1))
    z_rows[1::2] += (1e-6 * rng.standard_normal((N // 2, C))).astype(np.float32)
    rj = (np.arange(N) * 37 % delta).astype(np.int64)
    sel = _perturb(z_rows, E.astype(np.float32), B, hw, rj, delta)
    in_run = (sel >= 200) & (sel < 500)
    assert in_run.sum() > N // 4 and (~in_run).sum() > N // 4
    # ranks inside the run pick run codes in index order
    assert np.all(sel[(rj >= 50) & (np.arange(N) % 2 == 0)] == 200 + rj[(rj >= 50) & (np.arange(N) % 2 == 0)] - 50)


# ------------------------------------------------------------------------------------------
# multi-scale searches (ms_kernels.cu paths S and L): zero codes in the negative half-space, stride duplicates
# ------------------------------------------------------------------------------------------
def _vq2_indices(f, E, pn, zn):
    from imagefolder_b200 import VectorQuantizer2
    V, C = E.shape
    torch.manual_seed(V + C)
    q = VectorQuantizer2(V, C, using_znorm=zn, v_patch_nums=pn, num_latent_tokens=pn[-1] ** 2,
                         share_quant_resi=4).cuda().eval()
    q.embedding.weight.data.copy_(torch.from_numpy(E).cuda())
    mods = q.quant_resi.modules_list()
    with torch.no_grad():
        got = [_npy(t) for t in q.f_to_idxBl_or_fhat(torch.from_numpy(f).cuda(), to_fhat=False, v_patch_nums=pn)]
    want = xo.vq2_f_to_idxBl_or_fhat(f, E, np.stack([_npy(x.weight) for x in mods]),
                                     np.stack([_npy(x.bias) for x in mods]), pn, using_znorm=zn)
    for si in range(len(pn)):
        np.testing.assert_array_equal(got[si], want[si], err_msg=f"scale {si} (p = {pn[si]})")
    return got


PN10 = [1, 1, 2, 3, 3, 4, 5, 6, 8, 11]


@pytest.mark.parametrize("pn", [PN10, [1, 4, 16]])
@pytest.mark.parametrize("zn", [True, False])
def test_ms_zero_codes_negative_half_space(pn, zn):
    """F6 + F1: rows in the positive orthant, real codes in the negative one, zero and tiny codes at group / tile
    boundaries.  With using_znorm the key is -dot, so the zero code wins every row whose dots are all negative."""
    V, C, B = 1000, 32, 3
    rng = np.random.default_rng(21)
    _, E = m.f6_negative(V, C, 8)
    _, E1 = m.f1_zero_tiny(V, C, 8)
    special = np.linalg.norm(E1, axis=1) < 1e-12
    E[special] = E1[special]
    H = pn[-1]
    f = (np.abs(rng.standard_normal((B, C, H, H))) + 0.05).astype(np.float32)
    got = _vq2_indices(f, E, pn, zn)
    if zn:
        assert np.isin(got[0], np.nonzero(special)[0]).all()


@pytest.mark.parametrize("pn", [PN10, [1, 4, 16]])
@pytest.mark.parametrize("zn", [True, False])
def test_ms_stride_duplicates_take_first_index(pn, zn):
    """F7 at the search paths' strides: E[v] = E[v mod 64] for V = 512, so every code has copies at v + 64, v + 128
    (path L: one thread's two code columns and the next tile) and v + 384 (path S: one thread's two codes per step)."""
    V, C, B = 512, 16, 3
    rng = np.random.default_rng(22)
    base = rng.standard_normal((64, C)).astype(np.float32)
    E = base[np.arange(V) % 64]
    H = pn[-1]
    f = rng.standard_normal((B, C, H, H)).astype(np.float32)
    got = _vq2_indices(f, E, pn, zn)
    assert all(int(g.max()) < 64 for g in got)
