"""The fp16 twins of the ViT kernels (`*_f16` entry points: the same kernels instantiated for fp16 operands), for training
under fp16 autocast.  Each section mirrors the bf16 test of the same kernel (test_gpu_mlp_gemm.py, test_gpu_lora_mlp.py,
test_gpu_attn.py, test_gpu_vit_ops.py, test_vit_golden.py) so that the two can be read side by side.

Tolerances.  fp16 has an 11-bit significand: unit roundoff u = 2^-11 (bf16: 2^-8).
  * Fused MLP GEMMs: exact-grid operands ({-1, 0, 1} 2^-3 x {-1, 0, 1} 2^-2, K <= 1024) make every partial sum a multiple
    of 2^-5 below 2^5 -- exact in fp32 and, at 10 bits of magnitude, exact in fp16 too -- so `pre` equals fp16 of an fp64
    GEMM bit for bit, and act / d_pre equal the stand-alone f16 GELU kernels on the same `pre`.
  * Attention (fp32 explicit-softmax reference on the same fp16 inputs): the kernel rounds P and the output to fp16
    (forward: two roundings of relative size u on a convex combination -> |err| <= 2u max|o|, tested at 4u = 2^-9), and in
    the backward P, dS and the packed gradient (three roundings, one on dS whose terms cancel against delta; tested at
    8u = 2^-8 of the largest reference gradient).  Both are the bf16 test's bounds scaled from 2^-8 to 2^-11, with a factor
    two of margin for the fp32 accumulation and ex2.approx (2^-22 relative) that do not shrink with u.
  * Glue kernels against fp64: one fp16 rounding of each 16-bit output (u relative) plus fp32 arithmetic (1e-5 relative).
  * Model level (fused path vs the library path under the same fp16 autocast): both are fp16-GEMM pipelines through
    12 blocks that differ in rounding order; the bf16 test's bounds hold with room to spare at 8x the precision.
"""
import math
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

H16 = torch.float16
GUARD = 128
SENTINEL = -12345
SAT = 40.0
U = 2.0 ** -11
F16_MAX = 65504.0


def _lib():
    from imagefolder_b200 import _capi
    return _capi, _capi.lib()


def _nan(shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def _guarded(M, N):
    t = _nan((M + GUARD, N), H16)
    t[M:].view(torch.int16).fill_(SENTINEL)
    return t


def _assert_guard(t, M, what):
    bad = t[M:].view(torch.int16) != SENTINEL
    assert not bool(bad.any()), f"{what}: guard rows after row {M} overwritten"


def _assert_bits(a, b, what, zero_sign=False):
    bad = a.view(torch.int16) != b.view(torch.int16)
    if zero_sign:
        bad &= ~((a == 0) & (b == 0))
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {bad.numel()} elements differ"


def _assert_within(a, ref, tol, what):
    err = (a.double() - ref).abs()
    ok = err <= tol
    assert bool(ok.all()), f"{what}: {int((~ok).sum())} out of tolerance, max err {err.max().item():.3e}"


def _gelu64(u):
    return 0.5 * u * (1.0 + torch.erf(u / math.sqrt(2.0)))


def _grid(rows, cols, scale, gen):
    return torch.randint(-1, 2, (rows, cols), device="cuda", generator=gen).to(H16) * scale


def _bias(N, gen):
    b = torch.randn(N, device="cuda", generator=gen)
    kind = torch.arange(N, device="cuda") % 3
    b[kind == 0] = SAT
    b[kind == 1] = -SAT
    return b


# ---------------------------------------------------------------------------------------------------------------------
# fused MLP GEMMs (csrc/gemm_kernel.cu), bit for bit through the C ABI
# ---------------------------------------------------------------------------------------------------------------------
def _gemm_check(M, N, K, seed):
    _capi, L = _lib()
    p, s = _capi.ptr, _capi.stream_ptr()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x, w1 = _grid(M + GUARD, K, 2 ** -3, gen), _grid(N, K, 2 ** -2, gen)
    d_out, w2t = _grid(M + GUARD, K, 2 ** -3, gen), _grid(N, K, 2 ** -2, gen)
    b1 = _bias(N, gen)
    pos, neg = b1 == SAT, b1 == -SAT
    pre, act = _guarded(M, N), _guarded(M, N)
    _capi.check(L.xq_vit_fc1_gelu_fwd_f16(p(x), p(w1), p(b1), p(pre), p(act), M, N, K, s), "fc1_f16")
    d_pre, d_bias = _guarded(M, N), _nan((N,))
    _capi.check(L.xq_vit_fc2_dgelu_bwd_f16(p(d_out), p(w2t), p(pre), p(b1), p(d_pre), p(d_bias), M, N, K, s), "fc2_f16")
    pre_m, act_m, dp_m = pre[:M], act[:M], d_pre[:M]
    ref = x[:M].double() @ w1.double().t()
    _assert_bits(pre_m, ref.to(H16), "pre vs fp16(fp64 GEMM)", zero_sign=True)
    _assert_bits(act_m[:, pos], (pre_m[:, pos].float() + SAT).to(H16), "act on b1 = +40")
    assert bool((act_m[:, neg] == 0).all())
    g_fwd = _nan((M, N), H16)
    _capi.check(L.xq_vit_gelu_fwd_f16(p(pre_m), p(b1), p(g_fwd), M, N, s), "gelu_fwd_f16")
    _assert_bits(act_m, g_fwd, "act vs xq_vit_gelu_fwd_f16 on the same pre")
    gref = _gelu64(pre_m.double() + b1.double())
    _assert_within(act_m, gref, U * gref.abs() + 1e-6, "act vs fp64 GELU")
    gy = (d_out[:M].double() @ w2t.double().t()).to(H16)
    gx = _nan((M, N), H16)
    _capi.check(L.xq_vit_gelu_bwd_f16(p(pre_m), p(b1), p(gy), p(gx), None, M, N, s), "gelu_bwd_f16")
    _assert_bits(dp_m, gx, "d_pre vs xq_vit_gelu_bwd_f16", zero_sign=True)
    _assert_bits(dp_m[:, pos], gy[:, pos], "d_pre on b1 = +40", zero_sign=True)
    assert bool((dp_m[:, neg] == 0).all())
    # +40 columns: terms are multiples of 2^-5, sums exact in fp32 in any order
    assert torch.equal(d_bias[pos].double(), gy[:, pos].double().sum(0)), "d_bias on b1 = +40"
    assert bool((d_bias[neg] == 0).all())
    want = dp_m.double().sum(0)
    _assert_within(d_bias, want, 1e-5 * dp_m.double().abs().sum(0) + 1e-6, "d_bias vs fp64 column sums")
    for t, what in ((pre, "pre"), (act, "act"), (d_pre, "d_pre")):
        _assert_guard(t, M, what)
    return x, w1, b1, d_out, w2t, pre, act, d_pre, d_bias


@pytest.mark.parametrize("B", [128, 1])
@pytest.mark.parametrize("S", [513, 514, 769, 499, 379])
def test_fused_mlp_f16_training_rows(B, S):
    """ViT-B MLP at the shipped sequence lengths: B = 128 walks ~100 row blocks per CTA; B = 1 leaves a tail tile ending
    inside either warpgroup (M % 128 = 1, 2, 1, 115, 123)."""
    _gemm_check(B * S, 3072, 768, seed=B * 1000 + S)


@pytest.mark.parametrize("C,H,M", [(384, 1536, 3 * 499), (1024, 4096, 2 * 513), (768, 3072, 64 * 513)])
def test_fused_mlp_f16_widths_and_tails(C, H, M):
    """ViT-S / ViT-L widths; 64 x 513 leaves M % 128 = 64 (the tail ends where the second warpgroup starts)."""
    _gemm_check(M, H, C, seed=C + M)


@pytest.mark.parametrize("R", [8, 16, 64])
def test_lora_f16_rank_stage_equals_plain_kernel_on_concatenated_operands(R):
    """xq_vit_fc1_lora_gelu_fwd_f16 / xq_vit_fc2_lora_dgelu_bwd_f16 == the plain f16 kernels on [x | u], [w | b] (zero-padded
    to K + 64), bit for bit: exact-grid operands make the order of the fp32 sums irrelevant."""
    _capi, L = _lib()
    p, s = _capi.ptr, _capi.stream_ptr()
    M, N, K = 3 * 513, 3072, 768
    gen = torch.Generator(device="cuda").manual_seed(R)
    x, w, u, bl = (_grid(M, K, 2 ** -3, gen), _grid(N, K, 2 ** -2, gen), _grid(M, R, 2 ** -3, gen),
                   _grid(N, R, 2 ** -2, gen))
    g, w2t, v, a2t = (_grid(M, K, 2 ** -3, gen), _grid(N, K, 2 ** -2, gen), _grid(M, R, 2 ** -3, gen),
                      _grid(N, R, 2 ** -2, gen))
    b1 = _bias(N, gen)

    def cat(a, b):
        out = torch.zeros(a.shape[0], K + 64, dtype=H16, device="cuda")
        out[:, :K], out[:, K:K + R] = a, b
        return out

    pre, act, pre2, act2 = (_nan((M, N), H16) for _ in range(4))
    _capi.check(L.xq_vit_fc1_lora_gelu_fwd_f16(p(x), p(w), p(u), p(bl), p(b1), p(pre), p(act), M, N, K, R, s), "lora fwd")
    # the concatenated operands are held by name until the kernels have run: a temporary would go back to the caching
    # allocator as soon as its pointer is taken, and the next one could be built in the same memory before the launch
    xu, wb = cat(x, u), cat(w, bl)
    _capi.check(L.xq_vit_fc1_gelu_fwd_f16(p(xu), p(wb), p(b1), p(pre2), p(act2), M, N, K + 64, s), "fwd")
    _assert_bits(pre, pre2, "pre", zero_sign=True)
    _assert_bits(act, act2, "act", zero_sign=True)
    dp, db, dp2, db2 = _nan((M, N), H16), _nan((N,)), _nan((M, N), H16), _nan((N,))
    _capi.check(L.xq_vit_fc2_lora_dgelu_bwd_f16(p(g), p(w2t), p(v), p(a2t), p(pre), p(b1), p(dp), p(db), M, N, K, R, s), "bwd")
    gv, wa = cat(g, v), cat(w2t, a2t)
    _capi.check(L.xq_vit_fc2_dgelu_bwd_f16(p(gv), p(wa), p(pre), p(b1), p(dp2), p(db2), M, N, K + 64, s), "b")
    _assert_bits(dp, dp2, "d_pre", zero_sign=True)
    pos = b1 == SAT
    assert torch.equal(db[pos], db2[pos])


# ---------------------------------------------------------------------------------------------------------------------
# attention (csrc/attn_kernel.cu)
# ---------------------------------------------------------------------------------------------------------------------
def _attn_ref(qkv32, H):
    B, N, _ = qkv32.shape
    x = qkv32.view(B, N, 3, H, 64).permute(2, 0, 3, 1, 4)
    q, k, v = x[0], x[1], x[2]
    s = (q @ k.transpose(-1, -2)) * 0.125
    o = torch.softmax(s, -1) @ v
    return o.transpose(1, 2).reshape(B, N, H * 64), torch.logsumexp(s, -1) * math.log2(math.e)


def _attn_check(B, N, H, amp, gscale=1.0, seed=0):
    from imagefolder_b200 import vit_ops
    torch.manual_seed(seed)
    qkv = (torch.randn(B, N, 3 * H * 64, device="cuda") * amp).to(H16)
    g_true = torch.randn(B, N, H * 64, device="cuda") / gscale
    g = (g_true * gscale).to(H16)                               # what a GradScaler-scaled backward hands the node
    q32 = qkv.float().requires_grad_(True)
    o_ref, lse_ref = _attn_ref(q32, H)
    (o_ref * (g.float() / gscale)).sum().backward()
    out, lse2 = vit_ops.attn_tc_forward(qkv, H)
    dqkv = vit_ops.attn_tc_backward(qkv, out, lse2, g, H)
    assert out.dtype == H16 and dqkv.dtype == H16
    assert torch.isfinite(out.float()).all() and torch.isfinite(dqkv.float()).all()
    assert (out.float() - o_ref).abs().max().item() <= 4 * U * max(1.0, o_ref.abs().max().item())
    assert (lse2 - lse_ref.detach()).abs().max().item() <= 1e-3 * max(1.0, lse_ref.abs().max().item())
    gr = q32.grad.view(B, N, 3, H * 64)
    d = (dqkv.float() / gscale).view(B, N, 3, H * 64)
    for i, name in enumerate("qkv"):
        m = max(1e-3 / gscale, gr[:, :, i].abs().max().item())     # N = 1: dq = dk = 0
        err = (d[:, :, i] - gr[:, :, i]).abs().max().item()
        assert err <= 8 * U * m, f"d{name}: err {err:.3e} vs max {m:.3e}"
    dq2, db = vit_ops.attn_tc_backward(qkv, out, lse2, g, H, want_bias_grad=True)
    want = dq2.float().sum((0, 1))
    assert (db - want).abs().max().item() <= 2e-3 * max(1.0, want.abs().max().item()) + 1e-4 * B * N ** 0.5 * gscale


@pytest.mark.parametrize("B,N,H", [(2, 513, 3), (2, 514, 2), (1, 769, 2), (2, 499, 2), (2, 379, 3), (3, 1, 1), (1, 16, 2),
                                   (2, 128, 2), (2, 129, 1), (1, 1024, 1), (1, 333, 12),
                                   (5, 513, 12), (7, 300, 12), (40, 130, 12), (13, 100, 12),
                                   (2, 131, 2), (1, 132, 12), (2, 133, 3), (1, 387, 12), (2, 388, 2)])
@pytest.mark.parametrize("amp", [1.0, 2.5])
def test_attention_f16_matches_fp32_reference(B, N, H, amp):
    """the shapes of test_gpu_attn.py: every trailing-key count N mod 128 = 1 .. 5, more backward CTAs than SMs"""
    _attn_check(B, N, H, amp, seed=N * 7 + H)


@pytest.mark.parametrize("B,N,H", [(2, 513, 12), (2, 131, 2)])
def test_attention_f16_gradscaler_scaled_gradients_do_not_underflow(B, N, H):
    """true gradients of size 2^-16 (their fp16 dS terms would sit at the bottom of the subnormal range), scaled by 2^16 as
    GradScaler's default scale does: unscaled, the kernel's gradient matches the fp32 reference at the same relative bound
    as unit gradients, i.e. nothing was lost to underflow."""
    _attn_check(B, N, H, 1.0, gscale=2.0 ** 16, seed=N)


# ---------------------------------------------------------------------------------------------------------------------
# glue kernels (csrc/vit_kernels.cu) against fp64
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [384, 768, 1024])
@pytest.mark.parametrize("M", [8 * 3 + 5, 128 * 513])
def test_residual_ln_f16_fwd_bwd(D, M):
    _capi, L = _lib()
    p, s = _capi.ptr, _capi.stream_ptr()
    S = 513 if M % 513 == 0 else M
    torch.manual_seed(D + M)
    x = torch.randn(M, D, device="cuda")
    br = torch.randn(M, D, device="cuda").to(H16)
    bb, gam = torch.randn(D, device="cuda") * 0.1, torch.rand(D, device="cuda") + 0.5
    rs = (torch.rand(M // S, device="cuda") > 0.2).float() / 0.8
    w, b = torch.rand(D, device="cuda") + 0.5, torch.randn(D, device="cuda") * 0.1
    x_out, y, mean, rstd = _nan((M, D)), _nan((M, D), H16), _nan((M,)), _nan((M,))
    _capi.check(L.xq_vit_residual_ln_fwd_f16(p(x), p(br), p(bb), p(gam), p(rs), S, p(w), p(b), 1e-6, M, D, p(x_out), p(y),
                                             p(mean), p(rstd), s), "ln fwd f16")
    xd = x.double() + rs.double().repeat_interleave(S)[:, None] * gam.double() * (br.double() + bb.double())
    _assert_within(x_out, xd, 1e-5 * xd.abs() + 1e-5, "x_out")
    mu, var = xd.mean(1, keepdim=True), xd.var(1, unbiased=False, keepdim=True)
    yd = (xd - mu) / torch.sqrt(var + 1e-6) * w.double() + b.double()
    _assert_within(y, yd, U * yd.abs() + 1e-4, "y")
    # backward: integer-valued g_y makes d ln_b (its column sums) exact
    g_xout = torch.randn(M, D, device="cuda")
    g_y = torch.randint(-3, 4, (M, D), device="cuda").to(H16)
    ws = _capi.workspace(L.xq_vit_ln_bwd_workspace_bytes(D), x.device)
    g_x, g_br = _nan((M, D)), _nan((M, D), H16)
    g_w, g_b, g_g, g_bb = _nan((D,)), _nan((D,)), _nan((D,)), _nan((D,))
    _capi.check(L.xq_vit_residual_ln_bwd_f16(p(g_xout), p(g_y), p(x_out), p(mean), p(rstd), p(w), p(br), p(bb), p(gam), p(rs),
                                             S, M, D, p(g_x), p(g_br), p(g_w), p(g_b), p(g_g), p(g_bb), p(ws), ws.numel(), s),
                "ln bwd f16")
    assert torch.equal(g_b.double(), g_y.double().sum(0)), "d ln_b: integer column sums"
    xo = x_out.double().requires_grad_(True)
    mu, var = xo.mean(1, keepdim=True), xo.var(1, unbiased=False, keepdim=True)
    yy = (xo - mu) / torch.sqrt(var + 1e-6) * w.double()
    (yy * g_y.double()).sum().backward()
    G = g_xout.double() + xo.grad
    _assert_within(g_x, G, 1e-4 * G.abs().max() + 1e-5, "g_x")
    gbr = G * rs.double().repeat_interleave(S)[:, None] * gam.double()
    _assert_within(g_br, gbr, U * gbr.abs() + 1e-4 * gbr.abs().max(), "g_branch")


@pytest.mark.parametrize("M,C", [(128 * 513, 3072), (5, 1536)])
def test_gelu_f16_fwd_bwd(M, C):
    _capi, L = _lib()
    p, s = _capi.ptr, _capi.stream_ptr()
    torch.manual_seed(M)
    x = (torch.randn(M, C, device="cuda") * 2).to(H16)
    bias = torch.randn(C, device="cuda")
    bias[::3] = SAT
    y = _nan((M, C), H16)
    _capi.check(L.xq_vit_gelu_fwd_f16(p(x), p(bias), p(y), M, C, s), "gelu fwd f16")
    ref = _gelu64(x.double() + bias.double())
    _assert_within(y, ref, U * ref.abs() + 1e-6, "gelu")
    gy = torch.randint(-4, 5, (M, C), device="cuda").to(H16)
    gx, gb = _nan((M, C), H16), _nan((C,))
    _capi.check(L.xq_vit_gelu_bwd_f16(p(x), p(bias), p(gy), p(gx), p(gb), M, C, s), "gelu bwd f16")
    u = x.double() + bias.double()
    dref = gy.double() * (0.5 * (1 + torch.erf(u / math.sqrt(2))) + u * torch.exp(-u * u / 2) / math.sqrt(2 * math.pi))
    _assert_within(gx, dref, U * dref.abs() + 4e-6 * gy.double().abs(), "gelu'")
    sat = bias == SAT                          # GELU' == 1 exactly there: integer column sums, exact
    assert torch.equal(gb[sat].double(), gy[:, sat].double().sum(0))


def test_patchify_and_assemble_f16():
    _capi, L = _lib()
    p, s = _capi.ptr, _capi.stream_ptr()
    torch.manual_seed(5)
    B, Cin, Hh, W, P = 3, 3, 64, 48, 16
    x = torch.randn(B, Cin, Hh, W, device="cuda")
    M, K = B * (Hh // P) * (W // P), Cin * P * P
    out = _nan((M, K), H16)
    _capi.check(L.xq_vit_patchify_f16(p(x), p(out), B, Cin, Hh, W, P, s), "patchify f16")
    want = x.view(B, Cin, Hh // P, P, W // P, P).permute(0, 2, 4, 1, 3, 5).reshape(M, K).to(H16)
    _assert_bits(out, want, "patches")
    Bn, Ls, T, D, t0 = 9, 5, 8, 16, 2
    src = torch.randn(Bn, Ls, D, device="cuda").to(H16)
    table = torch.randn(T, D, device="cuda")
    o = _nan((Bn, T, D))
    _capi.check(L.xq_vit_assemble_fwd(p(src), 2, p(table), Bn, Ls, T, D, t0, p(o), s), "assemble fwd f16")
    want = table.expand(Bn, T, D).clone()
    want[:, t0:t0 + Ls] += src.float()
    assert torch.equal(o, want)
    g = torch.randint(-5, 6, (Bn, T, D), device="cuda").float()
    d_src, d_tab = _nan((Bn, Ls, D), H16), _nan((T, D))
    _capi.check(L.xq_vit_assemble_bwd(p(g), Bn, Ls, T, D, t0, p(d_src), 2, p(d_tab), s), "assemble bwd f16")
    assert torch.equal(d_src, g[:, t0:t0 + Ls].to(H16)) and torch.equal(d_tab, g.sum(0))


# ---------------------------------------------------------------------------------------------------------------------
# overflow is inf, never a clamp to +-65504
# ---------------------------------------------------------------------------------------------------------------------
def _overflowed(row, what):
    r = row.float()
    assert bool((~torch.isfinite(r)).any()), f"{what}: no inf / NaN in the overflowing row"
    assert not bool((r.abs() == F16_MAX).any()), f"{what}: saturated to 65504"


def test_overflow_gives_inf_in_every_f16_entry_point():
    _capi, L = _lib()
    p, s = _capi.ptr, _capi.stream_ptr()
    torch.manual_seed(0)
    # patchify: one image row above the fp16 range
    x = torch.randn(1, 3, 16, 16, device="cuda")
    x[0, 0, 0, :4] = 1e5
    pt = _nan((1, 768), H16)
    _capi.check(L.xq_vit_patchify_f16(p(x), p(pt), 1, 3, 16, 16, 16, s), "patchify")
    _overflowed(pt[0], "patchify")
    # GELU forward: 65504 + 40 rounds past the largest finite fp16
    xg = torch.zeros(2, 8, device="cuda", dtype=H16)
    xg[1] = F16_MAX
    bias = torch.full((8,), SAT, device="cuda")
    yg = _nan((2, 8), H16)
    _capi.check(L.xq_vit_gelu_fwd_f16(p(xg), p(bias), p(yg), 2, 8, s), "gelu fwd")
    _overflowed(yg[1], "gelu_fwd")
    # GELU backward: GELU'(x) > 1 for x ~ 1 times a gradient at the top of the range
    xb = torch.ones(2, 8, device="cuda", dtype=H16)
    gyb = torch.zeros(2, 8, device="cuda", dtype=H16)
    gyb[1] = F16_MAX
    gxb = _nan((2, 8), H16)
    _capi.check(L.xq_vit_gelu_bwd_f16(p(xb), None, p(gyb), p(gxb), None, 2, 8, s), "gelu bwd")
    _overflowed(gxb[1], "gelu_bwd")
    # residual LN forward (ln_w 1e5) / backward (ls_gamma 1e5)
    M, D = 16, 384
    xr = torch.randn(M, D, device="cuda")
    w = torch.ones(D, device="cuda")
    w[:8] = 1e6
    b = torch.zeros(D, device="cuda")
    x_out, y, mean, rstd = _nan((M, D)), _nan((M, D), H16), _nan((M,)), _nan((M,))
    br = torch.zeros(M, D, device="cuda", dtype=H16)
    gam = torch.ones(D, device="cuda")
    _capi.check(L.xq_vit_residual_ln_fwd_f16(p(xr), p(br), None, p(gam), None, M, p(w), p(b), 1e-6, M, D, p(x_out), p(y),
                                             p(mean), p(rstd), s), "ln fwd")
    _overflowed(y[3], "residual_ln_fwd")
    gam[:8] = 1e6
    g_xout = torch.zeros(M, D, device="cuda")
    g_xout[3] = 1.0
    ws = _capi.workspace(L.xq_vit_ln_bwd_workspace_bytes(D), xr.device)
    g_x, g_br = _nan((M, D)), _nan((M, D), H16)
    _capi.check(L.xq_vit_residual_ln_bwd_f16(p(g_xout), None, p(x_out), p(mean), p(rstd), p(w), p(br), None, p(gam), None, M,
                                             M, D, p(g_x), p(g_br), None, None, None, None, p(ws), ws.numel(), s), "ln bwd")
    _overflowed(g_br[3], "residual_ln_bwd")
    # fused MLP GEMMs: one row of x / d_out at 1000 against weights of 0.25: 96000 over K = 384
    Mm, N, K = 130, 256, 384
    xa = torch.zeros(Mm, K, device="cuda", dtype=H16)
    xa[7] = 1000.0
    wa = torch.full((N, K), 0.25, device="cuda", dtype=H16)
    b1 = torch.zeros(N, device="cuda")
    pre, act = _nan((Mm, N), H16), _nan((Mm, N), H16)
    _capi.check(L.xq_vit_fc1_gelu_fwd_f16(p(xa), p(wa), p(b1), p(pre), p(act), Mm, N, K, s), "fc1")
    _overflowed(pre[7], "fc1 pre")
    _overflowed(act[7], "fc1 act")
    pre_ok = torch.ones(Mm, N, device="cuda", dtype=H16)
    dp, db = _nan((Mm, N), H16), _nan((N,))
    _capi.check(L.xq_vit_fc2_dgelu_bwd_f16(p(xa), p(wa), p(pre_ok), p(b1), p(dp), p(db), Mm, N, K, s), "fc2")
    _overflowed(dp[7], "fc2 d_pre")
    # attention backward: every query attends to key 0, whose dV is the sum of 513 output gradients of 1000
    from imagefolder_b200 import vit_ops
    Bq, Nq, Hq = 1, 513, 1
    qkv = torch.zeros(Bq, Nq, 3, 64, device="cuda")
    qkv[:, :, 0] = 1.0
    qkv[:, 0, 1] = 8.0
    qkv = qkv.view(Bq, Nq, 192).to(H16)
    out, lse2 = vit_ops.attn_tc_forward(qkv, Hq)
    g = torch.full((Bq, Nq, 64), 1000.0, device="cuda", dtype=H16)
    dq = vit_ops.attn_tc_backward(qkv, out, lse2, g, Hq)
    _overflowed(dq.view(Bq, Nq, 3, 64)[0, 0, 2], "attn_bwd dV")
    # token assembly backward: an fp32 gradient above the fp16 range
    ga = torch.zeros(2, 4, 8, device="cuda")
    ga[1, 1] = 1e6
    d_src = _nan((2, 4, 8), H16)
    _capi.check(L.xq_vit_assemble_bwd(p(ga), 2, 4, 4, 8, 0, p(d_src), 2, None, s), "assemble bwd")
    _overflowed(d_src[1, 1], "assemble_bwd")


# ---------------------------------------------------------------------------------------------------------------------
# model level
# ---------------------------------------------------------------------------------------------------------------------
def _spy_run(fn):
    from imagefolder_b200 import _capi
    calls = []
    real = _capi.call

    def spy(name, *a, **k):
        calls.append(name)
        return real(name, *a, **k)

    _capi.call = spy
    try:
        out = fn()
    finally:
        _capi.call = real
    return out, calls


def _set_fused(on):
    from imagefolder_b200 import vit_ops
    vit_ops.MLP_TC_ENABLED[0] = vit_ops.ATTN_TC_ENABLED[0] = vit_ops.ASSEMBLE_ENABLED[0] = on


@pytest.mark.parametrize("name", ["VQ-8192", "MSVR10P2-4096"])
def test_model_fp16_fused_path_matches_library_path(name):
    from test_model_cpu import small_model
    import torch.nn.functional as F
    model, _ = small_model(name)
    model = model.cuda().eval()          # no DropPath / codebook-drop draws: both paths see the same model
    for m in (model.encoder, model.decoder):
        for blk in m.model.blocks:
            blk.ls1.gamma.data.fill_(0.5)
            blk.ls2.gamma.data.fill_(0.5)
    x = (torch.rand(2, 3, 256, 256) * 2 - 1).cuda()

    def step():
        model.zero_grad(set_to_none=True)
        torch.manual_seed(3)
        with torch.autocast("cuda", dtype=H16):
            dec, (vq, commit, ent, usages), _, _, _ = model(x, 0, 0.0, 0.0, 100)
            loss = F.mse_loss(dec.float(), x) + vq + commit
        loss.backward()
        return (dec.detach().float(), float(loss.detach()),
                {n: q.grad.float().clone() for n, q in model.named_parameters() if q.grad is not None})

    step()                               # the token-assembly probe draws random numbers on the first fused call only
    (d1, l1, g1), calls = _spy_run(step)
    _set_fused(False)
    try:
        d0, l0, g0 = step()
    finally:
        _set_fused(True)
    for n in ("xq_vit_fc1_gelu_fwd_f16", "xq_vit_fc2_dgelu_bwd_f16", "xq_vit_attn_fwd_f16", "xq_vit_attn_bwd_f16",
              "xq_vit_residual_ln_fwd_f16", "xq_vit_residual_ln_bwd_f16"):
        assert n in calls, n
    # no bf16 entry point, and no stand-alone GELU left in the blocks
    assert not any(c.startswith("xq_vit_") and not c.endswith("_f16") and "assemble" not in c for c in calls), set(calls)
    assert "xq_vit_gelu_fwd_f16" not in calls and "xq_vit_gelu_bwd_f16" not in calls
    assert math.isfinite(l1) and abs(l1 - l0) <= 2e-2 * abs(l0) + 1e-4
    torch.testing.assert_close(d1, d0, rtol=3e-2, atol=3e-2 * float(d0.abs().max()))
    assert set(g1) == set(g0)
    # in norm: all gradients together within 10 %; each parameter within 25 % (the cls / latent tokens, whose gradient
    # reaches them only through 12 attention backwards and cancels over the batch, differ by about 12 % between the two
    # fp16 paths on this random-weight model, the other parameters by less than 10 %); the quantizer's codebook within
    # 50 %, since a token whose two nearest codes are within the paths' rounding difference moves its gradient from one
    # codebook row to another
    tot = sum(float(g0[n].double().square().sum()) for n in g0) ** 0.5
    dif = sum(float((g1[n] - g0[n]).double().square().sum()) for n in g0) ** 0.5
    assert dif <= 0.1 * tot, (dif, tot)
    for n in g0:
        m = float(g0[n].norm())
        err = float((g1[n] - g0[n]).norm())
        tol = 0.5 if n.startswith("quantize") else 0.25
        assert err <= tol * m + 1e-6, f"{n}: err {err:.3e} vs norm {m:.3e}"


def test_model_fp16_attention_uses_no_sdpa():
    """the blocks' attention runs on the f16 kernels, not scaled_dot_product_attention"""
    from test_model_cpu import small_model
    model, _ = small_model("VQ-8192")
    model = model.cuda().eval()
    x = (torch.rand(1, 3, 256, 256) * 2 - 1).cuda()
    real = torch.nn.functional.scaled_dot_product_attention
    n = [0]

    def sdpa(*a, **k):
        n[0] += 1
        return real(*a, **k)

    torch.nn.functional.scaled_dot_product_attention = sdpa
    try:
        with torch.no_grad(), torch.autocast("cuda", dtype=H16):
            model.decode(model.encode(x))
    finally:
        torch.nn.functional.scaled_dot_product_attention = real
    assert n[0] == 0


@pytest.mark.parametrize("name", ["vit_vq", "vit_vp2", "vit_ms", "vit_relpos"])
def test_fused_fp16_vit_matches_reference_golden(name):
    """test_vit_golden's GPU check under fp16 autocast; fp16 keeps 3 more bits than bf16, so the bf16 bounds halve"""
    import ast
    from imagefolder_b200 import config as xcfg
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.join(here, "golden"))
    from vit_det_init import apply_det_init, golden_inputs
    g = np.load(os.path.join(here, "golden", name + ".npz"))
    cfg = ast.literal_eval(str(g["cfg_json"]))
    args = xcfg.parse_args([])
    for k, v in cfg.items():
        setattr(args, k, v)
    torch.manual_seed(0)
    model = xcfg.build_vq_model(args).eval()
    apply_det_init(model)
    model = model.cuda()
    x, q = golden_inputs(int(g["q_shape"][1]), int(g["q_shape"][2]))
    (res, calls) = _spy_run(lambda: _golden_run(model, x, q))
    tok, h, dec = res
    assert "xq_vit_attn_fwd_f16" in calls and "xq_vit_residual_ln_fwd_f16" in calls
    for got, want in ((tok[:, ::4], g["tok_sub"]), (h.reshape(h.shape[0], h.shape[1], -1)[:, :, ::4], g["h_sub"]),
                      (dec[:, :, ::4, ::4], g["dec_sub"])):
        err = np.abs(got - want)
        assert err.max() < 0.075 and err.mean() < 0.01, (err.max(), err.mean())


def _golden_run(model, x, q):
    with torch.no_grad(), torch.autocast("cuda", dtype=H16):
        tok = model.encoder(x.cuda()).float().cpu().numpy()
        h = model.encode(x.cuda()).float().cpu().numpy()
        dec = model.decode(q.cuda()).float().cpu().numpy()
    return tok, h, dec


def test_lora_fp16_reaches_the_f16_lora_kernels():
    from imagefolder_b200.dino_enc import DINOv2Encoder
    kw = {'img_size': 224, 'patch_size': 14, 'drop_path_rate': 0.0}
    torch.manual_seed(1)
    enc = DINOv2Encoder(num_latent_tokens=32, model_name='vit_small_patch14_dinov2.lvd142m', model_kwargs=kw,
                        pretrained=False, tuning_method='lora').cuda().train()
    x = torch.rand(2, 3, 224, 224, device="cuda") * 2 - 1

    def run():
        with torch.autocast("cuda", dtype=H16):
            h = enc(x)
        h.float().square().sum().backward()
        return h

    h, calls = _spy_run(run)
    assert torch.isfinite(h.float()).all()
    assert calls.count("xq_vit_fc1_lora_gelu_fwd_f16") == 12 and calls.count("xq_vit_fc2_lora_dgelu_bwd_f16") == 12
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for n, p in enc.named_parameters()
               if p.requires_grad and "lora_" in n)


# ---------------------------------------------------------------------------------------------------------------------
# GradScaler + imagefolder_b200.optim.AdamW end to end
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fused", [True, False])
def test_gradscaler_skips_the_overflowing_step_and_then_trains(fused):
    from test_model_cpu import small_model
    from imagefolder_b200.optim import AdamW
    import torch.nn.functional as F
    model, _ = small_model("VQ-8192")
    model = model.cuda().train()
    opt = AdamW(model.parameters(), lr=1e-4)
    # init_scale large enough that the first backward overflows fp16; the back-off brings the scale to 2^16 at once
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 40, backoff_factor=2.0 ** -24)
    x = (torch.rand(2, 3, 256, 256) * 2 - 1).cuda()
    _set_fused(fused)
    try:
        losses, scales = [], []
        before = {n: q.detach().clone() for n, q in model.named_parameters()}
        for i in range(4):
            with torch.autocast("cuda", dtype=H16):
                dec, (vq, commit, ent, usages), _, _, _ = model(x, 0, 0.0, 0.0, 100)
                loss = F.mse_loss(dec.float(), x) + vq + commit
            opt.zero_grad(set_to_none=True)
            scaler.scale(loss).backward()
            scaler.step(opt)
            scaler.update()
            losses.append(float(loss))
            scales.append(scaler.get_scale())
            if i == 0:
                for n, q in model.named_parameters():
                    assert torch.equal(q.detach(), before[n]), f"{n} changed in the skipped step"
                assert scales[0] == 2.0 ** 16
    finally:
        _set_fused(True)
    assert all(math.isfinite(v) for v in losses)
    moved = any(not torch.equal(q.detach(), before[n]) for n, q in model.named_parameters())
    assert moved, "no step after the skipped one was taken"
