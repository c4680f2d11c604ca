"""Numerics of the ViT glue kernels against a plain PyTorch fp32 / fp64 reference of the same op
(floating-point kernels: tolerance set by the bf16 operands, written per assertion).

The persistent kernels (residual_ln_bwd, pack_qkv, gelu_bwd) hand out row tiles dynamically, so they are also run at row
counts where every CTA takes several tiles (the training encoder has 128 x 513 rows), through the C ABI with every output
buffer NaN-filled first: a tile that is never written fails, and column sums of integer-valued inputs are exact in fp32
in any order, so they are compared by equality and a tile counted twice fails too."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TRAIN_ROWS = 128 * 513          # encoder rows at a per-GPU batch of 128: cls + 256 image + 256 latent tokens per sample


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _nan(shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def _assert_within(a, ref, tol, what):
    """|a - ref| <= tol elementwise (tol broadcasts against ref); a NaN in `a` (an output never written) fails."""
    err = (a.double() - ref).abs()
    ok = err <= tol
    assert bool(ok.all()), f"{what}: {int((~ok).sum())} of {ok.numel()} elements out of tolerance, max err {err.max().item():.3e}"


def ref_residual_ln(x, branch, gamma, rs, w, b, eps, S, bbias=None):
    x = x.double()
    if branch is not None:
        s = rs.double().repeat_interleave(S).view(x.shape[0], x.shape[1], 1) if rs is not None else 1.0
        g = gamma.double() if gamma is not None else 1.0
        br = branch.double() + (bbias.double() if bbias is not None else 0.0)
        x = x + s * g * br
    y = F.layer_norm(x, (x.shape[-1],), w.double(), b.double(), eps)
    return x, y


@pytest.mark.parametrize("D,Bn,S", [(768, 3, 37), (384, 2, 513), (1024, 1, 9)])
@pytest.mark.parametrize("with_branch", [True, False])
def test_residual_ln_fwd_bwd(D, Bn, S, with_branch):
    from imagefolder_b200.vit_ops import residual_ln
    torch.manual_seed(D + S)
    dev = "cuda"
    x = torch.randn(Bn, S, D, device=dev, requires_grad=True)
    branch = (torch.randn(Bn, S, D, device=dev) * 2).to(torch.bfloat16).requires_grad_(True) if with_branch else None
    gamma = (torch.rand(D, device=dev) + 0.5).requires_grad_(True) if with_branch else None
    rs = torch.tensor([0.0, 1 / 0.9, 1 / 0.9][:Bn], device=dev) if with_branch else None
    w = (torch.rand(D, device=dev) + 0.5).requires_grad_(True)
    b = torch.randn(D, device=dev, requires_grad=True)
    bbias = torch.randn(D, device=dev, requires_grad=True) if with_branch else None
    x_out, y = residual_ln(x, branch, bbias, gamma, rs, w, b, 1e-6)
    assert x_out.dtype == torch.float32 and y.dtype == torch.bfloat16
    with torch.no_grad():
        xr, yr = ref_residual_ln(x.detach(), branch.detach() if with_branch else None, gamma, rs, w, b, 1e-6, S, bbias)
    np.testing.assert_allclose(x_out.detach().cpu().numpy(), xr.float().cpu().numpy(), rtol=1e-6, atol=1e-6)
    # y is rounded to bf16: 2^-8 relative
    np.testing.assert_allclose(y.float().detach().cpu().numpy(), yr.detach().float().cpu().numpy(), rtol=8e-3, atol=8e-3)
    g_xo = torch.randn_like(x_out)
    g_y = torch.randn_like(y)
    (x_out * g_xo).sum().add((y.float() * g_y.float()).sum()).backward()
    # fp64 autograd reference
    x2 = x.detach().double().requires_grad_(True)
    br2 = branch.detach().double().requires_grad_(True) if with_branch else None
    ga2 = gamma.detach().double().requires_grad_(True) if with_branch else None
    w2, b2 = w.detach().double().requires_grad_(True), b.detach().double().requires_grad_(True)
    bb2 = bbias.detach().double().requires_grad_(True) if with_branch else None
    xo2, y2 = ref_residual_ln(x2, br2, ga2, rs, w2, b2, 1e-6, S, bb2)
    (xo2 * g_xo.double()).sum().add((y2 * g_y.double()).sum()).backward()

    def chk(a, r, rtol):
        r = r.float().cpu().numpy()
        np.testing.assert_allclose(a.float().cpu().numpy(), r, rtol=rtol, atol=rtol * float(np.abs(r).max()))
    chk(x.grad, x2.grad, 1e-4)
    chk(w.grad, w2.grad, 1e-4)
    chk(b.grad, b2.grad, 1e-4)
    if with_branch:
        chk(branch.grad, br2.grad, 8e-3)       # bf16 output
        chk(gamma.grad, ga2.grad, 1e-4)
        chk(bbias.grad, bb2.grad, 1e-4)


def test_residual_ln_none_grads():
    """final norm: only y is used downstream -> g_xout is None."""
    from imagefolder_b200.vit_ops import residual_ln
    x = torch.randn(2, 5, 768, device="cuda", requires_grad=True)
    w = torch.ones(768, device="cuda", requires_grad=True)
    b = torch.zeros(768, device="cuda", requires_grad=True)
    _, y = residual_ln(x, None, None, None, None, w, b, 1e-6)
    g = torch.randn_like(y)
    y.backward(g)
    x2 = x.detach().double().requires_grad_(True)
    F.layer_norm(x2, (768,), w.detach().double(), b.detach().double(), 1e-6).backward(g.double())
    np.testing.assert_allclose(x.grad.cpu().numpy(), x2.grad.float().cpu().numpy(), rtol=1e-4, atol=1e-4 * float(x2.grad.abs().max()))


def _ln_bwd_stages(D):
    # residual_ln_bwd_kernel's ring: 3 stages of 8 rows (x_out, g_xout fp32; g_y, branch bf16; 128 B of row stats) when
    # they fit in 225 KiB of shared memory, else 2 (D = 1024)
    return 3 if 3 * (8 * D * 12 + 128) <= 225 * 1024 else 2


# (D, row count).  The backward hands out 8-row tiles: CTA i takes tile i, then tiles from an atomic counter through its
# ring of stages.  "tile_per_sm": 8 rows per SM, one tile per CTA, the grid not clamped (the partial-sum reduction reads
# every SM's partials).  "ring_twice": every CTA takes ~2 x stages tiles, so each stage is refilled (mbarrier parity
# flips) and most tiles come from the counter; +5 leaves a ragged last tile.  "training": the encoder at a batch of 128
# (8,208 tiles), 513 rows per sample, so tiles straddle samples.
_LN_ROWS = [(D, rows) for D in (384, 768, 1024) for rows in ("tile_per_sm", "ring_twice")] + [(768, "training")]


@pytest.mark.parametrize("D,rows", _LN_ROWS)
@pytest.mark.parametrize("call", ["norm1", "mid_block", "final_norm"])
def test_residual_ln_cabi_multi_tile(D, rows, call):
    """xq_vit_residual_ln_fwd / _bwd at row counts where the persistent backward's CTAs take several tiles, with the
    argument sets run_blocks passes: a block's first norm1 (no branch), a mid-block norm (branch + bias + LayerScale +
    per-sample rowscale) and the final norm (branch, but x_out unused: g_xout = NULL).  fp64 autograd reference."""
    from imagefolder_b200 import _capi
    L = _capi.lib()
    sms = _sms()
    M, S = {"tile_per_sm": (8 * sms, 37), "ring_twice": (8 * sms * 2 * _ln_bwd_stages(D) + 5, 37),
            "training": (TRAIN_ROWS, 513)}[rows]
    torch.manual_seed(M + D)
    dev = "cuda"
    eps = 1e-6
    x = torch.randn(M, D, device=dev) + 0.5 * torch.randn(M, 1, device=dev)     # row offsets: the mean is not ~0
    w = torch.rand(D, device=dev) + 0.5
    b = torch.randn(D, device=dev)
    branch = bbias = gamma = rs = None
    if call != "norm1":
        branch = (torch.randn(M, D, device=dev) * 2).to(torch.bfloat16)
        bbias = torch.randn(D, device=dev)
        gamma = torch.rand(D, device=dev) + 0.5
        rs = torch.rand((M + S - 1) // S, device=dev) * 1.5 + 0.25      # a different DropPath scale for every sample ...
        rs[::5] = 0.0                                                     # ... and dropped samples
    g_xout = torch.randn(M, D, device=dev) if call != "final_norm" else None
    g_y = torch.randint(-4, 5, (M, D), device=dev).to(torch.bfloat16)    # integer-valued: d ln_b = sum g_y is exact

    x_out, y, mean, rstd = _nan((M, D)), _nan((M, D), torch.bfloat16), _nan((M,)), _nan((M,))
    stream = _capi.stream_ptr(x.device)
    p = _capi.ptr
    _capi.check(L.xq_vit_residual_ln_fwd(p(x), p(branch), p(bbias), p(gamma), p(rs), S, p(w), p(b), eps, M, D, p(x_out),
                                         p(y), p(mean), p(rstd), stream), "xq_vit_residual_ln_fwd")
    g_x = _nan((M, D))
    g_w, g_b = _nan((D,)), _nan((D,))
    g_branch = _nan((M, D), torch.bfloat16) if branch is not None else None
    g_gamma = _nan((D,)) if branch is not None else None
    g_bbias = _nan((D,)) if branch is not None else None
    ws = torch.full((int(L.xq_vit_ln_bwd_workspace_bytes(D)),), 0xFF, dtype=torch.uint8, device=dev)   # NaN partials
    _capi.check(L.xq_vit_residual_ln_bwd(p(g_xout), p(g_y), p(x_out), p(mean), p(rstd), p(w), p(branch), p(bbias), p(gamma),
                                         p(rs), S, M, D, p(g_x), p(g_branch), p(g_w), p(g_b), p(g_gamma), p(g_bbias), p(ws),
                                         ws.numel(), stream), "xq_vit_residual_ln_bwd")

    # fp64 reference: x_new = x + s[row // S] * gamma * (branch + bias);  y = LayerNorm(x_new)
    x2 = x.double().requires_grad_(True)
    w2, b2 = w.double().requires_grad_(True), b.double().requires_grad_(True)
    xn = x2
    if branch is not None:
        br2, bb2, ga2 = (t.double().requires_grad_(True) for t in (branch, bbias, gamma))
        s_row = rs.double()[torch.arange(M, device=dev) // S].unsqueeze(1)
        xn = x2 + s_row * ga2 * (br2 + bb2)
    y2 = F.layer_norm(xn, (D,), w2, b2, eps)
    if g_xout is not None:
        torch.autograd.backward((y2, xn), (g_y.double(), g_xout.double()))
    else:
        y2.backward(g_y.double())
    with torch.no_grad():
        xn = xn.detach()
        mean2 = xn.mean(-1)
        rstd2 = (xn.var(-1, unbiased=False) + eps).rsqrt()
        xh = (xn - mean2.unsqueeze(1)) * rstd2.unsqueeze(1)

        # forward.  fp32 values: 1e-5 relative (of the row's mean |x_new| for the mean, a sum of D terms); bf16 y: 2^-8
        if branch is None:
            assert torch.equal(x_out, x)
        _assert_within(x_out, xn, 1e-5 * xn.abs().max(), "x_out")
        _assert_within(mean, mean2, 1e-5 * xn.abs().mean(-1), "mean")
        _assert_within(rstd, rstd2, 1e-5 * rstd2, "rstd")
        _assert_within(y.float(), y2.detach(), 2 ** -8 * y2.detach().abs().max(), "y")
        del y2
        # backward.  G = d x_new (= g_x); fp32 g_x: 1e-5 of its max; bf16 g_branch: 2^-8 of its max
        G = x2.grad
        _assert_within(g_x, G, 1e-5 * G.abs().max(), "g_x")
        # column sums over M rows in fp32: a lane sums its CTA's tiles (~60 at the training shape), then 8 warps, then
        # the per-SM partials 8 x 17 -- about 100 additions deep, 100 x 2^-24 < 1e-5 of sum |terms| of the column
        gy64 = g_y.double()
        _assert_within(g_w, w2.grad, 1e-5 * (gy64 * xh).abs().sum(0), "d ln_w")
        assert torch.equal(g_b, g_y.to(torch.int64).sum(0).to(torch.float32)), "d ln_b: a row counted twice or not at all"
        del gy64, xh
        if branch is not None:
            _assert_within(g_branch.float(), br2.grad, 2 ** -8 * br2.grad.abs().max(), "g_branch")
            Gs = G * s_row
            # the kernel sums G s branch and G s separately: d gamma = sum(G s branch) + bias sum(G s), d bias = gamma sum(G s)
            sum_gs = Gs.abs().sum(0)
            _assert_within(g_gamma, ga2.grad, 1e-5 * ((Gs * br2.detach()).abs().sum(0) + bb2.detach().abs() * sum_gs), "d gamma")
            _assert_within(g_bbias, bb2.grad, 1e-5 * ga2.detach().abs() * sum_gs, "d branch_bias")


def test_gelu_bf16():
    from imagefolder_b200.vit_ops import gelu_bias
    for C in (3072, 1536, 64):
        x = (torch.randn(4, 33, C, device="cuda") * 2).to(torch.bfloat16).requires_grad_(True)
        bias = torch.randn(C, device="cuda", requires_grad=True)
        y = gelu_bias(x, bias)
        x2 = x.detach().double().requires_grad_(True)
        b2 = bias.detach().double().requires_grad_(True)
        ref = F.gelu(x2 + b2)
        np.testing.assert_allclose(y.float().detach().cpu().numpy(), ref.detach().float().cpu().numpy(), rtol=8e-3, atol=2e-3)
        g = torch.randn_like(y)
        y.backward(g)
        ref.backward(g.double())
        np.testing.assert_allclose(x.grad.float().cpu().numpy(), x2.grad.float().cpu().numpy(), rtol=8e-3, atol=8e-3)
        # bias grad = column sums of bf16-rounded gx
        np.testing.assert_allclose(bias.grad.cpu().numpy(), b2.grad.float().cpu().numpy(), rtol=2e-2, atol=0.15)
    y = gelu_bias((torch.randn(2, 8, device="cuda")).to(torch.bfloat16), None)
    assert y.shape == (2, 8)

    # the backward at the training rows and the ViT-B MLP width: every CTA of the persistent kernel walks dozens of row
    # groups with the next group's loads in flight.  C ABI, NaN-filled outputs, fp64 reference in row chunks.
    from imagefolder_b200 import _capi
    L = _capi.lib()
    M, C = TRAIN_ROWS, 3072
    x = (torch.randn(M, C, device="cuda") * 2).to(torch.bfloat16)
    bias = torch.randn(C, device="cuda")
    gy = torch.randn(M, C, device="cuda").to(torch.bfloat16)
    gx, gb = _nan((M, C), torch.bfloat16), _nan((C,))
    _capi.check(L.xq_vit_gelu_bwd(_capi.ptr(x), _capi.ptr(bias), _capi.ptr(gy), _capi.ptr(gx), _capi.ptr(gb), M, C,
                                  _capi.stream_ptr(x.device)), "xq_vit_gelu_bwd")
    gb_ref, gb_abs, gy_abs = (torch.zeros(C, dtype=torch.float64, device="cuda") for _ in range(3))
    errs, maxs = [], []
    for r0 in range(0, M, 8192):
        u = x[r0:r0 + 8192].double() + bias.double()
        g64 = gy[r0:r0 + 8192].double()
        t = g64 * (0.5 * (1.0 + torch.erf(u / math.sqrt(2.0))) + u * torch.exp(-0.5 * u * u) / math.sqrt(2.0 * math.pi))
        errs.append((gx[r0:r0 + 8192].double() - t).abs().max())
        maxs.append(t.abs().max())
        gb_ref += t.sum(0)
        gb_abs += t.abs().sum(0)
        gy_abs += g64.abs().sum(0)
    err, tmax = torch.stack(errs).max(), torch.stack(maxs).max()
    assert bool(err <= 2 ** -8 * tmax), f"gx: max err {err.item():.3e} vs max {tmax.item():.3e}"     # bf16 output
    # d bias: fp32 sums of the unrounded terms (a thread's ~100 rows, then one atomicAdd per CTA): rounding well under 1e-5 of
    # sum |terms| of the column; the A&S erf inside gelu' adds at most ~5e-7 |gy| per term
    _assert_within(gb, gb_ref, 1e-5 * gb_abs + 5e-7 * gy_abs, "d bias")


def test_fused_blocks_match_module_path():
    """bf16-autocast encoder through the fused glue == the plain module path (same weights, eval)."""
    from imagefolder_b200.dino_enc import DINOv2Encoder
    from imagefolder_b200 import vit_ops
    kw = {'img_size': 256, 'patch_size': 16, 'drop_path_rate': 0.1}
    torch.manual_seed(0)
    enc = DINOv2Encoder(num_latent_tokens=256, model_name='vit_small_patch14_dinov2.lvd142m', model_kwargs=kw,
                        tuning_method='full', abs_pos_embed=True).cuda().eval()
    for blk in enc.model.blocks:            # make LayerScale matter
        blk.ls1.gamma.data.fill_(0.5)
        blk.ls2.gamma.data.fill_(0.5)
    x = torch.rand(2, 3, 256, 256, device="cuda") * 2 - 1
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y_fused = enc(x)
        orig = vit_ops.fused_path_ok
        vit_ops.fused_path_ok = lambda *a, **k: False
        try:
            y_plain = enc(x)
        finally:
            vit_ops.fused_path_ok = orig
    assert y_fused.dtype == torch.bfloat16
    a, b = y_fused.detach().float().cpu().numpy(), y_plain.detach().float().cpu().numpy()
    # both are bf16-GEMM pipelines; they differ only by rounding order
    assert np.abs(a - b).max() < 0.06 * np.abs(b).max()
    assert np.corrcoef(a.ravel(), b.ravel())[0, 1] > 0.9995


def test_packed_attention_matches_explicit_softmax():
    from imagefolder_b200.vit_ops import packed_attention
    torch.manual_seed(3)
    B, N, H, hd = 3, 77, 6, 64
    C = H * hd
    qkv = torch.randn(B, N, 3 * C, device="cuda").to(torch.bfloat16).requires_grad_(True)
    o = packed_attention(qkv, H)
    assert o.shape == (B, N, C)
    g = torch.randn_like(o)
    o.backward(g)
    q2 = qkv.detach().double().requires_grad_(True)
    t = q2.view(B, N, 3, H, hd).permute(2, 0, 3, 1, 4)
    att = ((t[0] * hd ** -0.5) @ t[1].transpose(-2, -1)).softmax(-1)
    ref = (att @ t[2]).transpose(1, 2).reshape(B, N, C)
    ref.backward(g.double())
    np.testing.assert_allclose(o.float().detach().cpu().numpy(), ref.detach().float().cpu().numpy(), rtol=2e-2, atol=2e-2)
    gr = q2.grad.float().cpu().numpy()
    np.testing.assert_allclose(qkv.grad.float().cpu().numpy(), gr, rtol=3e-2, atol=3e-2 * float(np.abs(gr).max()))


def test_qkv_attention_node_matches_linear_plus_attention():
    """_QKVAttention (projection + attention as one node; bias gradient from the pack kernel's column sums) against
    nn.Linear + packed_attention with autograd's own sum(0) bias gradient."""
    from imagefolder_b200.vit_ops import packed_attention, _QKVAttention
    torch.manual_seed(5)
    B, N, H, hd = 4, 131, 6, 64
    C = H * hd
    y = torch.randn(B, N, C, device="cuda").to(torch.bfloat16).requires_grad_(True)
    W = (torch.randn(3 * C, C, device="cuda") * C ** -0.5).requires_grad_(True)
    b = torch.randn(3 * C, device="cuda").requires_grad_(True)
    g = torch.randn(B, N, C, device="cuda").to(torch.bfloat16)
    o1 = _QKVAttention.apply(y, W, b, H, 0.0)
    gy1, gW1, gb1 = torch.autograd.grad(o1, (y, W, b), g)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        o2 = packed_attention(torch.nn.functional.linear(y, W, b), H)
    gy2, gW2, gb2 = torch.autograd.grad(o2, (y, W, b), g)
    assert torch.equal(o1, o2)                                   # same GEMM + same library attention
    assert gW1.dtype == torch.float32 and gb1.dtype == torch.float32
    np.testing.assert_allclose(gy1.float().cpu().numpy(), gy2.float().cpu().numpy(), rtol=0, atol=0)
    np.testing.assert_allclose(gW1.cpu().numpy(), gW2.cpu().numpy(), rtol=0, atol=0)
    # the fused bias gradient sums the bf16 d(qkv) in fp32 (autograd: bf16 reduce) -> equal up to bf16 rounding
    ref = gb2.cpu().numpy()
    np.testing.assert_allclose(gb1.cpu().numpy(), ref, rtol=1e-2, atol=1e-2 * float(np.abs(ref).max()))


def test_pack_qkv_cabi_ragged_rows_and_bias():
    from imagefolder_b200 import _capi
    L = _capi.lib()
    torch.manual_seed(6)
    sms = _sms()
    # the last two: the training encoder's rows (8,208 tiles, ~60 per CTA) and ~8 tiles per CTA at the widest C the kernel
    # takes -- every CTA's 4-stage ring wraps and most tiles come from the atomic counter
    for M, C in [(1, 8), (7, 64), (1031, 768), (4099, 384), (2500, 1024), (TRAIN_ROWS, 768), (8 * sms * 8 + 3, 1024)]:
        ws = torch.empty(int(L.xq_vit_pack_workspace_bytes()), dtype=torch.uint8, device="cuda")

        def pack(dq, dk, dv, gb):
            out = _nan((M, 3 * C), torch.bfloat16)
            _capi.check(L.xq_vit_pack_qkv(_capi.ptr(dq), _capi.ptr(dk), _capi.ptr(dv), _capi.ptr(out), _capi.ptr(gb), M, C,
                                          _capi.ptr(ws), ws.numel(), _capi.stream_ptr(out.device)), "xq_vit_pack_qkv")
            return out

        # integer-valued gradients: the fp32 column sums are exact in any order, so the bias gradient must equal the int64
        # sums -- a row counted twice or not at all fails at any M
        dq, dk, dv = (torch.randint(-4, 5, (M, C), device="cuda").to(torch.bfloat16) for _ in range(3))
        gb = torch.full((3 * C,), 7.0, device="cuda")                   # the launcher zeroes it
        ref = torch.cat([dq, dk, dv], dim=1)
        assert torch.equal(pack(dq, dk, dv, gb), ref)
        assert torch.equal(gb, ref.to(torch.int64).sum(0).to(torch.float32))
        # full-mantissa values for the copy, with and without the bias gradient
        dq, dk, dv = (torch.randn(M, C, device="cuda").to(torch.bfloat16) for _ in range(3))
        ref = torch.cat([dq, dk, dv], dim=1)
        assert torch.equal(pack(dq, dk, dv, gb), ref)
        # fp32 sums: a lane's tiles (<= ~60), 8 warps, one atomicAdd per CTA: ~200 additions deep, 200 x 2^-24 = 1.2e-5
        _assert_within(gb, ref.double().sum(0), 1.2e-5 * ref.double().abs().sum(0), "g_bias")
        assert torch.equal(pack(dq, dk, dv, None), ref)
    assert L.xq_vit_pack_qkv(None, None, None, None, None, 4, 8, None, 0, None) != 0


def test_patch_embed_gemm_matches_conv():
    """_PatchEmbed (patchify kernel + GEMM) vs the module's Conv2d under the same bf16 autocast; patchify itself is a
    pure permutation -> bit-exact against unfold."""
    from imagefolder_b200 import _capi
    from imagefolder_b200.dino_enc.vision_transformer import PatchEmbed
    from imagefolder_b200.vit_ops import patch_embed, patch_embed_ok
    torch.manual_seed(8)
    for B, Cin, HW, p, D in [(3, 3, 64, 16, 96), (2, 3, 256, 16, 768), (1, 4, 48, 8, 40), (2, 3, 56, 4, 64)]:
        pe = PatchEmbed(img_size=HW, patch_size=p, in_chans=Cin, embed_dim=D).cuda()
        x = torch.rand(B, Cin, HW, HW, device="cuda") * 2 - 1
        patches = torch.empty(B * (HW // p) ** 2, Cin * p * p, device="cuda", dtype=torch.bfloat16)
        L = _capi.lib()
        _capi.check(L.xq_vit_patchify(_capi.ptr(x), _capi.ptr(patches), B, Cin, HW, HW, p, _capi.stream_ptr(x.device)),
                    "xq_vit_patchify")
        ref = torch.nn.functional.unfold(x, kernel_size=p, stride=p).transpose(1, 2).reshape(patches.shape)
        assert torch.equal(patches, ref.to(torch.bfloat16))
        with torch.autocast("cuda", dtype=torch.bfloat16):
            assert patch_embed_ok(pe, x)
            y1 = patch_embed(pe, x)
            y2 = pe(x)
        assert y1.shape == y2.shape and y1.dtype == torch.bfloat16
        np.testing.assert_allclose(y1.detach().float().cpu().numpy(), y2.detach().float().cpu().numpy(), rtol=2e-2, atol=2e-2)
        g = torch.randn_like(y1)
        gW1, gb1 = torch.autograd.grad(y1, (pe.proj.weight, pe.proj.bias), g)
        gW2, gb2 = torch.autograd.grad(y2, (pe.proj.weight, pe.proj.bias), g)
        assert gW1.dtype == torch.float32 and gW1.shape == pe.proj.weight.shape
        sW, sb = float(gW2.abs().max()), float(gb2.abs().max())
        np.testing.assert_allclose(gW1.cpu().numpy(), gW2.cpu().numpy(), rtol=2e-2, atol=2e-2 * sW)
        np.testing.assert_allclose(gb1.cpu().numpy(), gb2.cpu().numpy(), rtol=2e-2, atol=2e-2 * sb)
    # not applicable (image needs a gradient / no autocast) -> the module's own conv
    xg = torch.rand(1, 3, 64, 64, device="cuda", requires_grad=True)
    pe = PatchEmbed(img_size=64, patch_size=16, in_chans=3, embed_dim=32).cuda()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        assert not patch_embed_ok(pe, xg)
    assert not patch_embed_ok(pe, xg.detach())
    L = _capi.lib()
    assert L.xq_vit_patchify(None, None, 1, 3, 64, 64, 16, None) != 0
    assert L.xq_vit_patchify(_capi.ptr(xg.detach()), _capi.ptr(xg.detach()), 1, 3, 64, 64, 6, None) != 0


@pytest.mark.parametrize("pq,abs_pe", [(1, True), (2, True), (1, False)])
def test_fused_token_assembly_equals_module_chain(pq, abs_pe):
    """encoder / decoder input sequence through xq_vit_assemble_* == the module's own cat / add chain: outputs and the
    gradients of every parameter that feeds the sequence (cls / mask / latent tokens, pos-embed, level embedding)."""
    from imagefolder_b200.dino_enc import DINOv2Decoder, DINOv2Encoder
    from imagefolder_b200 import vit_ops
    kw = {'img_size': 256, 'patch_size': 16, 'drop_path_rate': 0.0}   # the level-embedding table assumes 16 x 16 image tokens
    torch.manual_seed(pq)
    L = 16 * pq if pq > 1 else 16
    enc = DINOv2Encoder(num_latent_tokens=L, model_name='vit_small_patch14_dinov2.lvd142m', model_kwargs=kw, tuning_method='full',
                        abs_pos_embed=abs_pe, product_quant=pq).cuda().train()
    dec = DINOv2Decoder(num_latent_tokens=16, model_name='vit_small_patch14_dinov2.lvd142m', model_kwargs=kw, tuning_method='full',
                        abs_pos_embed=abs_pe).cuda().train()
    x = torch.rand(2, 3, 256, 256, device="cuda") * 2 - 1
    z = torch.randn(2, 16, dec.embed_dim, device="cuda").to(torch.bfloat16).requires_grad_(True)

    def run(fused):
        vit_ops.ASSEMBLE_ENABLED[0] = fused
        try:
            for m in (enc, dec):
                m.zero_grad(set_to_none=True)
            if z.grad is not None:
                z.grad = None
            with torch.autocast("cuda", dtype=torch.bfloat16):
                he = enc(x)
                hd = dec(z)
            torch.manual_seed(99)
            (he.float() * torch.randn_like(he.float())).sum().add((hd.float() * torch.randn_like(hd.float())).sum()).backward()
            grads = {n: p.grad.clone() for mod, tag in ((enc, "enc."), (dec, "dec.")) for n_, p in mod.named_parameters()
                     if p.grad is not None for n in [tag + n_]
                     if any(k in n_ for k in ("cls_token", "pos_embed", "latent_tokens", "lvl_embed", "mask_token", "latent_pos_embed",
                                              "patch_embed.proj"))}
            return he.detach().float(), hd.detach().float(), z.grad.clone().float(), grads
        finally:
            vit_ops.ASSEMBLE_ENABLED[0] = True

    he1, hd1, gz1, g1 = run(True)
    assert getattr(enc, "_assemble_ok", None) is True and getattr(dec, "_assemble_ok", None) is True
    he0, hd0, gz0, g0 = run(False)
    tol = dict(rtol=3e-2, atol=3e-2)          # bf16 pipelines: identical up to rounding order of the fp32 adds feeding bf16 GEMMs
    np.testing.assert_allclose(he1.cpu().numpy(), he0.cpu().numpy(), **tol)
    np.testing.assert_allclose(hd1.cpu().numpy(), hd0.cpu().numpy(), **tol)
    np.testing.assert_allclose(gz1.cpu().numpy(), gz0.cpu().numpy(), rtol=5e-2, atol=5e-2 * float(gz0.abs().max()))
    assert set(g1) == set(g0) and len(g1) >= 6
    for k in g0:
        a, b = g1[k].float().cpu().numpy(), g0[k].float().cpu().numpy()
        np.testing.assert_allclose(a, b, rtol=5e-2, atol=5e-2 * float(np.abs(b).max()) + 1e-6, err_msg=k)


def test_assemble_cabi_exact():
    from imagefolder_b200.vit_ops import _Assemble
    torch.manual_seed(0)
    for dt in (torch.float32, torch.bfloat16):
        src = torch.randn(5, 7, 24, device="cuda").to(dt).requires_grad_(True)
        table = torch.randn(12, 24, device="cuda", requires_grad=True)
        out = _Assemble.apply(src, table, 3)
        ref = table.detach().unsqueeze(0).repeat(5, 1, 1)
        ref[:, 3:10] += src.detach().float()
        assert torch.equal(out, ref)
        g = torch.randn_like(out)
        gs, gt = torch.autograd.grad(out, (src, table), g)
        assert gs.dtype == dt and torch.equal(gs, g[:, 3:10].to(dt))
        np.testing.assert_allclose(gt.cpu().numpy(), g.sum(0).cpu().numpy(), rtol=1e-6, atol=1e-6)
    # the backward at the encoder's sequence shape (cls + 256 image rows from src at t0 = 1 + 256 latents, D = 768) with
    # batches where assemble_bwd_kernel's 8-sample loop runs once exactly, once plus a ragged step, and 16 times.  C ABI,
    # NaN-filled outputs.  g on a 2^-8 grid with |g| <= 16: the cast to bf16 still rounds, and every partial sum over the
    # batch is a multiple of 2^-8 below 2^11, exact in fp32 in any order -> d_table must equal the integer sum.
    from imagefolder_b200 import _capi
    L = _capi.lib()
    T, Ls, t0, D = 513, 256, 1, 768
    for B in (8, 9, 128):
        gi = torch.randint(-4096, 4097, (B, T, D), device="cuda")
        g = gi.float() / 256
        d_table_ref = gi.sum(0).float() / 256
        for dt in (torch.float32, torch.bfloat16):
            d_src, d_table = _nan((B, Ls, D), dt), _nan((T, D))
            _capi.check(L.xq_vit_assemble_bwd(_capi.ptr(g), B, Ls, T, D, t0, _capi.ptr(d_src), int(dt == torch.bfloat16),
                                              _capi.ptr(d_table), _capi.stream_ptr(g.device)), "xq_vit_assemble_bwd")
            assert torch.equal(d_src, g[:, t0:t0 + Ls].to(dt)), (B, dt)
            assert torch.equal(d_table, d_table_ref), (B, dt)


@pytest.mark.parametrize("M,C,Hd", [(2 * 513, 384, 1536), (4 * 513, 768, 3072), (131, 768, 3072), (3 * 256, 384, 1536)])
def test_fused_mlp_gemm_epilogues_equal_library_gemm_plus_gelu_kernels(M, C, Hd):
    """xq_vit_fc1_gelu_fwd / xq_vit_fc2_dgelu_bwd (wgmma GEMMs with GELU / GELU' + bias-gradient epilogues) against the
    path they replace -- library GEMM + the stand-alone bias / GELU kernels -- for timm Mlp inside Block.forward
    (dino_enc/vision_transformer.py:336-339).  The epilogues apply the same device functions to the same rounded bf16 values, so the
    results agree to the last bit up to the accumulation order of the GEMMs (checked at bf16 resolution)."""
    from imagefolder_b200 import vit_ops
    torch.manual_seed(M + C)
    dev = torch.device("cuda")
    mlp = torch.nn.Module()
    mlp.fc1 = torch.nn.Linear(C, Hd).to(dev)
    mlp.fc2 = torch.nn.Linear(Hd, C).to(dev)
    y0 = torch.randn(M, C, device=dev).to(torch.bfloat16)
    g = torch.randn(M, C, device=dev).to(torch.bfloat16)

    def run(fused):
        vit_ops.MLP_TC_ENABLED[0] = fused
        for p in mlp.parameters():
            p.grad = None
        y = y0.clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = vit_ops.mlp_forward(mlp, y)
        out.backward(g)
        return out.detach(), y.grad, mlp.fc1.weight.grad, mlp.fc1.bias.grad, mlp.fc2.weight.grad

    try:
        assert vit_ops.mlp_tc_ok(y0, mlp.fc1, mlp.fc2)
        a = run(True)
        b = run(False)
    finally:
        vit_ops.MLP_TC_ENABLED[0] = True
    torch.cuda.synchronize()
    names = ["branch", "d_y", "d_W1", "d_b1", "d_W2"]
    for n, u, v in zip(names, a, b):
        assert u.shape == v.shape and torch.isfinite(u.float()).all(), n
        scale = max(1e-6, v.float().abs().max().item())
        err = (u.float() - v.float()).abs().max().item()
        assert err <= 8e-3 * scale, f"{n}: max err {err:.3e} vs max {scale:.3e}"
