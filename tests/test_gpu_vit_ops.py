"""Numerics of the ViT glue kernels against a plain PyTorch fp32 reference of the same op
(floating-point kernels: tolerance set by the bf16 operands, written per assertion)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


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
    for M, C in [(1, 8), (7, 64), (1031, 768), (4099, 384), (2500, 1024)]:
        dq, dk, dv = (torch.randn(M, C, device="cuda").to(torch.bfloat16) for _ in range(3))
        out = torch.empty(M, 3 * C, device="cuda", dtype=torch.bfloat16)
        gb = torch.full((3 * C,), 7.0, device="cuda")
        ws = torch.empty(int(L.xq_vit_pack_workspace_bytes()), dtype=torch.uint8, device="cuda")
        _capi.check(L.xq_vit_pack_qkv(_capi.ptr(dq), _capi.ptr(dk), _capi.ptr(dv), _capi.ptr(out), _capi.ptr(gb), M, C,
                                      _capi.ptr(ws), ws.numel(), _capi.stream_ptr(out.device)), "xq_vit_pack_qkv")
        ref = torch.cat([dq, dk, dv], dim=1)
        assert torch.equal(out, ref)
        np.testing.assert_allclose(gb.cpu().numpy(), ref.float().sum(0).cpu().numpy(), rtol=1e-4, atol=1e-3)
        out.zero_()
        _capi.check(L.xq_vit_pack_qkv(_capi.ptr(dq), _capi.ptr(dk), _capi.ptr(dv), _capi.ptr(out), None, M, C,
                                      _capi.ptr(ws), ws.numel(), _capi.stream_ptr(out.device)), "xq_vit_pack_qkv")
        assert torch.equal(out, ref)
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
