"""SwiGLU on the GPU: the stand-alone xq_vit_swiglu_fwd / _bwd and the D = 1536 LayerNorm glue against fp64, and the giant /
reg4 backbones end to end (library GEMMs + the stand-alone SwiGLU kernel)."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

DTYPES = {"bf16": (torch.bfloat16, ""), "f16": (torch.float16, "_f16")}
EPS = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}       # one rounding to the 16-bit type, relative
TINY = {torch.bfloat16: 2.0 ** -134, torch.float16: 2.0 ** -25}     # ... and absolute: half the subnormal spacing


def _lib():
    from imagefolder_b200 import _capi
    return _capi, _capi.lib()


def _nan(shape, dt):
    return torch.full(shape, float("nan"), dtype=dt, device="cuda")


def _assert_within(a, ref, tol, what):
    err = (a.double() - ref).abs()
    ok = err <= tol
    assert bool(ok.all()), f"{what}: {int((~ok).sum())} of {ok.numel()} out of tolerance, max err {err.max().item():.3e}"


# ---- stand-alone SwiGLU against fp64 -----------------------------------------------------------------------------
def _silu64(a):
    return a / (1.0 + torch.exp(-a))


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("M,H", [(128 * 517, 512), (517, 4096), (3, 8)])
def test_standalone_swiglu_against_fp64(M, H, dtn):
    dt, sfx = DTYPES[dtn]
    _capi, L = _lib()
    p, s = _capi.ptr, _capi.stream_ptr()
    gen = torch.Generator(device="cuda").manual_seed(M + H)
    pre = (3 * torch.randn(M, 2 * H, device="cuda", generator=gen)).to(dt)
    b = torch.randn(2 * H, device="cuda", generator=gen)
    g = torch.randn(M, H, device="cuda", generator=gen).to(dt)
    act, d_pre, d_b = _nan((M, H), dt), _nan((M, 2 * H), dt), _nan((2 * H,), torch.float32)
    _capi.check(getattr(L, "xq_vit_swiglu_fwd" + sfx)(p(pre), p(b), p(act), M, H, s), "swiglu_fwd")
    _capi.check(getattr(L, "xq_vit_swiglu_bwd" + sfx)(p(pre), p(b), p(g), p(d_pre), p(d_b), M, H, s), "swiglu_bwd")
    a, c, gd = pre[:, :H].double() + b[:H].double(), pre[:, H:].double() + b[H:].double(), g.double()
    sa = _silu64(a)
    sg = 1.0 / (1.0 + torch.exp(-a))
    eps, tiny = EPS[dt], TINY[dt]
    # one 16-bit rounding of the result, plus the fp32 arithmetic before it (a few 1e-7 relative to each product's factors)
    ref = sa * c
    _assert_within(act, ref, eps * ref.abs() + 4e-6 * (a.abs() + 1) * c.abs() + tiny, "act vs fp64")
    ra = gd * c * sg * (1.0 + a * (1.0 - sg))
    rc = gd * sa
    _assert_within(d_pre[:, :H], ra, eps * ra.abs() + 4e-6 * (a.abs() + 1) * (gd * c).abs() + tiny, "d_gate vs fp64")
    _assert_within(d_pre[:, H:], rc, eps * rc.abs() + 4e-6 * (a.abs() + 1) * gd.abs() + tiny, "d_up vs fp64")
    t = d_pre.double()
    _assert_within(d_b, t.sum(0), (M + 2) * 2.0 ** -24 * t.abs().sum(0), "d_b vs fp64 column sums of d_pre")


@pytest.mark.parametrize("dtn", list(DTYPES))
def test_standalone_swiglu_exact_on_integer_inputs(dtn):
    """gate + bias >= 32: silu is the identity and silu' is 1 in fp32 (exp(-32) < 2^-24), so with integer pre, bias and g
    every output is an integer of magnitude <= 176 (exact in bf16 and fp16), and every column sum (< 2^24) is exact in fp32
    in any order."""
    dt, sfx = DTYPES[dtn]
    _capi, L = _lib()
    p, s = _capi.ptr, _capi.stream_ptr()
    M, H = 128 * 517, 256
    gen = torch.Generator(device="cuda").manual_seed(5)
    pre = torch.randint(-3, 4, (M, 2 * H), device="cuda", generator=gen).to(dt)
    b = torch.cat([torch.full((H,), 40.0, device="cuda"), torch.randint(-1, 2, (H,), device="cuda", generator=gen).float()])
    g = torch.randint(-4, 5, (M, H), device="cuda", generator=gen).to(dt)
    act, d_pre, d_b = _nan((M, H), dt), _nan((M, 2 * H), dt), _nan((2 * H,), torch.float32)
    _capi.check(getattr(L, "xq_vit_swiglu_fwd" + sfx)(p(pre), p(b), p(act), M, H, s), "swiglu_fwd")
    _capi.check(getattr(L, "xq_vit_swiglu_bwd" + sfx)(p(pre), p(b), p(g), p(d_pre), p(d_b), M, H, s), "swiglu_bwd")
    a, c, gd = pre[:, :H].double() + 40.0, pre[:, H:].double() + b[H:].double(), g.double()
    assert float((a * c).abs().max()) <= 256 and float((gd * a).abs().max()) <= 256
    assert torch.equal(act.double(), a * c)
    assert torch.equal(d_pre[:, :H].double(), gd * c) and torch.equal(d_pre[:, H:].double(), gd * a)
    want = torch.cat([(gd * c).sum(0), (gd * a).sum(0)])
    assert float(torch.cat([(gd * c).abs().sum(0), (gd * a).abs().sum(0)]).max()) < 2 ** 24
    assert torch.equal(d_b.double(), want)


@pytest.mark.parametrize("dtn", list(DTYPES))
def test_silu_special_values_match_torch(dtn):
    """silu at +-0, large +-x, where exp(-x) overflows, and at +-inf / NaN: the stand-alone kernel's arithmetic against torch.nn.functional.silu on the same fp32 inputs, probed as act = silu(-0 + b) * (1 + 0) (-0 + b is b,
    -0 included)"""
    dt, sfx = DTYPES[dtn]
    _capi, L = _lib()
    p, s = _capi.ptr, _capi.stream_ptr()
    vals = [0.0, -0.0, 1e-30, -1e-30, 0.5, -0.5, 20.0, -20.0, 88.0, -88.0, 89.0, -89.0, 100.0, -100.0, 1e4, -1e4, 3e38,
            -3e38, float("inf"), -float("inf"), float("nan")]
    H = 8 * ((len(vals) + 7) // 8)
    a = torch.zeros(H, device="cuda")
    a[:len(vals)] = torch.tensor(vals, device="cuda")
    b = torch.cat([a, torch.zeros(H, device="cuda")])
    pre = torch.cat([torch.full((1, H), -0.0), torch.ones(1, H)], 1).to(dt).cuda()
    act = _nan((1, H), dt)
    _capi.check(getattr(L, "xq_vit_swiglu_fwd" + sfx)(p(pre), p(b), p(act), 1, H, s), "swiglu_fwd")
    want = torch.nn.functional.silu(a).to(dt)
    same = (act[0].view(torch.int16) == want.view(torch.int16)) | (torch.isnan(act[0]) & torch.isnan(want))
    assert bool(same.all()), (a[~same].tolist(), act[0][~same].tolist(), want[~same].tolist())
    assert float(act[0, 1].view(torch.int16)) == float(want[1].view(torch.int16))       # silu(-0) keeps its sign


# ---- LayerNorm glue at D = 1536 ----------------------------------------------------------------------------------
@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("B,S", [(128, 517), (3, 513), (1, 5)])
def test_residual_ln_d1536_against_fp64(B, S, dtn):
    """xq_vit_residual_ln_fwd / _bwd at the giant width (one staged tile in flight in the backward) through vit_ops"""
    from imagefolder_b200 import vit_ops
    dt = DTYPES[dtn][0]
    D = 1536
    gen = torch.Generator(device="cuda").manual_seed(B * S)
    x = torch.randn(B, S, D, device="cuda", generator=gen, requires_grad=True)
    br = torch.randn(B, S, D, device="cuda", generator=gen).to(dt).requires_grad_()
    bb = (0.1 * torch.randn(D, device="cuda", generator=gen)).requires_grad_()
    gm = (0.3 + 0.1 * torch.randn(D, device="cuda", generator=gen)).requires_grad_()
    rs = torch.rand(B, device="cuda", generator=gen) * 2
    w = (1 + 0.1 * torch.randn(D, device="cuda", generator=gen)).requires_grad_()
    lb = (0.1 * torch.randn(D, device="cuda", generator=gen)).requires_grad_()
    gx = torch.randn(B, S, D, device="cuda", generator=gen)
    gy = torch.randn(B, S, D, device="cuda", generator=gen).to(dt)
    with torch.autocast("cuda", dtype=dt):
        xo, y = vit_ops.residual_ln(x, br, bb, gm, rs, w, lb, 1e-6)
    torch.autograd.backward([xo, y], [gx, gy])
    leaves = [x, br, bb, gm, w, lb]
    got = [t.grad.double() for t in leaves]
    d = [t.detach().double().requires_grad_() for t in leaves]
    xo64 = d[0] + rs.double()[:, None, None] * d[3] * (d[1] + d[2])
    y64 = torch.nn.functional.layer_norm(xo64, (D,), d[4], d[5], 1e-6)
    torch.autograd.backward([xo64, y64], [gx.double(), gy.double()])
    _assert_within(xo, xo64.detach(), 1e-5 * xo64.detach().abs() + 1e-5, "x_out vs fp64")
    _assert_within(y, y64.detach(), EPS[dt] * y64.detach().abs() + 1e-4, "y vs fp64")
    for gt, t, name in zip(got, d, ["x", "branch", "branch_bias", "ls_gamma", "ln_w", "ln_b"]):
        ref = t.grad
        scale = float(ref.abs().max())
        tol = (EPS[dt] if name == "branch" else 1e-4) * ref.abs() + 2e-4 * scale
        _assert_within(gt, ref, tol, f"d {name} vs fp64")


# ---- model level ---------------------------------------------------------------------------------------------------
GIANT = "vit_giant_patch14_dinov2.lvd142m"
REG4 = "vit_small_patch14_reg4_dinov2.lvd142m"


def _build(cfg, depth, monkeypatch, det=True):
    from imagefolder_b200 import config as xcfg
    from imagefolder_b200.dino_enc import vision_transformer as vt
    from vit_det_init import apply_det_init
    for name in (GIANT, GIANT.replace("_patch14_", "_patch14_reg4_")):
        monkeypatch.setitem(vt._ARCH, name, dict(vt._ARCH[name], depth=depth))
    args = xcfg.parse_args([])
    for k, v in cfg.items():
        setattr(args, k, v)
    torch.manual_seed(0)
    model = xcfg.build_vq_model(args)
    if det:
        apply_det_init(model)
    return model


def _count_swiglu(monkeypatch):
    """counts the stand-alone SwiGLU nodes (vit_ops._SwiGLUBias) the model runs"""
    from imagefolder_b200 import vit_ops
    n = {"swiglu": 0}
    lib = vit_ops._SwiGLUBias.apply
    monkeypatch.setattr(vit_ops._SwiGLUBias, "apply", lambda *a: (n.__setitem__("swiglu", n["swiglu"] + 1), lib(*a))[1])
    return n


def _giant_cfg(abs_pos_embed=True):
    return dict(codebook_size=8192, codebook_embed_dim=32, v_patch_nums=[16], num_latent_tokens=256, product_quant=1,
                abs_pos_embed=abs_pos_embed, enc_type="dinov2", dec_type="dinov2", semantic_guide="none",
                detail_guide="none", encoder_model=GIANT, decoder_model=GIANT)


@pytest.mark.parametrize("name", ["vit_giant_vq", "vit_giant_relpos", "vit_reg4_relpos"])
def test_fused_path_matches_reference_golden(name, monkeypatch):
    import ast
    g = np.load(os.path.join(HERE, "golden", name + ".npz"))
    cfg = ast.literal_eval(str(g["cfg_json"]))
    model = _build(cfg, int(g["giant_depth"]), monkeypatch).cuda().eval()
    from vit_det_init import golden_inputs
    x, q = golden_inputs(int(g["q_shape"][1]), int(g["q_shape"][2]))
    n = _count_swiglu(monkeypatch)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        tok = model.encoder(x.cuda()).float().cpu().numpy()
        h = model.encode(x.cuda()).float().cpu().numpy()
        dec = model.decode(q.cuda()).float().cpu().numpy()
    if "giant" in name:
        assert n["swiglu"] > 0
    st = int(g["token_stride"])
    for got, want in ((tok[:, ::st], g["tok_sub"]), (h.reshape(h.shape[0], h.shape[1], -1)[:, :, ::4], g["h_sub"]),
                      (dec[:, :, ::4, ::4], g["dec_sub"])):
        err = np.abs(got - want)
        assert err.max() < 0.15 and err.mean() < 0.02, (err.max(), err.mean())


def _enc_dec_loss(model, x, q, r1, r2):
    return (model.encoder(x).float() * r1).sum() + (model.decode(q).float() * r2).sum()


@pytest.mark.parametrize("dtn", list(DTYPES))
def test_giant_parameter_gradients_against_fp64(dtn, monkeypatch):
    """every parameter gradient of the giant encoder + decoder (depth cut to 2, DropPath off) on the fused ViT path (SwiGLU
    MLP: library GEMMs + the stand-alone kernel) against the same modules run in fp64 (module path, no kernels of this
    library); fp16 through GradScaler"""
    dt = DTYPES[dtn][0]
    model = _build(_giant_cfg(), 2, monkeypatch).cuda().train()
    for m in model.modules():
        if hasattr(m, "drop_prob"):
            m.drop_prob = 0.0
    ref = _build(_giant_cfg(), 2, monkeypatch).cuda().double().train()
    ref.load_state_dict(model.state_dict())
    for m in ref.modules():
        if hasattr(m, "drop_prob"):
            m.drop_prob = 0.0
    gen = torch.Generator(device="cuda").manual_seed(3)
    x = torch.rand(2, 3, 256, 256, device="cuda", generator=gen) * 2 - 1
    q = torch.randn(2, 32, 16, 16, device="cuda", generator=gen)
    r1 = torch.randn(2, 256, 1536, device="cuda", generator=gen) / 256
    r2 = torch.randn(2, 3, 256, 256, device="cuda", generator=gen) / 256
    n = _count_swiglu(monkeypatch)
    scaler = torch.amp.GradScaler("cuda", init_scale=1024.0, enabled=dt == torch.float16)
    with torch.autocast("cuda", dtype=dt):
        loss = _enc_dec_loss(model, x, q, r1, r2)
    scaler.scale(loss).backward()
    inv = 1.0 / scaler.get_scale() if dt == torch.float16 else 1.0
    assert n["swiglu"] == 4                                # the two blocks of the encoder and of the decoder
    loss64 = _enc_dec_loss(ref, x.double(), q.double(), r1.double(), r2.double())
    loss64.backward()
    ref_grads = dict(ref.named_parameters())
    checked = 0
    for name, p in model.named_parameters():
        g64 = ref_grads[name].grad
        if g64 is None or not (name.startswith("encoder.") or name.startswith("decoder.") or name.startswith("quant_conv")
                                or name.startswith("post_quant_conv")):
            continue
        assert p.grad is not None, name
        gg = p.grad.double() * inv
        assert bool(torch.isfinite(gg).all()), name
        rel = float((gg - g64).norm() / g64.norm().clamp_min(1e-30))
        assert rel < 5e-2, (name, rel)
        checked += 1
    assert checked > 40


def test_full_depth_giant_fused_matches_library_path(monkeypatch):
    """the 40-block giant encoder + decoder at batch 2, forward and backward under bf16 autocast on the fused ViT path (SwiGLU
    MLP: library GEMMs + the stand-alone kernel): the tokens, the image and the picked gradients are finite"""
    model = _build(_giant_cfg(), 40, monkeypatch, det=False).cuda().train()
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith(".gamma"):
                p.fill_(0.1)
    for m in model.modules():
        if hasattr(m, "drop_prob"):
            m.drop_prob = 0.0
    gen = torch.Generator(device="cuda").manual_seed(4)
    x = torch.rand(2, 3, 256, 256, device="cuda", generator=gen) * 2 - 1
    q = torch.randn(2, 32, 16, 16, device="cuda", generator=gen)
    r1 = torch.randn(2, 256, 1536, device="cuda", generator=gen) / 256
    r2 = torch.randn(2, 3, 256, 256, device="cuda", generator=gen) / 256
    picks = ["encoder.model.blocks.0.mlp.fc1.weight", "encoder.model.blocks.39.mlp.fc2.weight",
             "decoder.model.blocks.20.mlp.fc1.bias", "decoder.model.blocks.0.attn.qkv.weight"]
    n = _count_swiglu(monkeypatch)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        tok = model.encoder(x).float()
        dec = model.decode(q).float()
        loss = (tok * r1).sum() + (dec * r2).sum()
    loss.backward()
    assert n["swiglu"] == 2 * 40
    params = dict(model.named_parameters())
    for a, what in [(tok, "tokens"), (dec, "image")] + [(params[k].grad, k) for k in picks]:
        assert bool(torch.isfinite(a).all()), what


def test_reg4_model_training_step(monkeypatch):
    cfg = dict(_giant_cfg(abs_pos_embed=False), encoder_model=REG4, decoder_model=REG4)
    model = _build(cfg, 2, monkeypatch).cuda().train()
    assert model.encoder.num_prefix_tokens == 5
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4)
    gen = torch.Generator(device="cuda").manual_seed(6)
    x = torch.rand(2, 3, 256, 256, device="cuda", generator=gen) * 2 - 1
    before = {k: v.detach().clone() for k, v in model.named_parameters()}
    with torch.autocast("cuda", dtype=torch.bfloat16):
        dec = model.decode(model.encode(x))
        loss = (dec.float() - x).square().mean()
    loss.backward()
    assert model.encoder.model.reg_token.grad is not None and bool(torch.isfinite(model.encoder.model.reg_token.grad).all())
    for name, p in model.named_parameters():
        if p.grad is not None:
            assert bool(torch.isfinite(p.grad).all()), name
    opt.step()
    assert not torch.equal(before["encoder.model.reg_token"], model.encoder.model.reg_token)


def test_lora_giant_takes_library_path_and_matches(monkeypatch):
    model = _build(_giant_cfg(), 2, monkeypatch).cuda().eval()
    torch.manual_seed(7)
    model.encoder.finetine("lora", {"r": 8})
    for name, p in model.encoder.named_parameters():
        if "lora_B" in name:
            with torch.no_grad():
                p.normal_(0, 0.02)                      # nonzero adapters: the LoRA term contributes
    gen = torch.Generator(device="cuda").manual_seed(8)
    x = torch.rand(2, 3, 256, 256, device="cuda", generator=gen) * 2 - 1
    n = _count_swiglu(monkeypatch)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        tok = model.encoder(x).float()
    assert n["swiglu"] == 2
    with torch.no_grad():
        ref = model.encoder.double()(x.double())
    rel = float((tok.double() - ref).norm() / ref.norm())
    assert rel < 3e-2, rel
