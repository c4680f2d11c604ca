"""The frozen guide teachers on the sm_90a kernels: the inference form of the fused fc1 GEMMs (`pre` = NULL), the
class-token attention xq_vit_attn_fwd_cls, VisionTransformer.forward / forward_features on the frozen fused path
(vit_ops.frozen_forward) against an fp64 module path, its routing, and the VQModel losses that read the teachers.

Teacher bound: the fused frozen path's largest error against the float64 module path (run on the GPU) must be at most
twice the largest error of the library module path under the same autocast."""
import copy
import math
import warnings

import pytest
import torch

pytestmark = pytest.mark.gpu

XQ_ERR_ARG, XQ_ERR_UNSUPPORTED = -1, -4
GUARD = 128
DTYPES = [torch.bfloat16, torch.float16]


def _lib():
    from imagefolder_b200 import _capi
    return _capi, _capi.lib()


def _fn(L, name, dt):
    return getattr(L, name + ("_f16" if dt == torch.float16 else ""))


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ---------------------------------------------------------------------------------------------------------------- 1. pre = NULL
def _grid(rows, cols, scale, gen, dt):
    """entries in {-1, 0, 1} * scale (exact in both 16-bit types; every partial sum of a product is exact in fp32)"""
    return (torch.randint(-1, 2, (rows, cols), device="cuda", generator=gen).float() * scale).to(dt)


def _bias(N, gen):
    b = torch.randn(N, device="cuda", generator=gen)
    kind = torch.arange(N, device="cuda") % 3
    b[kind == 0] = 40.0
    b[kind == 1] = -40.0
    return b


def _out(M, N, dt):
    """[M + GUARD, N]: rows < M NaN, the guard rows a sentinel"""
    t = torch.full((M + GUARD, N), float("nan"), dtype=dt, device="cuda")
    t[M:].view(torch.int16).fill_(-12345)
    return t


def _same_bits(a, b, what):
    bad = a.view(torch.int16) != b.view(torch.int16)
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {bad.numel()} elements differ"


MS = [128 * 257, 3 * 257, 128, 1]


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("kind", ["gelu", "lora"])
def test_fc1_without_pre_is_bit_identical(kind, M, dt):
    """act of the call with pre = NULL equals act of the call with pre given, bit for bit, and neither writes past row M"""
    C, L = _lib()
    gen = torch.Generator(device="cuda").manual_seed(M + len(kind))
    K, N, R = 768, 3072, 8 if kind == "lora" else 0
    x = _grid(M + GUARD, K, 0.125, gen, dt)           # extra rows after M: a read past M would show in no output
    w = _grid(N, K, 0.25, gen, dt)
    b = _bias(N, gen)
    u = _grid(M + GUARD, R, 0.125, gen, dt) if R else None
    bl = _grid(N, R, 0.25, gen, dt) if R else None
    acts = []
    for with_pre in (True, False):
        pre = _out(M, N, dt) if with_pre else None
        act = _out(M, N, dt)
        p = pre.data_ptr() if with_pre else None
        if kind == "gelu":
            rc = _fn(L, "xq_vit_fc1_gelu_fwd", dt)(x.data_ptr(), w.data_ptr(), b.data_ptr(), p, act.data_ptr(), M, N, K, _stream())
        else:
            rc = _fn(L, "xq_vit_fc1_lora_gelu_fwd", dt)(x.data_ptr(), w.data_ptr(), u.data_ptr(), bl.data_ptr(), b.data_ptr(),
                                                        p, act.data_ptr(), M, N, K, R, _stream())
        assert rc == 0, C.lib().xq_strerror(rc)
        torch.cuda.synchronize()
        assert not bool(act[:M].isnan().any()), "an act tile was skipped"
        assert bool((act[M:].view(torch.int16) == -12345).all()), "act written past row M"
        if with_pre:
            assert not bool(pre[:M].isnan().any()) and bool((pre[M:].view(torch.int16) == -12345).all())
        acts.append(act)
    _same_bits(acts[0], acts[1], f"{kind} M={M}")


@pytest.mark.parametrize("dt", DTYPES)
def test_fc1_null_operands_still_refused(dt):
    C, L = _lib()
    M, N, K = 128, 256, 64
    t = torch.zeros(M * max(N, K) + 64, dtype=dt, device="cuda")
    b = torch.zeros(N, device="cuda")
    a = t.data_ptr()
    f = _fn(L, "xq_vit_fc1_gelu_fwd", dt)
    for args in [(None, a, b.data_ptr(), None, a), (a, None, b.data_ptr(), None, a), (a, a, None, None, a),
                 (a, a, b.data_ptr(), None, None)]:
        assert f(*args, M, N, K, _stream()) == XQ_ERR_ARG
    assert f(a, a, b.data_ptr(), a + 2, a, M, N, K, _stream()) == XQ_ERR_ARG          # a misaligned pre is still refused
    g = _fn(L, "xq_vit_fc2_dgelu_bwd", dt)
    assert g(a, a, None, b.data_ptr(), a, b.data_ptr(), M, N, K, _stream()) == XQ_ERR_ARG  # the backward needs pre


# ---------------------------------------------------------------------------------------------------------------- 2. class attention
CLS_SHAPES = [(128, 257, 12), (3, 257, 6), (2, 261, 16), (1, 1, 1), (2, 2, 12), (2, 129, 24), (2, 513, 12), (1, 1029, 2)]


def _ulp16(x, dt):
    """spacing of the 16-bit type at |x| (subnormal floor included)"""
    mant, emin = (7, -126) if dt == torch.bfloat16 else (10, -14)
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** emin))).clamp_min(emin)
    return torch.exp2(e - mant)


def _cls_ref(qkv, H):
    B, N, _ = qkv.shape
    q5 = qkv.double().view(B, N, 3, H, 64)
    q, k, v = q5[:, 0, 0], q5[:, :, 1], q5[:, :, 2]                    # [B,H,64], [B,N,H,64]
    s = torch.einsum("bhd,bnhd->bhn", q, k) * 0.125
    p = torch.softmax(s, dim=-1)
    return torch.einsum("bhn,bnhd->bhd", p, v), v.abs().amax(dim=(1, 3))   # [B,H,64], max|v| per (b,h)


def _cls_inputs(B, N, H, dt, mode, gen):
    qkv = torch.randn(B, N, 3, H, 64, device="cuda", generator=gen)
    if mode == "onehot":
        # q = k_last scaled: score of the last key exceeds every other by >= ~100 in the exponent
        qkv[:, :, 1] *= 0.05
        qkv[:, -1, 1] = torch.randn(B, H, 64, device="cuda", generator=gen).sign() * 2.0
        qkv[:, 0, 0] = qkv[:, -1, 1] * 2.0
    elif mode == "tie":
        qkv[:, :, 1] = qkv[:, :1, 1]                                      # every key equal: uniform softmax
    return qkv.reshape(B, N, 3 * H * 64).to(dt).contiguous()


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("shape", CLS_SHAPES)
def test_attn_cls_against_fp64(shape, dt):
    C, L = _lib()
    B, N, H = shape
    f = _fn(L, "xq_vit_attn_fwd_cls", dt)
    gen = torch.Generator(device="cuda").manual_seed(B * 7919 + N * 31 + H)
    for mode in ("random", "onehot", "tie"):
        qkv = _cls_inputs(B, N, H, dt, mode, gen)
        outs = []
        for _ in range(2):
            out = torch.full((B, H * 64), float("nan"), dtype=dt, device="cuda")
            assert f(qkv.data_ptr(), out.data_ptr(), B, N, H, 64, 0.125, _stream()) == 0
            outs.append(out)
        torch.cuda.synchronize()
        _same_bits(outs[0], outs[1], f"{mode}: two calls")
        ref, vmax = _cls_ref(qkv, H)
        got = outs[0].view(B, H, 64).double()
        assert not bool(got.isnan().any()), f"{mode}: unwritten output"
        bound = 0.5 * _ulp16(ref, dt) + 1e-5 * vmax[..., None]
        err = (got - ref).abs()
        assert bool((err <= bound).all()), f"{mode}: max excess {float((err - bound).max()):.3e}"
        if mode == "onehot" and N > 1:
            _same_bits(outs[0].view(B, H, 64), qkv.view(B, N, 3, H, 64)[:, -1, 2], "one-hot: the last key's v")


@pytest.mark.parametrize("dt", DTYPES)
def test_attn_cls_refusals_write_nothing(dt):
    C, L = _lib()
    f = _fn(L, "xq_vit_attn_fwd_cls", dt)
    B, N, H = 2, 9, 3
    qkv = torch.randn(B, N, 3 * H * 64, device="cuda").to(dt)
    out = torch.full((B, H * 64), float("nan"), dtype=dt, device="cuda")
    q, o, s = qkv.data_ptr(), out.data_ptr(), _stream()
    assert f(None, o, B, N, H, 64, 0.125, s) == XQ_ERR_ARG
    assert f(q, None, B, N, H, 64, 0.125, s) == XQ_ERR_ARG
    assert f(q + 2, o, B, N, H, 64, 0.125, s) == XQ_ERR_ARG
    assert f(q, o + 2, B, N, H, 64, 0.125, s) == XQ_ERR_ARG
    for b_, n_, h_ in [(0, N, H), (B, 0, H), (B, N, 0), (-1, N, H)]:
        assert f(q, o, b_, n_, h_, 64, 0.125, s) == XQ_ERR_ARG
    assert f(q, o, B, N, H, 32, 0.125, s) == XQ_ERR_UNSUPPORTED
    assert f(q, o, 1, 8193, 1, 64, 0.125, s) == XQ_ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert bool(out.isnan().all()), "a refused call wrote its output"


# ---------------------------------------------------------------------------------------------------------------- 3. teachers
def _teacher(name, depth=None, seed=0):
    from imagefolder_b200.dino_enc.vision_transformer import create_model
    torch.manual_seed(seed)
    kw = dict(img_size=256, patch_size=16, drop_path_rate=0.0)
    if depth is not None:
        kw["depth"] = depth
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = create_model(name, pretrained=False, **kw)
    g = torch.Generator().manual_seed(seed + 1)
    for mod in m.modules():
        if hasattr(mod, "gamma"):                        # LayerScale of order 0.1 - 1: every block matters
            with torch.no_grad():
                mod.gamma.copy_(torch.rand(mod.gamma.shape, generator=g) * 0.9 + 0.1)
        if isinstance(mod, torch.nn.LayerNorm):
            with torch.no_grad():
                mod.weight.copy_(1 + 0.2 * torch.randn(mod.weight.shape, generator=g))
                mod.bias.copy_(0.1 * torch.randn(mod.bias.shape, generator=g))
    m.eval()
    for p in m.parameters():
        p.requires_grad = False
    return m.cuda()


class _Module:
    """the module path for calls inside the block (the routing test answers no)"""

    def __enter__(self):
        from imagefolder_b200.dino_enc import vision_transformer as vt
        self.vt, self.saved = vt, vt.frozen_path_ok
        vt.frozen_path_ok = lambda vit, x: False

    def __exit__(self, *exc):
        self.vt.frozen_path_ok = self.saved


def _run(m, x, call, dt):
    with torch.no_grad(), torch.autocast("cuda", dtype=dt):
        return (m(x) if call == "forward" else m.forward_features(x)).float()


def _ref64(m, x, call):
    m64 = copy.deepcopy(m).double()
    with torch.no_grad():
        r = m64(x.double()) if call == "forward" else m64.forward_features(x.double())
    del m64
    return r


def _frozen_calls():
    from imagefolder_b200 import vit_ops
    n = [0]
    saved = vit_ops.frozen_forward

    def counting(*a, **k):
        n[0] += 1
        return saved(*a, **k)
    return n, saved, counting


TEACHERS = [("vit_base_patch14_dinov2.lvd142m", None, 128, "forward"),
            ("vit_base_patch14_dinov2.lvd142m", None, 128, "forward_features"),
            ("vit_base_patch16_clip_224.openai", None, 128, "forward_features"),
            ("vit_small_patch14_reg4_dinov2.lvd142m", None, 3, "forward"),
            ("vit_small_patch14_reg4_dinov2.lvd142m", None, 3, "forward_features"),
            ("vit_large_patch14_dinov2.lvd142m", None, 2, "forward"),
            ("vit_large_patch14_dinov2.lvd142m", None, 2, "forward_features"),
            ("vit_giant_patch14_dinov2.lvd142m", 2, 2, "forward"),
            ("vit_giant_patch14_dinov2.lvd142m", 2, 2, "forward_features")]


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("name,depth,B,call", TEACHERS)
def test_teacher_against_fp64(name, depth, B, call, dt, monkeypatch):
    from imagefolder_b200.dino_enc import vision_transformer as vt
    m = _teacher(name, depth)
    x = torch.rand(B, 3, 256, 256, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3)) * 2 - 1
    ref = _ref64(m, x, call)
    n, _, counting = _frozen_calls()
    monkeypatch.setattr(vt, "frozen_forward", counting)
    fused = _run(m, x, call, dt)
    assert n[0] == 1, "the frozen fused path was not taken"
    with _Module():
        module = _run(m, x, call, dt)
    assert n[0] == 1
    assert fused.shape == module.shape == ref.shape
    e_mod = float((module.double() - ref).abs().max())
    e_fus = float((fused.double() - ref).abs().max())
    assert e_fus <= 2 * e_mod, f"fused error {e_fus:.3e} > 2 x module error {e_mod:.3e}"
    if call == "forward":
        # the class tail against row 0 of the full fused forward_features, within the same bound
        ff = _run(m, x, "forward_features", dt)[:, 0]
        assert float((fused - ff).abs().max()) <= 2 * e_mod
        assert float((ff.double() - ref).abs().max()) <= 2 * e_mod


# ---------------------------------------------------------------------------------------------------------------- 4. routing
def test_routing_conditions(monkeypatch):
    from imagefolder_b200.dino_enc import vision_transformer as vt
    m = _teacher("vit_small_patch14_dinov2.lvd142m")
    x = torch.rand(2, 3, 256, 256, device="cuda") * 2 - 1
    n, _, counting = _frozen_calls()
    monkeypatch.setattr(vt, "frozen_forward", counting)
    with torch.no_grad():
        m(x)                                              # fp32, no autocast: module path
        assert n[0] == 0
        with torch.autocast("cuda", dtype=torch.bfloat16):
            m(x)
            assert n[0] == 1
            m.forward_features(x)
            assert n[0] == 2
    with torch.autocast("cuda", dtype=torch.bfloat16):
        m(x.clone().requires_grad_(True))                 # the image needs a gradient: module path
        assert n[0] == 2
    # one unfrozen parameter: the module path runs and its gradient is filled
    m.blocks[0].mlp.fc1.weight.requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        (m(x).float() * torch.randn(2, 384, device="cuda")).sum().backward()
    assert n[0] == 2
    g = m.blocks[0].mlp.fc1.weight.grad
    assert g is not None and bool(g.abs().sum() > 0)


def test_frozen_path_peak_memory_not_above_module_path():
    m = _teacher("vit_base_patch14_dinov2.lvd142m")
    x = torch.rand(128, 3, 256, 256, device="cuda") * 2 - 1

    def peak(fn):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = fn()
        torch.cuda.synchronize()
        r = torch.cuda.max_memory_allocated() - base
        del out
        return r
    for call in ("forward", "forward_features"):
        fn = (lambda: _run(m, x, call, torch.bfloat16))
        fn()
        with _Module():
            fn()
            p_mod = peak(fn)
        p_fus = peak(fn)
        assert p_fus <= p_mod, f"{call}: fused peak {p_fus / 2**20:.0f} MB > module {p_mod / 2**20:.0f} MB"


# ---------------------------------------------------------------------------------------------------------------- 5. model level
def _model(name, **over):
    from imagefolder_b200 import config as xcfg
    c = dict(xcfg.SHIPPED_CONFIGS[name])
    # a ViT-B encoder: quant_conv reads the 768-wide teacher features (xqgan_model.py reshapes them to 768 channels)
    c.update(encoder_model="vit_base_patch14_dinov2.lvd142m", decoder_model="vit_small_patch14_dinov2.lvd142m",
             semantic_guide="dinov2")
    c.update(over)
    a = xcfg.parse_args([])
    for k, v in c.items():
        setattr(a, k, v)
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model = xcfg.build_vq_model(a).cuda()
    g = torch.Generator().manual_seed(9)
    for t in ("semantic_model", "detail_model"):
        te = getattr(model, t, None)
        if te is None:
            continue
        for mod in te.modules():
            if hasattr(mod, "gamma"):
                with torch.no_grad():
                    mod.gamma.copy_(torch.rand(mod.gamma.shape, generator=g) * 0.9 + 0.1)
    return model, a


class _Teachers64:
    """the teachers' forward / forward_features replaced by a float64 copy on the module path (the fp64 reference)"""

    def __init__(self, model):
        self.model, self.saved = model, []

    def __enter__(self):
        for t in ("semantic_model", "detail_model"):
            te = getattr(self.model, t, None)
            if te is None:
                continue
            t64 = copy.deepcopy(te).double()

            def fwd(x, t64=t64):
                with torch.autocast("cuda", enabled=False):
                    return t64(x.double()).float()

            def ff(x, t64=t64):
                with torch.autocast("cuda", enabled=False):
                    return t64.forward_features(x.double()).float()
            self.saved.append((te, te.__dict__.get("forward"), te.__dict__.get("forward_features")))
            te.forward, te.forward_features = fwd, ff

    def __exit__(self, *exc):
        for te, f, ff in self.saved:
            del te.forward, te.forward_features


@pytest.mark.parametrize("name,over", [("VQ-8192", {}), ("MSBR10P2-16384", dict(detail_guide="clip", guide_type_2="patch"))])
def test_model_losses_and_quant_conv_grads(name, over):
    model, a = _model(name, **over)
    model.train()
    model.encoder.eval(), model.decoder.eval()
    x = torch.rand(4, 3, 256, 256, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2)) * 2 - 1

    def run():
        torch.manual_seed(5)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            dec, (vq, commit, ent, _), sem, det, dep = model(x, 0, 0.0, 0.0, 100)
        losses = [t for t in (sem, det) if t is not None]
        g = torch.autograd.grad(sum(losses), [model.quant_conv.weight, model.quant_conv.bias])
        return [float(t) for t in losses], [t.detach().double() for t in g], dec

    fused = run()
    with _Module():
        module = run()
    with _Module(), _Teachers64(model):
        ref = run()
    assert len(fused[0]) == (2 if "detail_guide" in over else 1)
    for f, m_, r in zip(fused[0], module[0], ref[0]):
        floor = 1e-6 * abs(r)
        assert abs(f - r) <= 2 * abs(m_ - r) + floor, (f, m_, r)
    for f, m_, r in zip(fused[1], module[1], ref[1]):
        floor = 1e-5 * float(r.abs().max())
        assert float((f - r).abs().max()) <= 2 * float((m_ - r).abs().max()) + floor
    # the whole backward runs with the fused teachers in the graph
    model.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        dec, (vq, commit, ent, _), sem, det, dep = model(x, 0, 0.0, 0.0, 100)
        loss = (dec.float() - x).pow(2).mean() + vq + commit + ent + sem + (det if det is not None else 0.0)
    loss.backward()
    assert model.quant_conv.weight.grad is not None and bool(torch.isfinite(model.quant_conv.weight.grad).all())
    assert all(p.grad is None for p in model.semantic_model.parameters())
    assert not math.isnan(float(loss))
