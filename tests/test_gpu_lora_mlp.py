"""LoRA on the fused MLP GEMMs: xq_vit_fc1_lora_gelu_fwd / xq_vit_fc2_lora_dgelu_bwd (csrc/gemm_kernel.cu), the LoRA MLP autograd
node (vit_ops._LoRAMLP), the LoRA-wrapped DINOv2 encoder / decoder on the fused path, and their EMA copy.

The entry points are checked bit for bit against the plain entry points run on the operands concatenated along K ([x | u | 0],
[w | b_lora | 0], K + 64 columns): on the exact grid of tests/test_gpu_mlp_gemm.py (A entries {-1, 0, 1} * 2^-3, B entries
{-1, 0, 1} * 2^-2, K + 64 <= 1024) every partial sum is exact in fp32, so both must give the same bits whatever the order.
Outputs start NaN-filled and are followed by sentinel rows; the inputs carry nonzero rows past M.
"""
import copy
import math

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu

GUARD = 128
SENTINEL = -12345
EPS = 2.0 ** -8                # one bf16 rounding, relative (generous: round-to-nearest gives 2^-9)


def _lib():
    from imagefolder_b200 import _capi
    return _capi, _capi.lib()


def _grid(rows, cols, scale, gen):
    return torch.randint(-1, 2, (rows, cols), device="cuda", generator=gen).to(torch.bfloat16) * scale


def _guarded(M, N):
    t = torch.full((M + GUARD, N), float("nan"), dtype=torch.bfloat16, device="cuda")
    t[M:].view(torch.int16).fill_(SENTINEL)
    return t


def _assert_guard(t, M, what):
    assert bool((t[M:].view(torch.int16) == SENTINEL).all()), f"{what}: guard rows after row {M} overwritten"


def _cat_k(a, b, K):
    """[a | b | 0] with K + 64 columns"""
    out = torch.zeros(a.shape[0], K + 64, dtype=torch.bfloat16, device="cuda")
    out[:, :K], out[:, K:K + b.shape[1]] = a, b
    return out


def _fwd(x, w, b, M, N, K, u=None, bl=None, R=0):
    _capi, L = _lib()
    p, s = _capi.ptr, _capi.stream_ptr(x.device)
    pre, act = _guarded(M, N), _guarded(M, N)
    if R:
        _capi.check(L.xq_vit_fc1_lora_gelu_fwd(p(x), p(w), p(u), p(bl), p(b), p(pre), p(act), M, N, K, R, s), "lora fwd")
    else:
        _capi.check(L.xq_vit_fc1_gelu_fwd(p(x), p(w), p(b), p(pre), p(act), M, N, K, s), "fwd")
    return pre, act


def _bwd(d_out, w2t, pre, b, M, N, K, v=None, a2t=None, R=0):
    _capi, L = _lib()
    p, s = _capi.ptr, _capi.stream_ptr(d_out.device)
    d_pre, d_bias = _guarded(M, N), torch.full((N,), float("nan"), device="cuda")
    if R:
        _capi.check(L.xq_vit_fc2_lora_dgelu_bwd(p(d_out), p(w2t), p(v), p(a2t), p(pre), p(b), p(d_pre), p(d_bias), M, N, K, R, s),
                    "lora bwd")
    else:
        _capi.check(L.xq_vit_fc2_dgelu_bwd(p(d_out), p(w2t), p(pre), p(b), p(d_pre), p(d_bias), M, N, K, s), "bwd")
    return d_pre, d_bias


def _assert_dbias(a, b, d_pre, M, what):
    """equal up to the order of the fp32 atomic adds: within 2^-20 of the column sums of |d_pre|"""
    tol = d_pre[:M].float().abs().sum(0) * 2.0 ** -20 + 1e-30
    assert bool(((a - b).abs() <= tol).all()), f"{what}: max diff {float((a - b).abs().max()):.3e}"


@pytest.mark.parametrize("M", [128 * 513, 3 * 513, 513])
@pytest.mark.parametrize("R", [8, 16, 64])
def test_lora_entry_points_equal_plain_kernel_on_k_concatenated_operands(M, R):
    N, K = 3072, 768
    gen = torch.Generator(device="cuda").manual_seed(1000 * R + M % 1000)
    x, u = _grid(M + GUARD, K, 2.0 ** -3, gen), _grid(M + GUARD, R, 2.0 ** -3, gen)
    w1, b1l = _grid(N, K, 2.0 ** -2, gen), _grid(N, R, 2.0 ** -2, gen)
    b1 = torch.randn(N, device="cuda", generator=gen)
    pre, act = _fwd(x, w1, b1, M, N, K, u, b1l, R)
    pre_c, act_c = _fwd(_cat_k(x, u, K), _cat_k(w1, b1l, K), b1, M, N, K + 64)
    for t, what in ((pre, "pre"), (act, "act")):
        _assert_guard(t, M, what)
    assert torch.equal(pre[:M], pre_c[:M]) and torch.equal(act[:M], act_c[:M])
    # backward on the forward's own `pre`
    d_out, v = _grid(M + GUARD, K, 2.0 ** -3, gen), _grid(M + GUARD, R, 2.0 ** -3, gen)
    w2t, a2t = _grid(N, K, 2.0 ** -2, gen), _grid(N, R, 2.0 ** -2, gen)
    d_pre, d_bias = _bwd(d_out, w2t, pre, b1, M, N, K, v, a2t, R)
    d_pre_c, d_bias_c = _bwd(_cat_k(d_out, v, K), _cat_k(w2t, a2t, K), pre, b1, M, N, K + 64)
    _assert_guard(d_pre, M, "d_pre")
    assert torch.equal(d_pre[:M], d_pre_c[:M])
    _assert_dbias(d_bias, d_bias_c, d_pre, M, "d_bias")


def test_zero_adapter_equals_plain_entry_points():
    M, N, K, R = 3 * 513, 3072, 768, 8
    torch.manual_seed(3)
    x = torch.randn(M + GUARD, K, device="cuda").to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda") * 0.03).to(torch.bfloat16)
    u = torch.randn(M + GUARD, R, device="cuda").to(torch.bfloat16)
    zero = torch.zeros(N, R, dtype=torch.bfloat16, device="cuda")
    b = torch.randn(N, device="cuda")
    pre, act = _fwd(x, w, b, M, N, K, u, zero, R)
    pre0, act0 = _fwd(x, w, b, M, N, K)
    assert torch.equal(pre[:M], pre0[:M]) and torch.equal(act[:M], act0[:M])
    d_pre, d_bias = _bwd(x, w, pre, b, M, N, K, u, zero, R)
    d_pre0, d_bias0 = _bwd(x, w, pre, b, M, N, K)
    assert torch.equal(d_pre[:M], d_pre0[:M])
    _assert_dbias(d_bias, d_bias0, d_pre, M, "d_bias")


def test_refused_lora_calls_write_nothing():
    _capi, L = _lib()
    M, N, K = 256, 256, 128
    x = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    w = torch.randn(N, K, device="cuda").to(torch.bfloat16)
    u = torch.zeros(M, 72, dtype=torch.bfloat16, device="cuda")
    bl = torch.zeros(N, 72, dtype=torch.bfloat16, device="cuda")
    b = torch.zeros(N, device="cuda")
    p, s = _capi.ptr, _capi.stream_ptr(x.device)
    pre, act = _guarded(M, N), _guarded(M, N)
    d_bias = torch.full((N,), 7.0, device="cuda")
    before = [t.clone() for t in (pre, act, d_bias)]
    for R, up in ((4, p(u)), (72, p(u)), (8, p(u) + 8), (8, None)):
        assert L.xq_vit_fc1_lora_gelu_fwd(p(x), p(w), up, p(bl), p(b), p(pre), p(act), M, N, K, R, s) == -1
        assert L.xq_vit_fc2_lora_dgelu_bwd(p(x), p(w), up, p(bl), p(pre), p(b), p(act), p(d_bias), M, N, K, R, s) == -1
    torch.cuda.synchronize()
    for t, t0 in zip((pre, act, d_bias), before):
        assert torch.equal(t.view(torch.int16) if t.dtype == torch.bfloat16 else t,
                           t0.view(torch.int16) if t0.dtype == torch.bfloat16 else t0)


# ---- the autograd node ---------------------------------------------------------------------------------------------------
class _Mlp(nn.Module):
    def __init__(self, fc1, fc2):
        super().__init__()
        self.fc1, self.fc2 = fc1, fc2


def _lora_mlp(D, H, r, alpha, seed):
    from imagefolder_b200.dino_enc import lora
    torch.manual_seed(seed)
    fc1, fc2 = nn.Linear(D, H), nn.Linear(H, D)
    for fc in (fc1, fc2):
        nn.init.normal_(fc.weight, std=0.02)
        nn.init.normal_(fc.bias, std=0.5)
    m = _Mlp(lora.Linear(fc1, r, alpha, 0.0), lora.Linear(fc2, r, alpha, 0.0))
    for fc in (m.fc1, m.fc2):
        fc.base_layer.requires_grad_(False)                    # what LoRA wrapping leaves frozen
        nn.init.normal_(fc.lora_B["default"].weight, std=0.2)
    return m.cuda()


def _mm_outputs(fn):
    """output shapes of every aten::mm / aten::addmm that `fn` runs (forward and autograd backward)"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU], record_shapes=True) as prof:
        fn()
    out = []
    for e in prof.events():
        sh = e.input_shapes
        if e.name == "aten::mm":
            out.append((sh[0][0], sh[1][1]))
        elif e.name == "aten::addmm":
            out.append((sh[1][0], sh[2][1]))
    return out


def _gelu64(t):
    return 0.5 * t * (1.0 + torch.erf(t / math.sqrt(2.0)))


def _dgelu64(t):
    return 0.5 * (1.0 + torch.erf(t / math.sqrt(2.0))) + t * torch.exp(-0.5 * t * t) / math.sqrt(2.0 * math.pi)


def _assert_bound(got, ref, q, what, c=8.0):
    """|got - ref| <= c 2^-8 (|ref| + q) elementwise.  q is the root-sum-square of the terms of the output's last contraction,
    taken over the error scales of its operands (each operand's own value plus what its upstream roundings can move it):
    bf16 rounding errors of independent terms add like random variables, so c = 8 (16 unit roundoffs) is a wide margin
    that a missing or wrongly scaled adapter term still exceeds."""
    err = (got.double() - ref).abs()
    lim = c * EPS * (ref.abs() + q) + 1e-30
    bad = err > lim
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {bad.numel()} beyond the bound, worst ratio {float((err / lim).max()):.2f}"
    return lim


def _rss(a, b):
    """sqrt(a^2 @ b^2): root-sum-square magnitude of the terms of a @ b"""
    return ((a * a) @ (b * b)).sqrt()


@pytest.mark.parametrize("M,r,alpha", [(128 * 513, 8, 16), (3 * 513, 12, 8)])
def test_lora_mlp_node_matches_fp64_peft_formula(M, r, alpha):
    from imagefolder_b200 import _capi, vit_ops
    D, H = 768, 3072
    m = _lora_mlp(D, H, r, alpha, seed=M + r)
    s = alpha / r
    torch.manual_seed(7)
    y = torch.randn(M, D, device="cuda").to(torch.bfloat16).requires_grad_(True)
    g = torch.randn(M, D, device="cuda").to(torch.bfloat16)
    calls = []
    real_call = _capi.call

    def spy(name, *a, **k):
        calls.append(name)
        return real_call(name, *a, **k)

    _capi.call = spy
    try:
        branch = vit_ops.mlp_forward(m, y)
        assert type(branch.grad_fn).__name__ == "_LoRAMLPBackward"
        branch.backward(g)
    finally:
        _capi.call = real_call
    assert calls == ["xq_vit_fc1_lora_gelu_fwd", "xq_vit_fc2_lora_dgelu_bwd"]
    assert m.fc1.weight.grad is None and m.fc2.weight.grad is None and m.fc1.bias.grad is None

    # fp64 of the peft formula on the bf16 operands the node uses (autocast casts the parameters to bf16)
    d = lambda t: t.detach().to(torch.bfloat16).double()
    W1, b1, W2 = d(m.fc1.weight), m.fc1.bias.detach().double(), d(m.fc2.weight)
    A1, B1 = d(m.fc1.lora_A["default"].weight), d(m.fc1.lora_B["default"].weight)
    A2, B2 = d(m.fc2.lora_A["default"].weight), d(m.fc2.lora_B["default"].weight)
    Y, G = y.detach().double(), g.double()
    u = s * Y @ A1.t()
    pre = Y @ W1.t() + u @ B1.t()
    act = _gelu64(pre + b1)
    act_sc = act.abs() + 1.13 * (pre.abs() + _rss(u, B1.t()))        # act and what the roundings of u / pre move it by
    h2 = s * act @ A2.t()
    h2_sc = s * _rss(act_sc, A2.t())
    lora2 = h2 @ B2.t()
    out = act @ W2.t() + lora2
    lim = _assert_bound(branch.detach(), out, _rss(act_sc, W2.t()) + _rss(h2.abs() + h2_sc, B2.t()), "branch")
    assert bool((lora2.abs() > lim).any()), "the fc2 adapter term must exceed the bound somewhere"
    del lora2, lim
    v = s * G @ B2
    dact = G @ W2 + v @ A2
    dact_sc = dact.abs() + _rss(G, W2) + _rss(v, A2)
    dpre = dact * _dgelu64(pre + b1)
    dpre_sc = dpre.abs() + 1.13 * dact_sc + 0.8 * dact.abs() * act_sc     # |GELU'| <= 1.13, |GELU''| <= 0.8
    del dact, dact_sc
    t1 = s * dpre @ B1
    t1_sc = s * _rss(dpre_sc, B1)
    _assert_bound(y.grad, dpre @ W1 + t1 @ A1, _rss(dpre_sc, W1) + _rss(t1.abs() + t1_sc, A1), "dy")
    _assert_bound(m.fc1.lora_A["default"].weight.grad, t1.t() @ Y, _rss((t1.abs() + t1_sc).t(), Y), "d lora_A fc1")
    _assert_bound(m.fc1.lora_B["default"].weight.grad, dpre.t() @ u, _rss(dpre_sc.t(), u), "d lora_B fc1")
    _assert_bound(m.fc2.lora_A["default"].weight.grad, v.t() @ act, _rss(v.t(), act_sc), "d lora_A fc2")
    _assert_bound(m.fc2.lora_B["default"].weight.grad, G.t() @ h2, _rss(G.t(), h2.abs() + h2_sc), "d lora_B fc2")
    db1, db1_sc = dpre.sum(0), (dpre_sc * dpre_sc).sum(0).sqrt()
    del t1, t1_sc, dpre, dpre_sc

    # the fc1 bias trainable: its gradient, and still no weight-gradient GEMM while W1 / W2 are frozen
    m.fc1.bias.requires_grad_(True)
    y.grad = None
    for p in m.parameters():
        p.grad = None
    shapes = _mm_outputs(lambda: vit_ops.mlp_forward(m, y).backward(g))
    _assert_bound(m.fc1.bias.grad, db1, db1_sc, "d b1")
    assert (H, D) not in shapes and (D, H) not in shapes, shapes
    # ... and with them trainable, the two dW GEMMs are there (the check above sees the backward's GEMMs)
    m.fc1.base_layer.weight.requires_grad_(True)
    m.fc2.base_layer.weight.requires_grad_(True)
    shapes = _mm_outputs(lambda: vit_ops.mlp_forward(m, y).backward(g))
    assert (H, D) in shapes and (D, H) in shapes, shapes


# ---- the ViT-S encoder + decoder ------------------------------------------------------------------------------------------
def _lora_pair(seed):
    from imagefolder_b200.dino_enc import DINOv2Decoder, DINOv2Encoder, lora
    kw = {'img_size': 224, 'patch_size': 14, 'drop_path_rate': 0.0}
    torch.manual_seed(seed)
    enc = DINOv2Encoder(num_latent_tokens=32, model_name='vit_small_patch14_dinov2.lvd142m', model_kwargs=dict(kw),
                        pretrained=False, tuning_method='lora')
    dec = DINOv2Decoder(num_latent_tokens=32, model_name='vit_small_patch14_dinov2.lvd142m', model_kwargs=dict(kw),
                        pretrained=False, tuning_method='lora')
    for m in (enc, dec):
        for mod in m.modules():
            if isinstance(mod, lora.Linear):
                nn.init.normal_(mod.lora_B["default"].weight, std=0.2)
        for blk in m.model.blocks:                           # make the blocks' branches count (DINOv2 init: 1e-5)
            blk.ls1.gamma.data.fill_(0.5)
            blk.ls2.gamma.data.fill_(0.5)
    return enc.cuda().train(), dec.cuda().train()


def test_lora_encoder_decoder_fused_path_matches_module_path():
    from imagefolder_b200 import _capi, vit_ops
    enc, dec = _lora_pair(11)
    torch.manual_seed(12)
    x = torch.rand(4, 3, 224, 224, device="cuda") * 2 - 1

    def run(fused):
        vit_ops.MLP_TC_ENABLED[0] = fused
        calls = []
        real_call = _capi.call

        def spy(name, *a, **k):
            calls.append(name)
            return real_call(name, *a, **k)

        _capi.call = spy
        try:
            for m in (enc, dec):
                m.zero_grad(set_to_none=True)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                h = enc(x)
                img = dec(h)
            torch.manual_seed(13)
            (img.float() * torch.randn_like(img.float())).sum().backward()
        finally:
            _capi.call = real_call
            vit_ops.MLP_TC_ENABLED[0] = True
        grads = {tag + n: p.grad.float().clone() for m, tag in ((enc, "enc."), (dec, "dec.")) for n, p in m.named_parameters()
                 if p.requires_grad}
        return h.detach().float(), img.detach().float(), grads, calls

    h1, i1, g1, c1 = run(True)
    h0, i0, g0, c0 = run(False)
    assert c1.count("xq_vit_fc1_lora_gelu_fwd") == 24 and c1.count("xq_vit_fc2_lora_dgelu_bwd") == 24
    assert "xq_vit_fc1_gelu_fwd" not in c1 and not any("lora" in n for n in c0)
    assert c1.count("xq_vit_attn_fwd") == 24                  # the wrapped q_norm / k_norm keep the attention kernels
    # bf16 pipelines through 12 blocks: the same arithmetic up to where the adapter terms are rounded
    torch.testing.assert_close(h1, h0, rtol=3e-2, atol=3e-2 * float(h0.abs().max()))
    torch.testing.assert_close(i1, i0, rtol=3e-2, atol=3e-2 * float(i0.abs().max()))
    assert set(g1) == set(g0) and any(".lora_A." in k for k in g1)
    for k in g0:
        assert g1[k] is not None and torch.isfinite(g1[k]).all(), k
        scale = float(g0[k].abs().max()) + 1e-12
        err = float((g1[k] - g0[k]).abs().max())
        assert err <= 5e-2 * scale, f"{k}: max err {err:.3e} vs max |grad| {scale:.3e}"
    frozen = [n for n, p in enc.named_parameters() if ".base_layer." in n]
    assert frozen and all(dict(enc.named_parameters())[n].grad is None for n in frozen)


def test_lora_ema_copy_steps_and_round_trips():
    """the EMA copy is deep-copied before `finetune` and must get the same call; update_ema then steps it unchanged"""
    from imagefolder_b200.dino_enc import DINOv2Encoder
    from imagefolder_b200.ema import update_ema
    kw = {'img_size': 56, 'patch_size': 14, 'drop_path_rate': 0.0}
    torch.manual_seed(21)
    model = DINOv2Encoder(num_latent_tokens=4, model_name='vit_small_patch14_dinov2.lvd142m', model_kwargs=kw, pretrained=False,
                          tuning_method='full').cuda()
    ema = copy.deepcopy(model)
    model.finetine('lora')
    with pytest.raises(KeyError):
        update_ema(ema, model, decay=0)
    ema.finetine('lora')
    update_ema(ema, model, decay=0)
    for (n, e), (_, p) in zip(ema.named_parameters(), model.named_parameters()):
        assert torch.equal(e, p), n
    with torch.no_grad():
        for p in model.parameters():
            if p.requires_grad:
                p.add_(torch.randn_like(p) * 0.01)
    want = {n: e.detach().clone().mul_(0.99).add_(p.detach(), alpha=1 - 0.99)
            for (n, e), (_, p) in zip(ema.named_parameters(), model.named_parameters())}
    update_ema(ema, model, decay=0.99)
    for n, e in ema.named_parameters():
        assert torch.equal(e, want[n]), n
    fresh = DINOv2Encoder(num_latent_tokens=4, model_name='vit_small_patch14_dinov2.lvd142m', model_kwargs=kw, pretrained=False,
                          tuning_method='lora').cuda()
    fresh.load_state_dict(ema.state_dict())
    for (k, a), (_, b) in zip(ema.state_dict().items(), fresh.state_dict().items()):
        assert torch.equal(a, b), k
