"""The RoPE decoder on the GPU: xq_vit_rope_fwd / _bwd (csrc/rope_kernel.cu) against fp64, DINOv2Decoder(use_rope=True)
under bf16 / fp16 autocast against the fp32 module path, the reference's goldens and fp64 gradients, and the trainer pieces
(AdamW, clip_grad_norm_, update_ema) on its complex64 `freqs_1d`.

Bounds of the kernels against fp64 (u = 2^-8 for bf16, 2^-11 for fp16; 16-bit ulp(y) = 2u at |y|'s binade):
  * rotated q / k: half a 16-bit ulp of the exact product (one rounding) + the fp32 error of theta, sincosf and the complex
    product before it, at most 8 * 2^-24 (1 + |theta|) (|x_r| + |x_i|);
  * d(qkv): the same with g for x (the angle is the forward's);
  * the reductions (qkv bias, d freqs, d freqs_1d): fp32 sums of n terms, |err| <= n 2^-24 sum|terms| (+ the terms' own fp32
    error, far smaller), with n the number of terms in one output."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)

IMG = 256
DT = {"bf16": torch.bfloat16, "f16": torch.float16}
SUFFIX = {"bf16": "", "f16": "_f16"}
GUARD = 4096                  # NaN guard elements before and after every output


def _lib():
    from imagefolder_b200 import _capi
    return _capi


def _ulp16(y, dt):
    """the 16-bit spacing at |y| (subnormals floored at the smallest normal's spacing)"""
    mant = 7 if dt == torch.bfloat16 else 10
    tiny = 2.0 ** (-126 if dt == torch.bfloat16 else -14)
    e = torch.floor(torch.log2(y.abs().clamp_min(tiny)))
    return torch.exp2(e - mant)


def _inputs(B, N, H, P, L, dt, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = torch.randn(B, N, 3 * H * 64, generator=g, device="cuda").to(dt)
    freqs = torch.randn(2, H * 32, generator=g, device="cuda") * 0.3
    f1 = torch.randn(L, 32, 2, generator=g, device="cuda")
    return qkv, freqs, f1


def _guarded(shape, dtype):
    buf = torch.full((GUARD + int(np.prod(shape)) + GUARD,), float("nan"), dtype=dtype, device="cuda")
    return buf, buf[GUARD:GUARD + int(np.prod(shape))].view(shape)


def _cis64(freqs, f1, H, P, N):
    """c [N, H, 32] complex128: theta formed as the kernel forms it (fp32 products and sum), then exact polar"""
    L = N - P - IMG
    i = torch.arange(IMG, device="cuda")
    tx, ty = (i % 16).float()[:, None, None], (i // 16).float()[:, None, None]
    fr = freqs.view(2, 1, H, 32)
    theta = (tx * fr[0] + ty * fr[1]).double()                   # fp32 products, fp32 sum: the kernel's theta
    c = torch.ones(N, H, 32, dtype=torch.complex128, device="cuda")
    c[P:P + IMG] = torch.polar(torch.ones_like(theta), theta)
    c[P + IMG:] = torch.view_as_complex(f1.double().contiguous())[:, None, :].expand(L, H, 32)
    th = torch.zeros(N, H, 32, dtype=torch.float64, device="cuda")
    th[P:P + IMG] = theta
    return c, th


def _qk_pairs(t, B, N, H):
    """[B, N, 3*H*64] -> complex128 q / k pairs [2, B, N, H, 32]"""
    return torch.view_as_complex(t.double().view(B, N, 3, H, 32, 2)[:, :, :2].permute(2, 0, 1, 3, 4, 5).contiguous())


def _rope_fwd(qkv, freqs, f1, H, P, dtn):
    B, N, _ = qkv.shape
    buf, out = _guarded(qkv.shape, qkv.dtype)
    C = _lib()
    name = "xq_vit_rope_fwd" + SUFFIX[dtn]
    C.check(getattr(C.lib(), name)(qkv.data_ptr(), out.data_ptr(), freqs.data_ptr(), f1.data_ptr(), B, N, H, 64, P, IMG,
                                   f1.shape[0], C.stream_ptr()), name)
    torch.cuda.synchronize()
    assert torch.isnan(buf[:GUARD].float()).all() and torch.isnan(buf[-GUARD:].float()).all(), "write outside the output"
    return out


def _rope_bwd(qkv, g, freqs, f1, H, P, dtn):
    B, N, C3 = qkv.shape
    L = f1.shape[0]
    C = _lib()
    bufs = [_guarded(qkv.shape, qkv.dtype), _guarded((C3,), torch.float32), _guarded(freqs.shape, torch.float32),
            _guarded(f1.shape, torch.float32)]
    ws = torch.full((C.lib().xq_vit_rope_bwd_workspace_bytes(B, N, H, L),), 0xFF, dtype=torch.uint8, device="cuda")
    name = "xq_vit_rope_bwd" + SUFFIX[dtn]
    C.check(getattr(C.lib(), name)(qkv.data_ptr(), g.data_ptr(), freqs.data_ptr(), f1.data_ptr(), B, N, H, 64, P, IMG, L,
                                   *[b[1].data_ptr() for b in bufs], ws.data_ptr(), ws.numel(), C.stream_ptr()), name)
    torch.cuda.synchronize()
    for buf, _ in bufs:
        assert torch.isnan(buf[:GUARD].float()).all() and torch.isnan(buf[-GUARD:].float()).all(), "write outside an output"
    return [b[1] for b in bufs]


def _check_rotation(got, x, c, th, B, N, H, P, dt, conj=False):
    """q / k pairs of `got` against x * c (or conj(c)) in fp64, v and prefix rows bit-equal to x"""
    xg = x.view(B, N, 3, H * 64)
    gg = got.view(B, N, 3, H * 64)
    assert torch.equal(gg[:, :, 2].view(torch.int16), xg[:, :, 2].view(torch.int16)), "v changed"
    assert torch.equal(gg[:, :P].view(torch.int16), xg[:, :P].view(torch.int16)), "prefix rows changed"
    xp = _qk_pairs(x, B, N, H)
    want = xp * (c.conj() if conj else c)                        # [2, B, N, H, 32]
    gp = _qk_pairs(got, B, N, H)
    eps = 8 * 2.0 ** -24 * (1 + th.abs()) * (xp.real.abs() + xp.imag.abs())
    for part in ("real", "imag"):
        w, y = getattr(want, part)[:, :, P:], getattr(gp, part)[:, :, P:]
        bound = 0.5 * _ulp16(w.abs() + eps[:, :, P:], dt) + eps[:, :, P:]
        err = (y - w).abs()
        assert bool((err <= bound).all()), f"{part}: {int((err > bound).sum())} outside, max err {err.max().item():.3e}"


# (B, H, L, P): every value of B in {1, 3, 128}, H in {6, 12, 16, 24}, L in {1, 60, 121, 256}, P in {1, 5} appears
SHAPES = [(1, 6, 1, 1), (3, 12, 60, 5), (3, 16, 121, 1), (1, 24, 256, 5), (128, 12, 256, 1), (128, 6, 60, 5),
          (3, 24, 1, 1), (1, 16, 256, 1)]


@pytest.mark.parametrize("dtn", ["bf16", "f16"])
@pytest.mark.parametrize("B,H,L,P", SHAPES)
def test_rope_fwd_against_fp64(B, H, L, P, dtn):
    from imagefolder_b200.dino_enc.vision_transformer import apply_rotary_emb, compute_mixed_cis, init_t_xy
    dt = DT[dtn]
    N = P + IMG + L
    qkv, freqs, f1 = _inputs(B, N, H, P, L, dt)
    out = _rope_fwd(qkv, freqs, f1, H, P, dtn)
    c, th = _cis64(freqs, f1, H, P, N)
    _check_rotation(out, qkv, c, th, B, N, H, P, dt)
    # torch's own fp32 expression (the reference's apply_rotary_emb), rounded to the 16-bit dtype
    q5 = qkv.view(B, N, 3, H, 64).permute(2, 0, 3, 1, 4)
    t_x, t_y = (t.cuda() for t in init_t_xy(16, 16))
    cis = compute_mixed_cis(freqs, t_x, t_y, H)
    qi, ki = apply_rotary_emb(q5[0][:, :, P:N - L], q5[1][:, :, P:N - L], cis)
    ql, kl = apply_rotary_emb(q5[0][:, :, N - L:], q5[1][:, :, N - L:], torch.view_as_complex(f1.contiguous()))
    o5 = out.view(B, N, 3, H, 64).permute(2, 0, 3, 1, 4)
    diff = sum(int((a.view(torch.int16) != b.view(torch.int16)).sum())
               for a, b in ((o5[0][:, :, P:N - L], qi), (o5[1][:, :, P:N - L], ki), (o5[0][:, :, N - L:], ql),
                            (o5[1][:, :, N - L:], kl)))
    total = 2 * B * H * (IMG + L) * 64
    print(f"rope_fwd {dtn} B={B} H={H} L={L} P={P}: {diff} of {total} rotated elements differ from torch's fp32 "
          f"apply_rotary_emb rounded to {dtn}")
    assert diff <= 1e-3 * total


@pytest.mark.parametrize("dtn", ["bf16", "f16"])
@pytest.mark.parametrize("B,H,L,P", SHAPES)
def test_rope_bwd_against_fp64_and_deterministic(B, H, L, P, dtn):
    dt = DT[dtn]
    N = P + IMG + L
    qkv, freqs, f1 = _inputs(B, N, H, P, L, dt)
    g = torch.randn(qkv.shape, generator=torch.Generator(device="cuda").manual_seed(7), device="cuda").to(dt)
    dq, db, dfr, d1 = _rope_bwd(qkv, g, freqs, f1, H, P, dtn)
    c, th = _cis64(freqs, f1, H, P, N)
    _check_rotation(dq, g, c, th, B, N, H, P, dt, conj=True)
    # reductions against fp64 of the same terms
    n_rows = B * N
    db64 = dq.double().sum((0, 1))
    assert bool(((db.double() - db64).abs() <= n_rows * 2.0 ** -24 * dq.double().abs().sum((0, 1))).all()), "bias"
    xp, gp = _qk_pairs(qkv, B, N, H), _qk_pairs(g, B, N, H)
    y = xp * c
    dth = (gp.imag * y.real - gp.real * y.imag)[:, :, P:P + IMG]           # [2, B, 256, H, 32]
    i = torch.arange(IMG, device="cuda", dtype=torch.float64)
    t = torch.stack([i % 16, torch.div(i, 16, rounding_mode="floor")])[:, None, None, :, None, None]
    terms = t * dth[None]                                                   # [2(x/y), 2(q/k), B, 256, H, 32]
    want = terms.sum((1, 2, 3)).reshape(2, H * 32)
    nt = 2 * B * IMG
    assert bool(((dfr.double() - want).abs() <= nt * 2.0 ** -24 * terms.abs().sum((1, 2, 3)).reshape(2, H * 32)
                 + 1e-6 * want.abs()).all()), "d freqs"
    u = (xp.conj() * gp)[:, :, P + IMG:]                                    # [2, B, L, H, 32]
    w1 = torch.view_as_real(u.sum((0, 1, 3)))
    a1 = torch.view_as_real(u).abs().sum((0, 1, 3))
    assert bool(((d1.double() - w1).abs() <= 2 * B * H * 2.0 ** -24 * a1 + 1e-6 * w1.abs()).all()), "d freqs_1d"
    again = _rope_bwd(qkv, g, freqs, f1, H, P, dtn)
    for a, b in zip((dq, db, dfr, d1), again):
        assert torch.equal(a.view(torch.int16) if a.element_size() == 2 else a.view(torch.int32),
                           b.view(torch.int16) if b.element_size() == 2 else b.view(torch.int32)), "not deterministic"


@pytest.mark.parametrize("dtn", ["bf16", "f16"])
@pytest.mark.parametrize("B,H,L,P", [(128, 12, 256, 1), (3, 6, 60, 5), (33, 16, 121, 1)])
def test_rope_bwd_sums_are_exact_on_integer_inputs(B, H, L, P, dtn):
    """angle 0 and freqs_1d = 1: d(qkv) = g exactly, and with small integers every sum is an exact fp32 integer, so a row
    counted twice or missed by the partials or the fixed-order pass shows as a wrong integer"""
    dt = DT[dtn]
    N = P + IMG + L
    gen = torch.Generator(device="cuda").manual_seed(3)
    qkv = torch.randint(-3, 4, (B, N, 3 * H * 64), generator=gen, device="cuda").to(dt)
    g = torch.randint(-3, 4, (B, N, 3 * H * 64), generator=gen, device="cuda").to(dt)
    freqs = torch.zeros(2, H * 32, device="cuda")
    f1 = torch.zeros(L, 32, 2, device="cuda")
    f1[..., 0] = 1
    dq, db, dfr, d1 = _rope_bwd(qkv, g, freqs, f1, H, P, dtn)
    assert torch.equal(dq.view(torch.int16), g.view(torch.int16))
    assert torch.equal(db, g.long().sum((0, 1)).float())
    xp = qkv.long().view(B, N, 3, H, 32, 2)[:, :, :2]
    gp = g.long().view(B, N, 3, H, 32, 2)[:, :, :2]
    dth = (gp[..., 1] * xp[..., 0] - gp[..., 0] * xp[..., 1])[:, P:P + IMG]          # [B, 256, 2, H, 32]
    i = torch.arange(IMG, device="cuda")
    want = torch.stack([((i % 16)[None, :, None, None, None] * dth).sum((0, 1, 2)),
                        ((i // 16)[None, :, None, None, None] * dth).sum((0, 1, 2))]).view(2, H * 32)
    assert torch.equal(dfr, want.float())
    xl, gl = xp[:, P + IMG:], gp[:, P + IMG:]
    re = (xl[..., 0] * gl[..., 0] + xl[..., 1] * gl[..., 1]).sum((0, 2, 3))
    im = (xl[..., 0] * gl[..., 1] - xl[..., 1] * gl[..., 0]).sum((0, 2, 3))
    assert torch.equal(d1, torch.stack([re, im], -1).float())


# ---- decoder level -----------------------------------------------------------------------------------------------------
def _decoder(name, seeded=True, **kw):
    import make_vit_rope_golden as mrg
    from imagefolder_b200.dino_enc.dinov2 import DINOv2Decoder
    torch.manual_seed(0)
    dec = DINOv2Decoder(**dict(mrg.decoder_kwargs(name), **kw))
    if seeded:
        mrg.det_init_rope(dec)
    return dec.cuda().eval()


def _count_rope_calls(monkeypatch):
    from imagefolder_b200 import vit_ops
    calls = [0]
    orig = vit_ops.rope_forward

    def counted(*a, **k):
        calls[0] += 1
        return orig(*a, **k)
    monkeypatch.setattr(vit_ops, "rope_forward", counted)
    return calls


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("amp", ["bf16", "f16"])
@pytest.mark.parametrize("name", ["vit_rope_l256", "vit_rope_l60", "vit_rope_reg4"])
def test_decoder_autocast_matches_fp32_and_reference_golden(name, amp, monkeypatch):
    import make_vit_rope_golden as mrg
    g = np.load(os.path.join(HERE, "golden", name + ".npz"))
    dec = _decoder(name)
    z, w = mrg.golden_io(name, dec.embed_dim)
    z, w = z.cuda(), w.cuda()
    calls = _count_rope_calls(monkeypatch)
    with torch.no_grad():
        out32 = dec(z)
        with torch.autocast("cuda", dtype=DT[amp]):
            out = dec(z).float()
    assert calls[0] == len(dec.model.blocks), "the RoPE kernels did not run"
    want = torch.from_numpy(g["out_sub"]).cuda()
    torch.testing.assert_close(out32[:, :, ::4, ::4], want, rtol=1e-3, atol=1e-3)
    assert _rel(out, out32) <= 2e-2, _rel(out, out32)
    assert _rel(out[:, :, ::4, ::4], want) <= 2e-2


@pytest.mark.parametrize("amp", ["bf16", "f16"])
@pytest.mark.parametrize("name", ["vit_rope_l256", "vit_rope_reg4"])
def test_decoder_gradients_against_fp64(name, amp, monkeypatch):
    """every parameter gradient of a training step under autocast on the fused path against the fp64 restatement"""
    import make_vit_rope_golden as mrg
    import rope_oracle
    dec = _decoder(name).train()
    z, w = mrg.golden_io(name, dec.embed_dim)
    z, w = z.cuda(), w.cuda()
    calls = _count_rope_calls(monkeypatch)
    with torch.autocast("cuda", dtype=DT[amp]):
        out = dec(z)
    (out.float() * w).sum().backward()
    assert calls[0] == len(dec.model.blocks)
    sd = rope_oracle.fp64_state(dec)
    (rope_oracle.rope_decoder_forward(sd, z.double(), dec.model.blocks[0].attn.num_heads) * w.double()).sum().backward()
    tol = 5e-2 if amp == "bf16" else 2e-2
    worst = {}
    for n, p in dec.named_parameters():
        ref = sd[n].grad
        if ref is None:
            assert p.grad is None, n
            continue
        got = torch.view_as_real(p.grad) if p.grad.is_complex() else p.grad
        want = torch.view_as_real(ref) if ref.is_complex() else ref
        worst[n] = _rel(got, want)
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:5]
    print(f"{name} {amp}: largest relative gradient errors {top}")
    assert all(v <= tol for v in worst.values()), top


def test_fp16_gradscaler_skips_an_overflowing_step(monkeypatch):
    """torch's GradScaler cannot unscale a complex64 grad (_amp_foreach_non_finite_check_and_unscale_ has no ComplexFloat
    kernel, for the reference's model too), so freqs_1d stays out of the scaled optimizer here; every other parameter,
    freqs included, goes through the fp16 RoPE kernels and the skipped step"""
    import make_vit_rope_golden as mrg
    from imagefolder_b200.optim import AdamW
    dec = _decoder("vit_rope_l60").train()
    opt = AdamW([p for p in dec.parameters() if p.requires_grad and not p.is_complex()], lr=1e-3)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 40)
    z, w = mrg.golden_io("vit_rope_l60", dec.embed_dim)
    before = {n: p.detach().clone() for n, p in dec.named_parameters()}
    calls = _count_rope_calls(monkeypatch)
    with torch.autocast("cuda", dtype=torch.float16):
        out = dec(z.cuda())
    scaler.scale((out.float() * w.cuda()).sum()).backward()
    scaler.step(opt)
    scaler.update()
    assert calls[0] == len(dec.model.blocks)
    assert scaler.get_scale() < 2.0 ** 40
    for n, p in dec.named_parameters():
        assert torch.equal(p.detach(), before[n]), n


# ---- trainer pieces on the complex64 parameter ---------------------------------------------------------------------------
def _as_int(t):
    return (torch.view_as_real(t) if t.is_complex() else t).detach().contiguous().view(torch.int32)


def test_adamw_is_bit_identical_to_torch_on_a_rope_decoder():
    from imagefolder_b200.optim import AdamW
    a = _decoder("vit_rope_l60", tuning_method="full").train()
    b = _decoder("vit_rope_l60", tuning_method="full").train()
    pa = [p for p in a.parameters() if p.requires_grad]
    pb = [p for p in b.parameters() if p.requires_grad]
    assert any(p.is_complex() for p in pa)
    oa = AdamW(pa, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.05)
    ob = torch.optim.AdamW(pb, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.05)
    gen = torch.Generator(device="cuda").manual_seed(11)
    for _ in range(5):
        for x, y in zip(pa, pb):
            gr = torch.randn(x.shape, dtype=x.dtype, generator=gen, device="cuda")
            x.grad, y.grad = gr.clone(), gr.clone()
        oa.step()
        ob.step()
    for x, y in zip(pa, pb):
        assert torch.equal(_as_int(x), _as_int(y))
    for x, y in zip(pa, pb):
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(_as_int(oa.state[x][k]), _as_int(ob.state[y][k])), k


def test_clip_grad_norm_on_a_complex_grad():
    """the total norm of a complex64 grad is that of its real view; prints whether torch's complex _foreach_norm gives the
    same bits, and how the grads compare after scaling"""
    from imagefolder_b200.optim import clip_grad_norm_
    gen = torch.Generator(device="cuda").manual_seed(5)
    shapes = [(60, 32), (256, 32)]
    params = [torch.zeros(2, 384, device="cuda", requires_grad=True)] + [
        torch.zeros(s, dtype=torch.complex64, device="cuda", requires_grad=True) for s in shapes]
    grads = [torch.randn(p.shape, dtype=p.dtype, generator=gen, device="cuda") for p in params]
    ours = [p.detach().clone().requires_grad_() for p in params]
    for p, o, g in zip(params, ours, grads):
        p.grad, o.grad = g.clone(), g.clone()
    cg = [g for g in grads if g.is_complex()]
    n_c = torch._foreach_norm(cg)
    n_r = torch._foreach_norm([torch.view_as_real(g) for g in cg])
    same = [bool(torch.equal(a.view(torch.int32), b.view(torch.int32))) for a, b in zip(n_c, n_r)]
    tn_t = torch.nn.utils.clip_grad_norm_(params, 1.0)
    tn_o = clip_grad_norm_(ours, 1.0)
    print(f"torch._foreach_norm(complex) == norm of the real view, bit for bit: {same}; total norm torch "
          f"{tn_t.item()!r} ours {tn_o.item()!r}")
    assert torch.equal(tn_o.view(torch.int32), tn_t.view(torch.int32)) or not all(same)
    assert abs(tn_o.item() - tn_t.item()) <= 4 * 2.0 ** -24 * tn_t.item()
    for p, o in zip(params, ours):
        if all(same):
            assert torch.equal(_as_int(o.grad), _as_int(p.grad))
        else:
            assert torch.allclose(torch.view_as_real(o.grad) if o.grad.is_complex() else o.grad,
                                  torch.view_as_real(p.grad) if p.grad.is_complex() else p.grad, rtol=4e-7, atol=0)


def test_update_ema_matches_the_reference_loop_on_complex_parameters():
    """ema.mul_(decay).add_(param, alpha=1 - decay) (utils/ema.py) against the real-view kernel.  fp32 parameters: bit for bit.
    complex64 `freqs_1d`: torch's complex add rounds alpha * param and the sum separately where the kernel (like torch's fp32
    add_) rounds once, so a component may differ by one fp32 ulp of the result; at decay 0 the two are equal."""
    from imagefolder_b200.ema import update_ema
    m = _decoder("vit_rope_l60", tuning_method="full")
    e1 = _decoder("vit_rope_l60", tuning_method="full")
    e2 = _decoder("vit_rope_l60", tuning_method="full")
    gen = torch.Generator(device="cuda").manual_seed(9)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(torch.randn(p.shape, dtype=p.dtype, generator=gen, device="cuda"))
    for decay in (0.0, 0.9999, 0.5):
        update_ema(e1, m, decay=decay)
        with torch.no_grad():
            mp = dict(m.named_parameters())
            for n, p in e2.named_parameters():
                p.mul_(decay).add_(mp[n].data, alpha=1 - decay)
        n_diff, worst = 0, 0.0
        for (n, a), (_, b) in zip(e1.named_parameters(), e2.named_parameters()):
            if not a.is_complex() or decay == 0.0:
                assert torch.equal(_as_int(a), _as_int(b)), (n, decay)
                continue
            ra, rb = torch.view_as_real(a).detach(), torch.view_as_real(b).detach()
            ulp = torch.finfo(torch.float32).eps * torch.exp2(torch.floor(torch.log2(rb.abs().clamp_min(2.0 ** -126))))
            err = (ra - rb).abs()
            assert bool((err <= ulp).all()), (n, decay, float((err / ulp).max()))
            n_diff += int((ra != rb).sum())
            worst = max(worst, float((err / ulp).max()))
            with torch.no_grad():
                a.copy_(b)                          # both sides continue from the reference's values
        print(f"update_ema decay={decay}: {n_diff} complex components differ from torch's complex update, "
              f"at most {worst} ulp")
