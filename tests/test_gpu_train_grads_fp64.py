"""Every parameter gradient of one bf16 / fp16 training step, fused ViT path and library path, against fp64.

The step is the benchmarked one: `mse(dec, x) + vq + commit (+ entropy)` on a ViT-B encoder and decoder (D = 768, 12
heads, guides off) in train mode, B = 4 at 256 x 256, with DropPath on (drop_path_rate 0.1) and LayerScale gammas random
in [0.25, 1] so that a gradient sent to the wrong branch, or scaled by gamma twice, shows.  The multi-scale cases raise
`codebook_drop` to 0.5, so two of the four samples lose scales.

The step is checked segment by segment, so that a discrete index choice never enters a float comparison:
  decoder    fp64 `post_quant_conv` + decoder (oracle/vit_ref.py) with the DropPath multipliers the product drew, on the
             product's own `quant`, with its own MSE: every decoder / post_quant_conv gradient and d(quant);
  quantizer  the fp32 C oracle on the product's own quantizer input with the product's d(quant) upstream: indices bit for
             bit, codebook / Phi gradients and d(h) at the quantizer tests' 1e-4 bar;
  encoder    fp64 encoder + `quant_conv` on the same x with the recorded multipliers, back-propagated from the product's
             own d(h): every encoder / quant_conv gradient.
The fused path must be no worse than the library path (every fused ViT kernel off, `torch.nn` modules, library attention)
measured the same way: for each parameter tensor, with e = |g - g64| / |g64|,
    e_fused <= 2 e_lib + u,        u = 2^-8 (bf16), 2^-11 (fp16).
Named mutants (fp64 gradients with one routing bug) must fail that bound.  `pytest -s` prints the measured errors.

fp16 runs the step with the loss scaled by 2^16 (GradScaler's initial scale) and divides every gradient by it, as a
GradScaler run does.  Without the scale the decoder's pixel gradients (about 1e-6) are fp16 subnormals on both paths:
the cls / latent-token gradients are then 10-24 % off fp64 on both paths (the fused one being the closer), which is the
gap that the unscaled fp16 fused-vs-library comparison in test_gpu_fp16_vit.py sees.

Measured on an H100 80GB HBM3 (700 W power limit): the largest e_fused / (2 e_lib + u) over every parameter and case is
0.43, and in every printed parameter class e_fused and e_lib are close to each other (the cls / latent tokens: about
7e-3 in bf16, 8e-4 in fp16, on both paths).  Every mutant exceeds its bound at least 3.5x (the decoder's latent-slot
pos-embed mutant is the closest).
The file takes about 45 s and at most 5.6 GiB of extra device memory.
"""
import contextlib
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import vit_ref, xq_oracle as xo
from test_model_cpu import small_model

pytestmark = pytest.mark.gpu

VIT_B = "vit_base_patch14_dinov2.lvd142m"
U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
LOSS_SCALE = {torch.bfloat16: 1.0, torch.float16: 2.0 ** 16}
B = 4
SEED = 7


def _segment(name):
    if name.startswith(("encoder.", "quant_conv.")):
        return "encoder"
    if name.startswith(("decoder.", "post_quant_conv.")):
        return "decoder"
    assert name.startswith("quantize"), name
    return "quantizer"


def _rel(g, g64):
    return float((g.double() - g64).norm() / g64.norm())


def _cls(name):
    return re.sub(r"\.blocks\.\d+\.", ".blocks.*.", name)


# ------------------------------------------------------------------------------------------------------------------
# the product's step
# ------------------------------------------------------------------------------------------------------------------
def _spy_calls():
    from imagefolder_b200 import _capi
    calls, real = [], _capi.call

    def spy(name, *a, **k):
        calls.append(name)
        return real(name, *a, **k)

    @contextlib.contextmanager
    def ctx():
        _capi.call = spy
        try:
            yield calls
        finally:
            _capi.call = real
    return ctx()


@contextlib.contextmanager
def _library_path(model, masks):
    """every fused ViT path off (the switches of oracle/eager_ref.EagerTokenizer plus the three kernel flags), with the
    DropPath modules forced to the multipliers `masks` (module -> [B] or None) the fused run drew"""
    from imagefolder_b200 import vit_ops
    saved = (vit_ops.fused_path_ok, vit_ops.patch_embed_ok)
    flags = (vit_ops.ASSEMBLE_ENABLED, vit_ops.MLP_TC_ENABLED, vit_ops.ATTN_TC_ENABLED)
    vit_ops.fused_path_ok = vit_ops.patch_embed_ok = lambda *a, **k: False
    for f in flags:
        f[0] = False
    mods = [m for m in masks if masks[m] is not None]
    for m in mods:
        m.forward = lambda x, k=masks[m]: x * k.to(x.dtype).view(-1, *([1] * (x.dim() - 1)))
    try:
        yield
    finally:
        vit_ops.fused_path_ok, vit_ops.patch_embed_ok = saved
        for f in flags:
            f[0] = True
        for m in mods:
            del m.forward


@contextlib.contextmanager
def _record_droppath(masks):
    from imagefolder_b200 import vit_ops
    real = vit_ops._droppath_scale

    def rec(mod, batch, device):
        t = real(mod, batch, device)
        masks[mod] = None if t is None else t.clone()
        return t

    vit_ops._droppath_scale = rec
    try:
        yield
    finally:
        vit_ops._droppath_scale = real


def _product_step(model, x, dt):
    """one training step; -> (param grads, h, d h, quant, d quant), every gradient divided by the loss scale"""
    S = LOSS_SCALE[dt]
    cap = {}

    def keep_h(mod, inp, out):
        out.retain_grad()
        cap["h"] = out

    def keep_q(mod, inp):
        inp[0].retain_grad()
        cap["quant"] = inp[0]

    hooks = [model.quant_conv.register_forward_hook(keep_h), model.post_quant_conv.register_forward_pre_hook(keep_q)]
    model.zero_grad(set_to_none=True)
    try:
        torch.manual_seed(SEED)                          # the CPU generator draws dropout_rand (xqgan_model.py:274)
        with torch.autocast("cuda", dtype=dt):
            dec, (vq, commit, ent, _), _, _, _ = model(x, 0, 0.0, 0.0, 100)
            loss = F.mse_loss(dec.float(), x) + vq + commit + ent
        (loss * S).backward()
    finally:
        for hk in hooks:
            hk.remove()
    grads = {n: p.grad.float() / S for n, p in model.named_parameters() if p.grad is not None}
    model.zero_grad(set_to_none=True)
    h, q = cap["h"], cap["quant"]
    return grads, h.detach(), h.grad.double() / S, q.detach(), q.grad.double() / S


def _keep_lists(model, masks):
    out = {}
    for seg, vit in (("encoder", model.encoder.model), ("decoder", model.decoder.model)):
        out[seg] = [[masks.get(dp) for dp in (blk.drop_path1, blk.drop_path2)] for blk in vit.blocks]
    return out


# ------------------------------------------------------------------------------------------------------------------
# fp64 segments
# ------------------------------------------------------------------------------------------------------------------
def _ref_grads(rt, prefixes):
    out = {}
    for k, v in rt.sd.items():
        if k.startswith(prefixes) and v.requires_grad:
            out[k] = v.grad.clone() if v.grad is not None else torch.zeros_like(v)
            v.grad = None
    return out


def _ref_decoder(rt, quant, x, keep):
    """fp64 post_quant_conv + decoder on the product's quant, its own MSE; one sample at a time (the loss is a sum over
    samples), which keeps the fp64 activations of ViT-B small"""
    q64 = quant.double().requires_grad_(True)
    n = x.numel()
    for b in range(x.shape[0]):
        kb = [[None if m is None else m[b:b + 1] for m in pair] for pair in keep]
        dec = rt.decode(q64[b:b + 1], kb)
        ((dec - x[b:b + 1].double()).square().sum() / n).backward()
    return _ref_grads(rt, ("decoder.", "post_quant_conv.")), q64.grad


def _ref_encoder(rt, x, dh, keep):
    for b in range(x.shape[0]):
        kb = [[None if m is None else m[b:b + 1] for m in pair] for pair in keep]
        rt.encode(x[b:b + 1].double(), kb).backward(dh[b:b + 1])
    return _ref_grads(rt, ("encoder.", "quant_conv."))


def _ref_quantizer(rt, h, dquant, dropout):
    h64 = h.double().requires_grad_(True)
    quant, (vq, cm, en) = rt.quantize(h64, dropout)
    ((quant * dquant).sum() + vq + cm + en).backward()
    return _ref_grads(rt, ("quantize",)), h64.grad, quant.detach()


def _check_indices(model, rt, h, dropout):
    """the product's token indices equal the C oracle's on the product's own quantizer input"""
    cfg = rt.cfg
    pn = list(cfg["v_patch_nums"])
    for qm, hb in zip(model._quantizers(), rt._branches(h.float().cpu())):
        hbn = np.ascontiguousarray(hb.numpy())
        if len(pn) == 1:
            idx = xo.vq_forward(hbn, qm.embedding.weight.detach().cpu().numpy(), cfg["beta"], cfg["codebook_l2_norm"])["idx"]
            np.testing.assert_array_equal(qm.last_idx.cpu().numpy(), idx)
            continue
        mods = qm.quant_resi.modules_list()
        pw = np.stack([m.weight.detach().cpu().numpy() for m in mods])
        pb = np.stack([m.bias.detach().cpu().numpy() for m in mods])
        if cfg["lfq"]:
            fw = xo.lfq_forward(hbn, pw, pb, pn, using_znorm=cfg["codebook_l2_norm"], codebook_drop=cfg["codebook_drop"],
                                dropout=dropout, scaler=qm.scaler.cpu().numpy(), entropy_weight=cfg["entropy_weight"])
        else:
            fw = xo.vq2_forward(hbn, qm.embedding.weight.detach().cpu().numpy(), pw, pb, pn, using_znorm=True,
                                codebook_drop=cfg["codebook_drop"], dropout=dropout)
        for si in range(len(pn)):
            np.testing.assert_array_equal(qm.last_idx_Bl[si].cpu().numpy().astype(np.int64), np.asarray(fw["idx"][si]))


def _measure(model, rt, x, dt, keep_of, dropout):
    """run the product step (fused or library, as set up by the caller) and its fp64 segments with the DropPath
    multipliers keep_of() gives after the step -> (per-parameter relative error, the fp64 gradients, the product's
    (h, d h, quant, d quant), the multipliers)"""
    grads, h, dh, quant, dquant = _product_step(model, x, dt)
    keep = keep_of()
    g64, dq64 = _ref_decoder(rt, quant, x, keep["decoder"])
    gq, dh64, quant64 = _ref_quantizer(rt, h, dquant, dropout)
    g64.update(gq)
    g64.update(_ref_encoder(rt, x, dh, keep["encoder"]))
    trainable = {n for n, p in model.named_parameters() if p.requires_grad}
    assert set(grads) == trainable and set(g64) == trainable, (set(grads) ^ trainable, set(g64) ^ trainable)
    # quantizer segment: the oracle's own bar (1e-4), plus d h's one rounding to the latent's 16-bit dtype
    _check_indices(model, rt, h, dropout)
    ulp = U[dt] * 2
    for n in trainable:
        if _segment(n) == "quantizer":
            torch.testing.assert_close(grads[n].double(), g64[n], rtol=1e-4, atol=1e-4 * float(g64[n].abs().max()), msg=n)
    tiny = 2.0 ** -24 / LOSS_SCALE[dt] if dt == torch.float16 else 0.0
    torch.testing.assert_close(dh, dh64, rtol=1e-4 + ulp, atol=1e-4 * float(dh64.abs().max()) + tiny)
    # d quant: the decoder's input gradient, fp64 reference on the same quant
    e = {n: _rel(grads[n], g64[n]) for n in trainable if _segment(n) != "quantizer"}
    e["d(quant)"] = _rel(dquant, dq64)
    return e, g64, (h, dh, quant, dquant), keep


# ------------------------------------------------------------------------------------------------------------------
# mutants: fp64 gradients with one routing bug each
# ------------------------------------------------------------------------------------------------------------------
def _mutant_block(target, branch, kind):
    """vit_ref._block with one bug in `branch` (0 attention, 1 MLP) of block `target`:
    'droppath'  the DropPath multiplier applied in the forward only: a + (a*keep - a).detach();
    'gamma'     LayerScale gamma applied twice in the backward (forward unchanged)"""
    real = vit_ref._block

    def scaled(a, gamma, keep, br):
        if kind == "gamma" and br == branch:
            twice = a * gamma * gamma.detach()
            a = twice + (a * gamma - twice).detach()
        else:
            a = a * gamma
        if keep is None:
            return a
        if kind == "droppath" and br == branch:
            return a + (a * keep[br] - a).detach()
        return a * keep[br]

    def block(x, sd, prefix, num_heads, keep=None):
        if prefix != target:
            return real(x, sd, prefix, num_heads, keep)
        a = vit_ref._attention(vit_ref._ln(x, sd, prefix + ".norm1"), sd, prefix + ".attn", num_heads)
        x = x + scaled(a, sd[prefix + ".ls1.gamma"], keep, 0)
        m = F.linear(vit_ref._ln(x, sd, prefix + ".norm2"), sd[prefix + ".mlp.fc1.weight"], sd[prefix + ".mlp.fc1.bias"])
        m = F.linear(F.gelu(m), sd[prefix + ".mlp.fc2.weight"], sd[prefix + ".mlp.fc2.bias"])
        return x + scaled(m, sd[prefix + ".ls2.gamma"], keep, 1)
    return block


def _pos_embed_without_latents():
    """vit_ref._pos_embed whose pos-embed gets no gradient from the latent-token grids (the 4-D calls)"""
    real = vit_ref._pos_embed

    def pos_embed(x, sd, prefix):
        if x.dim() == 4:
            sd = dict(sd)
            sd[prefix + ".pos_embed"] = sd[prefix + ".pos_embed"].detach()
        return real(x, sd, prefix)
    return pos_embed


@contextlib.contextmanager
def _patched(name, fn):
    real = getattr(vit_ref, name)
    setattr(vit_ref, name, fn)
    try:
        yield
    finally:
        setattr(vit_ref, name, real)


def _caught(g_mut, g64, e_lib, u):
    """names whose mutant gradient breaks the bound"""
    return [n for n in g_mut if _rel(g_mut[n], g64[n]) > 2 * e_lib[n] + u]


def _run_mutants(model, rt, x, keep, g64, prod, e_lib, u):
    h, dh, quant, dquant = prod
    PQ = rt.cfg["product_quant"]
    mut = {}

    def rerun(seg, name, fn):
        with _patched(name, fn):
            if seg == "decoder":
                return _ref_decoder(rt, quant, x, keep["decoder"])[0]
            return _ref_encoder(rt, x, dh, keep["encoder"])

    # DropPath mask ignored in the backward of one branch where a sample was dropped
    seg, i, br = next((s, i, br) for s in ("decoder", "encoder") for i, pair in enumerate(keep[s])
                      for br, k in enumerate(pair) if k is not None and bool((k == 0).any()))
    mut[f"droppath-ignored-in-bwd {seg}.blocks.{i}.{'attn' if br == 0 else 'mlp'}"] = rerun(
        seg, "_block", _mutant_block(f"{seg}.model.blocks.{i}", br, "droppath"))
    # LayerScale gamma applied twice in the backward of one block's attention branch
    mut["gamma-twice decoder.blocks.5.attn"] = rerun("decoder", "_block", _mutant_block("decoder.model.blocks.5", 0, "gamma"))
    # pos-embed gradient without the latent-token slots
    mut["pos-embed-no-latent-slots decoder"] = rerun("decoder", "_pos_embed", _pos_embed_without_latents())
    mut["pos-embed-no-latent-slots encoder"] = rerun("encoder", "_pos_embed", _pos_embed_without_latents())
    # the last block's fc2 bias gradient lost (it is folded into the final norm)
    for s in ("encoder", "decoder"):
        n = f"{s}.model.blocks.11.mlp.fc2.bias"
        mut[f"last-fc2-bias-lost {s}"] = {n: torch.zeros_like(g64[n])}
    # lvl-embed gradient missing one product-quant branch
    if PQ > 1:
        g = g64["encoder.lvl_embed.weight"].clone()
        g[PQ] = 0
        mut["lvl-embed-missing-last-branch encoder"] = {"encoder.lvl_embed.weight": g}
    out = {}
    for name, gm in mut.items():
        bad = _caught(gm, g64, e_lib, u)
        out[name] = bad
        worst = max(gm, key=lambda n: _rel(gm[n], g64[n]) / (2 * e_lib[n] + u))
        print(f"  mutant {name:52s} caught by {len(bad):3d} tensors, worst {worst}: "
              f"e {_rel(gm[worst], g64[worst]):.2e} > bound {2 * e_lib[worst] + u:.2e}")
    return out


# ------------------------------------------------------------------------------------------------------------------
# the test
# ------------------------------------------------------------------------------------------------------------------
CASES = [("VQ-8192", torch.bfloat16), ("MSVR10P2-4096", torch.bfloat16), ("MSBR10P2-16384", torch.bfloat16),
         ("VQ-8192", torch.float16), ("MSVR10P2-4096", torch.float16)]


@pytest.mark.parametrize("name,dt", CASES, ids=[f"{n}-{str(d)[6:]}" for n, d in CASES])
def test_train_step_grads_vs_fp64(name, dt):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    over = dict(encoder_model=VIT_B, decoder_model=VIT_B)
    if name.startswith("MS"):
        over["codebook_drop"] = 0.5
    model, _ = small_model(name, **over)
    model = model.cuda().train()
    gen = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for vit in (model.encoder.model, model.decoder.model):
            for blk in vit.blocks:
                for ls in (blk.ls1, blk.ls2):
                    ls.gamma.copy_(0.25 + 0.75 * torch.rand(ls.gamma.shape, generator=gen))
    x = (torch.rand(B, 3, 256, 256, generator=gen) * 2 - 1).cuda()
    u = U[dt]
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()

    cfg = vit_ref.cfg_from_model_args(model.config, num_heads=12)
    rt = vit_ref.RefTokenizer(model.state_dict(), cfg, requires_grad=True, dtype=torch.float64, device="cuda")
    SN = len(cfg["v_patch_nums"])
    torch.manual_seed(SEED)
    dropout = torch.randint(model.start_drop, SN + 1, (B,)).numpy() if SN > 1 else None
    if SN > 1:
        assert int(B * cfg["codebook_drop"]) >= 1 and (dropout[:int(B * cfg["codebook_drop"])] < SN + 1).all()

    # fused step: the product draws the DropPath multipliers, the recorder keeps them for the references and the library run
    masks = {}
    keep_of = lambda: _keep_lists(model, masks)
    with _record_droppath(masks), _spy_calls() as calls:
        e_fused, g64, prod, keep = _measure(model, rt, x, dt, keep_of, dropout)
    for n in ("xq_vit_attn_fwd", "xq_vit_attn_bwd", "xq_vit_fc1_gelu_fwd", "xq_vit_fc2_dgelu_bwd", "xq_vit_residual_ln_fwd",
              "xq_vit_residual_ln_bwd", "xq_vit_patchify", "xq_vit_assemble_fwd", "xq_vit_assemble_bwd"):
        n = n + "_f16" if dt == torch.float16 and "assemble" not in n else n
        assert n in calls, n
    n_drop = sum(int((k == 0).sum()) for s in keep.values() for pair in s for k in pair if k is not None)
    assert n_drop >= 1, "no sample was dropped in any block: pick another seed"

    # library path with the same multipliers: no fused ViT entry point may run
    with _library_path(model, masks), _spy_calls() as calls:
        e_lib, _, _, _ = _measure(model, rt, x, dt, keep_of, dropout)
    assert not [c for c in calls if c.startswith("xq_vit_")], sorted(set(calls))

    # per parameter class: the worst ratio over the blocks
    print(f"\n{name} {str(dt)[6:]}: {n_drop} dropped (sample, branch) pairs; peak extra device memory "
          f"{(torch.cuda.max_memory_allocated() - base) / 2 ** 30:.2f} GiB")
    classes = {}
    for n in e_fused:
        c = _cls(n)
        r = e_fused[n] / (2 * e_lib[n] + u)
        if c not in classes or r > classes[c][2]:
            classes[c] = (e_fused[n], e_lib[n], r)
    for c in sorted(classes):
        ef, el, r = classes[c]
        print(f"  {c:48s} e_fused {ef:.2e}  e_lib {el:.2e}  e_fused/(2 e_lib + u) {r:.2f}")
    caught = _run_mutants(model, rt, x, keep, g64, prod, e_lib, u)

    bad = {n: (e_fused[n], e_lib[n]) for n in e_fused if e_fused[n] > 2 * e_lib[n] + u}
    assert not bad, bad
    assert all(caught.values()), [m for m, b in caught.items() if not b]
    assert torch.cuda.max_memory_allocated() - base < 8 * 2 ** 30
