"""The quantizers' binding of the C ABI (include/xqb200.h): torch.library ops for the single-scale VQ and the usage EMA,
autograd.Function wrappers for the latent perturbation and the multi-scale quantizers.

PyTorch is plumbing here: it owns the device memory and the stream; every arithmetic step of the
quantizer path happens inside libxqb200.so.  Gradients are the closed forms of SURVEY.md
Appendix A (hand-written backward kernels), not autograd traces.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import torch
from torch import Tensor

from . import _capi as C


def _f32c(t):
    """contiguous fp32 view or copy of t (None stays None)."""
    if t is None:
        return None
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


# ----------------------------------------------------------------------------------------------
# single-scale VQ: torch.library ops, so that torch.compile(fullgraph=True) traces VectorQuantizer.forward without graph
# breaks and CUDA graphs capture it (SURVEY.md section 8b: "loaded as PyTorch custom ops through a thin C-ABI")
#
#     torch.ops.xqb200.vq_forward(z, E, beta, codebook_norm)                       -> (out, loss[2], idx, hist)
#     torch.ops.xqb200.vq_backward(z, E, idx, g_out, g_loss, beta, codebook_norm)  -> (gz, gE)
#     torch.ops.xqb200.usage_ema_(ema, hit, counter, margin)                       -> usage[rows]  (mutates ema and counter)
# ----------------------------------------------------------------------------------------------
def _vq_search(z, E, codebook_norm: bool, train: bool, beta: float = 0.0):
    """one xq_vq_forward call.  train: straight-through output, {vq, commit} losses and code histogram
    (xqgan_model.py:745-801); otherwise the codes themselves, no losses (xqgan_model.py:803-833)."""
    z, E = _f32c(z), _f32c(E)
    B, Cc = z.shape[0], z.shape[1]
    HW = z[0, 0].numel()
    V = E.shape[0]
    dev = z.device
    idx = torch.empty(B * HW, dtype=torch.int64, device=dev)
    out = torch.empty_like(z)
    loss = torch.empty(2, dtype=torch.float32, device=dev) if train else None
    hist = torch.zeros(V, dtype=torch.float32, device=dev) if train else None
    L = C.lib()
    ws = C.workspace(L.xq_vq_workspace_bytes(B, Cc, HW, V), dev)
    name, nk = ("xq_vq_forward", 3) if train else ("xq_vq_lookup", 2)
    C.call(name, nk, L.xq_vq_forward, C.ptr(z), C.ptr(E), B, Cc, HW, V, int(codebook_norm), int(train), float(beta),
           C.ptr(idx), C.ptr(out), C.ptr(loss), C.ptr(hist), C.ptr(ws), ws.numel(), C.stream_ptr(dev))
    return out, loss, idx, hist


@torch.library.custom_op("xqb200::vq_forward", mutates_args=())
def _vq_forward(z: Tensor, E: Tensor, beta: float, codebook_norm: bool) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    return _vq_search(z, E, codebook_norm, train=True, beta=beta)


@_vq_forward.register_fake
def _(z, E, beta, codebook_norm):
    n = z.shape[0] * z[0, 0].numel()
    return (torch.empty_like(z, dtype=torch.float32, memory_format=torch.contiguous_format), z.new_empty(2, dtype=torch.float32),
            z.new_empty(n, dtype=torch.int64), z.new_empty(E.shape[0], dtype=torch.float32))


@torch.library.custom_op("xqb200::vq_backward", mutates_args=())
def _vq_backward(z: Tensor, E: Tensor, idx: Tensor, g_out: Tensor, g_loss: Tensor, beta: float,
                codebook_norm: bool) -> Tuple[Tensor, Tensor]:
    z, E, g_out, g_loss = _f32c(z), _f32c(E), _f32c(g_out), _f32c(g_loss)
    B, Cc = z.shape[0], z.shape[1]
    HW = z[0, 0].numel()
    V = E.shape[0]
    gz = torch.empty_like(z)
    gE = torch.empty_like(E)
    L = C.lib()
    C.call("xq_vq_backward", 1, L.xq_vq_backward, C.ptr(z), C.ptr(E), C.ptr(idx), C.ptr(g_out), C.ptr(g_loss),
           C.ptr(g_loss) + 4, B, Cc, HW, V, int(codebook_norm), float(beta), C.ptr(gz), C.ptr(gE), C.stream_ptr(z.device))
    return gz, gE


@_vq_backward.register_fake
def _(z, E, idx, g_out, g_loss, beta, codebook_norm):
    return (torch.empty_like(z, dtype=torch.float32, memory_format=torch.contiguous_format),
            torch.empty_like(E, dtype=torch.float32, memory_format=torch.contiguous_format))


def _vq_setup(ctx, inputs, output):
    z, E, beta, codebook_norm = inputs
    ctx.save_for_backward(z, E, output[2])
    ctx.beta, ctx.codebook_norm = beta, codebook_norm


def _vq_bwd(ctx, g_out, g_loss, _g_idx, _g_hist):
    z, E, idx = ctx.saved_tensors
    if g_out is None:
        g_out = torch.zeros_like(z, dtype=torch.float32)
    if g_loss is None:
        g_loss = z.new_zeros(2, dtype=torch.float32)
    gz, gE = torch.ops.xqb200.vq_backward(z, E, idx, g_out, g_loss, ctx.beta, ctx.codebook_norm)
    return gz, gE, None, None


torch.library.register_autograd("xqb200::vq_forward", _vq_bwd, setup_context=_vq_setup)


def vq_forward(z, E, beta=0.25, codebook_norm=True, want_hist=True):
    """(z[B,C,H,W], E[V,C]) -> out, vq_loss, commit_loss, idx, hist|None   (xqgan_model.py:745-801)."""
    out, loss, idx, hist = torch.ops.xqb200.vq_forward(z, E, beta, codebook_norm)
    return out, loss[0], loss[1], idx, (hist.detach() if want_hist else None)    # statistics only: no gradient


@torch.no_grad()
def vq_lookup(z, E, codebook_norm=True) -> Tuple[torch.Tensor, torch.Tensor]:
    """inference: (q[B,C,H,W], idx[N])  (xqgan_model.py:803-833)."""
    out, _, idx, _ = _vq_search(z, E, codebook_norm, train=False)
    return out, idx


@torch.library.custom_op("xqb200::usage_ema_", mutates_args=("ema", "counter"))
def usage_ema_(ema: Tensor, hit: Tensor, counter: Tensor, margin: float) -> Tensor:
    """in-place EMA update of ema [rows, V] or [V] from hit (same shape) + usage percentages (device tensor [rows]).
    counter: int64 [2] on the device, the quantizer's step counter and the kernel's scratch word (see xq_usage_ema_dev)."""
    rows = 1 if ema.dim() == 1 else ema.shape[0]
    V = ema.shape[-1]
    usage = torch.empty(rows, dtype=torch.float32, device=ema.device)
    L = C.lib()
    C.call("xq_usage_ema", 1, L.xq_usage_ema_dev, C.ptr(ema), C.ptr(hit.contiguous()), rows, V, C.ptr(counter),
           float(margin), C.ptr(usage), C.stream_ptr(ema.device))
    return usage


@usage_ema_.register_fake
def _(ema, hit, counter, margin):
    return ema.new_empty(1 if ema.dim() == 1 else ema.shape[0], dtype=torch.float32)


# ----------------------------------------------------------------------------------------------
# latent perturbation
# ----------------------------------------------------------------------------------------------
class _Perturb(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z, z_q, E, rand_u, rand_j, codebook_norm: bool, alpha: float, n_perturb: int, delta: int):
        z, z_q, E = _f32c(z), _f32c(z_q), _f32c(E)
        B, Cc = z.shape[0], z.shape[1]
        HW = z[0, 0].numel()
        V = E.shape[0]
        dev = z.device
        out = torch.empty_like(z)
        L = C.lib()
        ws = C.workspace(L.xq_perturb_workspace_bytes(B, Cc, HW, V), dev)
        ru = rand_u.float().contiguous() if rand_u is not None else None
        rj = rand_j.to(torch.int64).contiguous() if rand_j is not None else None
        nk = (1 if n_perturb < B else 0) + (2 if n_perturb > 0 else 0)
        C.call("xq_perturb_forward", nk, L.xq_perturb_forward, C.ptr(z), C.ptr(z_q), C.ptr(E), C.ptr(ru), C.ptr(rj),
               B, Cc, HW, V, int(codebook_norm), float(alpha), int(n_perturb), int(delta), C.ptr(out), None,
               C.ptr(ws), ws.numel(), C.stream_ptr(dev))
        ctx.save_for_backward(z)
        ctx.codebook_norm, ctx.n_perturb = bool(codebook_norm), int(n_perturb)
        return out

    @staticmethod
    def backward(ctx, g):
        (z,) = ctx.saved_tensors
        g = _f32c(g)
        B, Cc = z.shape[0], z.shape[1]
        HW = z[0, 0].numel()
        gz = torch.empty_like(z)
        gzq = torch.empty_like(z)
        L = C.lib()
        C.call("xq_perturb_backward", 1, L.xq_perturb_backward, C.ptr(z), C.ptr(g), B, Cc, HW,
               int(ctx.codebook_norm), ctx.n_perturb, C.ptr(gz), C.ptr(gzq), C.stream_ptr(z.device))
        return gz, gzq, None, None, None, None, None, None, None


def perturb(z, z_q, E, rand_u, rand_j, codebook_norm, alpha, n_perturb, delta):
    return _Perturb.apply(z, z_q, E, rand_u, rand_j, codebook_norm, alpha, n_perturb, delta)


# ----------------------------------------------------------------------------------------------
# multi-scale residual (VQ2 / BSQ)
# ----------------------------------------------------------------------------------------------
def _ms_idx_buffer(L, desc, dev) -> torch.Tensor:
    """the int64 token buffer of every scale (checks the descriptor)."""
    total = L.xq_ms_total_tokens(desc)
    if total < 0:
        raise ValueError("xq_ms_forward: invalid multi-scale descriptor")
    return torch.empty(total, dtype=torch.int64, device=dev)


class _MSForward(torch.autograd.Function):
    """(f, E|None, phi_w|None, phi_b|None) -> out, vq, commit, entropy, idx_all, hist."""

    @staticmethod
    def forward(ctx, f, E, phi_w, phi_b, n_quantizers, desc, want_hist: bool):
        f, E, phi_w, phi_b, nq = map(_f32c, (f, E, phi_w, phi_b, n_quantizers))
        dev = f.device
        L = C.lib()
        idx_all = _ms_idx_buffer(L, desc, dev)
        out = torch.empty_like(f)
        loss = torch.empty(3, dtype=torch.float32, device=dev)
        hist = torch.zeros(desc.SN, desc.V, dtype=torch.float32, device=dev) if want_hist else None
        saved = C.workspace(L.xq_ms_saved_bytes(desc), dev)
        ws = C.workspace(L.xq_ms_workspace_bytes(desc), dev)
        nk = 2 + (1 if desc.channel_norm else 0) + (1 if E is not None else 1) + (1 if desc.mode == C.XQ_MS_BSQ_HARD else 0)
        try:
            C.call("xq_ms_forward", nk, L.xq_ms_forward, desc, C.ptr(f), C.ptr(E), C.ptr(phi_w), C.ptr(phi_b), C.ptr(nq),
                   1, C.ptr(out), C.ptr(idx_all), None, C.ptr(loss), C.ptr(hist), C.ptr(saved), C.ptr(ws), ws.numel(),
                   C.stream_ptr(dev))
        except C.XqError as e:
            # most refusals are shape limits (one image's forward or backward working set in shared memory)
            raise C.XqError(f"{e} (B = {desc.B}, C = {desc.C}, last scale {desc.H} x {desc.W})") from None
        ctx.desc = desc
        ctx.has = (E is not None, phi_w is not None)
        ctx.save_for_backward(f, E, phi_w, phi_b, nq, idx_all, saved)
        ctx.mark_non_differentiable(idx_all)
        if hist is not None:
            ctx.mark_non_differentiable(hist)
        return out, loss[0], loss[1], loss[2], idx_all, hist

    @staticmethod
    def backward(ctx, g_out, g_vq, g_commit, g_ent, _gi, _gh):
        f, E, phi_w, phi_b, nq, idx_all, saved = ctx.saved_tensors
        desc = ctx.desc
        dev = f.device
        L = C.lib()
        g_out, g_vq, g_commit, g_ent = map(_f32c, (g_out, g_vq, g_commit, g_ent))
        gf = torch.empty_like(f)
        gE = torch.empty_like(E) if E is not None else None
        gw = torch.empty_like(phi_w) if phi_w is not None else None
        gb = torch.empty_like(phi_b) if phi_b is not None else None
        ws = C.workspace(L.xq_ms_workspace_bytes(desc), dev)
        nk = 1 + (2 if phi_w is not None else 0) + (1 if (E is None and g_ent is not None) else 0)
        nk += 1 if (desc.mode == C.XQ_MS_BSQ_HARD and g_ent is not None) else 0
        C.call("xq_ms_backward", nk, L.xq_ms_backward, desc, C.ptr(f), C.ptr(E), C.ptr(phi_w), C.ptr(phi_b), C.ptr(nq),
               C.ptr(idx_all), C.ptr(saved), C.ptr(g_out), C.ptr(g_vq), C.ptr(g_commit), C.ptr(g_ent), C.ptr(gf),
               C.ptr(gE), C.ptr(gw), C.ptr(gb), C.ptr(ws), ws.numel(), C.stream_ptr(dev))
        return gf, gE, gw, gb, None, None, None


def ms_forward(f, E, phi_w, phi_b, n_quantizers, desc, want_hist=True):
    return _MSForward.apply(f, E, phi_w, phi_b, n_quantizers, desc, want_hist)


def split_scales(idx_all: torch.Tensor, B: int, patch_nums: Sequence[int]) -> List[torch.Tensor]:
    out, off = [], 0
    for p in patch_nums:
        n = B * p * p
        out.append(idx_all[off:off + n].view(B, p * p))
        off += n
    return out


@torch.no_grad()
def ms_lookup(f, E, phi_w, phi_b, desc, want_fhat_scales: bool):
    """inference loop (quant.py:182-223): returns (f_hat_last, idx_all, fhat_scales|None)."""
    f, E, phi_w, phi_b = map(_f32c, (f, E, phi_w, phi_b))
    dev = f.device
    L = C.lib()
    idx_all = _ms_idx_buffer(L, desc, dev)
    out = torch.empty_like(f)
    fs = torch.empty((desc.SN,) + tuple(f.shape), dtype=torch.float32, device=dev) if want_fhat_scales else None
    ws = C.workspace(L.xq_ms_workspace_bytes(desc), dev)
    nk = 1 + (1 if desc.channel_norm else 0) + (1 if E is not None else 0)
    C.call("xq_ms_lookup", nk, L.xq_ms_forward, desc, C.ptr(f), C.ptr(E), C.ptr(phi_w), C.ptr(phi_b), None, 0,
           C.ptr(out), C.ptr(idx_all), C.ptr(fs), None, None, None, C.ptr(ws), ws.numel(), C.stream_ptr(dev))
    return out, idx_all, fs


@torch.no_grad()
def ms_decode(idx_all, E, phi_w, phi_b, desc, want_out=True, want_fhat_scales=False, want_var_input=False):
    """indices -> f_hat / per-scale f_hat / next-scale inputs (quant.py:148-180, 226-244)."""
    dev = idx_all.device
    E, phi_w, phi_b = map(_f32c, (E, phi_w, phi_b))
    shape = (desc.B, desc.C, desc.H, desc.W)
    out = torch.empty(shape, dtype=torch.float32, device=dev) if want_out else None
    fs = torch.empty((desc.SN,) + shape, dtype=torch.float32, device=dev) if want_fhat_scales else None
    Lv = sum(int(desc.patch_nums[i]) ** 2 for i in range(1, desc.SN))
    var = torch.empty(desc.B, Lv, desc.C, dtype=torch.float32, device=dev) if (want_var_input and Lv > 0) else None
    L = C.lib()
    C.call("xq_ms_decode", 1, L.xq_ms_decode, desc, C.ptr(idx_all.contiguous()), C.ptr(E), C.ptr(phi_w), C.ptr(phi_b),
           C.ptr(out), C.ptr(fs), C.ptr(var), C.stream_ptr(dev))
    return out, fs, var


@torch.no_grad()
def ms_embed(h_all, phi_w, phi_b, desc, si0: int, si1: int, f_hat=None, want_scales=False, want_next=False):
    """feature-map form of the per-scale step (quant.py:148-166, 247-258): for si in [si0, si1)
    f_hat += Phi_si(bicubic_up(h_si)).  `f_hat` (fp32 [B,C,H,W], contiguous) is updated IN PLACE when given, as the
    reference's f_hat.add_ does.  -> (f_hat, per-scale cumulative f_hat [si1-si0,B,C,H,W] | None, next | None)"""
    dev = h_all.device
    phi_w, phi_b = _f32c(phi_w), _f32c(phi_b)
    shape = (desc.B, desc.C, desc.H, desc.W)
    if f_hat is not None:
        if tuple(f_hat.shape) != shape or f_hat.dtype != torch.float32 or not f_hat.is_contiguous():
            raise ValueError(f"f_hat must be a contiguous float32 tensor of shape {shape}")
        out, fin = f_hat, f_hat
    else:
        out, fin = torch.empty(shape, dtype=torch.float32, device=dev), None
    fs = torch.empty((si1 - si0,) + shape, dtype=torch.float32, device=dev) if want_scales else None
    nxt = None
    if want_next and si1 < desc.SN:
        pn = int(desc.patch_nums[si1])
        nxt = torch.empty(desc.B, desc.C, pn, pn, dtype=torch.float32, device=dev)
    L = C.lib()
    C.call("xq_ms_embed", 1, L.xq_ms_embed, desc, int(si0), int(si1), C.ptr(h_all), C.ptr(phi_w), C.ptr(phi_b),
           C.ptr(fin), C.ptr(out), C.ptr(fs), C.ptr(nxt), C.stream_ptr(dev))
    return out, fs, nxt
