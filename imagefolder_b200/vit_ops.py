"""Fused ViT block glue over libxqb200 (csrc/vit_kernels.cu).

`run_blocks(vit, x)` walks `vit.blocks` + `vit.norm` exactly like the reference
(dino_enc/dinov2.py:183-190 -> vision_transformer.py:336-339) but replaces every chain
   [+ residual] -> LayerScale -> DropPath -> add -> LayerNorm -> cast-to-bf16
by ONE kernel (`xq_vit_residual_ln_fwd`), GELU by one bf16 kernel and attention by the wgmma / TMA flash
kernels of csrc/attn_kernel.cu (`xq_vit_attn_fwd/bwd`, reading the packed qkv projection in place and writing d(qkv)
in the packed layout); the projection GEMMs stay on cuBLAS.  Blocks the attention kernels do not cover (head dims other
than 64, attention dropout > 0 in training, qk_norm; no shipped config) run the module's own Attention.forward for
their attention.  The residual stream is fp32 and the GEMM operands are the autocast dtype, bf16 or fp16: the
`_f16` twin of every entry point runs the same kernel instantiated for fp16.  That is what bf16 / fp16 autocast gives the
reference, so the numerics are the reference's.  Without autocast (or under another autocast dtype) `run_blocks` takes the
module path.  `frozen_forward` runs a frozen VisionTransformer (the guide teachers) on the same block body (`block_forward`),
without saved activations, and with a class-token-only last block for `forward`.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _capi as C

_SUPPORTED_D = (384, 768, 1024, 1536)
_HALF = (torch.bfloat16, torch.float16)       # the GEMM operand dtypes the kernels are instantiated for


def _autocast_half():
    """the CUDA autocast dtype when autocast is on and it is bf16 or fp16, else None"""
    if not torch.is_autocast_enabled():
        return None
    dt = torch.get_autocast_dtype("cuda")
    return dt if dt in _HALF else None


def _op_dtype():
    """16-bit operand dtype of a glue kernel whose inputs do not fix it: fp16 under fp16 autocast, else bf16"""
    return torch.float16 if _autocast_half() == torch.float16 else torch.bfloat16


def _entry(name: str, dt):
    """(symbol name, function) of entry point `name` for 16-bit dtype `dt`: its `_f16` twin for fp16, else the bf16 one"""
    if dt == torch.float16:
        name += "_f16"
    return name, getattr(C.lib(), name)


def _lora():
    from .dino_enc import lora          # imported here: dino_enc imports this module
    return lora


def _live(m):
    """the module that runs `m`'s forward: the trainable copy of a LoRA `modules_to_save` wrapper (dino_enc/lora.py), else `m`"""
    return _lora().active_module(m)


class _ResidualLN(torch.autograd.Function):
    """(x, branch, branch_bias, ls_gamma, rowscale, ln_w, ln_b) -> (x_out fp32, y 16-bit)
    x_out = x + rowscale * ls_gamma * (branch + branch_bias);  y = LayerNorm(x_out).
    branch / y are fp16 under fp16 autocast, else bf16 (_op_dtype)."""

    @staticmethod
    def forward(ctx, x, branch, branch_bias, ls_gamma, rowscale, ln_w, ln_b, eps: float):
        Bn, S, D = x.shape
        M = Bn * S
        dt = _op_dtype()
        x = x.contiguous()
        if x.dtype != torch.float32:
            x = x.float()
        if branch is not None:
            branch = branch.contiguous()
            if branch.dtype != dt:
                branch = branch.to(dt)
        x_out = torch.empty_like(x)
        y = torch.empty(x.shape, dtype=dt, device=x.device)
        mean = torch.empty(M, dtype=torch.float32, device=x.device)
        rstd = torch.empty(M, dtype=torch.float32, device=x.device)
        name, fn = _entry("xq_vit_residual_ln_fwd", dt)
        C.call(name, 1, fn, C.ptr(x), C.ptr(branch), C.ptr(branch_bias),
               C.ptr(ls_gamma), C.ptr(rowscale), S, C.ptr(ln_w), C.ptr(ln_b), float(eps), M, D, C.ptr(x_out), C.ptr(y),
               C.ptr(mean), C.ptr(rstd), C.stream_ptr(x.device),
               nbytes=M * D * (10 + (2 if branch is not None else 0)))
        ctx.save_for_backward(x_out, mean, rstd, ln_w, branch, branch_bias, ls_gamma, rowscale)
        ctx.shape = (Bn, S, D)
        ctx.dt = dt
        ctx.set_materialize_grads(False)
        return x_out, y

    @staticmethod
    def backward(ctx, g_xout, g_y):
        x_out, mean, rstd, ln_w, branch, branch_bias, ls_gamma, rowscale = ctx.saved_tensors
        Bn, S, D = ctx.shape
        M = Bn * S
        dev = x_out.device
        if g_xout is not None:
            g_xout = g_xout.contiguous()
            if g_xout.dtype != torch.float32:
                g_xout = g_xout.float()
        if g_y is not None:
            g_y = g_y.contiguous()
            if g_y.dtype != ctx.dt:
                g_y = g_y.to(ctx.dt)
        g_x = torch.empty_like(x_out)
        g_branch = torch.empty_like(branch) if branch is not None else None
        g_w = torch.empty_like(ln_w)
        g_b = torch.empty_like(ln_w)
        g_g = torch.empty_like(ls_gamma) if (branch is not None and ls_gamma is not None) else None
        g_bb = torch.empty_like(branch_bias) if (branch is not None and branch_bias is not None) else None
        L = C.lib()
        ws = C.workspace(L.xq_vit_ln_bwd_workspace_bytes(D), dev)
        name, fn = _entry("xq_vit_residual_ln_bwd", ctx.dt)
        C.call(name, 2, fn, C.ptr(g_xout), C.ptr(g_y), C.ptr(x_out),
               C.ptr(mean), C.ptr(rstd), C.ptr(ln_w), C.ptr(branch), C.ptr(branch_bias), C.ptr(ls_gamma),
               C.ptr(rowscale), S, M, D, C.ptr(g_x), C.ptr(g_branch), C.ptr(g_w), C.ptr(g_b), C.ptr(g_g), C.ptr(g_bb),
               C.ptr(ws), ws.numel(), C.stream_ptr(dev),
               nbytes=M * D * (8 + (4 if g_xout is not None else 0) + (2 if g_y is not None else 0)
                               + (4 if branch is not None else 0)))
        return g_x, g_branch, g_bb, g_g, None, g_w, g_b, None


def residual_ln(x, branch, branch_bias, ls_gamma, rowscale, ln_w, ln_b, eps=1e-6):
    return _ResidualLN.apply(x, branch, branch_bias, ls_gamma, rowscale, ln_w, ln_b, eps)


class _GeluBias(torch.autograd.Function):
    """y = GELU(x + bias), x bf16 or fp16 [..., C] (the fc1 GEMM output WITHOUT its bias), bias fp32 [C]."""

    @staticmethod
    def forward(ctx, x, bias):
        x = x.contiguous()
        Cc = x.shape[-1]
        M = x.numel() // Cc
        y = torch.empty_like(x)
        name, fn = _entry("xq_vit_gelu_fwd", x.dtype)
        C.call(name, 1, fn, C.ptr(x), C.ptr(bias), C.ptr(y), M, Cc, C.stream_ptr(x.device),
               nbytes=M * Cc * 4)
        ctx.save_for_backward(x, bias)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, bias = ctx.saved_tensors
        gy = gy.contiguous()
        dt = torch.float16 if x.dtype == torch.float16 else torch.bfloat16
        if gy.dtype != dt:
            gy = gy.to(dt)
        Cc = x.shape[-1]
        M = x.numel() // Cc
        gx = torch.empty_like(x)
        gb = torch.empty_like(bias) if bias is not None else None
        name, fn = _entry("xq_vit_gelu_bwd", dt)
        C.call(name, 1, fn, C.ptr(x), C.ptr(bias), C.ptr(gy), C.ptr(gx), C.ptr(gb), M, Cc,
               C.stream_ptr(x.device), nbytes=M * Cc * 6)
        return gx, gb


def gelu_bias(x, bias=None):
    return _GeluBias.apply(x, bias)


MLP_TC_ENABLED = [True]       # the wgmma GEMMs with fused GELU / GELU' epilogues (csrc/gemm_kernel.cu)
_SM_COUNT = {}                # device index -> multiprocessor count


def _sm_count(device) -> int:
    idx = device.index if device.index is not None else torch.cuda.current_device()
    n = _SM_COUNT.get(idx)
    if n is None:
        n = _SM_COUNT[idx] = torch.cuda.get_device_properties(idx).multi_processor_count
    return n


def mlp_tc_ok(y, fc1, fc2) -> bool:
    """xq_vit_fc1_gelu_fwd / xq_vit_fc2_dgelu_bwd (and their _f16 twins) cover the shipped widths: bf16 or fp16 tokens,
    hidden % 256 == 0, embed % 64 == 0,
    out % 64 == 0 (the K of the backward GEMM), and at most one CTA column per SM (hidden / 128 <= SM count)."""
    return (MLP_TC_ENABLED[0] and y.is_cuda and y.dtype in _HALF and fc1.bias is not None
            and fc1.weight.shape[0] % 256 == 0 and fc1.weight.shape[1] % 64 == 0
            and fc2.weight.shape[1] == fc1.weight.shape[0] and fc2.weight.shape[0] % 64 == 0
            and fc1.weight.shape[0] // 128 <= _sm_count(y.device))


def _keeps_pre(ctx) -> bool:
    """whether a fused fc1 forward must store and save its pre-activation: only when some input needs a gradient.  A
    forward whose inputs all do without one (a frozen teacher, a model with every parameter frozen) passes NULL for `pre`
    -- the kernel then stores `act` only, the same bits -- and saves nothing for a backward that cannot run."""
    return any(ctx.needs_input_grad)


class _FusedMLP(torch.autograd.Function):
    """branch = fc2(GELU(fc1(y)))  WITHOUT the fc2 bias (folded into the next residual_ln), timm Mlp as called from Block.forward
    (dino_enc/vision_transformer.py:336-339).  The fc1 GEMM carries bias + GELU in its epilogue, the fc2 input-gradient GEMM carries
    GELU' and the fc1-bias gradient; the other GEMMs are library calls.  Same bits as F.linear + gelu_bias (the epilogues apply
    the same device functions to the same rounded 16-bit values).  Operands, weights and outputs in y's dtype, bf16 or fp16.
    When no input needs a gradient (a frozen teacher) the fc1 GEMM writes no `pre` and nothing is saved (_keeps_pre)."""

    @staticmethod
    def forward(ctx, y, W1, b1, W2):
        K = W1.shape[1]
        N = W1.shape[0]
        y2 = y.reshape(-1, K)
        if not y2.is_contiguous():
            y2 = y2.contiguous()
        M = y2.shape[0]
        dt = y.dtype
        W1b = W1.to(dt)
        W2b = W2.to(dt)
        b1f = b1.float()
        keep = _keeps_pre(ctx)
        pre = torch.empty(M, N, dtype=dt, device=y.device) if keep else None
        act = torch.empty(M, N, dtype=dt, device=y.device)
        name, fn = _entry("xq_vit_fc1_gelu_fwd", dt)
        C.call(name, 1, fn, C.ptr(y2), C.ptr(W1b), C.ptr(b1f), C.ptr(pre), C.ptr(act), M, N, K,
               C.stream_ptr(y.device), nbytes=M * K * 2 + N * K * 2 + M * N * (4 if keep else 2), nflops=2.0 * M * N * K)
        branch = act @ W2b.t()
        if keep:
            ctx.save_for_backward(y2, pre, act, W1b, W2b, b1f)
        ctx.out_shape = y.shape[:-1] + (W2.shape[0],)
        ctx.in_shape = y.shape
        return branch.view(ctx.out_shape)

    @staticmethod
    def backward(ctx, g):
        y2, pre, act, W1b, W2b, b1f = ctx.saved_tensors
        M, N = pre.shape
        Ko = W2b.shape[0]
        g2 = g.reshape(M, Ko)
        if g2.dtype != pre.dtype:
            g2 = g2.to(pre.dtype)
        if not g2.is_contiguous():
            g2 = g2.contiguous()
        dW2 = (g2.t() @ act).float() if ctx.needs_input_grad[3] else None
        W2t = W2b.t().contiguous()                      # [hidden, out]: the K-major B operand of d_act = g W2
        dpre = torch.empty_like(pre)
        db1 = torch.empty(N, dtype=torch.float32, device=pre.device)
        name, fn = _entry("xq_vit_fc2_dgelu_bwd", pre.dtype)
        C.call(name, 1, fn, C.ptr(g2), C.ptr(W2t), C.ptr(pre), C.ptr(b1f), C.ptr(dpre), C.ptr(db1),
               M, N, Ko, C.stream_ptr(pre.device), nbytes=M * Ko * 2 + N * Ko * 2 + M * N * 4, nflops=2.0 * M * N * Ko)
        dW1 = (dpre.t() @ y2).float() if ctx.needs_input_grad[1] else None
        dy = (dpre @ W1b).view(ctx.in_shape) if ctx.needs_input_grad[0] else None
        return dy, dW1, (db1 if ctx.needs_input_grad[2] else None), dW2


class _SwiGLUBias(torch.autograd.Function):
    """act = silu(a) * c with a = x[..., :H] + bias[:H], c = x[..., H:] + bias[H:], x bf16 or fp16 [..., 2H] (the fc1 GEMM
    output WITHOUT its bias), bias fp32 [2H] (timm GluMlp, gate_last=False)."""

    @staticmethod
    def forward(ctx, x, bias):
        x = x.contiguous()
        H = x.shape[-1] // 2
        M = x.numel() // (2 * H)
        act = torch.empty(x.shape[:-1] + (H,), dtype=x.dtype, device=x.device)
        name, fn = _entry("xq_vit_swiglu_fwd", x.dtype)
        C.call(name, 1, fn, C.ptr(x), C.ptr(bias), C.ptr(act), M, H, C.stream_ptr(x.device), nbytes=M * H * 6)
        ctx.save_for_backward(x, bias)
        return act

    @staticmethod
    def backward(ctx, g):
        x, bias = ctx.saved_tensors
        g = g.contiguous()
        if g.dtype != x.dtype:
            g = g.to(x.dtype)
        H = x.shape[-1] // 2
        M = x.numel() // (2 * H)
        gx = torch.empty_like(x)
        gb = torch.empty_like(bias) if bias is not None else None
        name, fn = _entry("xq_vit_swiglu_bwd", x.dtype)
        C.call(name, 1, fn, C.ptr(x), C.ptr(bias), C.ptr(g), C.ptr(gx), C.ptr(gb), M, H, C.stream_ptr(x.device),
               nbytes=M * H * 10)
        return gx, gb


def swiglu_bias(x, bias=None):
    return _SwiGLUBias.apply(x, bias)


def _scaled_mm(a, b, s: float):
    """16-bit(s * (a @ b)) in a's dtype: the scale applied to the fp32 accumulator, one rounding"""
    return torch.addmm(a.new_zeros(()), a, b, beta=0, alpha=s)


def _pad_rank(t, dim: int, R: int):
    """zero rows (dim 0) / columns (dim 1) up to rank R: the kernel's rank stage needs R % 8 == 0"""
    n = t.shape[dim]
    if n == R:
        return t.contiguous()
    return F.pad(t, (0, R - n) if dim == 1 else (0, 0, 0, R - n))


class _LoRAMLP(torch.autograd.Function):
    """branch = fc2(GELU(fc1(y))) WITHOUT the fc2 bias, fc1 / fc2 LoRA-wrapped (dino_enc/lora.py, lora_dropout inactive):
    fc(x) = x W^T + b + s (x A^T) B^T.  With u = 16-bit(s1 y A1^T) and v = 16-bit(s2 g B2) (rank-r library GEMMs; every
    16-bit tensor in y's dtype, bf16 or fp16):
      forward   pre = y W1^T + u B1^T, act = GELU(pre + b1)      xq_vit_fc1_lora_gelu_fwd (u B1^T: one more K stage)
                branch = act W2^T + s2 (act A2^T) B2^T           library
      backward  d_pre = (g W2 + v A2) * GELU'(pre + b1), d_b1   xq_vit_fc2_lora_dgelu_bwd
                dy = d_pre W1 + s1 (d_pre B1) A1, the four adapter gradients, and dW1 / dW2 / d_b1 only for parameters that
                require grad (LoRA freezes them: their GEMMs are not run).
    The base and rank-r products of `pre` / `d_act` share one fp32 accumulator and one rounding (DESIGN.md section 8).
    No `pre` and nothing saved when no input needs a gradient (_keeps_pre)."""

    @staticmethod
    def forward(ctx, y, W1, b1, W2, A1, B1, A2, B2, s1: float, s2: float):
        K, N = W1.shape[1], W1.shape[0]
        y2 = y.reshape(-1, K)
        if not y2.is_contiguous():
            y2 = y2.contiguous()
        M = y2.shape[0]
        r = A1.shape[0]
        R = -(-r // 8) * 8
        bf = y.dtype
        W1b, W2b, b1f = W1.to(bf), W2.to(bf), b1.float()
        A1b, B1b = _pad_rank(A1.to(bf), 0, R), _pad_rank(B1.to(bf), 1, R)           # [R, K], [N, R]
        A2b, B2b = _pad_rank(A2.to(bf), 0, R), _pad_rank(B2.to(bf), 1, R)           # [R, N], [Ko, R]
        u = _scaled_mm(y2, A1b.t(), s1)
        keep = _keeps_pre(ctx)
        pre = torch.empty(M, N, dtype=bf, device=y.device) if keep else None
        act = torch.empty(M, N, dtype=bf, device=y.device)
        name, fn = _entry("xq_vit_fc1_lora_gelu_fwd", bf)
        C.call(name, 1, fn, C.ptr(y2), C.ptr(W1b), C.ptr(u), C.ptr(B1b), C.ptr(b1f),
               C.ptr(pre), C.ptr(act), M, N, K, R, C.stream_ptr(y.device),
               nbytes=M * (K + R) * 2 + N * (K + R) * 2 + M * N * (4 if keep else 2), nflops=2.0 * M * N * (K + R))
        h2 = _scaled_mm(act, A2b.t(), s2)
        branch = torch.addmm(act @ W2b.t(), h2, B2b.t())
        if keep:
            ctx.save_for_backward(y2, pre, act, u, h2, W1b, W2b, b1f, A1b, B1b, A2b, B2b)
        ctx.cfg = (s1, s2, r)
        ctx.out_shape = y.shape[:-1] + (W2.shape[0],)
        ctx.in_shape = y.shape
        return branch.view(ctx.out_shape)

    @staticmethod
    def backward(ctx, g):
        y2, pre, act, u, h2, W1b, W2b, b1f, A1b, B1b, A2b, B2b = ctx.saved_tensors
        s1, s2, r = ctx.cfg
        need = ctx.needs_input_grad
        M, N = pre.shape
        Ko, R = W2b.shape[0], A1b.shape[0]
        g2 = g.reshape(M, Ko)
        if g2.dtype != pre.dtype:
            g2 = g2.to(pre.dtype)
        if not g2.is_contiguous():
            g2 = g2.contiguous()
        v = _scaled_mm(g2, B2b, s2)                     # [M, R]
        W2t = W2b.t().contiguous()                      # [hidden, out]: the K-major B operand of d_act = g W2
        A2t = A2b.t().contiguous()                      # [hidden, R]: the K-major adapter of the rank stage v A2
        dpre = torch.empty_like(pre)
        db1 = torch.empty(N, dtype=torch.float32, device=pre.device)
        name, fn = _entry("xq_vit_fc2_lora_dgelu_bwd", pre.dtype)
        C.call(name, 1, fn, C.ptr(g2), C.ptr(W2t), C.ptr(v), C.ptr(A2t), C.ptr(pre),
               C.ptr(b1f), C.ptr(dpre), C.ptr(db1), M, N, Ko, R, C.stream_ptr(pre.device),
               nbytes=M * (Ko + R) * 2 + N * (Ko + R) * 2 + M * N * 4, nflops=2.0 * M * N * (Ko + R))
        t1 = _scaled_mm(dpre, B1b, s1)                  # [M, R] = s1 d_pre B1
        dy = torch.addmm(dpre @ W1b, t1, A1b).view(ctx.in_shape) if need[0] else None
        dW1 = (dpre.t() @ y2).float() if need[1] else None
        dW2 = (g2.t() @ act).float() if need[3] else None
        dA1 = (t1.t() @ y2).float()[:r] if need[4] else None
        dB1 = (dpre.t() @ u).float()[:, :r] if need[5] else None
        dA2 = (v.t() @ act).float()[:r] if need[6] else None
        dB2 = (g2.t() @ h2).float()[:, :r] if need[7] else None
        return dy, dW1, (db1 if need[2] else None), dW2, dA1, dB1, dA2, dB2, None, None


def _lora_off(fc) -> bool:
    """a LoRA Linear whose lora_dropout does nothing"""
    d = fc.lora_dropout[fc.active_adapter]
    return isinstance(d, nn.Identity) or not d.training or d.p == 0.0


def _linear_no_bias(fc, x):
    """fc(x) without its bias, for an nn.Linear or a LoRA Linear"""
    out = F.linear(x, fc.weight)
    return out + fc.lora_delta(x) if isinstance(fc, _lora().Linear) else out


def mlp_forward(mlp, y):
    """timm Mlp (fc1 -> GELU -> fc2, drop = 0) or GluMlp (fc1 -> SwiGLU -> fc2) without the fc2 bias.  Mlp: fused wgmma path
    when the shapes allow, else library GEMMs + the stand-alone bias / GELU kernel; LoRA-wrapped fc1 and fc2 with inactive
    lora_dropout and r <= 64 take the LoRA form of the fused path.  GluMlp: library GEMMs + the stand-alone SwiGLU kernel.  Any
    LoRA Linear off the fused path adds its `lora_delta` to a library GEMM."""
    fc1, fc2 = mlp.fc1, mlp.fc2
    lora = _lora()
    from .dino_enc.vision_transformer import GluMlp      # imported here: dino_enc imports this module
    if isinstance(mlp, GluMlp):
        # timm GluMlp (the giant backbones), plain or LoRA-wrapped fc1 / fc2: library GEMMs + the stand-alone SwiGLU kernel
        return _linear_no_bias(fc2, swiglu_bias(_linear_no_bias(fc1, y), fc1.bias))
    if isinstance(fc1, lora.Linear) or isinstance(fc2, lora.Linear):
        if (isinstance(fc1, lora.Linear) and isinstance(fc2, lora.Linear) and _lora_off(fc1) and _lora_off(fc2)
                and fc1.r[fc1.active_adapter] <= 64 and fc2.r[fc2.active_adapter] == fc1.r[fc1.active_adapter]
                and mlp_tc_ok(y, fc1, fc2)):
            a1, a2 = fc1.active_adapter, fc2.active_adapter
            return _LoRAMLP.apply(y, fc1.weight, fc1.bias, fc2.weight, fc1.lora_A[a1].weight, fc1.lora_B[a1].weight,
                                  fc2.lora_A[a2].weight, fc2.lora_B[a2].weight, fc1.scaling[a1], fc2.scaling[a2])
        return _linear_no_bias(fc2, gelu_bias(_linear_no_bias(fc1, y), fc1.bias))
    if mlp_tc_ok(y, fc1, fc2):
        return _FusedMLP.apply(y, fc1.weight, fc1.bias, fc2.weight)
    h = gelu_bias(F.linear(y, fc1.weight), fc1.bias)
    return F.linear(h, fc2.weight)


# The wgmma attention kernels (csrc/attn_kernel.cu).  False runs every block's attention through the module's own
# Attention.forward.  bench.py reads it: while it is True, the benchmarked step must show the attention kernels.
ATTN_TC_ENABLED = [True]


def attn_tc_ok(attn, y) -> bool:
    """xq_vit_attn_fwd/bwd (and their _f16 twins) cover what the shipped configs run: bf16 or fp16 CUDA tokens, head_dim 64, no qk_norm, no mask and
    an attention dropout of 0 where it applies (training)."""
    p = attn.attn_drop.p if attn.training else 0.0
    return (ATTN_TC_ENABLED[0] and y.is_cuda and y.dtype in _HALF and p == 0.0 and attn.head_dim == 64
            and isinstance(_live(attn.q_norm), nn.Identity) and isinstance(_live(attn.k_norm), nn.Identity))


def attn_tc_forward(qkv, num_heads: int):
    """qkv bf16 or fp16 [B,N,3*H*64] (packed projection, read in place) -> (out [B,N,H*64] in qkv's dtype, lse2 fp32 [B,H,N])."""
    B, N, C3 = qkv.shape
    qkv = qkv.contiguous()
    out = torch.empty(B, N, C3 // 3, dtype=qkv.dtype, device=qkv.device)
    lse2 = torch.empty(B, num_heads, N, dtype=torch.float32, device=qkv.device)
    name, fn = _entry("xq_vit_attn_fwd", qkv.dtype)
    C.call(name, 1, fn, C.ptr(qkv), C.ptr(out), C.ptr(lse2), B, N, num_heads, 64, 0.125,
           C.stream_ptr(qkv.device), nbytes=qkv.numel() * 2 + out.numel() * 2 + lse2.numel() * 4,
           nflops=4.0 * B * num_heads * N * N * 64)
    return out, lse2


def attn_cls_forward(qkv, num_heads: int):
    """qkv bf16 or fp16 [B,N,3*H*64] -> the attention output of query row 0 only, [B,H*64] in qkv's dtype
    (xq_vit_attn_fwd_cls: fp32 on CUDA cores, fixed summation order).  Inference only: there is no backward."""
    B, N, C3 = qkv.shape
    qkv = qkv.contiguous()
    out = torch.empty(B, C3 // 3, dtype=qkv.dtype, device=qkv.device)
    name, fn = _entry("xq_vit_attn_fwd_cls", qkv.dtype)
    C.call(name, 1, fn, C.ptr(qkv), C.ptr(out), B, N, num_heads, 64, 0.125, C.stream_ptr(qkv.device),
           nbytes=B * N * (C3 // 3) * 4 + out.numel() * 2)
    return out


def attn_tc_backward(qkv, out, lse2, g, num_heads: int, want_bias_grad: bool = False):
    """d(out) [B,N,H*64] -> d(qkv) [B,N,3*H*64] in qkv's dtype (bf16 or fp16), written directly in the packed layout
    (+ its column sums = the qkv-bias gradient, fp32 [3*H*64], when asked for)."""
    B, N, C3 = qkv.shape
    g = g.contiguous()
    if g.dtype != qkv.dtype:
        g = g.to(qkv.dtype)
    dqkv = torch.empty_like(qkv)
    db = torch.empty(C3, dtype=torch.float32, device=qkv.device) if want_bias_grad else None
    nbytes = int(C.lib().xq_vit_attn_bwd_workspace_bytes(B, N, num_heads))
    ws = C.stream_workspace("xq_vit_attn_bwd", nbytes, qkv.device)
    name, fn = _entry("xq_vit_attn_bwd", qkv.dtype)
    C.call(name, 3, fn, C.ptr(qkv), C.ptr(out), C.ptr(g), C.ptr(lse2), C.ptr(dqkv), C.ptr(db), B, N, num_heads,
           64, 0.125, C.ptr(ws), ws.numel(), C.stream_ptr(qkv.device),
           nbytes=qkv.numel() * 4 + out.numel() * 4 + lse2.numel() * 4, nflops=10.0 * B * num_heads * N * N * 64)
    return (dqkv, db) if want_bias_grad else dqkv


def _qkv_projection(y, W, b):
    """(W in y's dtype, qkv = y W^T (+ b) [B,N,3D]) for y [B,N,D]: the packed qkv projection as one library GEMM in y's dtype
    (autocast semantics)"""
    B, N, D = y.shape
    Wb = W.to(y.dtype)
    y2 = y.reshape(B * N, D)
    return Wb, (torch.addmm(b.to(y.dtype), y2, Wb.t()) if b is not None else y2 @ Wb.t()).view(B, N, 3 * D)


class _QKVAttention(torch.autograd.Function):
    """qkv = y W^T (+ b) ; attention(qkv)   (vision_transformer.py:175-191) as ONE autograd node on the wgmma kernels, so that
    the bias gradient is the column sum the attention backward already has in registers (no separate sum(0) pass over
    d(qkv)).  y [B,N,C] bf16 or fp16, W [3C,C] / b [3C] (or None) fp32 parameters; GEMMs are library calls in y's dtype
    (autocast semantics)."""

    @staticmethod
    def forward(ctx, y, W, b, num_heads: int):
        Wb, qkv = _qkv_projection(y, W, b)
        out, lse2 = attn_tc_forward(qkv, num_heads)
        ctx.save_for_backward(y, Wb, qkv, out, lse2)
        ctx.heads = num_heads
        return out

    @staticmethod
    def backward(ctx, g):
        y, Wb, qkv, out, lse2 = ctx.saved_tensors
        B, N, C = y.shape
        if ctx.needs_input_grad[2]:
            dqkv, db = attn_tc_backward(qkv, out, lse2, g, ctx.heads, want_bias_grad=True)
        else:
            dqkv, db = attn_tc_backward(qkv, out, lse2, g, ctx.heads), None
        d2 = dqkv.view(B * N, 3 * C)
        dy = (d2 @ Wb).view(B, N, C) if ctx.needs_input_grad[0] else None
        dW = (d2.t() @ y.reshape(B * N, C)).float() if ctx.needs_input_grad[1] else None
        return dy, dW, db, None


_ROPE_IMG = 256                # image tokens xq_vit_rope_fwd / _bwd cover (a 16 x 16 grid)


def rope_forward(qkv, freqs, freqs_1d_real, num_heads: int, P: int):
    """q / k of the packed qkv bf16 or fp16 [B,N,3*H*64] rotated (xq_vit_rope_fwd) into a new packed tensor; freqs fp32
    [2,H*32], freqs_1d_real fp32 [L,32,2] (view_as_real of the complex table)."""
    B, N, _ = qkv.shape
    out = torch.empty_like(qkv)
    name, fn = _entry("xq_vit_rope_fwd", qkv.dtype)
    C.call(name, 1, fn, C.ptr(qkv), C.ptr(out), C.ptr(freqs), C.ptr(freqs_1d_real), B, N, num_heads, 64, P, _ROPE_IMG,
           freqs_1d_real.shape[0], C.stream_ptr(qkv.device), nbytes=qkv.numel() * 4)
    return out


def rope_backward(qkv, g, freqs, freqs_1d_real, num_heads: int, P: int):
    """d(rotated qkv) -> (d(qkv) in qkv's dtype, qkv-bias gradient fp32 [3*H*64], d freqs fp32 [2,H*32], d freqs_1d fp32
    [L,32,2]) through xq_vit_rope_bwd: deterministic sums, no atomics."""
    B, N, C3 = qkv.shape
    L = freqs_1d_real.shape[0]
    g = g.contiguous()
    dqkv = torch.empty_like(qkv)
    db = torch.empty(C3, dtype=torch.float32, device=qkv.device)
    dfreqs = torch.empty_like(freqs)
    d1 = torch.empty_like(freqs_1d_real)
    nbytes = int(C.lib().xq_vit_rope_bwd_workspace_bytes(B, N, num_heads, L))
    ws = C.stream_workspace("xq_vit_rope_bwd", nbytes, qkv.device)
    name, fn = _entry("xq_vit_rope_bwd", qkv.dtype)
    C.call(name, 2, fn, C.ptr(qkv), C.ptr(g), C.ptr(freqs), C.ptr(freqs_1d_real), B, N, num_heads, 64, P, _ROPE_IMG, L,
           C.ptr(dqkv), C.ptr(db), C.ptr(dfreqs), C.ptr(d1), C.ptr(ws), ws.numel(), C.stream_ptr(qkv.device),
           nbytes=qkv.numel() * 6 + ws.numel() * 2)
    return dqkv, db, dfreqs, d1


class _RoPEQKVAttention(torch.autograd.Function):
    """RoPEAttention.forward (vision_transformer.py:238-270) up to the proj GEMM as one autograd node: qkv = y W^T (+ b)
    [library GEMM] -> q / k rotated [xq_vit_rope_fwd] -> attention [xq_vit_attn_fwd]; the backward runs xq_vit_attn_bwd,
    xq_vit_rope_bwd and the two library GEMMs.  The qkv-bias gradient is the column sum of the gradient BEFORE the rotation,
    which the RoPE backward computes; the attention backward's column sums (of the rotated gradient) are not used.  Saves the
    unrotated qkv next to the rotated one: one more [B,N,3C] 16-bit tensor per layer (DESIGN.md section 0)."""

    @staticmethod
    def forward(ctx, y, W, b, freqs, freqs_1d_real, num_heads: int, P: int):
        Wb, qkv = _qkv_projection(y, W, b)
        freqs, freqs_1d_real = freqs.contiguous(), freqs_1d_real.contiguous()
        rot = rope_forward(qkv, freqs, freqs_1d_real, num_heads, P)
        out, lse2 = attn_tc_forward(rot, num_heads)
        ctx.save_for_backward(y, Wb, qkv, rot, out, lse2, freqs, freqs_1d_real)
        ctx.cfg = (num_heads, P)
        return out

    @staticmethod
    def backward(ctx, g):
        y, Wb, qkv, rot, out, lse2, freqs, freqs_1d_real = ctx.saved_tensors
        H, P = ctx.cfg
        B, N, C = y.shape
        drot = attn_tc_backward(rot, out, lse2, g, H)
        dqkv, db, dfreqs, d1 = rope_backward(qkv, drot, freqs, freqs_1d_real, H, P)
        d2 = dqkv.view(B * N, 3 * C)
        need = ctx.needs_input_grad
        dy = (d2 @ Wb).view(B, N, C) if need[0] else None
        dW = (d2.t() @ y.reshape(B * N, C)).float() if need[1] else None
        return dy, dW, (db if need[2] else None), (dfreqs if need[3] else None), (d1 if need[4] else None), None, None


def rope_tc_ok(attn, y) -> bool:
    """the RoPE kernels cover what DINOv2Decoder(use_rope=True) builds: the attn_tc_ok gates, mixed frequencies, a 16 x 16
    image grid and a sequence of exactly prefix + 256 + latent tokens"""
    P, L = attn.num_prefix_tokens, attn.num_latent_tokens
    return (attn_tc_ok(attn, y) and attn.rope_mixed and attn.num_image_tokens == _ROPE_IMG and P >= 0 and L >= 1
            and y.shape[1] == P + _ROPE_IMG + L and attn.num_heads <= 64
            and tuple(attn.freqs.shape) == (2, attn.num_heads * 32) and tuple(attn.freqs_1d.shape) == (L, 32))


def attention_forward(attn, y):
    """Attention.forward (vision_transformer.py:173-197, no mask) or RoPEAttention.forward (:238-270) -> (branch, bias to fold
    into the next residual_ln).  On the wgmma (and RoPE) kernels the proj GEMM leaves its bias to the caller; otherwise the
    module's own forward, bias included."""
    from .dino_enc.vision_transformer import RoPEAttention      # imported here: dino_enc imports this module
    if isinstance(attn, RoPEAttention):
        if not rope_tc_ok(attn, y):
            return attn(y), None
        o = _RoPEQKVAttention.apply(y, attn.qkv.weight, attn.qkv.bias, attn.freqs, torch.view_as_real(attn.freqs_1d),
                                    attn.num_heads, attn.num_prefix_tokens)
        return F.linear(o, attn.proj.weight), attn.proj.bias
    if not attn_tc_ok(attn, y):
        return attn(y), None
    o = _QKVAttention.apply(y, attn.qkv.weight, attn.qkv.bias, attn.num_heads)
    return F.linear(o, attn.proj.weight), attn.proj.bias


class _PatchEmbed(torch.autograd.Function):
    """timm PatchEmbed (Conv2d(kernel = stride = p) -> flatten(2).transpose(1,2)) as im2col-permutation + ONE GEMM.
    x fp32 [B,Cin,H,W] (no gradient), W [D,Cin,p,p] / b [D] fp32 parameters -> tokens [B, gh*gw, D] in the autocast dtype
    (bf16 or fp16)."""

    @staticmethod
    def forward(ctx, x, W, b):
        Bn, Cin, H, Wd = x.shape
        D, p = W.shape[0], W.shape[2]
        x = x.contiguous()
        M, K = Bn * (H // p) * (Wd // p), Cin * p * p
        dt = _op_dtype()
        patches = torch.empty(M, K, dtype=dt, device=x.device)
        name, fn = _entry("xq_vit_patchify", dt)
        C.call(name, 1, fn, C.ptr(x), C.ptr(patches), Bn, Cin, H, Wd, p, C.stream_ptr(x.device),
               nbytes=x.numel() * 6)
        Wb = W.reshape(D, K).to(dt)
        if b is not None:
            y = torch.addmm(b.to(dt), patches, Wb.t())
        else:
            y = patches @ Wb.t()
        ctx.save_for_backward(patches)
        ctx.wshape = tuple(W.shape)
        ctx.has_bias = b is not None
        return y.view(Bn, M // Bn, D)

    @staticmethod
    def backward(ctx, g):
        (patches,) = ctx.saved_tensors
        D = ctx.wshape[0]
        g2 = g.reshape(-1, D)
        if g2.dtype != patches.dtype:
            g2 = g2.to(patches.dtype)
        dW = (g2.t() @ patches).float().view(ctx.wshape) if ctx.needs_input_grad[1] else None
        db = g2.float().sum(0) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        return None, dW, db


def patch_embed_ok(pe, x) -> bool:
    p = pe.patch_size[0]
    proj = _live(pe.proj)
    return (x.is_cuda and x.dtype == torch.float32 and not x.requires_grad and _autocast_half() is not None
            and isinstance(_live(pe.norm), nn.Identity)
            and pe.patch_size[0] == pe.patch_size[1] and p % 4 == 0 and x.shape[2] % p == 0 and x.shape[3] % p == 0
            and tuple(proj.stride) == tuple(proj.kernel_size) and tuple(proj.padding) == (0, 0))


def patch_embed(pe, x):
    """PatchEmbed.forward on the fused path when it applies (bf16 or fp16 autocast, fp32 CUDA image that needs no gradient,
    patch % 4 == 0, no norm); otherwise the module's own conv."""
    if patch_embed_ok(pe, x):
        proj = _live(pe.proj)
        return _PatchEmbed.apply(x, proj.weight, proj.bias)
    return pe(x)


_ASSEMBLE_TYPE = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}    # src_type of xq_vit_assemble_fwd/bwd


class _Assemble(torch.autograd.Function):
    """out[b,t] = table[t] + (t0 <= t < t0+Ls ? src[b,t-t0] : 0)  -- the encoder / decoder token assembly as one pass."""

    @staticmethod
    def forward(ctx, src, table, t0: int):
        src = src.contiguous()
        if src.dtype not in _ASSEMBLE_TYPE:
            src = src.float()
        table = table.float().contiguous()
        B, Ls, D = src.shape
        T = table.shape[-2]
        out = torch.empty(B, T, D, dtype=torch.float32, device=src.device)
        L = C.lib()
        C.call("xq_vit_assemble_fwd", 1, L.xq_vit_assemble_fwd, C.ptr(src), _ASSEMBLE_TYPE[src.dtype], C.ptr(table), B, Ls, T,
               D, int(t0), C.ptr(out), C.stream_ptr(src.device), nbytes=out.numel() * 4 + src.numel() * src.element_size())
        ctx.cfg = (B, Ls, T, D, int(t0), src.dtype, tuple(table.shape))
        return out

    @staticmethod
    def backward(ctx, g):
        B, Ls, T, D, t0, sdt, tshape = ctx.cfg
        g = g.contiguous()
        if g.dtype != torch.float32:
            g = g.float()
        d_src = torch.empty(B, Ls, D, dtype=sdt, device=g.device) if ctx.needs_input_grad[0] else None
        d_tab = torch.empty(tshape, dtype=torch.float32, device=g.device) if ctx.needs_input_grad[1] else None
        L = C.lib()
        C.call("xq_vit_assemble_bwd", 1, L.xq_vit_assemble_bwd, C.ptr(g), B, Ls, T, D, t0, C.ptr(d_src),
               _ASSEMBLE_TYPE[sdt], C.ptr(d_tab), C.stream_ptr(g.device),
               nbytes=g.numel() * 4 + (d_src.numel() * d_src.element_size() if d_src is not None else 0))
        return d_src, d_tab, None


ASSEMBLE_ENABLED = [True]      # bench.py --impl eager switches the fused assembly off together with the other fused paths


def assemble_tokens(owner, path_fn, src, t0: int):
    """Token assembly through the fused kernel when it applies, else `path_fn(src)` (the module's own cat / add chain).

    `path_fn` maps the batch-dependent rows src [B,Ls,D] to the full fp32 sequence [B,T,D] and must be affine in `src` with
    the identity on rows [t0, t0+Ls) -- true for dinov2.py:151-170 / 318-336 whatever the configuration (prefix tokens,
    product quantisation, level embeddings).  That assumption is CHECKED once per module instance on a random probe; if it
    does not hold (a configuration not anticipated here) the module path is used from then on.  Active dropout on the
    sequence makes the assembly batch-dependent: module path."""
    ok = (ASSEMBLE_ENABLED[0] and src.is_cuda and src.dim() == 3 and src.shape[-1] % 4 == 0 and torch.is_autocast_enabled()
          and src.dtype in _ASSEMBLE_TYPE)
    if ok and getattr(owner, "_assemble_ok", None) is None:
        with torch.no_grad():
            probe = torch.randn(2, src.shape[1], src.shape[2], device=src.device)
            full, base = path_fn(probe).float(), path_fn(torch.zeros_like(probe[:1])).float()
            want = base.expand(2, -1, -1).clone()
            ok_shape = base.dim() == 3 and t0 + src.shape[1] <= base.shape[1]
            if ok_shape:
                want[:, t0:t0 + src.shape[1]] += probe
            owner._assemble_ok = bool(ok_shape and torch.allclose(full, want, rtol=1e-5, atol=1e-6))
    if not ok or not owner._assemble_ok:
        return path_fn(src)
    table = path_fn(torch.zeros(1, src.shape[1], src.shape[2], dtype=torch.float32, device=src.device))[0]
    return _Assemble.apply(src, table, t0)


def _droppath_scale(mod, batch: int, device):
    """DropPath (timm): per-sample keep mask / keep_prob, or None when inactive."""
    p = getattr(mod, "drop_prob", 0.0)
    if p == 0.0 or not mod.training:
        return None
    keep = 1.0 - p
    t = torch.empty(batch, dtype=torch.float32, device=device).bernoulli_(keep)
    if keep > 0.0 and getattr(mod, "scale_by_keep", True):
        t.div_(keep)
    return t


_NO_BRANCH = (None, None, None, None)


def _mlp_tail(blk, x, y):
    """the MLP half of Block.forward from norm2's output y: (branch, fc2 bias, ls2 gamma, drop-path scale) -- the residual add
    that block_forward leaves to the next residual_ln"""
    branch = mlp_forward(blk.mlp, y)              # fc1 bias in the GELU epilogue / kernel; fc2 bias folded into the next residual_ln
    gamma = blk.ls2.gamma if hasattr(blk.ls2, "gamma") else None
    return branch, blk.mlp.fc2.bias, gamma, _droppath_scale(blk.drop_path2, x.shape[0], x.device)


def block_forward(blk, x, pending):
    """Block.forward (vision_transformer.py:336-339) on the fused glue.  x: the fp32 residual stream [B,S,D] WITHOUT the
    previous block's MLP branch, which arrives in `pending` = (branch, bias, ls gamma, drop-path scale) and is added by this
    block's first residual_ln (_NO_BRANCH for the first block).  Returns (x, pending) in the same sense for the next block or
    the final norm."""
    Bn, dev = x.shape[0], x.device
    x, y = residual_ln(x, *pending, blk.norm1.weight, blk.norm1.bias, blk.norm1.eps)
    a, a_bias = attention_forward(blk.attn, y)
    g1 = blk.ls1.gamma if hasattr(blk.ls1, "gamma") else None
    x, y = residual_ln(x, a, a_bias, g1,
                       _droppath_scale(blk.drop_path1, Bn, dev), blk.norm2.weight, blk.norm2.bias, blk.norm2.eps)
    return x, _mlp_tail(blk, x, y)


def fused_path_ok(vit, x) -> bool:
    return (x.is_cuda and _autocast_half() is not None
            and vit.embed_dim in _SUPPORTED_D and isinstance(vit.norm_pre, nn.Identity))


def run_blocks(vit, x, attn_mask=None):
    """x: [B,S,D] token stream after pos-embed (fp32).  Returns norm(blocks(x)) in the autocast dtype (bf16 or fp16) on the
    fused path, or the plain module path result otherwise (fp32 parity runs, CPU)."""
    if attn_mask is not None or not fused_path_ok(vit, x):
        x = x.to(torch.matmul(x.new_ones(8, 8), x.new_ones(8, 8)).dtype)   # dinov2.py:177-179
        x = vit.norm_pre(x)
        if attn_mask is not None:
            for blk in vit.blocks:
                x = blk(x, attn_mask)
        else:
            x = vit.blocks(x)
        return vit.norm(x)
    x = x.float()
    pending = _NO_BRANCH
    for blk in vit.blocks:
        x, pending = block_forward(blk, x, pending)
    norm = _live(vit.norm)
    _, y = residual_ln(x, *pending, norm.weight, norm.bias, norm.eps)
    return y


def frozen_path_ok(vit, x) -> bool:
    """VisionTransformer.forward / forward_features take the frozen fused path (frozen_forward) when the model is a frozen
    teacher under bf16 / fp16 autocast: x a CUDA fp32 image that needs no gradient, a supported width, and no parameter
    that requires grad.  Anything else -- CPU, fp32 runs, a teacher a user has unfrozen -- runs the module path."""
    return (x.is_cuda and x.dtype == torch.float32 and not x.requires_grad and _autocast_half() is not None
            and vit.embed_dim in _SUPPORTED_D and not any(p.requires_grad for p in vit.parameters()))


def _cls_tail_ok(vit, blk, y) -> bool:
    """the class-token tail covers a plain Attention on the wgmma kernels with the class token in row 0"""
    from .dino_enc.vision_transformer import RoPEAttention      # imported here: dino_enc imports this module
    return (vit.has_class_token and not isinstance(blk.attn, RoPEAttention) and attn_tc_ok(blk.attn, y)
            and y.shape[1] <= _ATTN_CLS_MAX_N)


_ATTN_CLS_MAX_N = 8192         # sequence lengths xq_vit_attn_fwd_cls covers (include/xqb200.h)


def frozen_forward(vit, x, cls_only: bool = False):
    """VisionTransformer.forward_features of a frozen model (frozen_path_ok) on the fused kernels: image x fp32 [B,3,H,W] ->
    norm(blocks(norm_pre(pos_embed(patch_embed(x))))) [B,S,D] in the autocast dtype, as run_blocks returns it.  Nothing is
    saved for a backward and the fused MLP GEMMs write no pre-activation.

    cls_only: row 0 only, [B,D] -- what forward() reads with global_pool 'token'.  The last block then computes its qkv GEMM
    over every token (keys and values need them all), the attention of the class query alone (xq_vit_attn_fwd_cls), and the
    proj GEMM, residual_ln, MLP and final norm on the B class rows."""
    x = patch_embed(vit.patch_embed, x)
    x = assemble_tokens(vit, vit._pos_embed, x, vit.num_prefix_tokens)
    x = vit.patch_drop(x)
    if isinstance(vit.norm_pre, nn.LayerNorm):
        # the CLIP teacher: torch's layer_norm on the fp32 stream, the fp32 result autocast gives the module path
        x = F.layer_norm(x.float(), vit.norm_pre.normalized_shape, vit.norm_pre.weight, vit.norm_pre.bias, vit.norm_pre.eps)
    else:
        x = vit.norm_pre(x)
    x = x.float()
    blocks = list(vit.blocks)
    norm = _live(vit.norm)
    pending = _NO_BRANCH
    for blk in blocks[:-1] if cls_only else blocks:
        x, pending = block_forward(blk, x, pending)
    if cls_only:
        blk = blocks[-1]
        x_in = x
        x, y = residual_ln(x_in, *pending, blk.norm1.weight, blk.norm1.bias, blk.norm1.eps)
        if not _cls_tail_ok(vit, blk, y):
            x, pending = block_forward(blk, x_in, pending)       # the whole last block, then row 0 of the norm
            _, y = residual_ln(x, *pending, norm.weight, norm.bias, norm.eps)
            return y[:, 0]
        attn = blk.attn
        Bn, _, D = y.shape
        _, qkv = _qkv_projection(y, attn.qkv.weight, attn.qkv.bias)
        a = F.linear(attn_cls_forward(qkv, attn.num_heads), attn.proj.weight).view(Bn, 1, D)
        g1 = blk.ls1.gamma if hasattr(blk.ls1, "gamma") else None
        x, y = residual_ln(x[:, :1], a, attn.proj.bias, g1, _droppath_scale(blk.drop_path1, Bn, x.device),
                           blk.norm2.weight, blk.norm2.bias, blk.norm2.eps)
        pending = _mlp_tail(blk, x, y)
    _, y = residual_ln(x, *pending, norm.weight, norm.bias, norm.eps)
    return y[:, 0] if cls_only else y
