"""AdamW step of the tokenizer trainer -- drop-in for torch.optim.AdamW as xqgan_train.py builds it (:344-347).

The reference steps the tokenizer (`optimizer.step()` via `scaler.step`, :459) and the discriminator (`optimizer_disc.step()`,
:474) with `torch.optim.AdamW(params, lr, betas=(beta1, beta2), weight_decay=...)`.  On CUDA that is torch's foreach
implementation: seven or eight multi-tensor kernels per step and a full fp32 copy of every second moment for its square root.
Here `step()` is one launch of csrc/adamw_kernel.cu per param group (for up to XQ_ADAMW_MAX_TENSORS tensors), one pass over
param, grad and both moments, with the same bits:

    from imagefolder_b200.optim import AdamW          # instead of: torch.optim.AdamW

The class keeps torch's constructor, `param_groups`, `state` layout and `state_dict` / `load_state_dict`, so checkpoints move
both ways between it and torch.optim.AdamW, and LR schedulers that write `group['lr']` work unchanged.

With --max_grad_norm set, the trainer clips between `scaler.unscale_` and `scaler.step` (:456-458, 471-473).
`clip_grad_norm_` is torch.nn.utils.clip_grad_norm_ with the same signature, return value and bits; its two passes over the
grads are csrc/clip_kernel.cu launches instead of torch's foreach chains:

    from imagefolder_b200.optim import clip_grad_norm_  # instead of: torch.nn.utils.clip_grad_norm_
"""
from __future__ import annotations

import math
import types
import warnings

import numpy as np
import torch
from torch.utils._foreach_utils import _group_tensors_by_device_and_dtype

from . import _capi

__all__ = ["AdamW", "clip_grad_norm_"]

_UNSUPPORTED = ("amsgrad", "maximize", "capturable", "differentiable")


def _real(t):
    """t itself when fp32; its fp32 [..., 2] view when complex64 -- how torch's foreach AdamW (`_view_as_real`) and the
    kernels see a complex tensor, element for element"""
    return torch.view_as_real(t) if t.dtype == torch.complex64 else t


def _check_group(group):
    """raise on a group option the kernel does not reproduce (the reference sets none of them)"""
    for k in _UNSUPPORTED:
        if group[k]:
            raise ValueError(f"AdamW: {k}=True is not supported")
    if group["fused"]:
        raise ValueError("AdamW: fused=True is torch's own kernel; this class always runs its own")
    if group["foreach"] is False:
        raise ValueError("AdamW: foreach=False (torch's per-tensor loop) rounds differently; the kernel reproduces the "
                         "foreach implementation that torch picks for CUDA tensors by default")
    if not group["decoupled_weight_decay"]:
        raise ValueError("AdamW: decoupled_weight_decay=False (Adam's L2 penalty) is not supported")
    for k in ("lr", "eps", "weight_decay"):
        if torch.is_tensor(group[k]):
            raise ValueError(f"AdamW: a tensor {k} is not supported")
    if any(torch.is_tensor(b) for b in group["betas"]):
        raise ValueError("AdamW: tensor betas are not supported")
    # torch's constructor ranges, checked again because schedulers and users write the groups; with them every scalar the
    # kernel receives is finite, so the launch cannot be refused after the step counters have advanced
    beta1, beta2 = group["betas"]
    if not (0.0 <= group["lr"] < math.inf and 0.0 <= group["eps"] < math.inf and 0.0 <= group["weight_decay"] < math.inf
            and 0.0 <= beta1 < 1.0 and 0.0 <= beta2 < 1.0):
        raise ValueError(f"AdamW: lr {group['lr']}, betas {group['betas']}, eps {group['eps']} or weight_decay "
                         f"{group['weight_decay']} out of range")


class AdamW(torch.optim.AdamW):
    """torch.optim.AdamW whose step() runs one sm_90a kernel per param group, bit-identical to torch's foreach step.

    Supported: fp32 or complex64 dense CUDA params on one device per group, with contiguous grads and state.  A complex64
    param (the RoPE decoder's `freqs_1d`) is stepped through its real view, as torch's foreach step does.  Anything else
    raises before any tensor is written: there is no CPU or eager fallback."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, *,
                 maximize=False, foreach=None, capturable=False, differentiable=False, fused=None):
        super().__init__(params, lr, betas, eps, weight_decay, amsgrad, maximize=maximize, foreach=foreach,
                         capturable=capturable, differentiable=differentiable, fused=fused)
        for group in self.param_groups:
            _check_group(group)

    def _plan_group(self, group):
        """the group's (param, grad) pairs in param order, checked; nothing is written"""
        pairs, device = [], None
        for i, p in enumerate(group["params"]):
            g = p.grad
            if g is None:
                continue
            if g.is_sparse or g.layout != torch.strided or p.layout != torch.strided:
                raise ValueError(f"AdamW: param {i}: sparse params or grads are not supported")
            if p.dtype not in (torch.float32, torch.complex64) or g.dtype != p.dtype:
                raise ValueError(f"AdamW: param {i}: fp32 or complex64 params with grads of the same dtype are required "
                                 f"(param {p.dtype}, grad {g.dtype})")
            if not p.is_cuda or not g.is_cuda:
                raise _capi.XqError(f"AdamW: param {i}: CUDA tensors are required, there is no CPU path "
                                    f"(param on {p.device}, grad on {g.device})")
            device = p.device if device is None else device
            tensors = [p, g]
            st = self.state.get(p)
            if st:
                tensors += [st["exp_avg"], st["exp_avg_sq"]]
                if not torch.is_tensor(st["step"]):
                    raise ValueError(f"AdamW: param {i}: state['step'] must be a tensor")
            for t in tensors:
                if t.device != device:
                    raise ValueError(f"AdamW: param {i}: tensors on {t.device}, expected {device}")
                if t.dtype != p.dtype or t.shape != p.shape:
                    raise ValueError(f"AdamW: param {i}: state {tuple(t.shape)} {t.dtype} does not match the param")
                if not t.is_contiguous():
                    raise ValueError(f"AdamW: param {i}: param, grad and state must be contiguous")
            pairs.append((p, g))
        return pairs, device

    @torch.no_grad()
    def step(self, closure=None):
        """One AdamW step for every param with a grad, bit-identical to torch.optim.AdamW's default (foreach) step.

        Every group is checked before anything is written, then each group is one launch (or several, in order, past
        XQ_ADAMW_MAX_TENSORS params) on the current stream of its device."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        plans = []
        for group in self.param_groups:
            _check_group(group)
            plans.append((group, *self._plan_group(group)))
        L = _capi.lib()
        for group, pairs, device in plans:
            if not pairs:
                continue
            steps, ps, gs, ms, vs = [], [], [], [], []
            for p, g in pairs:
                st = self.state[p]
                if len(st) == 0:                     # torch's lazy initialisation (Adam._init_group)
                    st["step"] = torch.tensor(0.0, dtype=torch.float32)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                steps.append(st["step"])
                ps.append(_real(p))
                gs.append(_real(g))
                ms.append(_real(st["exp_avg"]))
                vs.append(_real(st["exp_avg_sq"]))
            # the step counters and scalars exactly as torch/optim/adam.py::_multi_tensor_adam computes them
            if steps[0].is_cpu:
                torch._foreach_add_(steps, torch.tensor(1.0, device="cpu"), alpha=1.0)
            else:
                torch._foreach_add_(steps, 1)
            lr, (beta1, beta2), eps, wd = group["lr"], group["betas"], group["eps"], group["weight_decay"]
            ts = [s.item() for s in steps]
            step_size = np.array([(lr / (1 - beta1 ** t)) * -1 for t in ts], dtype=np.float64)
            bc2_sqrt = np.array([(1 - beta2 ** t) ** 0.5 for t in ts], dtype=np.float64)
            wd_factor = 1 - lr * wd if wd != 0 else 1.0
            arr = lambda ts_: np.array([t.data_ptr() for t in ts_], dtype=np.uint64)
            p_arr, g_arr, m_arr, v_arr = arr(ps), arr(gs), arr(ms), arr(vs)
            n_arr = np.array([p.numel() for p in ps], dtype=np.int64)
            n = len(ps)
            with torch.cuda.device(device):
                _capi.call("xq_adamw_step", -(-n // _capi.XQ_ADAMW_MAX_TENSORS), L.xq_adamw_step, p_arr.ctypes.data,
                           g_arr.ctypes.data, m_arr.ctypes.data, v_arr.ctypes.data, n_arr.ctypes.data,
                           step_size.ctypes.data, bc2_sqrt.ctypes.data, n, float(wd_factor), float(1 - beta1),
                           float(beta2), float(1 - beta2), float(eps), _capi.stream_ptr(device),
                           nbytes=28 * int(n_arr.sum()))
            # the kernel writes through raw pointers: bump the version counters as torch's in-place foreach ops do
            torch.autograd.graph.increment_version(ps + ms + vs)
        return loss


def _clip_tables(numels):
    """(start, stop, launches of xq_grad_norm, launches of xq_grad_scale) of each XQ_CLIP_MAX_TENSORS-entry table of a call"""
    T = _capi.XQ_CLIP_MAX_TENSORS
    tables = []
    for i0 in range(0, len(numels), T):
        nonempty = any(int(k) > 0 for k in numels[i0:i0 + T])
        tables.append((i0, min(i0 + T, len(numels)), 1 + nonempty, int(nonempty)))
    return tables


def _check_grads(grads):
    """the device of `grads`, after refusing anything the kernels do not reproduce; nothing is written"""
    for i, g in enumerate(grads):
        if g.is_sparse or g.layout != torch.strided:
            raise ValueError(f"clip_grad_norm_: grad {i}: sparse grads are not supported")
        if g.dtype not in (torch.float32, torch.complex64):
            raise ValueError(f"clip_grad_norm_: grad {i}: fp32 or complex64 grads are required (got {g.dtype})")
        if not g.is_contiguous():
            raise ValueError(f"clip_grad_norm_: grad {i}: contiguous grads are required")
    for i, g in enumerate(grads):
        if not g.is_cuda:
            raise _capi.XqError(f"clip_grad_norm_: grad {i}: CUDA tensors are required, there is no CPU path "
                                f"(grad on {g.device})")
        if g.device != grads[0].device:
            raise ValueError(f"clip_grad_norm_: grad {i} is on {g.device}, expected {grads[0].device}: one device "
                             "per call")
    return grads[0].device


@torch.no_grad()
def clip_grad_norm_(parameters, max_norm, norm_type=2.0, error_if_nonfinite=False, foreach=None):
    """torch.nn.utils.clip_grad_norm_ (torch 2.11) for fp32 CUDA grads on one device, with the same bits.

    A complex64 grad counts as its real view (the norm of a complex tensor is that of its real and imaginary parts) and is
    scaled component-wise (DESIGN.md section 8 states where that differs from torch's complex multiply).
    The per-tensor norms are one xq_grad_norm call (bit-identical to torch._foreach_norm), the total norm and the clip
    coefficient are torch's own ops on them, and the grads are scaled by one xq_grad_scale call that reads the coefficient on
    the device, so nothing synchronises unless `error_if_nonfinite` asks to.  Returns the total norm, as torch does.

    Raises before anything is written on norm_type != 2, foreach=False, grads neither fp32 nor complex64, sparse or
    non-contiguous grads, grads on more
    than one device, and CPU grads (_capi.XqError: there is no CPU path)."""
    if isinstance(parameters, torch.Tensor):
        parameters = [parameters]
    else:
        is_generator = isinstance(parameters, types.GeneratorType)
        parameters = list(parameters)                  # a generator is consumed once
        if is_generator and len(parameters) == 0:
            warnings.warn("`parameters` is an empty generator, no gradient clipping will occur.", stacklevel=3)
    grads = [p.grad for p in parameters if p.grad is not None]
    norm_type = float(norm_type)
    if norm_type != 2.0:
        raise ValueError(f"clip_grad_norm_: norm_type {norm_type} is not supported; the kernels reproduce the L2 norm")
    if foreach is False:
        raise ValueError("clip_grad_norm_: foreach=False (torch's per-tensor vector_norm loop) rounds differently; the kernels "
                         "reproduce the foreach implementation that torch picks for CUDA grads by default")
    if len(grads) == 0:
        return torch.tensor(0.0)
    max_norm = float(max_norm)
    device = _check_grads(grads)
    # the order of torch's per-dtype groups, which is the order of the norms its total norm sums (one group for fp32 grads)
    grads = [_real(g) for ([gs], _) in _group_tensors_by_device_and_dtype([grads]).values() for g in gs]
    ptrs = np.array([g.data_ptr() for g in grads], dtype=np.uint64)
    numel = np.array([g.numel() for g in grads], dtype=np.int64)
    n = len(grads)
    tables = _clip_tables(numel)
    L = _capi.lib()
    with torch.cuda.device(device):
        stream = _capi.stream_ptr(device)
        ws_bytes = L.xq_grad_norm_workspace_bytes(n, numel.ctypes.data)
        ws = _capi.workspace(ws_bytes, device)
        norms = torch.empty(n, dtype=torch.float32, device=device)    # what torch.stack(torch._foreach_norm(grads)) holds
        _capi.call("xq_grad_norm", sum(t[2] for t in tables), L.xq_grad_norm, ptrs.ctypes.data, numel.ctypes.data, n,
                   norms.data_ptr(), ws.data_ptr(), ws.numel(), stream, nbytes=4 * int(numel.sum()))
        # torch/nn/utils/clip_grad.py, _get_total_norm and _clip_grads_with_norm_, op for op
        total_norm = torch.linalg.vector_norm(norms, norm_type)
        if error_if_nonfinite and torch.logical_or(total_norm.isnan(), total_norm.isinf()):
            raise RuntimeError(
                f"The total norm of order {norm_type} for gradients from "
                "`parameters` is non-finite, so it cannot be clipped. To disable "
                "this error and scale the gradients by the non-finite norm anyway, "
                "set `error_if_nonfinite=False`"
            )
        clip_coef = max_norm / (total_norm + 1e-6)
        clip_coef_clamped = torch.clamp(clip_coef, max=1.0)
        _capi.call("xq_grad_scale", sum(t[3] for t in tables), L.xq_grad_scale, ptrs.ctypes.data, numel.ctypes.data, n,
                   clip_coef_clamped.data_ptr(), stream, nbytes=8 * int(numel.sum()))
    # the kernel writes through raw pointers: bump the version counters as torch's in-place _foreach_mul_ does
    torch.autograd.graph.increment_version(grads)
    return total_norm
