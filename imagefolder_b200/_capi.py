"""ctypes binding of libxqb200.so (include/xqb200.h).

There is NO fallback: if the CUDA library is missing or a call fails, this module raises.
The product never imports anything under oracle/.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_double, c_float, c_int, c_int64, c_size_t, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libxqb200.so")
XQ_MAX_SCALES = 32
XQ_EMA_MAX_TENSORS = 1020      # entries of one xq_ema_update launch (include/xqb200.h)
XQ_ADAMW_MAX_TENSORS = 584     # entries of one xq_adamw_step launch (include/xqb200.h)
XQ_CLIP_MAX_TENSORS = 1360     # entries of one xq_grad_norm / xq_grad_scale table (include/xqb200.h)
XQ_GRAD_NORM_CHUNK = 65536     # floats per partial of xq_grad_norm: torch's _foreach_norm chunk (csrc/clip_kernel.cu)
XQ_METRIC_STRIP_ROWS = 32      # image rows per CTA of xq_recon_psnr_ssim (include/xqb200.h)

XQ_MS_VQ_ZNORM, XQ_MS_VQ_L2, XQ_MS_BSQ, XQ_MS_BSQ_HARD = 0, 1, 2, 3


class XqMsDesc(ctypes.Structure):
    _fields_ = [
        ("B", c_int), ("C", c_int), ("H", c_int), ("W", c_int),
        ("V", c_int), ("K", c_int), ("SN", c_int), ("mode", c_int),
        ("patch_nums", c_int * XQ_MAX_SCALES),
        ("phi_map", c_int * XQ_MAX_SCALES),
        ("scaler", c_float * XQ_MAX_SCALES),
        ("resi_ratio", c_float), ("beta", c_float),
        ("loss_div_sn_all", c_int), ("channel_norm", c_int),
        ("entropy_weight", c_float), ("w_sample", c_float), ("w_batch", c_float),
    ]


class XqError(RuntimeError):
    pass


_lib = None
# ViT entry points with an `_f16` twin (include/xqb200.h): same arguments, fp16 instead of bf16 data
F16_TWINS = [
    "xq_vit_residual_ln_fwd", "xq_vit_residual_ln_bwd", "xq_vit_patchify", "xq_vit_gelu_fwd", "xq_vit_gelu_bwd",
    "xq_vit_attn_fwd", "xq_vit_attn_bwd", "xq_vit_fc1_gelu_fwd", "xq_vit_fc2_dgelu_bwd", "xq_vit_fc1_lora_gelu_fwd",
    "xq_vit_fc2_lora_dgelu_bwd",
]


def lib() -> ctypes.CDLL:
    """Load libxqb200.so; fail loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise XqError(
            f"{LIB_PATH} not found: the sm_90a CUDA library is required (there is no CPU/PyTorch fallback). "
            "Build it with `python -c 'import __graft_entry__ as g; g.build()'` or imagefolder_b200/csrc/build.sh")
    L = ctypes.CDLL(LIB_PATH)
    vp, f32p, i64p = c_void_p, c_void_p, c_void_p  # device pointers are passed as integers
    L.xq_strerror.restype = ctypes.c_char_p
    L.xq_strerror.argtypes = [c_int]
    L.xq_last_cuda_error.restype = ctypes.c_char_p
    L.xq_abi_version.restype = c_int
    L.xq_vq_workspace_bytes.restype = c_size_t
    L.xq_vq_workspace_bytes.argtypes = [c_int] * 4
    L.xq_vq_forward.restype = c_int
    L.xq_vq_forward.argtypes = [f32p, f32p, c_int, c_int, c_int, c_int, c_int, c_int, c_float, i64p, f32p, f32p, f32p,
                                vp, c_size_t, vp]
    L.xq_vq_backward.restype = c_int
    L.xq_vq_backward.argtypes = [f32p, f32p, i64p, f32p, f32p, f32p, c_int, c_int, c_int, c_int, c_int, c_float, f32p,
                                 f32p, vp]
    L.xq_perturb_workspace_bytes.restype = c_size_t
    L.xq_perturb_workspace_bytes.argtypes = [c_int] * 4
    L.xq_perturb_forward.restype = c_int
    L.xq_perturb_forward.argtypes = [f32p, f32p, f32p, f32p, i64p, c_int, c_int, c_int, c_int, c_int, c_float, c_int,
                                     c_int, f32p, i64p, vp, c_size_t, vp]
    L.xq_perturb_backward.restype = c_int
    L.xq_perturb_backward.argtypes = [f32p, f32p, c_int, c_int, c_int, c_int, c_int, f32p, f32p, vp]
    dp = POINTER(XqMsDesc)
    L.xq_ms_workspace_bytes.restype = c_size_t
    L.xq_ms_workspace_bytes.argtypes = [dp]
    L.xq_ms_saved_bytes.restype = c_size_t
    L.xq_ms_saved_bytes.argtypes = [dp]
    L.xq_ms_total_tokens.restype = c_int64
    L.xq_ms_total_tokens.argtypes = [dp]
    L.xq_ms_forward.restype = c_int
    L.xq_ms_forward.argtypes = [dp, f32p, f32p, f32p, f32p, f32p, c_int, f32p, i64p, f32p, f32p, f32p, vp, vp,
                                c_size_t, vp]
    L.xq_ms_backward.restype = c_int
    L.xq_ms_backward.argtypes = [dp, f32p, f32p, f32p, f32p, f32p, i64p, vp, f32p, f32p, f32p, f32p, f32p, f32p, f32p,
                                 f32p, vp, c_size_t, vp]
    L.xq_ms_decode.restype = c_int
    L.xq_ms_decode.argtypes = [dp, i64p, f32p, f32p, f32p, f32p, f32p, f32p, vp]
    L.xq_ms_embed.restype = c_int
    L.xq_ms_embed.argtypes = [dp, c_int, c_int, f32p, f32p, f32p, f32p, f32p, f32p, f32p, vp]
    L.xq_usage_ema_dev.restype = c_int
    L.xq_usage_ema_dev.argtypes = [f32p, f32p, c_int, c_int, i64p, c_float, f32p, vp]
    L.xq_vit_residual_ln_fwd.restype = c_int
    L.xq_vit_residual_ln_fwd.argtypes = [f32p, vp, f32p, f32p, f32p, c_int, f32p, f32p, c_float, c_int, c_int, f32p, vp,
                                         f32p, f32p, vp]
    L.xq_vit_ln_bwd_workspace_bytes.restype = c_size_t
    L.xq_vit_ln_bwd_workspace_bytes.argtypes = [c_int]
    L.xq_vit_residual_ln_bwd.restype = c_int
    L.xq_vit_residual_ln_bwd.argtypes = [f32p, vp, f32p, f32p, f32p, f32p, vp, f32p, f32p, f32p, c_int, c_int, c_int,
                                         f32p, vp, f32p, f32p, f32p, f32p, vp, c_size_t, vp]
    L.xq_vit_patchify.restype = c_int
    L.xq_vit_patchify.argtypes = [f32p, vp, c_int, c_int, c_int, c_int, c_int, vp]
    L.xq_vit_assemble_fwd.restype = c_int
    L.xq_vit_assemble_fwd.argtypes = [vp, c_int, f32p, c_int, c_int, c_int, c_int, c_int, f32p, vp]
    L.xq_vit_assemble_bwd.restype = c_int
    L.xq_vit_assemble_bwd.argtypes = [f32p, c_int, c_int, c_int, c_int, c_int, vp, c_int, f32p, vp]
    L.xq_vit_gelu_fwd.restype = c_int
    L.xq_vit_gelu_fwd.argtypes = [vp, f32p, vp, c_int, c_int, vp]
    L.xq_vit_gelu_bwd.restype = c_int
    L.xq_vit_gelu_bwd.argtypes = [vp, f32p, vp, vp, f32p, c_int, c_int, vp]
    L.xq_vit_attn_fwd.restype = c_int
    L.xq_vit_attn_fwd.argtypes = [vp, vp, f32p, c_int, c_int, c_int, c_int, c_float, vp]
    L.xq_vit_attn_bwd_workspace_bytes.restype = c_size_t
    L.xq_vit_attn_bwd_workspace_bytes.argtypes = [c_int, c_int, c_int]
    L.xq_vit_attn_bwd.restype = c_int
    L.xq_vit_attn_bwd.argtypes = [vp, vp, vp, f32p, vp, f32p, c_int, c_int, c_int, c_int, c_float, vp, c_size_t, vp]
    L.xq_vit_fc1_gelu_fwd.restype = c_int
    L.xq_vit_fc1_gelu_fwd.argtypes = [vp, vp, f32p, vp, vp, c_int, c_int, c_int, vp]
    L.xq_vit_fc2_dgelu_bwd.restype = c_int
    L.xq_vit_fc2_dgelu_bwd.argtypes = [vp, vp, vp, f32p, vp, f32p, c_int, c_int, c_int, vp]
    L.xq_vit_fc1_lora_gelu_fwd.restype = c_int
    L.xq_vit_fc1_lora_gelu_fwd.argtypes = [vp, vp, vp, vp, f32p, vp, vp, c_int, c_int, c_int, c_int, vp]
    L.xq_vit_fc2_lora_dgelu_bwd.restype = c_int
    L.xq_vit_fc2_lora_dgelu_bwd.argtypes = [vp, vp, vp, vp, vp, f32p, vp, f32p, c_int, c_int, c_int, c_int, vp]
    # fp16 twins of the 16-bit ViT entry points: the same argument lists
    for name in F16_TWINS:
        twin = getattr(L, name + "_f16")
        twin.restype = c_int
        twin.argtypes = getattr(L, name).argtypes
    L.xq_lpips_workspace_bytes.restype = c_size_t
    L.xq_lpips_workspace_bytes.argtypes = [c_int, c_int]
    L.xq_lpips_layer_forward.restype = c_int
    L.xq_lpips_layer_forward.argtypes = [vp, vp, c_int, f32p, c_int, c_int, c_int, c_float, c_int, f32p, vp, c_size_t, vp]
    L.xq_lpips_layer_backward.restype = c_int
    L.xq_lpips_layer_backward.argtypes = [vp, vp, c_int, f32p, c_int, c_int, c_int, c_float, f32p, vp, vp]
    L.xq_diffaug_forward.restype = c_int
    L.xq_diffaug_forward.argtypes = [f32p, f32p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, f32p, f32p, vp]
    L.xq_diffaug_backward.restype = c_int
    L.xq_diffaug_backward.argtypes = [f32p, f32p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, f32p, f32p, vp]
    # image transforms (csrc/img_kernels.cu): src / offs / plan / out are device pointers, except plan_host / ws_off_host
    L.xq_img_workspace_bytes.restype = c_size_t
    L.xq_img_workspace_bytes.argtypes = [vp, c_int, c_int, vp]
    L.xq_img_box_halve.restype = c_int
    L.xq_img_box_halve.argtypes = [vp, c_size_t, vp, vp, c_int, c_int, c_int, c_int, c_int, vp, c_size_t, vp]
    L.xq_img_resize_crop_normalize.restype = c_int
    L.xq_img_resize_crop_normalize.argtypes = [vp, c_size_t, vp, vp, c_int, c_int, vp, c_size_t, f32p, vp]
    # weight EMA (csrc/ema_kernel.cu): ema / param / numel are HOST arrays of device pointers and sizes
    L.xq_ema_update.restype = c_int
    L.xq_ema_update.argtypes = [vp, vp, vp, c_int, c_float, c_float, vp]
    # AdamW step (csrc/adamw_kernel.cu): every array is a HOST array (of device pointers, sizes or per-tensor doubles)
    L.xq_adamw_step.restype = c_int
    L.xq_adamw_step.argtypes = [vp, vp, vp, vp, vp, vp, vp, c_int, c_double, c_double, c_double, c_double, c_double, vp]
    # gradient-norm clipping (csrc/clip_kernel.cu): grad / numel are HOST arrays of device pointers and sizes
    L.xq_grad_norm_workspace_bytes.restype = c_size_t
    L.xq_grad_norm_workspace_bytes.argtypes = [c_int, vp]
    L.xq_grad_norm.restype = c_int
    L.xq_grad_norm.argtypes = [vp, vp, c_int, f32p, vp, c_size_t, vp]
    L.xq_grad_scale.restype = c_int
    L.xq_grad_scale.argtypes = [vp, vp, c_int, f32p, vp]
    # reconstruction metrics (csrc/metric_kernels.cu)
    L.xq_recon_psnr_ssim_workspace_bytes.restype = c_size_t
    L.xq_recon_psnr_ssim_workspace_bytes.argtypes = [c_int] * 4
    L.xq_recon_psnr_ssim.restype = c_int
    L.xq_recon_psnr_ssim.argtypes = [vp, c_int, f32p, c_int, c_int, c_int, c_int, vp, vp, vp, c_size_t, vp]
    _lib = L
    return L


# --- instrumentation used by bench.py (off by default) ---------------------------------------
TIMING = None        # dict name -> [(start_event, end_event, algorithmic_bytes, tensor_flops), ...] when enabled
LAUNCHES = [0]       # number of libxqb200 kernels launched (counted per C call)


def call(name: str, n_kernels: int, fn, *args, nbytes: int = 0, nflops: float = 0.0) -> None:
    """invoke a C-ABI entry point, map its return code, count its kernel launches and (when
    TIMING is enabled) bracket it with CUDA events on the current stream.  `nbytes` = the call's algorithmic
    HBM bytes (what it must read + write once), `nflops` = its tensor-core FLOPs (contractions only), recorded for
    bench.py's per-kernel roofline table."""
    LAUNCHES[0] += n_kernels
    if TIMING is None:
        check(fn(*args), name)
        return
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    rc = fn(*args)
    e.record()
    TIMING.setdefault(name, []).append((s, e, nbytes, nflops))
    check(rc, name)


def check(rc: int, what: str) -> None:
    if rc == 0:
        return
    L = lib()
    msg = L.xq_strerror(rc).decode()
    if rc == -3:
        msg += ": " + L.xq_last_cuda_error().decode()
    if rc == -1:
        raise ValueError(f"{what}: {msg}")
    raise XqError(f"{what}: {msg}")


def ptr(t):
    """Device pointer of a tensor (None -> NULL).  The tensor must be a contiguous CUDA tensor."""
    if t is None:
        return None
    if not t.is_cuda:
        raise XqError("libxqb200 needs CUDA tensors: there is no CPU path (got a %s tensor)" % t.device)
    if not t.is_contiguous():
        raise XqError("libxqb200 needs contiguous tensors")
    return t.data_ptr()


def stream_ptr(device=None):
    return torch.cuda.current_stream(device).cuda_stream


def workspace(nbytes: int, device) -> torch.Tensor:
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def make_ms_desc(B, C, H, W, V, K, patch_nums, phi_map, mode, scaler=None, resi_ratio=0.5, beta=0.25,
                 loss_div_sn_all=False, channel_norm=False, entropy_weight=0.0, w_sample=1.0, w_batch=1.0) -> XqMsDesc:
    SN = len(patch_nums)
    if SN > XQ_MAX_SCALES:
        raise ValueError(f"at most {XQ_MAX_SCALES} scales are supported")
    d = XqMsDesc()
    d.B, d.C, d.H, d.W, d.V, d.K, d.SN, d.mode = int(B), int(C), int(H), int(W), int(V), int(K), SN, int(mode)
    for i, p in enumerate(patch_nums):
        d.patch_nums[i] = int(p)
        d.phi_map[i] = int(phi_map[i]) if K > 0 else -1
        d.scaler[i] = float(scaler[i]) if scaler is not None else 0.0
    d.resi_ratio, d.beta = float(resi_ratio), float(beta)
    d.loss_div_sn_all, d.channel_norm = int(bool(loss_div_sn_all)), int(bool(channel_norm))
    d.entropy_weight, d.w_sample, d.w_batch = float(entropy_weight), float(w_sample), float(w_batch)
    return d


EXPORTED_SYMBOLS = [
    "xq_strerror", "xq_abi_version", "xq_last_cuda_error", "xq_vq_workspace_bytes", "xq_vq_forward",
    "xq_vq_backward", "xq_perturb_workspace_bytes", "xq_perturb_forward", "xq_perturb_backward",
    "xq_ms_workspace_bytes", "xq_ms_saved_bytes", "xq_ms_total_tokens", "xq_ms_forward", "xq_ms_backward",
    "xq_ms_decode", "xq_ms_embed", "xq_usage_ema_dev", "xq_vit_residual_ln_fwd", "xq_vit_ln_bwd_workspace_bytes",
    "xq_vit_residual_ln_bwd", "xq_vit_gelu_fwd", "xq_vit_gelu_bwd", "xq_vit_patchify", "xq_vit_assemble_fwd", "xq_vit_assemble_bwd", "xq_vit_attn_fwd", "xq_vit_attn_bwd_workspace_bytes", "xq_vit_attn_bwd", "xq_vit_fc1_gelu_fwd", "xq_vit_fc2_dgelu_bwd", "xq_vit_fc1_lora_gelu_fwd", "xq_vit_fc2_lora_dgelu_bwd",
    "xq_lpips_workspace_bytes", "xq_lpips_layer_forward", "xq_lpips_layer_backward", "xq_diffaug_forward",
    "xq_diffaug_backward", "xq_img_workspace_bytes", "xq_img_box_halve", "xq_img_resize_crop_normalize",
    "xq_ema_update", "xq_adamw_step", "xq_grad_norm_workspace_bytes", "xq_grad_norm", "xq_grad_scale", "xq_recon_psnr_ssim_workspace_bytes", "xq_recon_psnr_ssim",
] + [n + "_f16" for n in F16_TWINS]
