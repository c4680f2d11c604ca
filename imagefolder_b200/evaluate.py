"""Reconstruction-evaluation loop of the tokenizer (the rFID data path) -- tokenizer/tokenizer_image/xqgan_train.py:517-535.

The reference, every `ckpt_every` steps: puts the model in eval mode, reconstructs the whole validation set with
`img_to_reconstructed_img`, converts both the reconstruction and the ground truth to NHWC uint8
(`clamp(127.5 * x + 128, 0, 255)`), ALL-GATHERs them across ranks (`dist.nn.all_gather`), and accumulates them on the host
for the (TensorFlow) Inception-statistics evaluator.  This module is that loop up to the evaluator boundary: it returns the
two uint8 arrays the reference hands to `Evaluator.read_activations` (the evaluator itself -- a frozen TF Inception graph
with downloaded weights -- is out of scope, SURVEY.md section 8).

Data-path notes: the gather moves uint8 (one byte per value, as the reference), is issued once per batch for each of the
two tensors, and every rank returns the same arrays (rank 0 is the one that evaluates).

`reconstruction_metrics` runs the same loop and scores it with PSNR and SSIM instead (the reference's replacement for rFID,
README.md:192; tokenizer/vqgan/reconstruction_vqgan_ddp.py:149-190), on the GPU (`psnr_ssim`, csrc/metric_kernels.cu)."""
from __future__ import annotations

import contextlib
from typing import Iterable, NamedTuple, Optional, Tuple

import numpy as np
import torch
import torch.distributed as dist

from . import _capi


def to_uint8_nhwc(x: torch.Tensor) -> torch.Tensor:
    """[-1, 1] float NCHW -> uint8 NHWC exactly as xqgan_train.py:527-528."""
    return torch.clamp(127.5 * x + 128.0, 0, 255).permute(0, 2, 3, 1).to(torch.uint8).contiguous()


def _all_gather_cat(t: torch.Tensor) -> torch.Tensor:
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return t
    parts = [torch.empty_like(t) for _ in range(dist.get_world_size())]
    dist.all_gather(parts, t)          # rank-major concatenation, like torch.cat(dist.nn.all_gather(t), dim=0)
    return torch.cat(parts, dim=0)


@contextlib.contextmanager
def _eval_mode(model):
    """eval mode for the duration of the block; `model` is a VQModel or a DDP wrapper of one; yields the VQModel"""
    core = getattr(model, "module", model)
    was_training = core.training
    core.eval()
    try:
        yield core
    finally:
        core.train(was_training)


def _reconstructions(core, loader: Iterable, device, max_batches: Optional[int], autocast_dtype: Optional[torch.dtype]):
    """(x on `device`, img_to_reconstructed_img(x)) for every batch of `loader` (up to `max_batches`)"""
    for bi, (x, _) in enumerate(loader):
        if max_batches is not None and bi >= max_batches:
            break
        x = x.to(device, non_blocking=True)
        if autocast_dtype is not None and x.is_cuda:
            with torch.autocast("cuda", dtype=autocast_dtype):
                rec = core.img_to_reconstructed_img(x)
        else:
            rec = core.img_to_reconstructed_img(x)
        yield x, rec


def _distributed() -> bool:
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


@torch.no_grad()
def reconstruct_for_fid(model, loader: Iterable, device=None, max_batches: Optional[int] = None,
                        autocast_dtype: Optional[torch.dtype] = None) -> Tuple[np.ndarray, np.ndarray, int]:
    """-> (samples uint8 [T,H,W,3], ground_truth uint8 [T,H,W,3], T)  with T = all ranks' images in rank-major batch order.

    `model` is a VQModel (or a DDP wrapper of one); its training flag is restored on exit.  `loader` yields (images, _)
    with images in [-1, 1]; every rank must yield the same number of equally sized batches (the reference's sampler
    guarantees that)."""
    samples, gt, total = [], [], 0
    with _eval_mode(model) as core:
        device = device if device is not None else next(core.parameters()).device
        for x, rec in _reconstructions(core, loader, device, max_batches, autocast_dtype):
            s8 = _all_gather_cat(to_uint8_nhwc(rec.float()))
            x8 = _all_gather_cat(to_uint8_nhwc(x.float()))
            samples.append(s8.cpu().numpy())
            gt.append(x8.cpu().numpy())
            total += s8.shape[0]
    if _distributed():
        dist.barrier()
    if not samples:
        return np.zeros((0, 0, 0, 3), np.uint8), np.zeros((0, 0, 0, 3), np.uint8), 0
    return np.concatenate(samples, axis=0), np.concatenate(gt, axis=0), total


def psnr_ssim(rec: torch.Tensor, x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Per-image PSNR and SSIM of the reference's reconstruction evaluation (reconstruction_vqgan_ddp.py:155-169) in one
    launch pair of csrc/metric_kernels.cu -> (psnr, ssim), fp64 device tensors [B].

    `rec` is `img_to_reconstructed_img(x)` (already clamped to [-1, 1]; fp32, or bf16 under autocast, read as its fp32
    widening) and `x` the fp32 model input in [-1, 1], both contiguous [B, C, H, W] CUDA tensors with H, W >= 7.  The
    reconstruction is quantised exactly as `to_uint8_nhwc` does, the ground truth is not: see oracle/metric_oracle.py for
    the definition.  There is no CPU path."""
    if rec.dim() != 4 or tuple(rec.shape) != tuple(x.shape):
        raise ValueError(f"psnr_ssim: rec {tuple(rec.shape)} and x {tuple(x.shape)} must be equal [B, C, H, W] shapes")
    if rec.dtype not in (torch.float32, torch.bfloat16) or x.dtype != torch.float32:
        raise ValueError(f"psnr_ssim: rec must be fp32 or bf16 and x fp32 (got {rec.dtype}, {x.dtype})")
    if rec.device != x.device:
        raise ValueError(f"psnr_ssim: rec on {rec.device}, x on {x.device}")
    rp, xp = _capi.ptr(rec), _capi.ptr(x)
    B, C, H, W = (int(v) for v in x.shape)
    L = _capi.lib()
    psnr = torch.empty(B, dtype=torch.float64, device=x.device)
    ssim = torch.empty(B, dtype=torch.float64, device=x.device)
    with torch.cuda.device(x.device):
        ws = _capi.workspace(L.xq_recon_psnr_ssim_workspace_bytes(B, C, H, W), x.device)
        _capi.call("xq_recon_psnr_ssim", 2, L.xq_recon_psnr_ssim, rp, int(rec.dtype == torch.bfloat16), xp, B, C, H, W,
                   _capi.ptr(psnr), _capi.ptr(ssim), ws.data_ptr(), ws.numel(), _capi.stream_ptr(x.device),
                   nbytes=rec.numel() * rec.element_size() + x.numel() * 4)
    return psnr, ssim


class ReconstructionMetrics(NamedTuple):
    psnr: float                  # sum(psnr_per_image) / count, as reconstruction_vqgan_ddp.py:186
    ssim: float
    psnr_per_image: np.ndarray   # fp64 [count], rank-major: all of rank 0's images in loader order, then rank 1's, ...
    ssim_per_image: np.ndarray
    count: int


@torch.no_grad()
def reconstruction_metrics(model, loader: Iterable, device=None, max_batches: Optional[int] = None,
                           autocast_dtype: Optional[torch.dtype] = None) -> ReconstructionMetrics:
    """PSNR and SSIM of the model's reconstructions over `loader`, with the reference's scikit-image conventions
    (reconstruction_vqgan_ddp.py:149-190): a checkpoint-ranking number that needs no Inception evaluator.

    Same loop contract as `reconstruct_for_fid`: eval mode for the loop, training flag restored on exit, every rank yields
    the same number of equally sized batches.  Each batch is scored on the device by `psnr_ssim`; only the per-image values
    (two doubles per image) cross ranks, in one all-gather at the end, and the order is the reference's `all_gather_object`
    + `chain`: rank-major.  Every rank returns the same result.  An empty loader gives NaN means and count 0."""
    parts = []
    with _eval_mode(model) as core:
        device = device if device is not None else next(core.parameters()).device
        for x, rec in _reconstructions(core, loader, device, max_batches, autocast_dtype):
            if rec.dtype not in (torch.float32, torch.bfloat16):
                rec = rec.float()                 # exact widening, as reconstruct_for_fid's rec.float()
            p, s = psnr_ssim(rec.contiguous(), x.float().contiguous())
            parts.append(torch.stack([p, s], dim=1))
    local = torch.cat(parts) if parts else torch.zeros(0, 2, dtype=torch.float64, device=device)
    vals = _all_gather_cat(local).cpu().numpy()
    if _distributed():
        dist.barrier()
    psnr_all, ssim_all = vals[:, 0].copy(), vals[:, 1].copy()
    n = len(psnr_all)
    if n == 0:
        return ReconstructionMetrics(float("nan"), float("nan"), psnr_all, ssim_all, 0)
    psnr_list, ssim_list = psnr_all.tolist(), ssim_all.tolist()
    return ReconstructionMetrics(sum(psnr_list) / len(psnr_list), sum(ssim_list) / len(ssim_list), psnr_all, ssim_all, n)
