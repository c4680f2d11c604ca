"""Input pipeline: the reference's training / validation image transforms with the pixel work on the GPU.

The reference's DataLoader workers run, per image (tokenizer/tokenizer_image/xqgan_train.py:225-230, :250-254):
    decode -> random_crop_arr | center_crop_arr (dataset/augmentation.py:29-50 | :8-26) -> RandomHorizontalFlip (train)
           -> ToTensor -> Normalize(0.5, 0.5)
Here the workers only decode and draw the random numbers (`GpuDecode`), `collate` packs the uint8 images into one buffer, and
`GpuTransformLoader` runs the BOX halvings, the BICUBIC resize on the crop window, the flip and the normalisation with the
kernels of csrc/img_kernels.cu.  The result is bit-identical (torch.equal) to the reference transform for the same draws:

    loader = DataLoader(ImageFolder(root, transform=GpuDecode(256)), batch_size=128, num_workers=8,
                        collate_fn=collate, pin_memory=True, drop_last=True)
    for x, y in GpuTransformLoader(loader, device="cuda"):
        ...                                   # x: fp32 [128, 3, 256, 256] on the device

The plan draws in the reference's order, in the process that calls it: random.randrange for the short side, random.randrange
for crop_y then crop_x, then torch.rand(1) < 0.5 for the flip.  Inside a DataLoader worker it therefore consumes the same worker
RNG streams as the reference transform would.
"""
from __future__ import annotations

import math
import random
from typing import Iterable, Sequence, Tuple

import numpy as np
import torch

from . import _capi

PLAN_COLUMNS = ("h", "w", "levels", "rs_h", "rs_w", "crop_y", "crop_x", "flip")


def _halve(h: int, w: int, short: int):
    # augmentation.py:37-40 (and :13-16): BOX-halve while the short side is at least twice the target
    levels = 0
    while min(h, w) >= 2 * short:
        h, w, levels = h // 2, w // 2, levels + 1
    scale = short / min(h, w)
    return levels, round(h * scale), round(w * scale)


def plan_random_crop(sizes: Iterable[Sequence[int]], image_size: int, min_crop_frac: float = 0.8,
                     max_crop_frac: float = 1.0, flip: bool = True) -> np.ndarray:
    """int32 [B, 8] plan (PLAN_COLUMNS) of random_crop_arr + RandomHorizontalFlip for images of (h, w) `sizes`.
    Draws per image, in order: randrange(min_s, max_s + 1), randrange(rs_h - S + 1), randrange(rs_w - S + 1), torch.rand(1)."""
    lo = math.ceil(image_size / max_crop_frac)
    hi = math.ceil(image_size / min_crop_frac)
    rows = []
    for h, w in sizes:
        short = random.randrange(lo, hi + 1)
        levels, rh, rw = _halve(int(h), int(w), short)
        cy = random.randrange(rh - image_size + 1)
        cx = random.randrange(rw - image_size + 1)
        f = int(torch.rand(1) < 0.5) if flip else 0
        rows.append((h, w, levels, rh, rw, cy, cx, f))
    return np.asarray(rows, np.int32).reshape(-1, len(PLAN_COLUMNS))


def plan_center_crop(sizes: Iterable[Sequence[int]], image_size: int) -> np.ndarray:
    """int32 [B, 8] plan of center_crop_arr (no random draws, no flip)."""
    rows = []
    for h, w in sizes:
        levels, rh, rw = _halve(int(h), int(w), image_size)
        rows.append((h, w, levels, rh, rw, (rh - image_size) // 2, (rw - image_size) // 2, 0))
    return np.asarray(rows, np.int32).reshape(-1, len(PLAN_COLUMNS))


class GpuDecode:
    """Dataset transform for the workers: PIL image -> (uint8 [h, w, 3] array, int32 [8] plan row).  `train` selects
    random_crop_arr + RandomHorizontalFlip (xqgan_train.py:225-230), otherwise center_crop_arr (:250-254)."""

    def __init__(self, image_size: int = 256, train: bool = True):
        self.image_size, self.train = int(image_size), bool(train)

    def __call__(self, pil_image):
        arr = np.asarray(pil_image.convert("RGB"))
        size = [arr.shape[:2]]
        plan = plan_random_crop(size, self.image_size) if self.train else plan_center_crop(size, self.image_size)
        return arr, plan[0]


def collate(batch):
    """[((uint8 [h, w, 3], plan row), label), ...] -> (packed uint8 [sum h*w*3], src offsets int64 [B], plan int32 [B, 8],
    labels int64 [B]).  The packed buffer is pinned by DataLoader(pin_memory=True) or by GpuTransformLoader."""
    imgs = [np.ascontiguousarray(s[0][0], dtype=np.uint8) for s in batch]
    for a in imgs:
        if a.ndim != 3 or a.shape[2] != 3:
            raise ValueError(f"expected RGB uint8 [h, w, 3] images, got {a.shape}")
    nbytes = np.array([a.size for a in imgs], np.int64)
    offs = np.zeros(len(imgs), np.int64)
    np.cumsum(nbytes[:-1], out=offs[1:])
    packed = torch.empty(int(nbytes.sum()), dtype=torch.uint8)
    flat = packed.numpy()
    for a, o in zip(imgs, offs):
        flat[o:o + a.size] = a.reshape(-1)
    plan = torch.from_numpy(np.stack([np.asarray(s[0][1], np.int32) for s in batch]))
    labels = torch.as_tensor([int(s[1]) for s in batch], dtype=torch.int64)
    return packed, torch.from_numpy(offs), plan, labels


def unpack(packed: torch.Tensor, offs: torch.Tensor, plan: torch.Tensor):
    """Inverse of collate's packing: the list of uint8 [h, w, 3] arrays."""
    out = []
    for o, p in zip(offs.tolist(), plan.tolist()):
        h, w = p[0], p[1]
        out.append(packed[o:o + h * w * 3].numpy().reshape(h, w, 3))
    return out


def gpu_transform(packed: torch.Tensor, offs, plan, image_size: int, out: torch.Tensor = None) -> torch.Tensor:
    """Run a batch's plan on the device, on the current stream.  packed: uint8 [N] on the device; offs (int64 [B]) and plan
    (int32 [B, 8]) on the host, as `collate` returns them: they size the workspace and the halving grids and are copied over.
    Returns fp32 [B, 3, S, S]."""
    L = _capi.lib()
    dev = packed.device
    S, B = int(image_size), int(plan.shape[0])
    plan_h = np.ascontiguousarray(np.asarray(plan), np.int32).reshape(-1, len(PLAN_COLUMNS))
    offs_h = np.ascontiguousarray(np.asarray(offs), np.int64).reshape(-1)
    if offs_h.shape[0] != B:
        raise ValueError("gpu_transform: one offset per plan row")
    ws_off = np.zeros(B, np.int64)
    nbytes = L.xq_img_workspace_bytes(plan_h.ctypes.data, B, S, ws_off.ctypes.data)
    if nbytes == 0:
        raise ValueError("gpu_transform: invalid plan (see include/xqb200.h, xq_img_* preconditions)")
    if int(offs_h.min()) < 0 or int((offs_h + plan_h[:, 0].astype(np.int64) * plan_h[:, 1] * 3).max()) > packed.numel():
        raise ValueError("gpu_transform: an image lies outside the packed buffer")
    # pinned staging: the copies stay asynchronous, and the host allocator keeps the buffers until they complete
    meta = torch.from_numpy(np.stack([offs_h, ws_off], 1)).pin_memory().to(dev, non_blocking=True)
    plan_d = torch.from_numpy(plan_h).pin_memory().to(dev, non_blocking=True)
    ws = _capi.workspace(nbytes, dev)
    if out is None:
        out = torch.empty(B, 3, S, S, dtype=torch.float32, device=dev)
    if out.shape != (B, 3, S, S) or out.dtype != torch.float32:
        raise ValueError(f"gpu_transform: out must be fp32 [{B}, 3, {S}, {S}]")
    st = _capi.stream_ptr(dev)
    src = _capi.ptr(packed)
    for level in range(1, int(plan_h[:, 2].max()) + 1):
        sel = plan_h[plan_h[:, 2] >= level]
        _capi.call("xq_img_box_halve", 1, L.xq_img_box_halve, src, packed.numel(), _capi.ptr(meta), _capi.ptr(plan_d), B, S,
                   level, int((sel[:, 0] >> level).max()), int((sel[:, 1] >> level).max()), _capi.ptr(ws), ws.numel(), st)
    _capi.call("xq_img_resize_crop_normalize", 1, L.xq_img_resize_crop_normalize, src, packed.numel(), _capi.ptr(meta),
               _capi.ptr(plan_d), B, S, _capi.ptr(ws), ws.numel(), _capi.ptr(out), st)
    return out


class GpuTransformLoader:
    """Wraps a DataLoader built with `collate`; yields (fp32 [B, 3, S, S] on `device`, labels) with the transforms run on a side
    stream.  The next batch's copy and kernels are issued before the current one is handed out, so they overlap the caller's
    step; the caller's stream waits on an event before it uses a batch, and the batch is recorded on that stream so the caching
    allocator does not reuse its memory early."""

    def __init__(self, loader, device="cuda", image_size: int = 256):
        self.loader, self.device, self.image_size = loader, torch.device(device), int(image_size)
        if self.device.type != "cuda":
            raise _capi.XqError("GpuTransformLoader needs a CUDA device: there is no CPU path")

    def __len__(self):
        return len(self.loader)

    def _issue(self, batch, stream):
        packed, offs, plan, labels = batch
        if not packed.is_pinned():
            packed = packed.pin_memory()
        with torch.cuda.stream(stream):
            src = packed.to(self.device, non_blocking=True)
            x = gpu_transform(src, offs, plan, self.image_size)
            done = torch.cuda.Event()
            done.record(stream)
        return x, labels, done

    def __iter__(self) -> Iterable[Tuple[torch.Tensor, torch.Tensor]]:
        side = torch.cuda.Stream(self.device)
        it = iter(self.loader)
        try:
            nxt = self._issue(next(it), side)
        except StopIteration:
            return
        while nxt is not None:
            x, labels, done = nxt
            try:
                nxt = self._issue(next(it), side)
            except StopIteration:
                nxt = None
            cur = torch.cuda.current_stream(self.device)
            cur.wait_event(done)
            x.record_stream(cur)
            yield x, labels
