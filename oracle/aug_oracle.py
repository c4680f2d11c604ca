"""CPU restatement of the reference's image transforms (dataset/augmentation.py:8-50 + RandomHorizontalFlip + ToTensor +
Normalize(0.5, 0.5), as composed at tokenizer/tokenizer_image/xqgan_train.py:225-230 and :250-254).

`resample` restates Pillow's 8-bit `Image.resize` (libImaging/Resample.c) in numpy:
  - separable; per output index xx the coefficients are computed in fp64:
      scale = in / out, filterscale = max(scale, 1), support = filter_support * filterscale,
      center = (xx + 0.5) * scale, xmin = int(center - support + 0.5) clamped to >= 0,
      xmax = int(center + support + 0.5) clamped to <= in, w_j = filter((j + xmin - center + 0.5) / filterscale)
      (the reciprocal is taken first and multiplied), normalised by their sum;
  - fixed point with PRECISION_BITS = 22, rounding half away from zero (`(int)(k * 2^22 +- 0.5)`);
  - out = clip8((1 << 21) + sum_j k_j * p_j >> 22), horizontal pass first into a uint8 intermediate, vertical second;
  - BICUBIC: a = -0.5, support 2; BOX: support 0.5, 1 on (-0.5, 0.5].
A pass whose size does not change is skipped by Pillow; its coefficients would be the identity, so running it gives the same
bits.  `apply_plan` runs a per-image plan row (h, w, levels, rs_h, rs_w, crop_y, crop_x, flip) with this resample; with
`use_pil=True` it calls `PIL.Image.resize` instead, which the CPU tests use to pin the restatement to Pillow itself.
"""
from __future__ import annotations

import numpy as np

PRECISION_BITS = 22
BOX, BICUBIC = "box", "bicubic"
_SUPPORT = {BOX: 0.5, BICUBIC: 2.0}


def _filter(kind, x):
    if kind == BOX:
        return np.where((x > -0.5) & (x <= 0.5), 1.0, 0.0)
    a = -0.5
    x = np.abs(x)
    near = ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    far = (((x - 5) * x + 8) * x - 4) * a
    return np.where(x < 1.0, near, np.where(x < 2.0, far, 0.0))


def coeffs(in_size: int, out_size: int, kind: str):
    """(xmin [out], fixed-point taps [out, ksize] int64): Pillow's precompute_coeffs + normalize_coeffs_8bpc."""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = _SUPPORT[kind] * filterscale
    ksize = int(np.ceil(support)) * 2 + 1
    center = (np.arange(out_size, dtype=np.float64) + 0.5) * scale
    ss = 1.0 / filterscale
    xmin = np.maximum((center - support + 0.5).astype(np.int64), 0)   # C (int) cast: truncation toward zero
    xmax = np.minimum((center + support + 0.5).astype(np.int64), in_size) - xmin
    j = np.arange(ksize)
    w = _filter(kind, ((j[None, :] + xmin[:, None]) - center[:, None] + 0.5) * ss)
    w = np.where(j[None, :] < xmax[:, None], w, 0.0)
    ww = np.zeros(out_size)
    for t in range(ksize):                  # the C loop's summation order
        ww = ww + w[:, t]
    w = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    k = np.where(w < 0, (-0.5 + w * (1 << PRECISION_BITS)), (0.5 + w * (1 << PRECISION_BITS)))
    return xmin, np.trunc(k).astype(np.int64)


def _pass(a: np.ndarray, out_size: int, kind: str, axis: int) -> np.ndarray:
    in_size = a.shape[axis]
    xmin, k = coeffs(in_size, out_size, kind)
    a = np.moveaxis(a, axis, 0).astype(np.int64)
    acc = np.full((out_size,) + a.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
    for t in range(k.shape[1]):
        idx = np.minimum(xmin + t, in_size - 1)
        acc += k[:, t].reshape((-1,) + (1,) * (a.ndim - 1)) * a[idx]
    out = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(out, 0, axis)


def resample(img: np.ndarray, out_hw, kind: str) -> np.ndarray:
    """uint8 [H, W, 3] -> uint8 [oh, ow, 3], Pillow's `Image.resize((ow, oh), BOX | BICUBIC)`."""
    oh, ow = int(out_hw[0]), int(out_hw[1])
    if img.shape[:2] == (oh, ow):
        return img.copy()
    t = img
    if ow != img.shape[1]:
        t = _pass(t, ow, kind, 1)
    if oh != img.shape[0]:
        t = _pass(t, oh, kind, 0)
    return t


def _pil_resize(img, out_hw, kind):
    from PIL import Image
    return np.asarray(Image.fromarray(img).resize((int(out_hw[1]), int(out_hw[0])),
                                                  resample=Image.BOX if kind == BOX else Image.BICUBIC))


def crop_u8(img: np.ndarray, plan_row, image_size: int, use_pil: bool = False) -> np.ndarray:
    """uint8 [H, W, 3] + one plan row (h, w, levels, rs_h, rs_w, crop_y, crop_x, flip) -> the uint8 [S, S, 3] crop the
    reference's random_crop_arr / center_crop_arr (+ RandomHorizontalFlip) returns for the same draws."""
    h, w, levels, rs_h, rs_w, cy, cx, flip = (int(v) for v in plan_row[:8])
    assert img.shape == (h, w, 3), (img.shape, h, w)
    rs = _pil_resize if use_pil else resample
    for _ in range(levels):
        img = rs(img, (img.shape[0] // 2, img.shape[1] // 2), BOX)
    img = rs(img, (rs_h, rs_w), BICUBIC)
    S = image_size
    out = img[cy:cy + S, cx:cx + S]
    return np.ascontiguousarray(out[:, ::-1] if flip else out)


def to_tensor_normalize(crop: np.ndarray) -> np.ndarray:
    """uint8 [S, S, 3] -> fp32 [3, S, S]: ToTensor (u / 255) then Normalize(0.5, 0.5), in fp32 like torchvision."""
    u = np.ascontiguousarray(crop.transpose(2, 0, 1)).astype(np.float32)
    return (u / np.float32(255.0) - np.float32(0.5)) / np.float32(0.5)


def apply_plan(img: np.ndarray, plan_row, image_size: int, use_pil: bool = False) -> np.ndarray:
    return to_tensor_normalize(crop_u8(img, plan_row, image_size, use_pil))


def synth_image(seed: int, h: int, w: int) -> np.ndarray:
    """Procedural uint8 [h, w, 3] test image: smooth colour ramps plus a sharp checker and uniform noise, so that the bicubic
    overshoot clips at both ends and odd/even taps differ.  Deterministic in (seed, h, w) on any numpy with PCG64."""
    rng = np.random.default_rng(seed)
    yy, xx = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    f = rng.uniform(0.005, 0.05, size=(3, 2))
    base = np.stack([127.5 + 127.5 * np.sin(f[c, 0] * yy + f[c, 1] * xx + c) for c in range(3)], -1)
    checker = (((yy // 7) + (xx // 5)) % 2)[..., None] * 120.0 - 60.0
    noise = rng.integers(-40, 41, size=(h, w, 3)).astype(np.float64)
    return np.clip(np.rint(base + checker + noise), 0, 255).astype(np.uint8)
