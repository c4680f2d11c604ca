"""Host restatement of the reference's reconstruction metrics (tokenizer/vqgan/reconstruction_vqgan_ddp.py:155-169), the
checker of csrc/metric_kernels.cu.

Per image, with x the loader's fp32 image in [-1, 1] and s the clamped reconstruction widened to fp32:
  g = (x + 1) / 2                                   fp32, not quantised
  r = uint8(clamp(127.5 * s + 128, 0, 255)) / 255   fp32; the evaluator's `to_uint8_nhwc`, +128 quirk included
  psnr = skimage peak_signal_noise_ratio(r, g)                  (data_range inferred from r: 1.0)
  ssim = skimage structural_similarity(r, g, data_range=2.0, channel_axis=-1)
         7x7 uniform window, sample covariance, K1 = 0.01, K2 = 0.03, all on fp32 planes
The moment filter is `scipy.ndimage.uniform_filter` (what skimage calls).  `uniform7` is the kernel's scheme for it: per axis
a 7-tap fp64 sum, divided by 7, rounded to fp32.  scikit-image itself is not a dependency: this file restates its algorithm
and is not pinned against a scikit-image run (DESIGN.md)."""
from __future__ import annotations

import numpy as np
from scipy.ndimage import uniform_filter

WIN = 7
PAD = (WIN - 1) // 2
K1, K2, DATA_RANGE = 0.01, 0.03, 2.0
# numpy rounds these Python floats to fp32 when they meet an fp32 array
COV_NORM = np.float32(WIN * WIN / (WIN * WIN - 1.0))
C1 = np.float32((K1 * DATA_RANGE) ** 2)
C2 = np.float32((K2 * DATA_RANGE) ** 2)


def to_uint8(s: np.ndarray) -> np.ndarray:
    """[-1, 1] fp32 -> uint8: clamp(127.5 * s + 128, 0, 255), two fp32 roundings, truncating cast (`to_uint8_nhwc`)."""
    s = np.asarray(s, dtype=np.float32)
    v = np.float32(127.5) * s + np.float32(128.0)
    return np.clip(v, np.float32(0), np.float32(255)).astype(np.uint8)


def restored(s: np.ndarray) -> np.ndarray:
    return to_uint8(s).astype(np.float32) / np.float32(255.0)


def ground_truth(x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, dtype=np.float32)
    return (x + np.float32(1.0)) / np.float32(2.0)


def uniform7(plane: np.ndarray) -> np.ndarray:
    """The kernel's 7x7 box mean of an fp32 [H, W] plane: axis 0, then axis 1, each tap sum in fp64 from the left, / 7,
    rounded to fp32.  Only the interior (rows and columns [3, n-3)) of the result is defined; the border is NaN."""
    p = np.asarray(plane, dtype=np.float32)
    out = p
    for axis in (0, 1):
        n = out.shape[axis]
        src = out.astype(np.float64)
        acc = np.zeros(src.shape, np.float64)
        core = [slice(None)] * 2
        core[axis] = slice(PAD, n - PAD)
        for k in range(-PAD, PAD + 1):
            sl = [slice(None)] * 2
            sl[axis] = slice(PAD + k, n - PAD + k)
            acc[tuple(core)] += src[tuple(sl)]
        res = np.full(src.shape, np.nan, np.float32)
        res[tuple(core)] = (acc[tuple(core)] / 7.0).astype(np.float32)
        if axis == 0:
            res[:PAD] = res[n - PAD:] = 0.0      # rows outside the interior never reach an interior output of axis 1
        out = res
    return out


def scipy_uniform(plane: np.ndarray) -> np.ndarray:
    """skimage's moment filter: scipy.ndimage.uniform_filter(plane, 7) on fp32 (fp32 output after every 1-D pass)."""
    return uniform_filter(np.asarray(plane, dtype=np.float32), size=WIN)


def ssim_channel(r: np.ndarray, g: np.ndarray, filt=uniform7) -> float:
    """skimage structural_similarity of two fp32 [H, W] planes as the reference calls it; fp64 mean of S over the interior."""
    r = np.asarray(r, np.float32)
    g = np.asarray(g, np.float32)
    ux, uy = filt(r), filt(g)
    uxx, uyy, uxy = filt(r * r), filt(g * g), filt(r * g)
    vx = COV_NORM * (uxx - ux * ux)
    vy = COV_NORM * (uyy - uy * uy)
    vxy = COV_NORM * (uxy - ux * uy)
    a1 = np.float32(2) * ux * uy + C1
    a2 = np.float32(2) * vxy + C2
    b1 = ux * ux + uy * uy + C1
    b2 = vx + vy + C2
    s = (a1 * a2) / (b1 * b2)
    return float(s[PAD:-PAD, PAD:-PAD].mean(dtype=np.float64))


def psnr_image(r: np.ndarray, g: np.ndarray) -> float:
    """peak_signal_noise_ratio(r, g): difference and square in fp32, mean in fp64, data_range 1; +inf when mse == 0."""
    d = np.asarray(r, np.float32) - np.asarray(g, np.float32)
    mse = float(np.mean(d * d, dtype=np.float64))
    with np.errstate(divide="ignore"):
        return float(10.0 * np.log10(1.0 / np.float64(mse)))


def psnr_ssim(rec: np.ndarray, x: np.ndarray, filt=uniform7):
    """rec, x: [B, C, H, W] (rec the clamped reconstruction, any float dtype, widened to fp32) -> (psnr [B], ssim [B]) fp64."""
    rec = np.asarray(rec, dtype=np.float32)
    x = np.asarray(x, dtype=np.float32)
    if rec.shape != x.shape or rec.ndim != 4:
        raise ValueError(f"expected two equal [B, C, H, W] arrays, got {rec.shape} and {x.shape}")
    B, C = rec.shape[:2]
    psnr = np.empty(B, np.float64)
    ssim = np.empty(B, np.float64)
    for b in range(B):
        r, g = restored(rec[b]), ground_truth(x[b])
        psnr[b] = psnr_image(r, g)
        ssim[b] = np.mean([ssim_channel(r[c], g[c], filt) for c in range(C)])
    return psnr, ssim
