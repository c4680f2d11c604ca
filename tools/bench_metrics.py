"""Reconstruction-metric cost: xq_recon_psnr_ssim (evaluate.psnr_ssim) on one validation batch vs the host restatement of the
reference's per-image scikit-image calls.

    python tools/bench_metrics.py [--batch 128] [--size 256] [--iters 50] [--warmup 5] [--oracle-images 4]

The reference scores reconstructions one image at a time on the host (reconstruction_vqgan_ddp.py:155-169).  Here a batch of
--batch images, 3 x --size x --size, is scored for fp32 and for bf16 reconstructions:
  kernel   CUDA events around --iters back-to-back psnr_ssim calls (both launches), after --warmup calls; algorithmic bytes
           per image = 3HW * (4 or 2) for the reconstruction + 3HW * 4 for the input, read once; GB/s = bytes / time
  oracle   oracle/metric_oracle.py (numpy + scipy.ndimage.uniform_filter, one image at a time as the reference) on
           --oracle-images images of the same batch, host seconds per image; the kernel's results on those images are
           compared with it
The card name, power limit and maximum SM clock are read in the same run.  Prints one JSON line.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--oracle-images", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_metrics.py measures on a CUDA device; none is available")
    from imagefolder_b200.evaluate import psnr_ssim
    from oracle import metric_oracle as mo
    B, C, H, W = a.batch, 3, a.size, a.size
    g = torch.Generator().manual_seed(0)
    x = torch.rand(B, C, H, W, generator=g) * 2 - 1
    rec = (x + 0.1 * torch.randn(B, C, H, W, generator=g)).clamp(-1, 1)
    xd = x.cuda()
    res = {"batch": B, "shape": [C, H, W], "iters": a.iters, "warmup": a.warmup, "rounds": a.rounds,
           "torch": torch.__version__, "arms": {}}
    for dtype in (torch.float32, torch.bfloat16):
        rd = rec.to(dtype).cuda()
        for _ in range(a.warmup):
            psnr_ssim(rd, xd)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ms = []
        for _ in range(a.rounds):
            e0.record()
            for _ in range(a.iters):
                psnr_ssim(rd, xd)
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1) / a.iters)
        p, s = psnr_ssim(rd, xd)
        n = a.oracle_images
        t0 = time.perf_counter()
        wp, ws = mo.psnr_ssim(rd[:n].float().cpu().numpy(), x[:n].numpy())
        host_s = (time.perf_counter() - t0) / n
        p, s = p[:n].cpu().numpy(), s[:n].cpu().numpy()
        nbytes = B * C * H * W * (rd.element_size() + 4)
        m = statistics.median(ms)
        res["arms"][str(dtype).replace("torch.", "")] = {
            "kernel_ms_per_batch": m, "ms_per_round": ms, "us_per_image": 1e3 * m / B, "alg_bytes": nbytes,
            "alg_GBps": nbytes / (m * 1e-3) / 1e9, "oracle_host_s_per_image": host_s,
            "oracle_images": n, "max_psnr_rel_err": float(np.max(np.abs(p - wp) / np.abs(wp))),
            "max_ssim_abs_err": float(np.max(np.abs(s - ws))), "mean_psnr": float(p.mean()), "mean_ssim": float(s.mean())}
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers stand without it
        smi = f"unavailable ({e})"
    res.update(device=torch.cuda.get_device_name(0), nvidia_smi=smi)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
