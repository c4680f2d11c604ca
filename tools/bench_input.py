"""Input-pipeline cost: the reference's per-image CPU transform vs decode-only workers + the GPU transform (data.py).

    python tools/bench_input.py [--batch 128] [--iters 50] [--cpu-images 64] [--rate 580]

Prints one JSON line:
  cpu_decode_ms_per_img        PIL JPEG decode + convert('RGB') (quality-90 JPEGs of ImageNet-like sizes), one thread
  cpu_reference_ms_per_img     the reference transform on the decoded image: BOX halvings + BICUBIC resize (PIL), crop, flip,
                               ToTensor, Normalize (written out as dataset/augmentation.py + xqgan_train.py:225-230 compose it)
  cpu_decode_pack_ms_per_img   decode + np.asarray + plan draws + collate packing (what a worker does with GpuDecode)
  gpu_ms_per_batch             gpu_transform on a resident packed batch (CUDA events, mean over --iters)
  gpu_h2d_ms_per_batch         the same including the pinned host-to-device copy of the packed batch
  cores_per_gpu_*              worker cores needed to feed one GPU at --rate img/s with each path
The GPU numbers need a CUDA device; the CPU numbers are per thread on whatever host runs the script.
"""
import argparse
import io
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def imagenet_like_sizes(n, rng):
    """short side 300-500 with the common 4:3 / 3:4 / 1:1 / 16:9 shapes, plus a few large photos"""
    out = []
    for k in range(n):
        short = int(rng.integers(300, 501)) if k % 16 else int(rng.integers(1000, 2200))
        ar = [4 / 3, 4 / 3, 4 / 3, 1.0, 16 / 9][k % 5]
        long_ = int(round(short * ar))
        out.append((short, long_) if k % 3 else (long_, short))
    return out


def jpeg_bytes(h, w, seed):
    from PIL import Image
    from oracle.aug_oracle import synth_image
    buf = io.BytesIO()
    Image.fromarray(synth_image(seed, h, w)).save(buf, format="JPEG", quality=90)
    return buf.getvalue()


def reference_transform(im, plan_row, S):
    """PIL pipeline of random_crop_arr + RandomHorizontalFlip + ToTensor + Normalize for a given plan row"""
    from PIL import Image
    from torchvision import transforms as T
    _, _, levels, rh, rw, cy, cx, flip = (int(v) for v in plan_row)
    for _ in range(levels):
        im = im.resize((im.size[0] // 2, im.size[1] // 2), resample=Image.BOX)
    im = im.resize((rw, rh), resample=Image.BICUBIC)
    arr = np.array(im)
    im = Image.fromarray(arr[cy:cy + S, cx:cx + S])
    if flip:
        im = im.transpose(Image.FLIP_LEFT_RIGHT)
    return T.Normalize(mean=[0.5] * 3, std=[0.5] * 3, inplace=True)(T.ToTensor()(im))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--cpu-images", type=int, default=64)
    ap.add_argument("--image-size", type=int, default=256)
    ap.add_argument("--rate", type=float, default=580.0, help="training img/s per GPU to feed")
    a = ap.parse_args()
    from PIL import Image
    from imagefolder_b200 import data
    torch.set_num_threads(1)
    S = a.image_size
    rng = np.random.default_rng(0)
    random.seed(0)
    torch.manual_seed(0)
    sizes = imagenet_like_sizes(a.batch, rng)
    blobs = [jpeg_bytes(h, w, k) for k, (h, w) in enumerate(sizes)]
    res = {"batch": a.batch, "image_size": S, "pillow": Image.__version__, "torch": torch.__version__}

    # --- CPU, one thread: decode, reference transform, decode + pack
    n = min(a.cpu_images, len(blobs))
    t0 = time.perf_counter()
    decoded = [Image.open(io.BytesIO(b)).convert("RGB") for b in blobs[:n]]
    t_dec = (time.perf_counter() - t0) / n
    plan = data.plan_random_crop([(im.size[1], im.size[0]) for im in decoded], S)
    reference_transform(decoded[0], plan[0], S)            # imports torchvision outside the timed loop
    t0 = time.perf_counter()
    for im, p in zip(decoded, plan):
        reference_transform(im, p, S)
    t_ref = (time.perf_counter() - t0) / n
    dec = data.GpuDecode(S)
    t0 = time.perf_counter()
    batch = [(dec(Image.open(io.BytesIO(b))), 0) for b in blobs[:n]]
    data.collate(batch)
    t_pack = (time.perf_counter() - t0) / n
    res.update(cpu_decode_ms_per_img=1e3 * t_dec, cpu_reference_ms_per_img=1e3 * t_ref,
               cpu_decode_pack_ms_per_img=1e3 * t_pack,
               cores_per_gpu_reference=a.rate * (t_dec + t_ref), cores_per_gpu_decode_pack=a.rate * t_pack)

    # --- GPU: the whole batch
    if not torch.cuda.is_available():
        res["gpu"] = "not measured: no CUDA device"
        print(json.dumps(res))
        return
    full = [(dec(Image.open(io.BytesIO(b))), 0) for b in blobs]
    packed, offs, plan_t, _ = data.collate(full)
    packed = packed.pin_memory()
    src = packed.cuda()
    out = torch.empty(a.batch, 3, S, S, device="cuda")
    for _ in range(5):
        data.gpu_transform(src, offs, plan_t, S, out=out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.iters):
        data.gpu_transform(src, offs, plan_t, S, out=out)
    e1.record()
    torch.cuda.synchronize()
    gpu_ms = e0.elapsed_time(e1) / a.iters
    e0.record()
    for _ in range(a.iters):
        src.copy_(packed, non_blocking=True)
        data.gpu_transform(src, offs, plan_t, S, out=out)
    e1.record()
    torch.cuda.synchronize()
    h2d_ms = e0.elapsed_time(e1) / a.iters
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers stand without it
        smi = f"unavailable ({e})"
    res.update(gpu_ms_per_batch=gpu_ms, gpu_h2d_ms_per_batch=h2d_ms, packed_MB=packed.numel() / 1e6,
               gpu_ms_per_img=gpu_ms / a.batch, halving_levels=sorted(set(plan_t[:, 2].tolist())),
               device=torch.cuda.get_device_name(0), nvidia_smi=smi)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
