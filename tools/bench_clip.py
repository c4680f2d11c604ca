"""Gradient-norm clipping on shipped gradient sets: imagefolder_b200.optim.clip_grad_norm_ vs torch.nn.utils.clip_grad_norm_.

    python tools/bench_clip.py [--sets VQ-8192 MSBR10P2-16384 DinoDisc] [--iters 20] [--warmup 3] [--rounds 5]

With --max_grad_norm set, xqgan_train.py:456-458 and :471-473 clip the tokenizer's and the discriminator's grads between
scaler.unscale_ and scaler.step.  Per gradient set (the trainable parameters of a shipped config, or the DinoDisc heads, with
seeded grads of training magnitude, so max_norm = 1 clips) each arm owns its own copy of the grads:
  xq      imagefolder_b200.optim.clip_grad_norm_: xq_grad_norm (4 B per element) + torch's scalar ops + xq_grad_scale (8 B)
  torch   torch.nn.utils.clip_grad_norm_ (the reference): _foreach_norm, stack, vector_norm, clamp, _foreach_mul_
Call time: CUDA events around --iters back-to-back calls, the arms alternated over --rounds windows.  Kernel time:
torch.profiler over 5 more calls in a separate pass, the device time of all kernels of a call, and of the xq kernels alone.
Launches: kernels per call from the same trace.  Host time: one call from an idle device to its return, median of 10.  Also
reports whether both arms give the same total norm and grads bit for bit from the same grads, and the data-sheet floor of
the two streaming passes (12 B per element at 3.35 TB/s).  Prints one JSON line with the card, power limit and max SM clock.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

HBM_TBPS = 3.35                                      # H100 SXM data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sets", nargs="+", default=["VQ-8192", "MSBR10P2-16384", "DinoDisc"])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--max_norm", type=float, default=1.0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_clip.py measures on a CUDA device; none is available")
    from bench_adamw import param_set
    from imagefolder_b200.optim import clip_grad_norm_
    fns = {"xq": clip_grad_norm_, "torch": torch.nn.utils.clip_grad_norm_}
    res = {"iters": a.iters, "warmup": a.warmup, "rounds": a.rounds, "max_norm": a.max_norm, "torch": torch.__version__,
           "sets": {}}
    for name in a.sets:
        base = param_set(name)
        numel = sum(p.numel() for p in base)
        g = torch.Generator(device="cuda").manual_seed(1)
        grads = [torch.randn(p.shape, generator=g, device="cuda") * 1e-3 for p in base]
        arms = {}
        for k in fns:
            ps = [torch.nn.Parameter(p.clone()) for p in base]
            for p, gr in zip(ps, grads):
                p.grad = gr.clone()
            arms[k] = ps
        del grads
        totals = {k: fns[k](ps, a.max_norm) for k, ps in arms.items()}  # one call each from the same grads: the bit check
        torch.cuda.synchronize()
        same = torch.equal(totals["xq"].view(torch.int32), totals["torch"].view(torch.int32)) and all(
            torch.equal(x.grad.view(torch.int32), y.grad.view(torch.int32)) for x, y in zip(arms["xq"], arms["torch"]))
        for k, ps in arms.items():
            for _ in range(a.warmup):
                fns[k](ps, a.max_norm)
        torch.cuda.synchronize()
        ms = {k: [] for k in arms}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(a.rounds):
            for k, ps in arms.items():
                e0.record()
                for _ in range(a.iters):
                    fns[k](ps, a.max_norm)
                e1.record()
                torch.cuda.synchronize()
                ms[k].append(e0.elapsed_time(e1) / a.iters)
        kernel, own, launches, host = {}, {}, {}, {}
        for k, ps in arms.items():
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    fns[k](ps, a.max_norm)
                torch.cuda.synchronize()
            dev = [e for e in prof.key_averages() if e.self_device_time_total > 0]
            launches[k] = round(sum(e.count for e in dev) / 5)
            kernel[k] = sum(e.self_device_time_total for e in dev) / 5 / 1e3
            own[k] = sum(e.self_device_time_total for e in dev if "grad_norm_" in e.key or "grad_scale_" in e.key) / 5 / 1e3
            t = []
            for _ in range(10):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fns[k](ps, a.max_norm)
                t.append(time.perf_counter() - t0)
            torch.cuda.synchronize()
            host[k] = 1e3 * statistics.median(t)
        row = {"tensors": len(arms["xq"]), "elements": numel, "bit_identical_to_torch": same,
               "floor_ms_at_12B": 12 * numel / (HBM_TBPS * 1e12) * 1e3}
        for k in arms:
            row[k] = {"ms_per_call": statistics.median(ms[k]), "ms_per_round": ms[k], "kernel_ms_per_call": kernel[k],
                      "kernels_per_call": launches[k], "host_ms_per_call": host[k],
                      "kernel_GBps_at_12B": 12 * numel / (kernel[k] * 1e-3) / 1e9}
        row["xq"]["xq_kernels_ms_per_call"] = own["xq"]
        row["speedup_vs_torch"] = row["torch"]["ms_per_call"] / row["xq"]["ms_per_call"]
        res["sets"][name] = row
        del arms, base
        torch.cuda.empty_cache()
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers stand without it
        smi = f"unavailable ({e})"
    res.update(device=torch.cuda.get_device_name(0), nvidia_smi=smi)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
