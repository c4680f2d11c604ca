"""AdamW step cost on shipped parameter sets: imagefolder_b200.optim.AdamW vs the reference's torch.optim.AdamW (foreach) vs
torch's fused=True kernel.

    python tools/bench_adamw.py [--sets VQ-8192 MSBR10P2-16384 DinoDisc] [--iters 20] [--warmup 3] [--rounds 3]

xqgan_train.py:344-347 builds two AdamW optimizers (tokenizer and discriminator) with no foreach / fused argument, so on CUDA
torch runs its foreach step.  Per parameter set (the trainable parameters of a shipped config, or the DinoDisc heads) each arm
owns its own copy of the params and state, steps the same fixed grads, and is warmed up (state allocated) before timing:
  xq        imagefolder_b200.optim.AdamW: one pass, 28 B per element
  foreach   torch.optim.AdamW(params, lr, betas, weight_decay)  (the reference)
  fused     torch.optim.AdamW(..., fused=True)
Call time: CUDA events around --iters back-to-back step() calls, the arms alternated --rounds times.  Kernel time:
torch.profiler over 5 more calls, device time of the kernels alone.  Host time: one step() from an idle device to its return
(no synchronise inside), median of 10.  Peak growth: torch.cuda.max_memory_allocated during one step over the memory allocated
before it.  Also reports whether each arm's params equal the foreach arm's bit for bit after the same steps.  Prints one JSON line.
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

HYPER = {"VQ-8192": dict(lr=1e-4, betas=(0.9, 0.95), weight_decay=0.0),
         "MSBR10P2-16384": dict(lr=1e-4, betas=(0.9, 0.95), weight_decay=5e-5),
         "DinoDisc": dict(lr=1e-4, betas=(0.9, 0.95), weight_decay=5e-4)}


def param_set(name):
    import warnings
    warnings.filterwarnings("ignore", message=".*RANDOM.*")
    torch.manual_seed(0)
    if name == "DinoDisc":
        from imagefolder_b200.discriminator_dino import DinoDisc
        module = DinoDisc(device="cuda")
    else:
        from imagefolder_b200 import config as xcfg
        args = xcfg.parse_args([])
        for k, v in xcfg.SHIPPED_CONFIGS[name].items():
            setattr(args, k, v)
        module = xcfg.build_vq_model(args)
    params = [p.detach().cuda() for p in module.parameters() if p.requires_grad]
    del module
    return params


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sets", nargs="+", default=["VQ-8192", "MSBR10P2-16384", "DinoDisc"])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_adamw.py measures on a CUDA device; none is available")
    from imagefolder_b200.optim import AdamW
    res = {"iters": a.iters, "warmup": a.warmup, "rounds": a.rounds, "torch": torch.__version__, "sets": {}}
    for name in a.sets:
        base = param_set(name)
        numel = sum(p.numel() for p in base)
        g = torch.Generator(device="cuda").manual_seed(1)
        grads = [torch.randn(p.shape, generator=g, device="cuda") * 1e-3 for p in base]
        kw = HYPER[name]
        arms = {}
        for arm, make in (("xq", lambda ps: AdamW(ps, **kw)), ("foreach", lambda ps: torch.optim.AdamW(ps, **kw)),
                          ("fused", lambda ps: torch.optim.AdamW(ps, fused=True, **kw))):
            ps = [torch.nn.Parameter(p.clone()) for p in base]
            for p, gr in zip(ps, grads):
                p.grad = gr
            arms[arm] = (ps, make(ps))
        del base
        for ps, opt in arms.values():                                # allocates the state; also the bit comparison's steps
            for _ in range(a.warmup):
                opt.step()
        torch.cuda.synchronize()
        same = {k: all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(ps, arms["foreach"][0]))
                for k, (ps, _) in arms.items()}
        ms = {k: [] for k in arms}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(a.rounds):
            for k, (_, opt) in arms.items():
                e0.record()
                for _ in range(a.iters):
                    opt.step()
                e1.record()
                torch.cuda.synchronize()
                ms[k].append(e0.elapsed_time(e1) / a.iters)
        kernel, launches, host, peak = {}, {}, {}, {}
        for k, (_, opt) in arms.items():
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    opt.step()
                torch.cuda.synchronize()
            dev = [e for e in prof.key_averages() if e.self_device_time_total > 0]
            count = sum(e.count for e in dev)
            launches[k] = round(count / 5)
            kernel[k] = sum(e.self_device_time_total for e in dev) / 5 / 1e3
            t = []
            for _ in range(10):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                opt.step()
                t.append(time.perf_counter() - t0)
            torch.cuda.synchronize()
            host[k] = 1e3 * statistics.median(t)
            torch.cuda.reset_peak_memory_stats()
            before = torch.cuda.memory_allocated()
            opt.step()
            torch.cuda.synchronize()
            peak[k] = (torch.cuda.max_memory_allocated() - before) / 2**20
        row = {"tensors": len(arms["xq"][0]), "elements": numel, "hyper": kw, "bit_identical_to_foreach": same}
        for k in arms:
            m = statistics.mean(ms[k])
            row[k] = {"ms_per_step": m, "ms_per_round": ms[k], "kernel_ms_per_step": kernel[k], "kernels_per_step": launches[k],
                      "host_ms_per_step": host[k], "peak_growth_MiB": peak[k],
                      "kernel_GBps_at_28B": 28 * numel / (kernel[k] * 1e-3) / 1e9}
        row["speedup_vs_foreach"] = row["foreach"]["ms_per_step"] / row["xq"]["ms_per_step"]
        row["speedup_vs_fused"] = row["fused"]["ms_per_step"] / row["xq"]["ms_per_step"]
        res["sets"][name] = row
        del arms, grads
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
