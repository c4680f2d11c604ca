"""Weight-EMA step cost on shipped parameter sets: the reference loop vs torch's foreach ops vs xq_ema_update (ema.py).

    python tools/bench_ema.py [--configs VQ-8192 MSBR10P2-16384] [--iters 50] [--warmup 5] [--rounds 3]

Every shipped config trains with `ema: true`, so xqgan_train.py:461-462 runs update_ema after every optimizer step.  Per config
(built as shipped, frozen teachers included, because the reference averages their parameters too) three arms update the same
EMA copy at decay 0.9999:
  reference   utils/ema.py:4-14: ema.mul_(decay).add_(param, alpha=1 - decay) per tensor (2 kernels, 20 B per element)
  foreach     torch._foreach_mul_ + torch._foreach_add_ over the same lists (20 B per element)
  xq          imagefolder_b200.ema.update_ema: one launch, one pass (12 B per element)
Call time: CUDA events around --iters back-to-back calls, the arms alternated --rounds times in this process (when the host
cannot enqueue a call as fast as the device runs it, this is the host's rate).  Kernel time: torch.profiler over 10 more calls,
the device time of the kernels alone.  Host time: the enqueue of one call (device idle before it, no synchronise inside),
median of 20.  Bandwidth is algorithmic bytes over call time and over kernel time, also given as a fraction of
MEASURED_PEAKS.json's hbm_gbs when that file exists, else of the H100 SXM data sheet's 3.35 TB/s.  Prints one JSON line.
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys
import time
from collections import OrderedDict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def hbm_peak():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        d = json.load(open(path))
        if "hbm_gbs" in d:
            return float(d["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    return 3350.0, "data sheet (H100 SXM 3.35 TB/s, not a measured peak)"


@torch.no_grad()
def reference_arm(ema_model, model, decay=0.9999):
    ema_params = OrderedDict(ema_model.named_parameters())
    for name, param in OrderedDict(model.named_parameters()).items():
        ema_params[name].mul_(decay).add_(param.data, alpha=1 - decay)


@torch.no_grad()
def foreach_arm(ema_model, model, decay=0.9999):
    ema_params = OrderedDict(ema_model.named_parameters())
    names = [n for n, _ in model.named_parameters()]
    e = [ema_params[n] for n in names]
    p = [q.data for q in model.parameters()]
    torch._foreach_mul_(e, decay)
    torch._foreach_add_(e, p, alpha=1 - decay)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["VQ-8192", "MSBR10P2-16384"])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ema.py measures on a CUDA device; none is available")
    import warnings
    from imagefolder_b200 import config as xcfg
    from imagefolder_b200.ema import update_ema
    warnings.filterwarnings("ignore", message=".*RANDOM.*")
    peak, peak_src = hbm_peak()
    arms = {"reference": (reference_arm, 20), "foreach": (foreach_arm, 20), "xq": (update_ema, 12)}
    res = {"iters": a.iters, "warmup": a.warmup, "rounds": a.rounds, "decay": 0.9999, "hbm_peak_GBps": peak,
           "hbm_peak_source": peak_src, "torch": torch.__version__, "configs": {}}
    for name in a.configs:
        args = xcfg.parse_args([])
        for k, v in xcfg.SHIPPED_CONFIGS[name].items():
            setattr(args, k, v)
        torch.manual_seed(0)
        model = xcfg.build_vq_model(args).cuda()
        ema = copy.deepcopy(model)
        params = list(model.parameters())
        numel = sum(p.numel() for p in params)
        # same bits as the reference at the timed size (one step from identical copies)
        with torch.no_grad():
            for p in params:
                p.add_(torch.randn_like(p) * 1e-2)
        ref = copy.deepcopy(ema)
        update_ema(ema, model)
        reference_arm(ref, model)
        torch.cuda.synchronize()
        identical = all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(ema.parameters(), ref.parameters()))
        del ref
        ms = {k: [] for k in arms}
        for fn, _ in arms.values():
            for _ in range(a.warmup):
                fn(ema, model)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(a.rounds):
            for k, (fn, _) in arms.items():
                e0.record()
                for _ in range(a.iters):
                    fn(ema, model)
                e1.record()
                torch.cuda.synchronize()
                ms[k].append(e0.elapsed_time(e1) / a.iters)
        kernel, launches = {}, {}
        for k, (fn, _) in arms.items():
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(10):
                    fn(ema, model)
                torch.cuda.synchronize()
            dev = [e for e in prof.key_averages() if e.self_device_time_total > 0]
            count = sum(e.count for e in dev)
            # mean kernel time x kernels per call: robust to the odd kernel record the profiler drops
            launches[k] = round(count / 10)
            kernel[k] = sum(e.self_device_time_total for e in dev) / count * launches[k] / 1e3
        host = {}
        for k, (fn, _) in arms.items():
            t = []
            for _ in range(20):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn(ema, model)
                t.append(time.perf_counter() - t0)
            torch.cuda.synchronize()
            host[k] = 1e3 * statistics.median(t)
        row = {"tensors": len(params), "elements": numel, "bit_identical_to_reference": identical}
        for k, (_, bpe) in arms.items():
            m = statistics.mean(ms[k])
            gbs = bpe * numel / (m * 1e-3) / 1e9
            kgbs = bpe * numel / (kernel[k] * 1e-3) / 1e9
            row[k] = {"ms_per_call": m, "ms_per_round": ms[k], "host_enqueue_ms": host[k], "kernel_ms_per_call": kernel[k],
                      "kernels_per_call": launches[k],
                      "alg_bytes": bpe * numel, "alg_GBps": gbs, "frac_of_hbm_peak": gbs / peak,
                      "kernel_alg_GBps": kgbs, "kernel_frac_of_hbm_peak": kgbs / peak}
        row["speedup_vs_reference"] = row["reference"]["ms_per_call"] / row["xq"]["ms_per_call"]
        row["speedup_vs_foreach"] = row["foreach"]["ms_per_call"] / row["xq"]["ms_per_call"]
        res["configs"][name] = row
        del model, ema, params
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
