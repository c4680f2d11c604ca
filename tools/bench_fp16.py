"""fp16 autocast on the fused ViT kernels: whole training step and per-call times, against bf16 and the library path.

Step arms (VQ-8192, per-GPU batch --batch, 256 x 256; one model and optimizer shared by the arms, which only switch the
autocast dtype and the fused paths):
  fp16_fused    fp16 autocast + GradScaler, the `_f16` kernels
  fp16_library  the same with MLP_TC_ENABLED / ATTN_TC_ENABLED / ASSEMBLE_ENABLED off (attention and MLP on the library)
  bf16_fused    bf16 autocast, the bf16 kernels (what bench.py measures)
Each arm is warmed up, then the arms run in alternating windows of --window steps (CUDA events around each window) for
--rounds rounds; the median ms / step per arm is reported.
Per call: xq_vit_attn_fwd / _bwd (B = 128, N = 513, H = 12) and xq_vit_fc1_gelu_fwd / xq_vit_fc2_dgelu_bwd (M = 128 x 513,
N = 3072, K = 768), f16 and bf16 alternating, median over --rounds windows of --calls launches.
The GPU name, power limit, clocks and throttle reasons are read before and after and printed with the numbers.
Prints one JSON object; --out also writes it to a file.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active,temperature.gpu"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        idx = torch.cuda.current_device()
        return dict(zip(q.split(","), [v.strip() for v in out[idx].split(",")]))
    except Exception as e:          # the numbers stand without it, but say why it is missing
        return {"error": repr(e)}


def time_windows(fns, window, rounds):
    """alternate the callables in windows of `window` calls; median ms per call of each"""
    ms = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(window):
                fn()
            e1.record()
            e1.synchronize()
            ms[k].append(e0.elapsed_time(e1) / window)
    return {k: statistics.median(v) for k, v in ms.items()}


def step_arms(a):
    import torch.nn.functional as F
    from imagefolder_b200 import config as xcfg, vit_ops
    cfg = dict(xcfg.SHIPPED_CONFIGS["VQ-8192"])
    cfg.update(semantic_guide="none", detail_guide="none")
    args = xcfg.parse_args([])
    for k, v in cfg.items():
        setattr(args, k, v)
    torch.manual_seed(0)
    model = xcfg.build_vq_model(args).cuda().train()
    opt = torch.optim.AdamW(model.parameters(), lr=3e-5, betas=(0.9, 0.95), weight_decay=0.0, fused=True)
    scaler = torch.amp.GradScaler("cuda")
    alpha, beta, delta = xcfg.perturbation_schedule(args, 0)
    g = torch.Generator(device="cuda").manual_seed(1234)
    x = torch.rand(a.batch, 3, 256, 256, device="cuda", generator=g) * 2 - 1

    def fused(on):
        vit_ops.MLP_TC_ENABLED[0] = vit_ops.ATTN_TC_ENABLED[0] = vit_ops.ASSEMBLE_ENABLED[0] = on

    def make(dtype, on, scaled):
        def step():
            fused(on)
            with torch.autocast("cuda", dtype=dtype):
                dec, (vq, commit, ent, usages), _, _, _ = model(x, 0, alpha, beta, delta)
                loss = F.mse_loss(dec.float(), x) + vq + commit + ent
            opt.zero_grad(set_to_none=True)
            if scaled:
                scaler.scale(loss).backward()
                scaler.step(opt)
                scaler.update()
            else:
                loss.backward()
                opt.step()
        return step

    arms = {"fp16_fused": make(torch.float16, True, True), "fp16_library": make(torch.float16, False, True),
            "bf16_fused": make(torch.bfloat16, True, False)}
    try:
        for fn in arms.values():
            for _ in range(a.warmup):
                fn()
        torch.cuda.synchronize()
        ms = time_windows(arms, a.window, a.rounds)
    finally:
        fused(True)
    return {k: {"ms_per_step": v, "images_per_s": a.batch * 1000.0 / v} for k, v in ms.items()}


def call_table(a):
    from imagefolder_b200 import _capi
    L = _capi.lib()
    p, s = _capi.ptr, _capi.stream_ptr()
    B, N, H = 128, 513, 12
    M, Nh, K = 128 * 513, 3072, 768
    rows = {}
    for dt, suf in ((torch.float16, "_f16"), (torch.bfloat16, "")):
        torch.manual_seed(0)
        qkv = torch.randn(B, N, 3 * H * 64, device="cuda").to(dt)
        out = torch.empty(B, N, H * 64, device="cuda", dtype=dt)
        lse = torch.empty(B, H, N, device="cuda")
        gout = torch.randn(B, N, H * 64, device="cuda").to(dt)
        dqkv = torch.empty_like(qkv)
        ws = torch.empty(int(L.xq_vit_attn_bwd_workspace_bytes(B, N, H)), dtype=torch.uint8, device="cuda")
        y = (torch.randn(M, K, device="cuda") * 0.5).to(dt)
        w1 = (torch.randn(Nh, K, device="cuda") * 0.03).to(dt)
        b1 = torch.randn(Nh, device="cuda") * 0.1
        pre, act = torch.empty(M, Nh, device="cuda", dtype=dt), torch.empty(M, Nh, device="cuda", dtype=dt)
        gy = torch.randn(M, K, device="cuda").to(dt)
        w2t = (torch.randn(Nh, K, device="cuda") * 0.03).to(dt)
        dpre, db = torch.empty(M, Nh, device="cuda", dtype=dt), torch.empty(Nh, device="cuda")
        f = {n: getattr(L, n + suf) for n in ("xq_vit_attn_fwd", "xq_vit_attn_bwd", "xq_vit_fc1_gelu_fwd",
                                               "xq_vit_fc2_dgelu_bwd")}
        keep = (qkv, out, lse, gout, dqkv, ws, y, w1, b1, pre, act, gy, w2t, dpre, db)
        tag = "f16" if suf else "bf16"
        rows[("xq_vit_attn_fwd", tag)] = lambda f=f, k=keep: _capi.check(
            f["xq_vit_attn_fwd"](p(k[0]), p(k[1]), p(k[2]), B, N, H, 64, 0.125, s), "attn_fwd")
        rows[("xq_vit_attn_bwd", tag)] = lambda f=f, k=keep: _capi.check(
            f["xq_vit_attn_bwd"](p(k[0]), p(k[1]), p(k[3]), p(k[2]), p(k[4]), None, B, N, H, 64, 0.125, p(k[5]), k[5].numel(), s),
            "attn_bwd")
        rows[("xq_vit_fc1_gelu_fwd", tag)] = lambda f=f, k=keep: _capi.check(
            f["xq_vit_fc1_gelu_fwd"](p(k[6]), p(k[7]), p(k[8]), p(k[9]), p(k[10]), M, Nh, K, s), "fc1")
        rows[("xq_vit_fc2_dgelu_bwd", tag)] = lambda f=f, k=keep: _capi.check(
            f["xq_vit_fc2_dgelu_bwd"](p(k[11]), p(k[12]), p(k[9]), p(k[8]), p(k[13]), p(k[14]), M, Nh, K, s), "fc2")
    for fn in rows.values():          # warm-up: module load, tensor maps, attribute set-up
        fn()
        fn()
    torch.cuda.synchronize()
    ms = time_windows(rows, a.calls, a.rounds)
    flops = {"xq_vit_attn_fwd": 4.0 * B * H * N * N * 64, "xq_vit_attn_bwd": 10.0 * B * H * N * N * 64,
             "xq_vit_fc1_gelu_fwd": 2.0 * M * Nh * K, "xq_vit_fc2_dgelu_bwd": 2.0 * M * Nh * K}
    table = []
    for name in flops:
        f16, bf = ms[(name, "f16")], ms[(name, "bf16")]
        table.append({"entry": name, "f16_ms": f16, "bf16_ms": bf, "f16_over_bf16": f16 / bf,
                      "f16_TFLOPs": flops[name] / f16 / 1e9, "bf16_TFLOPs": flops[name] / bf / 1e9})
    return table


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--window", type=int, default=3, help="steps per timed window")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20, help="launches per timed window of the per-call table")
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_fp16.py measures on the GPU; no CUDA device is visible")
    res = {"gpu_before": gpu_state(), "batch": a.batch}
    res["per_call"] = call_table(a)
    if not a.skip_step:
        res["step"] = step_arms(a)
    res["gpu_after"] = gpu_state()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
