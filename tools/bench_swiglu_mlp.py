"""Time the fused SwiGLU GEMMs against a library GEMM + the stand-alone SwiGLU kernel at the giant training shape.

    python tools/bench_swiglu_mlp.py [--windows 10] [--iters 20]

Shape: M = 32 * 513 tokens (batch 32, S = 513), fc1 1536 -> 8192 ([gate | up], H = 4096), fc2 K = 1536 in the backward.
  forward   xq_vit_fc1_swiglu_fwd           vs  y @ W1^T (cuBLAS) + xq_vit_swiglu_fwd
  backward  xq_vit_fc2_dswiglu_bwd          vs  g @ W2   (cuBLAS) + xq_vit_swiglu_bwd
Windows of `iters` calls alternate between the two forms (CUDA events around each window); the median window is reported.
The card's name, power limit and max SM clock are read in the same run and printed with the result (one JSON line).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from imagefolder_b200 import _capi  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the timing stands without it, but says so
        out = f"unavailable ({e})"
    return out


def window(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=10)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    L, p, s = _capi.lib(), _capi.ptr, _capi.stream_ptr()
    M, D, H = 32 * 513, 1536, 4096
    dt = torch.bfloat16
    g = torch.Generator(device="cuda").manual_seed(0)
    y = torch.randn(M, D, device="cuda", generator=g).to(dt)
    W1 = (torch.randn(2 * H, D, device="cuda", generator=g) / D ** 0.5).to(dt)
    b1 = torch.randn(2 * H, device="cuda", generator=g) * 0.1
    W2 = (torch.randn(D, H, device="cuda", generator=g) / H ** 0.5).to(dt)
    W2t = W2.t().contiguous()
    gb = torch.randn(M, D, device="cuda", generator=g).to(dt)
    pre, act = torch.empty(M, 2 * H, dtype=dt, device="cuda"), torch.empty(M, H, dtype=dt, device="cuda")
    dpre, db = torch.empty(M, 2 * H, dtype=dt, device="cuda"), torch.empty(2 * H, device="cuda")
    pre_l, act_l = torch.empty_like(pre), torch.empty_like(act)
    dpre_l, db_l = torch.empty_like(dpre), torch.empty_like(db)
    gact = torch.empty(M, H, dtype=dt, device="cuda")

    def fused_fwd():
        L.xq_vit_fc1_swiglu_fwd(p(y), p(W1), p(b1), p(pre), p(act), M, H, D, s)

    def lib_fwd():
        torch.matmul(y, W1.t(), out=pre_l)
        L.xq_vit_swiglu_fwd(p(pre_l), p(b1), p(act_l), M, H, s)

    def fused_bwd():
        L.xq_vit_fc2_dswiglu_bwd(p(gb), p(W2t), p(pre), p(b1), p(dpre), p(db), M, H, D, s)

    def lib_bwd():
        torch.matmul(gb, W2, out=gact)
        L.xq_vit_swiglu_bwd(p(pre), p(b1), p(gact), p(dpre_l), p(db_l), M, H, s)

    for fn in (fused_fwd, lib_fwd, fused_bwd, lib_bwd):
        fn()
    torch.cuda.synchronize()
    _capi.check(L.xq_vit_fc1_swiglu_fwd(p(y), p(W1), p(b1), p(pre), p(act), M, H, D, s), "fused fwd")
    res = {}
    for name, a, b in (("forward", fused_fwd, lib_fwd), ("backward", fused_bwd, lib_bwd)):
        for fn in (a, b):
            window(fn, args.iters)                               # warm-up window
        ta, tb = [], []
        for _ in range(args.windows):
            ta.append(window(a, args.iters))
            tb.append(window(b, args.iters))
        flops = 2.0 * M * D * (2 * H if name == "forward" else H)
        fa, fb = statistics.median(ta), statistics.median(tb)
        res[name] = {"fused_ms": round(fa, 4), "library_ms": round(fb, 4), "fused_tflops": round(flops / fa / 1e9, 1),
                     "library_gemm_plus_kernel_tflops": round(flops / fb / 1e9, 1),
                     "fused_spread_ms": [round(min(ta), 4), round(max(ta), 4)],
                     "library_spread_ms": [round(min(tb), 4), round(max(tb), 4)]}
    # outputs of the two forms on the same inputs (act / d_pre are equal up to the GEMMs' accumulation order)
    lib_fwd()
    fused_fwd()
    lib_bwd()
    fused_bwd()
    torch.cuda.synchronize()
    res["act_max_abs_diff"] = float((act.float() - act_l.float()).abs().max())
    res["d_pre_max_abs_diff"] = float((dpre.float() - dpre_l.float()).abs().max())
    res["card"] = card()
    res["shape"] = {"M": M, "K_fwd": D, "N_fwd": 2 * H, "K_bwd": D, "N_bwd": H}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
