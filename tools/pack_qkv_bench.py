"""CUDA-event timing of xq_vit_pack_qkv through the C ABI at a training shape: dq, dk, dv [128 * 513, 768] bf16 -> the packed
d(qkv) [128 * 513, 2304] and the qkv-bias gradient.  The ViT blocks only call it on the SDPA fallback path (head_dim != 64),
so bench.py's step does not time it.  Prints one JSON line: median and min / max of the per-launch times over --reps
windows of --iters launches."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from imagefolder_b200 import _capi  # noqa: E402


def make_call(M=128 * 513, C=768, seed=0):
    """a closure that runs one xq_vit_pack_qkv call on fixed random operands, and the outputs it writes"""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    dq, dk, dv = (torch.randn(M, C, device="cuda", generator=gen).to(torch.bfloat16) for _ in range(3))
    out = torch.empty(M, 3 * C, dtype=torch.bfloat16, device="cuda")
    g_bias = torch.empty(3 * C, device="cuda")
    ws = torch.empty(int(_capi.lib().xq_vit_pack_workspace_bytes()), dtype=torch.uint8, device="cuda")
    p = _capi.ptr

    def call():
        L = _capi.lib()
        _capi.check(L.xq_vit_pack_qkv(p(dq), p(dk), p(dv), p(out), p(g_bias), M, C, p(ws), ws.numel(), _capi.stream_ptr()),
                    "xq_vit_pack_qkv")
    return call, (out, g_bias)


def time_ms(call, iters=50, warm=5):
    for _ in range(warm):
        call()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        call()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    call, _ = make_call()
    ts = sorted(time_ms(call, args.iters) for _ in range(args.reps))
    print(json.dumps({"kernel": "pack_qkv_kernel", "rows": 128 * 513, "C": 768, "gpu": torch.cuda.get_device_name(),
                      "median_ms": ts[len(ts) // 2], "min_ms": ts[0], "max_ms": ts[-1]}))


if __name__ == "__main__":
    main()
