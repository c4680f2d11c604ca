"""dev tool: the fused MLP GEMMs (xq_vit_fc1_gelu_fwd / xq_vit_fc2_dgelu_bwd, csrc/gemm_kernel.cu) against the two-call sequences they
replace (library GEMM + stand-alone bias / GELU kernel), with a bit-level comparison.
   python tools/mlp_gemm_bench.py [M N K]
Without arguments: the ViT-B MLP (N = 3072, K = 768) at the flagship bench's encoder rows (M = 128 x 513) and at twice that.
Each timing is the median of REPS windows of CALLS calls (device events), the two arms alternating window by window; the
spread (min .. max) is printed beside it, and the card, its power limit and its maximum SM clock above everything."""
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from imagefolder_b200 import _capi as C, vit_ops  # noqa: E402

REPS, CALLS = 15, 5
dev = torch.device("cuda")
L = C.lib()
st = C.stream_ptr(dev)


def window(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(CALLS):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / CALLS


def compare(a, b):
    """medians and spreads of two arms, timed in alternating windows"""
    for fn in (a, b):
        for _ in range(3):
            fn()
    ta, tb = [], []
    for _ in range(REPS):
        ta.append(window(a))
        tb.append(window(b))
    return [(statistics.median(t), min(t), max(t)) for t in (ta, tb)]


def run(M, N, K):
    torch.manual_seed(0)
    y = torch.randn(M, K, device=dev).to(torch.bfloat16)
    W1 = (torch.randn(N, K, device=dev) * 0.03).to(torch.bfloat16)
    b1 = torch.randn(N, device=dev) * 0.1
    W2t = (torch.randn(N, K, device=dev) * 0.03).to(torch.bfloat16)     # fc2.weight^T
    g = torch.randn(M, K, device=dev).to(torch.bfloat16)
    pre = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
    act = torch.empty_like(pre)
    dpre = torch.empty_like(pre)
    db = torch.empty(N, device=dev)

    def fused_fwd():
        C.call("xq_vit_fc1_gelu_fwd", 1, L.xq_vit_fc1_gelu_fwd, C.ptr(y), C.ptr(W1), C.ptr(b1), C.ptr(pre), C.ptr(act), M, N, K, st)

    def fused_bwd():
        C.call("xq_vit_fc2_dgelu_bwd", 1, L.xq_vit_fc2_dgelu_bwd, C.ptr(g), C.ptr(W2t), C.ptr(pre), C.ptr(b1), C.ptr(dpre), C.ptr(db), M, N, K, st)

    def lib_fwd():
        p = y @ W1.t()
        return p, vit_ops.gelu_bias(p, b1)

    def lib_bwd():
        da = g @ W2t.t()
        gx = torch.empty_like(da)
        gb = torch.empty_like(b1)
        C.call("xq_vit_gelu_bwd", 1, L.xq_vit_gelu_bwd, C.ptr(pre), C.ptr(b1), C.ptr(da), C.ptr(gx), C.ptr(gb), M, N, st)
        return gx, gb

    fused_fwd()
    p_ref, a_ref = lib_fwd()
    fused_bwd()
    gx_ref, gb_ref = lib_bwd()
    torch.cuda.synchronize()
    print(f"M={M} N={N} K={K}")
    print("pre  identical:", torch.equal(pre, p_ref), "  act identical:", torch.equal(act, a_ref))
    exact = dpre.double().sum(0)
    print("dpre identical:", torch.equal(dpre, gx_ref),
          f"  d_bias vs fp64 column sums of d_pre (max err / max |sum|): fused {((db.double() - exact).abs().max() / exact.abs().max()).item():.2e}"
          f", stand-alone kernel {((gb_ref.double() - exact).abs().max() / exact.abs().max()).item():.2e}")
    del p_ref, a_ref, gx_ref, gb_ref, exact
    fl = 2.0 * M * N * K
    for name, fused, lib, kern in (("forward ", fused_fwd, lib_fwd, "gelu_fwd"), ("backward", fused_bwd, lib_bwd, "gelu_bwd")):
        (t, tlo, thi), (tl, llo, lhi) = compare(fused, lib)
        print(f"{name}: fused {t:.3f} ms [{tlo:.3f} .. {thi:.3f}] ({fl / t / 1e9:.0f} TFLOP/s)   "
              f"library GEMM + {kern} kernel {tl:.3f} ms [{llo:.3f} .. {lhi:.3f}]")


print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                     text=True).stdout.strip())
if len(sys.argv) > 3:
    run(*(int(v) for v in sys.argv[1:4]))
else:
    for M in (128 * 513, 2 * 128 * 513):
        run(M, 3072, 768)
