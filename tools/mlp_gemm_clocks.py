"""dev tool: where a tile's clocks go inside the fused MLP GEMMs (csrc/gemm_kernel.cu), measured by the kernel itself.
   python tools/mlp_gemm_clocks.py [--source FILE.cu] [M N K]
Compiles gemm_kernel.cu (or FILE.cu, a variant of it, with the csrc headers) with -DXQ_GM_CLOCKS into a temporary directory.
That option makes thread 0 (first MMA warp) and the first epilogue thread of every CTA add their clock64() laps to a device
buffer; the shipped library is built without it.  Prints, per entry point, the mean clocks per tile of each role:
  MMA warp       K loop (ring waits included) | wait for the staging tile | hand-off (round + stmatrix)
  epilogue warp  wait for a staged tile       | element-wise work and its TMA stores
and the kernel time with the card, its power limit and its maximum SM clock.  The two roles run side by side, so each role's
laps add up to the same time per tile."""
import ctypes
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "imagefolder_b200", "csrc")
SLOTS = ["K loop", "MMA: staging wait", "MMA: hand-off", "epilogue: wait", "epilogue: work", "tiles"]

args = sys.argv[1:]
source = os.path.join(CSRC, "gemm_kernel.cu")
if args[:1] == ["--source"]:
    source, args = args[1], args[2:]
M, N, K = (int(v) for v in args[:3]) if len(args) >= 3 else (128 * 513, 3072, 768)

print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                     text=True).stdout.strip())
with tempfile.TemporaryDirectory() as tmp:
    so = os.path.join(tmp, "gemm_clocks.so")
    subprocess.check_call(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--compiler-options", "-fPIC",
                           "-DXQ_GM_CLOCKS", "-I", CSRC, "-I", os.path.join(ROOT, "include"), "-shared", "-Xlinker", "-Bsymbolic", source, "-o", so, "-lcudart"])
    # the one-file build leaves the library's error bookkeeping (xq::record_cuda_error) to the built libxqb200.so, and is linked
    # -Bsymbolic so that its own kernels, not that library's of the same name, are the ones it launches
    ctypes.CDLL(os.path.join(ROOT, "imagefolder_b200", "lib", "libxqb200.so"), mode=ctypes.RTLD_GLOBAL)
    L = ctypes.CDLL(so)
    dev = torch.device("cuda")
    torch.manual_seed(0)
    y = torch.randn(M, K, device=dev).to(torch.bfloat16)
    g = torch.randn(M, K, device=dev).to(torch.bfloat16)
    W1 = (torch.randn(N, K, device=dev) * 0.03).to(torch.bfloat16)
    W2t = (torch.randn(N, K, device=dev) * 0.03).to(torch.bfloat16)
    b1 = torch.randn(N, device=dev) * 0.1
    pre = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
    act, dpre, db = torch.empty_like(pre), torch.empty_like(pre), torch.empty(N, device=dev)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    calls = {"xq_vit_fc1_gelu_fwd": lambda: L.xq_vit_fc1_gelu_fwd(p(y), p(W1), p(b1), p(pre), p(act), M, N, K, st),
             "xq_vit_fc2_dgelu_bwd": lambda: L.xq_vit_fc2_dgelu_bwd(p(g), p(W2t), p(pre), p(b1), p(dpre), p(db), M, N, K, st)}
    buf = (ctypes.c_ulonglong * (2 * len(SLOTS)))()
    reps = 20
    print(f"M={M} N={N} K={K}, {reps} calls each")
    for i, (name, fn) in enumerate(calls.items()):
        for _ in range(3):
            assert fn() == 0, name
        torch.cuda.synchronize()
        assert L.xq_gm_clocks_read(buf) == 0
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(reps):
            assert fn() == 0, name
        e.record()
        torch.cuda.synchronize()
        assert L.xq_gm_clocks_read(buf) == 0
        c = list(buf)[i * len(SLOTS):(i + 1) * len(SLOTS)]
        tiles = max(1, c[-1])
        print(f"{name}: {s.elapsed_time(e) / reps:.3f} ms per call (instrumented); clocks per tile: "
              + ", ".join(f"{n} {v / tiles:.0f}" for n, v in zip(SLOTS[:-1], c[:-1])))
