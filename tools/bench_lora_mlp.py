"""dev tool: the LoRA MLP of a ViT-B block (fc1 / fc2 LoRA-wrapped, base weights frozen) forward and backward, three arms:
  lora   vit_ops._LoRAMLP: the rank-r terms as one more K stage of the fused wgmma GEMMs (xq_vit_fc1_lora_gelu_fwd /
         xq_vit_fc2_lora_dgelu_bwd) + the rank-r library GEMMs
  plain  vit_ops._FusedMLP on the same frozen weights, no adapters: the floor the LoRA terms are added to
  peft   peft's module arithmetic under bf16 autocast: base_layer(x) + lora_B(lora_A(x)) * scaling for fc1 and fc2, GELU
         between, as library GEMMs and element-wise kernels, backward by autograd
   python tools/bench_lora_mlp.py [M N K r]
Default: M = 128 x 513 (the flagship bench's encoder rows), N = 3072, K = 768, r = 8.  Every timing is the median of REPS
windows of CALLS calls (device events around the forward, and around the backward alone), the arms alternating window by
window, with min .. max beside it; the card, its power limit and clocks are printed first, the SM clock again after the run."""
import os
import statistics
import subprocess
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from imagefolder_b200 import vit_ops  # noqa: E402
from imagefolder_b200.dino_enc import lora  # noqa: E402

REPS, CALLS = 15, 5
dev = torch.device("cuda")


def smi(fields):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True, text=True,
                              check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"nvidia-smi unavailable ({e})"


class Mlp(nn.Module):
    def __init__(self, K, N, r):
        super().__init__()
        self.fc1 = lora.Linear(nn.Linear(K, N), r, 8, 0.0)
        self.fc2 = lora.Linear(nn.Linear(N, K), r, 8, 0.0)
        for fc in (self.fc1, self.fc2):
            nn.init.normal_(fc.base_layer.weight, std=0.02)
            nn.init.normal_(fc.lora_B["default"].weight, std=0.02)
            fc.base_layer.requires_grad_(False)


def arms(m):
    fc1, fc2 = m.fc1, m.fc2
    return {
        "lora": lambda y: vit_ops.mlp_forward(m, y),
        "plain": lambda y: vit_ops._FusedMLP.apply(y, fc1.weight, fc1.bias, fc2.weight),
        "peft": lambda y: fc2(F.gelu(fc1(y))),
    }


def timed(fn, y, g):
    """(forward ms, backward ms) of one call"""
    e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    with torch.autocast("cuda", dtype=torch.bfloat16):
        e[0].record()
        out = fn(y)
        e[1].record()
    e[2].record()
    out.backward(g)
    e[3].record()
    torch.cuda.synchronize()
    return e[0].elapsed_time(e[1]), e[2].elapsed_time(e[3])


def main():
    M, N, K, r = (int(a) for a in sys.argv[1:5]) if len(sys.argv) > 4 else (128 * 513, 3072, 768, 8)
    print("card, power limit, max SM clock:", smi("name,power.limit,clocks.max.sm"))
    torch.manual_seed(0)
    m = Mlp(K, N, r).to(dev)
    y = torch.randn(M, K, device=dev).to(torch.bfloat16).requires_grad_(True)
    g = torch.randn(M, K, device=dev).to(torch.bfloat16)
    fns = arms(m)
    outs = {}
    for name, fn in fns.items():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            outs[name] = fn(y).detach().float()
    outs["peft"] -= m.fc2.bias.detach().to(torch.bfloat16).float()     # the fused arms leave it to the next LayerNorm kernel
    d = (outs["lora"] - outs["peft"]).abs()
    print(f"M={M} N={N} K={K} r={r}: |lora - peft| max {float(d.max()):.3e}, mean {float(d.mean()):.3e} "
          f"(max |out| {float(outs['peft'].abs().max()):.3e}); |lora - plain| max "
          f"{float((outs['lora'] - outs['plain']).abs().max()):.3e}")
    for fn in fns.values():
        for _ in range(3):
            timed(fn, y, g)
    res = {n: ([], []) for n in fns}
    for _ in range(REPS):
        for name, fn in fns.items():
            f = b = 0.0
            for _ in range(CALLS):
                tf, tb = timed(fn, y, g)
                f, b = f + tf, b + tb
            res[name][0].append(f / CALLS)
            res[name][1].append(b / CALLS)
    for name, (f, b) in res.items():
        print(f"{name:6s} forward {statistics.median(f):.3f} ms ({min(f):.3f} .. {max(f):.3f})   "
              f"backward {statistics.median(b):.3f} ms ({min(b):.3f} .. {max(b):.3f})")
    print("SM clock, power draw, throttle reasons after the run:",
          smi("clocks.sm,power.draw,clocks_throttle_reasons.active"))


if __name__ == "__main__":
    main()
