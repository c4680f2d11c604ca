"""dev tool: one launch set of a hot kernel at its bench shape, for `ncu --set full` captures (profiles/README.md):
     python tools/ncu_target.py attn [B N H]      wgmma attention forward + backward       (default 256 513 12 = VQ-8192, B=256)
     python tools/ncu_target.py vq   [B V C]      single-scale search, 16x16 tokens/image  (default 256 8192 32)
     python tools/ncu_target.py ms   [B V]        MSVR10P2 fused 10-scale kernel, training  (default 128 4096)"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from imagefolder_b200 import VectorQuantizer2, ops, vit_ops  # noqa: E402

what = sys.argv[1] if len(sys.argv) > 1 else "attn"
nums = [int(x) for x in sys.argv[2:]]
torch.manual_seed(0)
if what == "attn":
    B, N, H = nums if len(nums) == 3 else (256, 513, 12)
    qkv = torch.randn(B, N, 3 * H * 64, device="cuda").to(torch.bfloat16)
    g = torch.randn(B, N, H * 64, device="cuda").to(torch.bfloat16)
    for _ in range(2):
        out, lse = vit_ops.attn_tc_forward(qkv, H)
        dqkv = vit_ops.attn_tc_backward(qkv, out, lse, g, H)
    r = float(dqkv.float().abs().mean())
elif what == "vq":
    B, V, C = nums if len(nums) == 3 else (256, 8192, 32)
    z = torch.randn(B, C, 16, 16, device="cuda")
    E = torch.randn(V, C, device="cuda")
    for _ in range(2):
        zq = ops.vq_forward(z, E, 0.25, True, want_hist=True)[0]
    r = float(zq.abs().mean())
elif what == "ms":
    B, V = nums if len(nums) == 2 else (128, 4096)
    pn = [1, 1, 2, 3, 3, 4, 5, 6, 8, 11]
    q = VectorQuantizer2(V, 32, v_patch_nums=pn, num_latent_tokens=121, codebook_drop=0.1).cuda().train()
    f = torch.randn(B, 32, 11, 11, device="cuda")
    dr = torch.randint(3, 11, (B,))
    for _ in range(2):
        o = q(f, True, dr)
    r = float(o[0].abs().mean())
else:
    raise SystemExit(__doc__)
torch.cuda.synchronize()
print("done", what, r)
