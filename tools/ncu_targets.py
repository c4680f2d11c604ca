"""one launch of every libxqb200 ViT glue kernel at the B = 256 training shapes (for `ncu --set full -k regex:xqv`)."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from imagefolder_b200 import vit_ops
from imagefolder_b200.dino_enc.vision_transformer import PatchEmbed

B, S, D, H = 256, 513, 768, 12
dev = "cuda"
x = torch.randn(B, S, D, device=dev, requires_grad=True)
br = torch.randn(B, S, D, device=dev).to(torch.bfloat16).requires_grad_(True)
g = torch.rand(D, device=dev, requires_grad=True)
bb = torch.randn(D, device=dev, requires_grad=True)
w = torch.rand(D, device=dev, requires_grad=True)
b = torch.randn(D, device=dev, requires_grad=True)
rs = torch.ones(B, device=dev)
xo, y = vit_ops.residual_ln(x, br, bb, g, rs, w, b, 1e-6)                        # residual_ln_fwd_kernel
torch.autograd.grad((xo, y), (x, br, g, bb, w, b), (torch.randn_like(xo), torch.randn_like(y)))   # ln_bwd + reduce_parts
h = torch.randn(B, S, 4 * D, device=dev).to(torch.bfloat16).requires_grad_(True)
b1 = torch.randn(4 * D, device=dev, requires_grad=True)
yy = vit_ops.gelu_bias(h, b1)                                                    # gelu_fwd_kernel
torch.autograd.grad(yy, (h, b1), torch.randn_like(yy))                           # gelu_bwd_kernel
del h, yy
yq = torch.randn(B, S, D, device=dev).to(torch.bfloat16).requires_grad_(True)
Wq = (torch.randn(3 * D, D, device=dev) * D ** -0.5).requires_grad_(True)
bq = torch.randn(3 * D, device=dev, requires_grad=True)
o = vit_ops._QKVAttention.apply(yq, Wq, bq, H)                                  # attn_fwd_kernel
torch.autograd.grad(o, (yq, Wq, bq), torch.randn_like(o))                        # attention backward kernels
pe = PatchEmbed(img_size=256, patch_size=16, in_chans=3, embed_dim=D).cuda()
img = torch.rand(B, 3, 256, 256, device=dev)
with torch.autocast("cuda", dtype=torch.bfloat16):
    vit_ops.patch_embed(pe, img)                                                 # patchify_kernel
torch.cuda.synchronize()
print("ok")
