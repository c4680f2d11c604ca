"""small-shape run of the newer libxqb200 kernels for `compute-sanitizer --tool memcheck|racecheck|synccheck`."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from imagefolder_b200 import vit_ops, VectorQuantizer2
from imagefolder_b200.dino_enc.vision_transformer import PatchEmbed

dev = "cuda"
torch.manual_seed(0)
for (B, S, D, H) in [(2, 37, 768, 12), (3, 9, 384, 6), (1, 21, 1024, 16)]:
    x = torch.randn(B, S, D, device=dev, requires_grad=True)
    br = torch.randn(B, S, D, device=dev).to(torch.bfloat16).requires_grad_(True)
    g = torch.rand(D, device=dev, requires_grad=True)
    bb = torch.randn(D, device=dev, requires_grad=True)
    w = torch.rand(D, device=dev, requires_grad=True)
    b = torch.randn(D, device=dev, requires_grad=True)
    rs = torch.ones(B, device=dev)
    xo, y = vit_ops.residual_ln(x, br, bb, g, rs, w, b, 1e-6)
    torch.autograd.grad((xo, y), (x, br, g, bb, w, b), (torch.randn_like(xo), torch.randn_like(y)))
    _, y2 = vit_ops.residual_ln(x, None, None, None, None, w, b, 1e-6)
    torch.autograd.grad(y2, (x, w, b), torch.randn_like(y2))
    h = torch.randn(B, S, 4 * D, device=dev).to(torch.bfloat16).requires_grad_(True)
    b1 = torch.randn(4 * D, device=dev, requires_grad=True)
    yy = vit_ops.gelu_bias(h, b1)
    torch.autograd.grad(yy, (h, b1), torch.randn_like(yy))
    yq = torch.randn(B, S, D, device=dev).to(torch.bfloat16).requires_grad_(True)
    Wq = (torch.randn(3 * D, D, device=dev) * D ** -0.5).requires_grad_(True)
    bq = torch.randn(3 * D, device=dev, requires_grad=True)
    o = vit_ops._QKVAttention.apply(yq, Wq, bq, H)
    torch.autograd.grad(o, (yq, Wq, bq), torch.randn_like(o))
pe = PatchEmbed(img_size=64, patch_size=16, in_chans=3, embed_dim=96).cuda()
with torch.autocast("cuda", dtype=torch.bfloat16):
    vit_ops.patch_embed(pe, torch.rand(2, 3, 64, 64, device=dev))
pn = [1, 2, 3, 5, 8]
q = VectorQuantizer2(96, 12, v_patch_nums=pn, num_latent_tokens=64).cuda().eval()
hs = [torch.randn(3, 12, p, p, device=dev) for p in pn]
q.embed_to_fhat(hs, last_one=False)
f = torch.zeros(3, 12, 8, 8, device=dev)
for si in range(len(pn)):
    q.get_next_autoregressive_input(si, len(pn), f, hs[si])
torch.cuda.synchronize()
print("ok")
