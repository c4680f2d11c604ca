"""wgmma flash attention (csrc/attn_kernel.cu, xq_vit_attn_fwd / xq_vit_attn_bwd through the C-ABI) against a plain
PyTorch fp32 explicit-softmax reference of the same op: Attention.forward,
tokenizer/tokenizer_image/dino_enc/vision_transformer.py:173-197 (softmax(q k^T / sqrt(d)) v on the packed projection).

Tolerances (bf16 operands and bf16 P / dS inside the kernel, fp32 statistics and accumulation): forward 8e-3, gradients
1e-2, both relative to the largest reference magnitude of the tensor.  Sequence lengths are the ones the shipped
configs produce (513 / 514 VQ, 769 VP2, 499 / 379 multi-scale) plus edge cases (1, 16, 128, 129, 1024) and every
trailing-key count of the backward pre-pass (N mod 128 = 1 .. 4, and 5, which goes back to the tensor cores)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(qkv32, H):
    B, N, _ = qkv32.shape
    x = qkv32.view(B, N, 3, H, 64).permute(2, 0, 3, 1, 4)
    q, k, v = x[0], x[1], x[2]
    s = (q @ k.transpose(-1, -2)) * 0.125
    o = torch.softmax(s, -1) @ v
    return o.transpose(1, 2).reshape(B, N, H * 64), torch.logsumexp(s, -1) * math.log2(math.e)


@pytest.mark.parametrize("B,N,H", [(2, 513, 3), (2, 514, 2), (1, 769, 2), (2, 499, 2), (2, 379, 3), (3, 1, 1), (1, 16, 2),
                                   (2, 128, 2), (2, 129, 1), (1, 1024, 1), (1, 333, 12),
                                   # more backward CTAs (one per key block and batch*head) than SMs: several waves, and the
                                   # fp32 dQ atomics of one (batch, head) come from CTAs of different waves
                                   (5, 513, 12), (7, 300, 12), (40, 130, 12), (13, 100, 12),
                                   # N mod 128 = 3 / 4: the trailing keys on CUDA cores in the backward pre-pass
                                   # (attn_bwd_prep_kernel<3> / <4>); N mod 128 = 5: the first length that goes back to a
                                   # tensor-core key block for them
                                   (2, 131, 2), (1, 132, 12), (2, 133, 3), (1, 387, 12), (2, 388, 2)])
@pytest.mark.parametrize("amp", [1.0, 2.5])
def test_attention_forward_backward_match_fp32_reference(B, N, H, amp):
    from imagefolder_b200 import vit_ops
    torch.manual_seed(N * 7 + H)
    dev = torch.device("cuda")
    qkv = (torch.randn(B, N, 3 * H * 64, device=dev) * amp).to(torch.bfloat16)
    g = torch.randn(B, N, H * 64, device=dev).to(torch.bfloat16)
    q32 = qkv.float().requires_grad_(True)
    o_ref, lse_ref = _ref(q32, H)
    (o_ref * g.float()).sum().backward()
    out, lse2 = vit_ops.attn_tc_forward(qkv, H)
    dqkv = vit_ops.attn_tc_backward(qkv, out, lse2, g, H)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all() and torch.isfinite(dqkv.float()).all()
    scale_o = max(1.0, o_ref.abs().max().item())
    assert (out.float() - o_ref).abs().max().item() <= 8e-3 * scale_o
    assert (lse2 - lse_ref.detach()).abs().max().item() <= 1e-3 * max(1.0, lse_ref.abs().max().item())
    gr = q32.grad.view(B, N, 3, H * 64)
    d = dqkv.float().view(B, N, 3, H * 64)
    for i, name in enumerate("qkv"):
        m = max(1e-3, gr[:, :, i].abs().max().item())
        err = (d[:, :, i] - gr[:, :, i]).abs().max().item()
        assert err <= 1e-2 * m, f"d{name}: err {err:.3e} vs max {m:.3e}"
    # the fused qkv-bias gradient = column sums of the ROUNDED packed gradient the same call wrote
    dq2, db = vit_ops.attn_tc_backward(qkv, out, lse2, g, H, want_bias_grad=True)
    torch.cuda.synchronize()
    want = dq2.float().sum((0, 1))
    assert (db - want).abs().max().item() <= 2e-3 * max(1.0, want.abs().max().item()) + 1e-4 * B * N ** 0.5


def test_attention_autograd_node_uses_the_tc_kernels_and_matches_sdpa():
    """The autograd node the ViT blocks call (_QKVAttention, on the wgmma kernels) vs the library composition it replaces:
    F.linear -> q / k / v views -> F.scaled_dot_product_attention -> head merge, under autograd."""
    import torch.nn.functional as F
    from imagefolder_b200 import _capi, vit_ops
    torch.manual_seed(0)
    dev = torch.device("cuda")
    B, N, C, H = 2, 513, 384, 6
    y = torch.randn(B, N, C, device=dev).to(torch.bfloat16).requires_grad_(True)
    W = (torch.randn(3 * C, C, device=dev) * 0.05).requires_grad_(True)
    b = (torch.randn(3 * C, device=dev) * 0.05).requires_grad_(True)
    g = torch.randn(B, N, C, device=dev).to(torch.bfloat16)

    def library(y, W, b):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            q, k, v = F.linear(y, W, b).view(B, N, 3, H, C // H).permute(2, 0, 3, 1, 4).unbind(0)
            return F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, N, C)

    res = []
    for node in (lambda y, W, b: vit_ops._QKVAttention.apply(y, W, b, H), library):
        n0 = _capi.LAUNCHES[0]
        o = node(y, W, b)
        grads = torch.autograd.grad(o, (y, W, b), g)
        res.append((o.float(), [t.float() for t in grads], _capi.LAUNCHES[0] - n0))
    assert res[0][2] >= 4 and res[1][2] == 0                 # fwd (1) + bwd (3) kernels of libxqb200 ran; none in the library path
    assert (res[0][0] - res[1][0]).abs().max().item() < 2e-2
    for a, bb in zip(res[0][1], res[1][1]):
        assert (a - bb).abs().max().item() <= 2e-2 * max(1.0, bb.abs().max().item())
