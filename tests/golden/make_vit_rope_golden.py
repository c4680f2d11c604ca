"""Goldens of the RoPE decoder (DINOv2Decoder(use_rope=True), RoPEAttention) from the REFERENCE'S OWN modules (CPU).

    XQ_REFERENCE=<checkout> python tests/golden/make_vit_rope_golden.py     # writes tests/golden/vit_rope_*.npz

Same recipe as make_vit_golden.py (whose timm stand-ins it reuses): the reference's dino_enc/dinov2.py (DINOv2Decoder
:201-365) and its vendored vision_transformer.py (RoPEAttention :200-270, helpers :58-142, the attn_layer partial :728-731),
at ViT-S width with the depth cut to a few blocks.  Weights are seeded by name (vit_det_init.py); `det_init_rope` also seeds
the real and imaginary parts of the complex `freqs_1d`, which apply_det_init skips (it seeds floating-point tensors only).

Each file stores:
  - the fp32 forward output (subsampled + full sums) and the state_dict key list;
  - `freqs` / `freqs_1d` of every block as the constructor draws them after torch.manual_seed(0) (before the seeded weights);
  - every parameter gradient (sums; full tensors for the RoPE parameters and the first qkv bias) of a run under CPU bf16
    autocast.  The reference's `torch.cuda.amp.autocast(enabled=False)` blocks are mapped to the CPU autocast while it runs,
    so that its image-token angles and rotations are fp32 there as they are under CUDA autocast;
  - the error the reference's fp32 backward raises (the in-place rotation overwrites a tensor autograd saved).
"""
import contextlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from vit_det_init import apply_det_init, det_tensor  # noqa: E402

# name -> (model name, depth, num_latent_tokens, batch)
CASES = {
    "vit_rope_l256": ("vit_small_patch14_dinov2.lvd142m", 2, 256, 2),       # N = 1 + 256 + 256 = 513
    "vit_rope_l60": ("vit_small_patch14_dinov2.lvd142m", 3, 60, 2),         # odd latent count, N = 317
    "vit_rope_reg4": ("vit_small_patch14_reg4_dinov2.lvd142m", 2, 60, 2),   # P = 5, N = 321
}
MODEL_KWARGS = dict(img_size=256, patch_size=16, drop_path_rate=0.0)
FULL_GRADS = ("freqs", "freqs_1d", "attn.qkv.bias", "mask_token")


def decoder_kwargs(name):
    model_name, depth, L, _ = CASES[name]
    return dict(in_channels=3, model_name=model_name, model_kwargs=dict(MODEL_KWARGS, depth=depth), pretrained=False,
                tuning_method="full", num_latent_tokens=L, to_pixel="linear", use_rope=True, abs_pos_embed=False)


def det_init_rope(module):
    """apply_det_init, plus name-seeded real and imaginary parts for complex parameters"""
    apply_det_init(module)
    with torch.no_grad():
        for n, p in module.named_parameters():
            if p.is_complex():
                p.copy_(torch.complex(det_tensor(n + ".real", p.shape), det_tensor(n + ".imag", p.shape)))


def golden_io(name, D):
    """the latent input z [B, L, D] and the output weights of the loss sum(out * w)"""
    _, _, L, B = CASES[name]
    g = torch.Generator().manual_seed(4321)
    z = torch.randn(B, L, D, generator=g)
    w = torch.randn(B, 3, 256, 256, generator=g)
    return z, w


@contextlib.contextmanager
def cuda_autocast_exits_on_cpu():
    """torch.cuda.amp.autocast(enabled=False) turns the CPU autocast off too (for the bf16 run only)"""
    orig = torch.cuda.amp.autocast
    torch.cuda.amp.autocast = lambda enabled=True, **kw: torch.autocast("cpu", enabled=enabled, dtype=torch.bfloat16)
    try:
        yield
    finally:
        torch.cuda.amp.autocast = orig


def main():
    import make_vit_golden as mvg
    sys.path.insert(0, mvg.REF)
    mvg.install_stand_ins()
    from tokenizer.tokenizer_image.dino_enc.dinov2 import DINOv2Decoder
    for name in CASES:
        kw = decoder_kwargs(name)
        torch.manual_seed(0)
        dec = DINOv2Decoder(**kw)
        init = {}
        for n, p in dec.named_parameters():
            if n.endswith("attn.freqs") or n.endswith("attn.freqs_1d"):
                init["init_" + n] = (torch.view_as_real(p) if p.is_complex() else p).detach().numpy().copy()
        det_init_rope(dec)
        dec.eval()
        z, w = golden_io(name, dec.embed_dim)
        with torch.no_grad():
            out = dec(z)
        # fp32 backward: the reference's in-place rotation breaks it
        fp32_err = ""
        try:
            (dec(z) * w).sum().backward()
        except RuntimeError as e:
            fp32_err = str(e).split("\n")[0]
        dec.zero_grad(set_to_none=True)
        with cuda_autocast_exits_on_cpu(), torch.autocast("cpu", dtype=torch.bfloat16):
            out_bf = dec(z)
        (out_bf.float() * w).sum().backward()
        grads = {}
        for n, p in dec.named_parameters():
            if p.grad is None:                   # pos_embed: the RoPE decoder adds no absolute positions
                continue
            g = torch.view_as_real(p.grad) if p.grad.is_complex() else p.grad
            grads["gsum_" + n] = np.float64(g.double().sum())
            grads["gabs_" + n] = np.float64(g.double().abs().sum())
            if n.endswith(FULL_GRADS) and (".0." in n or "blocks" not in n or n.endswith(("freqs", "freqs_1d"))):
                grads["grad_" + n] = g.float().numpy()
        np.savez_compressed(os.path.join(HERE, name + ".npz"), kwargs_json=np.array(repr(kw)),
                            keys=np.array(list(dec.state_dict().keys())),
                            param_names=np.array([n for n, _ in dec.named_parameters()]),
                            out_sub=out[:, :, ::4, ::4].numpy(), out_sum=np.float64(out.double().sum()),
                            out_abs=np.float64(out.double().abs().sum()),
                            out_bf16_sub=out_bf.float()[:, :, ::4, ::4].detach().numpy(),
                            fp32_backward_error=np.array(fp32_err), **init, **grads)
        print(name, "out", tuple(out.shape), "|mean|", float(out.abs().mean()), "fp32 backward:", fp32_err[:80])


if __name__ == "__main__":
    main()
