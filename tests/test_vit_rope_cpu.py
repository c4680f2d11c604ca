"""DINOv2Decoder(use_rope=True) on the module path (CPU): the reference's fp32 outputs (tests/golden/vit_rope_*.npz, from the
reference's own modules), its state_dict keys and RNG-drawn frequencies, fp32 gradients against the fp64 restatement
(tests/rope_oracle.py), bf16-autocast gradients against the reference's, and the refused configurations."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)
import make_vit_rope_golden as mrg  # noqa: E402
import rope_oracle  # noqa: E402

CASES = list(mrg.CASES)


def _golden(name):
    return np.load(os.path.join(HERE, "golden", name + ".npz"))


def _decoder(name, seeded=True):
    from imagefolder_b200.dino_enc.dinov2 import DINOv2Decoder
    torch.manual_seed(0)
    dec = DINOv2Decoder(**mrg.decoder_kwargs(name))
    if seeded:
        mrg.det_init_rope(dec)
    return dec.eval()


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("name", CASES)
def test_fp32_forward_matches_reference_golden(name):
    g = _golden(name)
    dec = _decoder(name)
    z, _ = mrg.golden_io(name, dec.embed_dim)
    with torch.no_grad():
        out = dec(z)
        ref = rope_oracle.rope_decoder_forward(rope_oracle.fp64_state(dec, False), z.double(), dec.model.blocks[0].attn.num_heads)
    want = torch.from_numpy(g["out_sub"])
    torch.testing.assert_close(out[:, :, ::4, ::4], want, rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(ref[:, :, ::4, ::4].float(), want, rtol=1e-3, atol=1e-3)
    assert abs(float(out.double().sum()) - float(g["out_sum"])) <= 1e-3 * float(g["out_abs"])
    assert abs(float(ref.sum()) - float(g["out_sum"])) <= 1e-3 * float(g["out_abs"])


@pytest.mark.parametrize("name", CASES)
def test_state_dict_keys_and_initial_freqs_are_the_references(name):
    g = _golden(name)
    dec = _decoder(name, seeded=False)
    # the stand-in timm registry builds the reference's classifier head (num_classes 1000); the decoder never uses it, and
    # this package builds its backbones with num_classes = 0, as for every other decoder
    no_head = lambda keys: [str(k) for k in keys if not str(k).startswith("model.head.")]   # noqa: E731
    assert list(dec.state_dict().keys()) == no_head(g["keys"])
    assert [n for n, _ in dec.named_parameters()] == no_head(g["param_names"])
    inits = [k for k in g.files if k.startswith("init_")]
    assert len(inits) == 2 * len(dec.model.blocks)
    params = dict(dec.named_parameters())
    for k in inits:
        p = params[k[len("init_"):]].detach()
        p = torch.view_as_real(p) if p.is_complex() else p
        assert torch.equal(p.view(torch.int32), torch.from_numpy(g[k]).view(torch.int32)), k
    attn = dec.model.blocks[0].attn
    assert attn.freqs.dtype == torch.float32 and tuple(attn.freqs.shape) == (2, attn.num_heads * 32)
    assert attn.freqs_1d.dtype == torch.complex64 and tuple(attn.freqs_1d.shape) == (dec.num_latent_tokens, 32)
    assert not hasattr(dec, "latent_pos_embed") and not hasattr(dec, "lvl_embed")


@pytest.mark.parametrize("name", CASES)
def test_fp32_gradients_match_fp64_oracle(name):
    """every parameter gradient of the module path in fp32 (freqs and freqs_1d included) within 1e-4 of fp64.  The reference's
    fp32 backward raises here (its in-place rotation); the golden records that error."""
    g = _golden(name)
    assert "modified by an inplace operation" in str(g["fp32_backward_error"])
    dec = _decoder(name)
    z, w = mrg.golden_io(name, dec.embed_dim)
    (dec(z) * w).sum().backward()
    sd = rope_oracle.fp64_state(dec)
    (rope_oracle.rope_decoder_forward(sd, z.double(), dec.model.blocks[0].attn.num_heads) * w.double()).sum().backward()
    checked = 0
    for n, p in dec.named_parameters():
        ref = sd[n].grad
        if ref is None:
            assert p.grad is None, n                    # pos_embed: unused by the RoPE decoder
            continue
        got = torch.view_as_real(p.grad) if p.grad.is_complex() else p.grad
        want = torch.view_as_real(ref) if ref.is_complex() else ref
        assert _rel(got, want) <= 1e-4, (n, _rel(got, want))
        checked += 1
    assert checked >= 10 * len(dec.model.blocks)


@pytest.mark.parametrize("name", CASES)
def test_bf16_autocast_gradients_match_reference(name):
    g = _golden(name)
    dec = _decoder(name)
    z, w = mrg.golden_io(name, dec.embed_dim)
    with torch.autocast("cpu", dtype=torch.bfloat16):
        out = dec(z)
    torch.testing.assert_close(out.float()[:, :, ::4, ::4], torch.from_numpy(g["out_bf16_sub"]), rtol=0.05, atol=0.05)
    (out.float() * w).sum().backward()
    for n, p in dec.named_parameters():
        if "gsum_" + n not in g.files:
            assert p.grad is None, n                    # pos_embed
            continue
        got = torch.view_as_real(p.grad) if p.grad.is_complex() else p.grad
        assert abs(float(got.double().abs().sum()) - float(g["gabs_" + n])) <= 0.05 * float(g["gabs_" + n]), n
        if "grad_" + n in g.files:
            assert _rel(got, torch.from_numpy(g["grad_" + n])) <= 0.05, (n, _rel(got, torch.from_numpy(g["grad_" + n])))


def test_refused_configurations():
    from imagefolder_b200.dino_enc.dinov2 import DINOv2Decoder
    from imagefolder_b200.dino_enc.vision_transformer import RoPEAttention
    kw = mrg.decoder_kwargs("vit_rope_l60")
    with pytest.raises(ValueError, match="abs_pos_embed"):
        DINOv2Decoder(**dict(kw, abs_pos_embed=True))
    with pytest.raises(NotImplementedError, match="cond_latent"):
        DINOv2Decoder(**dict(kw, cond_latent=True))
    with pytest.raises(NotImplementedError, match="rope_mixed=False"):
        RoPEAttention(384, num_heads=6, qkv_bias=True, rope_mixed=False)


def test_lora_on_the_rope_decoder():
    from imagefolder_b200.dino_enc.dinov2 import DINOv2Decoder
    torch.manual_seed(0)
    dec = DINOv2Decoder(**dict(mrg.decoder_kwargs("vit_rope_l60"), tuning_method="lora"))
    trainable = {n for n, p in dec.named_parameters() if p.requires_grad}
    assert any("lora_A" in n for n in trainable) and not any(n.endswith("attn.freqs") for n in trainable)
    z, w = mrg.golden_io("vit_rope_l60", dec.embed_dim)
    (dec(z) * w).sum().backward()
    assert all(dec.get_parameter(n).grad is not None for n in trainable if "lora_" in n)
