"""CPU-side checks of the fp16 twins of the ViT entry points (`*_f16`, include/xqb200.h): each is exported, and refuses
NULL, misaligned and unsupported arguments with the same code as its bf16 sibling.  Every refusal below happens before any
CUDA call, so it runs without a device; each call is made on the bf16 sibling too and the codes compared."""
import pytest

XQ_ERR_ARG, XQ_ERR_WORKSPACE, XQ_ERR_UNSUPPORTED = -1, -2, -4
P = 4096                  # a non-null dummy device pointer, 256-byte aligned
MIS = 4096 + 8            # the same, misaligned for a 16-byte access


def _lib():
    from imagefolder_b200 import _capi
    return _capi.lib()


def test_every_twin_is_exported_with_the_siblings_signature():
    from imagefolder_b200 import _capi
    L = _lib()
    assert len(_capi.F16_TWINS) == 16
    for name in _capi.F16_TWINS:
        twin = getattr(L, name + "_f16")
        assert twin.argtypes == getattr(L, name).argtypes
        assert name + "_f16" in _capi.EXPORTED_SYMBOLS


# (entry point, arguments, expected code)
REFUSALS = [
    # fused MLP GEMMs
    ("xq_vit_fc1_gelu_fwd", (None, P, P, P, P, 128, 256, 64, None), XQ_ERR_ARG),
    ("xq_vit_fc1_gelu_fwd", (P, P, P, P, P, 0, 256, 64, None), XQ_ERR_ARG),
    ("xq_vit_fc1_gelu_fwd", (MIS, P, P, P, P, 128, 256, 64, None), XQ_ERR_ARG),
    ("xq_vit_fc1_gelu_fwd", (P, P, P, P, P, 128, 200, 64, None), XQ_ERR_UNSUPPORTED),
    ("xq_vit_fc1_gelu_fwd", (P, P, P, P, P, 128, 256, 96, None), XQ_ERR_UNSUPPORTED),
    ("xq_vit_fc2_dgelu_bwd", (P, P, P, P, P, None, 128, 256, 64, None), XQ_ERR_ARG),
    ("xq_vit_fc2_dgelu_bwd", (P, P, MIS, P, P, P, 128, 256, 64, None), XQ_ERR_ARG),
    ("xq_vit_fc2_dgelu_bwd", (P, P, P, P, P, P, 128, 192, 64, None), XQ_ERR_UNSUPPORTED),
    ("xq_vit_fc1_lora_gelu_fwd", (P, P, None, P, P, P, P, 128, 256, 64, 8, None), XQ_ERR_ARG),
    ("xq_vit_fc1_lora_gelu_fwd", (P, P, P, P, P, P, P, 128, 256, 64, 12, None), XQ_ERR_ARG),
    ("xq_vit_fc1_lora_gelu_fwd", (P, P, P, P, P, P, P, 128, 256, 64, 72, None), XQ_ERR_ARG),
    ("xq_vit_fc1_lora_gelu_fwd", (P, P, MIS, P, P, P, P, 128, 256, 64, 8, None), XQ_ERR_ARG),
    ("xq_vit_fc2_lora_dgelu_bwd", (P, P, P, P, P, P, P, None, 128, 256, 64, 8, None), XQ_ERR_ARG),
    ("xq_vit_fc2_lora_dgelu_bwd", (P, P, P, None, P, P, P, P, 128, 256, 64, 8, None), XQ_ERR_ARG),
    ("xq_vit_fc2_lora_dgelu_bwd", (P, P, P, P, P, P, P, P, 128, 256, 64, 4, None), XQ_ERR_ARG),
    # attention
    ("xq_vit_attn_fwd", (None, P, P, 1, 16, 1, 64, 0.125, None), XQ_ERR_ARG),
    ("xq_vit_attn_fwd", (P, P, P, 1, 16, 1, 32, 0.125, None), XQ_ERR_UNSUPPORTED),
    ("xq_vit_attn_fwd", (MIS, P, P, 1, 16, 1, 64, 0.125, None), XQ_ERR_ARG),
    ("xq_vit_attn_bwd", (P, P, P, P, P, None, 1, 16, 1, 64, 0.125, None, 1 << 20, None), XQ_ERR_ARG),
    ("xq_vit_attn_bwd", (P, P, P, P, P, None, 1, 16, 1, 48, 0.125, P, 1 << 20, None), XQ_ERR_UNSUPPORTED),
    ("xq_vit_attn_bwd", (P, P, P, P, P, None, 1, 16, 1, 64, 0.125, P + 16, 1 << 20, None), XQ_ERR_ARG),
    ("xq_vit_attn_bwd", (P, P, P, P, P, None, 1, 16, 1, 64, 0.125, P, 16, None), XQ_ERR_WORKSPACE),
    # glue
    ("xq_vit_residual_ln_fwd", (None, None, None, None, None, 1, P, P, 1e-6, 8, 768, P, P, P, P, None), XQ_ERR_ARG),
    ("xq_vit_residual_ln_fwd", (P, None, None, None, None, 1, None, P, 1e-6, 8, 768, P, P, P, P, None), XQ_ERR_ARG),
    ("xq_vit_residual_ln_fwd", (P, P, None, None, P, 0, P, P, 1e-6, 8, 768, P, P, P, P, None), XQ_ERR_ARG),
    ("xq_vit_residual_ln_bwd", (None, None, None, None, None, None, None, None, None, None, 1, 8, 768, None, None, None,
                                None, None, None, None, 0, None), XQ_ERR_ARG),
    ("xq_vit_residual_ln_bwd", (None, P, P, P, P, None, None, None, None, None, 1, 8, 768, P, None, None, None, None, None, P,
                                1 << 20, None), XQ_ERR_ARG),
    ("xq_vit_patchify", (None, P, 2, 3, 64, 64, 16, None), XQ_ERR_ARG),
    ("xq_vit_patchify", (P, P, 2, 3, 64, 64, 6, None), XQ_ERR_UNSUPPORTED),
    ("xq_vit_patchify", (P, P, 2, 3, 60, 64, 16, None), XQ_ERR_UNSUPPORTED),
    ("xq_vit_gelu_fwd", (None, None, P, 4, 64, None), XQ_ERR_ARG),
    ("xq_vit_gelu_fwd", (P, None, P, 4, 60, None), XQ_ERR_ARG),
    ("xq_vit_gelu_bwd", (P, None, None, P, None, 4, 64, None), XQ_ERR_ARG),
    ("xq_vit_gelu_bwd", (P, None, P, P, None, 0, 64, None), XQ_ERR_ARG),
]


@pytest.mark.parametrize("name,args,code", REFUSALS, ids=[f"{r[0]}-{i}" for i, r in enumerate(REFUSALS)])
def test_f16_twin_refuses_like_its_bf16_sibling(name, args, code):
    L = _lib()
    assert getattr(L, name)(*args) == code
    assert getattr(L, name + "_f16")(*args) == code


def test_assemble_takes_f16_as_src_type_2():
    """xq_vit_assemble_fwd / bwd: src_type 2 is fp16; its argument checks are those of the other source types"""
    L = _lib()
    assert L.xq_vit_assemble_fwd(P, 2, P, 2, 4, 6, 16, 3, P, None) == XQ_ERR_ARG       # t0 + Ls > T
    assert L.xq_vit_assemble_fwd(P, 2, P, 2, 4, 8, 18, 1, P, None) == XQ_ERR_ARG       # D % 4 != 0
    assert L.xq_vit_assemble_bwd(P, 2, 4, 8, 16, 1, None, 2, None, None) == XQ_ERR_ARG  # nothing to compute
