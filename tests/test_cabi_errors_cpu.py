"""Every CUDA failure of the ViT glue (csrc/vit_kernels.cu), loss (csrc/loss_kernels.cu) and image-transform
(csrc/img_kernels.cu) entry points is recorded: the call returns XQ_ERR_CUDA and xq_last_cuda_error() names the CUDA call
or kernel that failed, not whatever an earlier call left there.

Runs only where no GPU is usable: every call gets valid sizes and non-null dummy pointers, so it passes its argument checks
and fails at its first CUDA call.  Before each call another entry point records an unrelated failure (xq_vq_backward's
gradient memset), so a call that does not record its own failure leaves that message behind and fails the check.  The
workspace-size queries xq_lpips_workspace_bytes and xq_img_workspace_bytes make no CUDA call and are not listed."""
import pytest
import torch

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="dummy device pointers must never reach a real GPU")

XQ_ERR_CUDA = -3
P = 4096                  # a non-null dummy device pointer, 256-byte aligned
BIG = 1 << 30             # a workspace size no check refuses

# (entry point, arguments, expected start of xq_last_cuda_error())
CALLS = [
    # vit_kernels.cu
    ("xq_vit_residual_ln_fwd", (P, None, None, None, None, 1, None, None, 1e-6, 8, 768, P, None, None, None, None),
     "residual_ln_fwd_kernel"),
    ("xq_vit_residual_ln_bwd", (None, None, P, P, P, None, None, None, None, None, 1, 8, 768, P, None, None, None, None,
                                None, P, BIG, None), "cudaGetDevice"),
    ("xq_vit_assemble_fwd", (P, 1, P, 2, 4, 8, 16, 1, P, None), "assemble_fwd_kernel"),
    ("xq_vit_assemble_bwd", (P, 2, 4, 8, 16, 1, P, 0, P, None), "assemble_bwd_kernel"),
    ("xq_vit_patchify", (P, P, 2, 3, 64, 64, 16, None), "patchify_kernel"),
    ("xq_vit_gelu_fwd", (P, None, P, 4, 64, None), "gelu_fwd_kernel"),
    ("xq_vit_gelu_bwd", (P, None, P, P, None, 4, 64, None), "cudaGetDevice"),
    # loss_kernels.cu
    ("xq_lpips_layer_forward", (P, P, 0, P, 1, 8, 16, 1e-10, 0, P, P, BIG, None), "lpips_layer_fwd_kernel"),
    ("xq_lpips_layer_backward", (P, P, 0, P, 1, 8, 16, 1e-10, P, P, None), "lpips_layer_bwd_kernel"),
    ("xq_diffaug_forward", (P, P, 2, 3, 8, 8, 1, 2, 2, P, P, None), "diffaug_fwd_kernel"),
    ("xq_diffaug_forward", (P, P, 2, 3, 8, 8, 2, 2, 2, P, P, None), "diffaug_sum_kernel"),
    ("xq_diffaug_backward", (P, P, 2, 3, 8, 8, 1, 2, 2, P, P, None), "diffaug_bwd_kernel"),
    ("xq_diffaug_backward", (P, P, 2, 3, 8, 8, 2, 2, 2, P, P, None), "diffaug_sum_kernel"),
    # img_kernels.cu
    ("xq_img_box_halve", (P, BIG, P, P, 1, 16, 1, 8, 8, P, BIG, None), "img_box_halve_kernel"),
    ("xq_img_resize_crop_normalize", (P, BIG, P, P, 1, 16, P, BIG, P, None), "cudaGetDevice"),
]


def _stale_message(L):
    rc = L.xq_vq_backward(P, P, P, P, P, P, 1, 8, 4, 16, 1, 0.25, P, P, None)
    assert rc == XQ_ERR_CUDA
    msg = L.xq_last_cuda_error().decode()
    assert msg.startswith("cudaMemsetAsync(gE"), msg
    return msg


@pytest.mark.parametrize("name,args,expect", CALLS, ids=[f"{c[0]}-{c[2]}" for c in CALLS])
def test_cuda_failure_is_recorded(name, args, expect):
    from imagefolder_b200 import _capi
    L = _capi.lib()
    stale = _stale_message(L)
    assert getattr(L, name)(*args) == XQ_ERR_CUDA
    msg = L.xq_last_cuda_error().decode()
    assert msg != stale and msg.startswith(expect), f"{name}: {msg!r}"


def test_ln_bwd_workspace_query_reports_zero_and_the_cause():
    from imagefolder_b200 import _capi
    L = _capi.lib()
    _stale_message(L)
    assert L.xq_vit_ln_bwd_workspace_bytes(768) == 0
    assert L.xq_last_cuda_error().decode().startswith("cudaGetDevice")
