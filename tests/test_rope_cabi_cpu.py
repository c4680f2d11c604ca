"""Argument checks of the RoPE entry points (csrc/rope_kernel.cu, include/xqb200.h): every refusal returns before any CUDA
call, so these run without a GPU.  On a machine without one, a call that passes its checks fails at its first launch and
records the kernel's name."""
import pytest
import torch

XQ_ERR_ARG, XQ_ERR_WORKSPACE, XQ_ERR_CUDA, XQ_ERR_UNSUPPORTED = -1, -2, -3, -4
P = 4096                  # a non-null dummy device pointer, 256-byte aligned
BIG = 1 << 34             # a workspace size no check refuses

# (B, N, H, head_dim, P, I, L) of a valid ViT-S decoder sequence: cls + 256 image + 256 latent tokens
OK = (2, 513, 6, 64, 1, 256, 256)


def _fwd(L, name, shape, qkv=P, out=P, freqs=P, freqs_1d=P):
    return getattr(L, name)(qkv, out, freqs, freqs_1d, *shape, None)


def _bwd(L, name, shape, qkv=P, d_out=P, freqs=P, freqs_1d=P, d_qkv=P, ws=P, ws_bytes=BIG):
    return getattr(L, name)(qkv, d_out, freqs, freqs_1d, *shape, d_qkv, P, P, P, ws, ws_bytes, None)


REFUSED = [
    ("head_dim 32", (2, 513, 6, 32, 1, 256, 256), XQ_ERR_UNSUPPORTED),
    ("head_dim 128", (2, 513, 6, 128, 1, 256, 256), XQ_ERR_UNSUPPORTED),
    ("I = 196", (2, 453, 6, 64, 1, 196, 256), XQ_ERR_UNSUPPORTED),
    ("P + I + L > N", (2, 512, 6, 64, 1, 256, 256), XQ_ERR_ARG),
    ("P + I + L < N", (2, 514, 6, 64, 1, 256, 256), XQ_ERR_ARG),
    ("L = 0", (2, 257, 6, 64, 1, 256, 0), XQ_ERR_ARG),
    ("P < 0", (2, 511, 6, 64, -1, 256, 256), XQ_ERR_ARG),
    ("B = 0", (0, 513, 6, 64, 1, 256, 256), XQ_ERR_ARG),
    ("H = 0", (2, 513, 0, 64, 1, 256, 256), XQ_ERR_ARG),
    ("H = 65", (2, 513, 65, 64, 1, 256, 256), XQ_ERR_ARG),
]


@pytest.mark.parametrize("dt", ["", "_f16"])
@pytest.mark.parametrize("what,shape,rc", REFUSED, ids=[r[0] for r in REFUSED])
def test_shape_refusals(what, shape, rc, dt):
    from imagefolder_b200 import _capi
    L = _capi.lib()
    assert _fwd(L, "xq_vit_rope_fwd" + dt, shape) == rc
    assert _bwd(L, "xq_vit_rope_bwd" + dt, shape) == rc


@pytest.mark.parametrize("dt", ["", "_f16"])
@pytest.mark.parametrize("arg", ["qkv", "out", "freqs", "freqs_1d"])
@pytest.mark.parametrize("bad", [None, P + 8], ids=["null", "misaligned"])
def test_forward_pointer_refusals(arg, bad, dt):
    from imagefolder_b200 import _capi
    assert _fwd(_capi.lib(), "xq_vit_rope_fwd" + dt, OK, **{arg: bad}) == XQ_ERR_ARG


@pytest.mark.parametrize("dt", ["", "_f16"])
@pytest.mark.parametrize("arg", ["qkv", "d_out", "freqs", "freqs_1d", "d_qkv", "ws"])
@pytest.mark.parametrize("bad", [None, P + 4], ids=["null", "misaligned"])
def test_backward_pointer_refusals(arg, bad, dt):
    from imagefolder_b200 import _capi
    assert _bwd(_capi.lib(), "xq_vit_rope_bwd" + dt, OK, **{arg: bad}) == XQ_ERR_ARG


@pytest.mark.parametrize("dt", ["", "_f16"])
def test_backward_workspace_size(dt):
    from imagefolder_b200 import _capi
    L = _capi.lib()
    need = L.xq_vit_rope_bwd_workspace_bytes(*OK[:3], OK[-1])
    # per 32-row batch chunk: bias partials [N, 3*H*64], theta partials [256, H*32], latent partials [L, 64], fp32
    B, N, H, _, _, _, Lt = OK
    assert need >= 4 * (N * 3 * H * 64 + 256 * H * 32 + Lt * 64) and need % 256 == 0
    assert L.xq_vit_rope_bwd_workspace_bytes(33, N, H, Lt) >= 2 * 4 * N * 3 * H * 64
    assert _bwd(L, "xq_vit_rope_bwd" + dt, OK, ws_bytes=need - 1) == XQ_ERR_WORKSPACE
    for bad in [(0, N, H, Lt), (B, 0, H, Lt), (B, N, 0, Lt), (B, N, 65, Lt), (B, N, H, 0)]:
        assert L.xq_vit_rope_bwd_workspace_bytes(*bad) == 0


@pytest.mark.skipif(torch.cuda.is_available(), reason="dummy device pointers must never reach a real GPU")
@pytest.mark.parametrize("dt", ["", "_f16"])
def test_valid_call_reaches_its_launch(dt):
    from imagefolder_b200 import _capi
    L = _capi.lib()
    assert _fwd(L, "xq_vit_rope_fwd" + dt, OK) == XQ_ERR_CUDA
    assert L.xq_last_cuda_error().decode().startswith("rope_fwd_kernel")
    assert _bwd(L, "xq_vit_rope_bwd" + dt, OK) == XQ_ERR_CUDA
    assert L.xq_last_cuda_error().decode().startswith("rope_bwd_partials_kernel")
