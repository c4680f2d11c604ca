"""CPU checks of the gradient-norm clipping (imagefolder_b200/optim.py::clip_grad_norm_, csrc/clip_kernel.cu): host planning,
every refusal before anything is written, and argument refusal of the C ABI before any CUDA call."""
import math
import os
import re
import warnings

import numpy as np
import pytest
import torch

from imagefolder_b200 import _capi
from imagefolder_b200.optim import _clip_tables, clip_grad_norm_

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_ARG, ERR_WORKSPACE = -1, -2
CHUNK = _capi.XQ_GRAD_NORM_CHUNK
T = _capi.XQ_CLIP_MAX_TENSORS


def test_constants_match_header_and_kernel():
    text = open(os.path.join(ROOT, "include", "xqb200.h")).read()
    assert int(re.search(r"#define XQ_CLIP_MAX_TENSORS (\d+)", text).group(1)) == T
    src = open(os.path.join(ROOT, "imagefolder_b200", "csrc", "clip_kernel.cu")).read()
    assert int(re.search(r"constexpr int NORM_CHUNK = (\d+);", src).group(1)) == CHUNK == 65536


def test_exported_symbols():
    L = _capi.lib()
    for s in ("xq_grad_norm_workspace_bytes", "xq_grad_norm", "xq_grad_scale"):
        assert s in _capi.EXPORTED_SYMBOLS and hasattr(L, s)


def test_tables_split_at_the_max_tensor_constant():
    assert _clip_tables([]) == []
    assert _clip_tables([5] * T) == [(0, T, 2, 1)]
    assert _clip_tables([5] * (T + 1)) == [(0, T, 2, 1), (T, T + 1, 2, 1)]
    # a table of empty entries still writes their norms (0) but streams nothing
    assert _clip_tables([0] * T + [7]) == [(0, T, 1, 0), (T, T + 1, 2, 1)]
    assert _clip_tables([3] * (2 * T + 2)) == [(0, T, 2, 1), (T, 2 * T, 2, 1), (2 * T, 2 * T + 2, 2, 1)]


def test_workspace_bytes():
    L = _capi.lib()

    def ws(numels):
        a = np.array(numels, dtype=np.int64)
        return L.xq_grad_norm_workspace_bytes(len(numels), a.ctypes.data if len(numels) else None)

    assert ws([]) == 0
    assert ws([0, 0]) == 0
    assert ws([1]) == 4
    assert ws([CHUNK - 1, CHUNK, CHUNK + 1]) == 4 * (1 + 1 + 2)
    assert ws([3 * CHUNK, 0, 10_000_000]) == 4 * (3 + math.ceil(10_000_000 / CHUNK))
    assert ws([7] * (2 * T + 3)) == 4 * (2 * T + 3)
    assert ws([5, -1]) == 0                                                  # out of range
    assert L.xq_grad_norm_workspace_bytes(-1, None) == 0
    assert L.xq_grad_norm_workspace_bytes(2, None) == 0


def _arrays(ptrs, numels):
    return np.array(ptrs, dtype=np.uint64), np.array(numels, dtype=np.int64)


def _norm(ptrs, numels, norms=8192, ws=16384, ws_bytes=1 << 20):
    L = _capi.lib()
    p, n = _arrays(ptrs, numels)
    return L.xq_grad_norm(p.ctypes.data, n.ctypes.data, len(numels), norms, ws, ws_bytes, None)


def _scale(ptrs, numels, coef=8192):
    L = _capi.lib()
    p, n = _arrays(ptrs, numels)
    return L.xq_grad_scale(p.ctypes.data, n.ctypes.data, len(numels), coef, None)


def test_c_abi_refuses_bad_arguments_without_gpu():
    """every refusal happens before the first CUDA call, so none of these touches a device"""
    L = _capi.lib()
    p, n = _arrays([4096], [16])
    for fn, tail in ((L.xq_grad_norm, (8192, 16384, 1 << 20, None)), (L.xq_grad_scale, (8192, None))):
        assert fn(None, None, 0, *tail) == 0                                 # n == 0: no-op
        assert fn(p.ctypes.data, n.ctypes.data, -1, *tail) == ERR_ARG
        assert fn(None, n.ctypes.data, 1, *tail) == ERR_ARG                  # NULL arrays with n > 0
        assert fn(p.ctypes.data, None, 1, *tail) == ERR_ARG
    for call in (_norm, _scale):
        assert call([4096], [-1]) == ERR_ARG                                 # negative numel
        assert call([0], [16]) == ERR_ARG                                    # NULL pointer, non-empty entry
        assert call([4098], [16]) == ERR_ARG                                 # not 4-byte aligned
    assert _norm([4096], [16], norms=0) == ERR_ARG                           # NULL / misaligned norms
    assert _norm([4096], [16], norms=8194) == ERR_ARG
    assert _norm([4096], [16], ws=0) == ERR_ARG                              # NULL / misaligned workspace
    assert _norm([4096], [16], ws=16386) == ERR_ARG
    assert _norm([4096, 8192], [CHUNK, 1], ws_bytes=7) == ERR_WORKSPACE      # two partials need 8 bytes
    assert _scale([4096], [16], coef=0) == ERR_ARG                           # NULL / misaligned coefficient
    assert _scale([4096], [16], coef=8195) == ERR_ARG
    assert _scale([0, 0], [0, 0]) == 0                                       # only empty entries: nothing to launch


def test_c_abi_validates_every_entry_before_the_first_launch():
    """a bad entry after more than two tables' worth of valid ones is still refused with XQ_ERR_ARG (a launch on these dummy
    pointers would have been attempted first otherwise, and fail with a CUDA error on this host)"""
    m = 2 * T + 7
    good = [4096 + 64 * i for i in range(m)]
    for bad_ptr, bad_n in ((4097, 16), (0, 16), (4096, -3)):
        assert _norm(good + [bad_ptr], [16] * m + [bad_n]) == ERR_ARG
        assert _scale(good + [bad_ptr], [16] * m + [bad_n]) == ERR_ARG
    assert _norm(good, [16] * m, ws_bytes=4 * m - 4) == ERR_WORKSPACE


def _params(dtype=torch.float32, grads=True):
    torch.manual_seed(0)
    ps = [torch.nn.Parameter(torch.randn(*s, dtype=dtype)) for s in ((3, 4), (5,), (2, 2, 2))]
    if grads:
        for p in ps:
            p.grad = torch.randn_like(p)
    return ps


def _dense(t):
    return t.to_dense() if t.is_sparse else t


def _snapshot(ps):
    return [None if p.grad is None else (_dense(p.grad).clone(), p.grad._version) for p in ps]


def _unchanged(ps, snap):
    for p, s in zip(ps, snap):
        if s is None:
            assert p.grad is None
        else:
            assert torch.equal(_dense(p.grad), s[0]) and p.grad._version == s[1]


def test_empty_returns_torch_zero():
    for params in ([], _params(grads=False), iter(_params(grads=False))):
        got = clip_grad_norm_(params, 1.0)
        want = torch.nn.utils.clip_grad_norm_([], 1.0)
        assert got.device == want.device and got.dtype == want.dtype and torch.equal(got, want)


def test_none_grads_are_skipped():
    """params without a grad take no part: a CPU param with no grad next to them changes nothing, and only the grads present
    are checked (here the one CPU grad is refused)"""
    ps = _params(grads=False)
    ps[1].grad = torch.randn(5)
    snap = _snapshot(ps)
    with pytest.raises(_capi.XqError):
        clip_grad_norm_(ps, 1.0)
    _unchanged(ps, snap)
    assert ps[0].grad is None and ps[2].grad is None


def test_empty_generator_warns_as_torch_does():
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        assert torch.equal(clip_grad_norm_((p for p in []), 1.0), torch.tensor(0.0))
    assert any("empty generator" in str(x.message) for x in w)


def test_generator_is_consumed_once():
    ps = _params(grads=False)
    seen = []

    def gen():
        for p in ps:
            seen.append(p)
            yield p

    assert torch.equal(clip_grad_norm_(gen(), 1.0), torch.tensor(0.0))
    assert seen == ps


@pytest.mark.parametrize("kw", [dict(norm_type=1.0), dict(norm_type=math.inf), dict(norm_type=3), dict(foreach=False)])
def test_unsupported_options_raise_before_writing(kw):
    ps = _params()
    snap = _snapshot(ps)
    with pytest.raises(ValueError):
        clip_grad_norm_(ps, 1.0, **kw)
    _unchanged(ps, snap)


def _with_grad(data, grad):
    p = torch.nn.Parameter(data)
    p.grad = grad
    return p


def _fp16(ps):
    ps[2] = _with_grad(torch.randn(2, 2).half(), torch.randn(2, 2).half())


def _bf16(ps):
    ps[0] = _with_grad(torch.randn(3).bfloat16(), torch.randn(3).bfloat16())


def _noncontig(ps):
    ps[0].grad = torch.randn(4, 3).t()


def _sparse(ps):
    ps[1] = _with_grad(torch.randn(5).to_sparse(), torch.randn(5).to_sparse())


@pytest.mark.parametrize("make", [_fp16, _bf16, _noncontig, _sparse])
def test_bad_grads_raise_before_writing(make):
    ps = _params()
    make(ps)
    snap = _snapshot(ps)
    with pytest.raises(ValueError):
        clip_grad_norm_(ps, 1.0)
    _unchanged(ps, snap)


def test_cpu_grads_raise_before_writing():
    ps = _params()
    snap = _snapshot(ps)
    with pytest.raises(_capi.XqError):                                       # no CPU path
        clip_grad_norm_(ps, 1.0)
    with pytest.raises(_capi.XqError):
        clip_grad_norm_(ps[0], 1.0)                                          # a single tensor
    _unchanged(ps, snap)
