"""CPU checks of the weight EMA (imagefolder_b200/ema.py, csrc/ema_kernel.cu): argument refusal of xq_ema_update before any
CUDA call, the Python surface's checks, and the reference's `ema = deepcopy(vq_model)` for every shipped config."""
import copy
import os
import re

import numpy as np
import pytest
import torch

from imagefolder_b200 import _capi
from imagefolder_b200 import config as xcfg
from imagefolder_b200.ema import requires_grad, update_ema

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_ARG = -1


def _table(ptrs_e, ptrs_p, numels):
    e = np.array(ptrs_e, dtype=np.uint64)
    p = np.array(ptrs_p, dtype=np.uint64)
    n = np.array(numels, dtype=np.int64)
    return e, p, n


def _call(e, p, n, count=1):
    L = _capi.lib()
    count = len(n) if n is not None else count
    return L.xq_ema_update(e.ctypes.data if e is not None else None, p.ctypes.data if p is not None else None,
                           n.ctypes.data if n is not None else None, count, 0.9999, 1e-4, None)


def test_table_capacity_matches_header():
    text = open(os.path.join(ROOT, "include", "xqb200.h")).read()
    assert int(re.search(r"#define XQ_EMA_MAX_TENSORS (\d+)", text).group(1)) == _capi.XQ_EMA_MAX_TENSORS


def test_c_abi_refuses_bad_arguments_without_gpu():
    """every refusal happens before the first CUDA call, so none of these touches a device"""
    L = _capi.lib()
    assert L.xq_ema_update(None, None, None, 0, 0.5, 0.5, None) == 0             # n == 0: no-op
    assert L.xq_ema_update(None, None, None, -1, 0.5, 0.5, None) == ERR_ARG
    e, p, n = _table([4096], [8192], [16])
    assert _call(None, p, n) == ERR_ARG                                           # NULL arrays with n > 0
    assert _call(e, None, n) == ERR_ARG
    assert _call(e, p, None) == ERR_ARG
    assert _call(*_table([4096], [8192], [-1])) == ERR_ARG                        # negative numel
    assert _call(*_table([0], [8192], [16])) == ERR_ARG                           # NULL pointer on a non-empty entry
    assert _call(*_table([4096], [0], [16])) == ERR_ARG
    assert _call(*_table([4098], [8192], [16])) == ERR_ARG                        # not 4-byte aligned
    assert _call(*_table([4096], [8193], [16])) == ERR_ARG
    assert _call(*_table([0, 0], [0, 0], [0, 0])) == 0                            # only empty entries: nothing to launch


def test_c_abi_validates_every_entry_before_the_first_launch():
    """a bad entry after more than two launches' worth of valid ones is still refused with XQ_ERR_ARG (a launch on these dummy
    pointers would have been attempted first otherwise, and fail with a CUDA error on this host)"""
    m = 2 * _capi.XQ_EMA_MAX_TENSORS + 7
    good = [4096 + 64 * i for i in range(m)]
    for bad in ([0], [-3]):
        e, p, n = _table(good + [4096], good + [8192], [16] * m + bad)
        if bad == [0]:
            e[-1] = 4097
            n[-1] = 16
        assert _call(e, p, n) == ERR_ARG


def _pair():
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(4, 3), torch.nn.LayerNorm(3))
    return model, copy.deepcopy(model)


def test_update_ema_refuses_before_writing():
    model, ema = _pair()
    before = [p.detach().clone() for p in ema.parameters()]
    with pytest.raises(_capi.XqError):                                            # no CPU path
        update_ema(ema, model)
    other = torch.nn.Sequential(torch.nn.Linear(4, 3))
    with pytest.raises(KeyError):                                                 # the reference's ema_params[name]
        update_ema(other, model)
    bad_shape = torch.nn.Sequential(torch.nn.Linear(4, 3), torch.nn.LayerNorm(3))
    bad_shape[1].bias = torch.nn.Parameter(torch.zeros(1, 3))
    with pytest.raises(ValueError, match="shape"):
        update_ema(bad_shape, model)
    with pytest.raises(ValueError, match="fp32"):
        update_ema(copy.deepcopy(model).double(), model)
    with pytest.raises(ValueError, match="fp32"):
        update_ema(ema, copy.deepcopy(model).half())
    for b, p in zip(before, ema.parameters()):
        assert torch.equal(b, p.detach())


def test_requires_grad_flips_every_parameter():
    model, _ = _pair()
    requires_grad(model, False)
    assert not any(p.requires_grad for p in model.parameters())
    requires_grad(model)
    assert all(p.requires_grad for p in model.parameters())


def build_shipped(name):
    args = xcfg.parse_args([])
    for k, v in xcfg.SHIPPED_CONFIGS[name].items():
        setattr(args, k, v)
    torch.manual_seed(0)
    return xcfg.build_vq_model(args)


def _storages(m):
    out = set()
    for t in list(m.parameters()) + list(m.buffers()):
        s = t.untyped_storage()
        if s.nbytes():
            out.add(s.data_ptr())
    return out


@pytest.mark.parametrize("name", sorted(xcfg.SHIPPED_CONFIGS))
def test_deepcopy_of_shipped_config_is_independent(name):
    """xqgan_train.py:315-317: `ema = deepcopy(vq_model); requires_grad(ema, False)`, teachers included"""
    model = build_shipped(name)
    ema = copy.deepcopy(model)
    requires_grad(ema, False)
    assert list(ema.state_dict()) == list(model.state_dict())
    assert [n for n, _ in ema.named_parameters()] == [n for n, _ in model.named_parameters()]
    assert not _storages(model) & _storages(ema)
    assert any(p.requires_grad for p in model.parameters())                       # the original keeps its flags
    for k, v in model.state_dict().items():
        assert torch.equal(v, ema.state_dict()[k]), k
    teachers = [getattr(ema, t) for t in ("semantic_model", "detail_model") if hasattr(ema, t)]
    assert teachers
    ema.train()
    assert ema.training and ema.encoder.training and not any(t.training for t in teachers)
    assert model.training == model.encoder.training                               # untouched by the copy's mode
    ema.eval()
    assert not any(m.training for m in ema.modules())
    model.train()
    assert not ema.training
