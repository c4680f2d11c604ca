"""CPU checks of the AdamW step (imagefolder_b200/optim.py, csrc/adamw_kernel.cu): argument refusal of xq_adamw_step before any
CUDA call, and the parts of the optimizer that are torch.optim.AdamW's own (param_groups, state_dict, option checks)."""
import os
import re

import numpy as np
import pytest
import torch

from imagefolder_b200 import _capi
from imagefolder_b200.optim import AdamW

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_ARG = -1


def _table(ptrs, numels, scalars=None):
    """the same pointer for all four operands of an entry unless `ptrs` holds 4-tuples"""
    quads = [p if isinstance(p, tuple) else (p,) * 4 for p in ptrs]
    cols = [np.array([q[k] for q in quads], dtype=np.uint64) for k in range(4)]
    n = np.array(numels, dtype=np.int64)
    ss = np.full(len(numels), -1e-3, dtype=np.float64) if scalars is None else np.array(scalars[0], dtype=np.float64)
    bc = np.full(len(numels), 0.5, dtype=np.float64) if scalars is None else np.array(scalars[1], dtype=np.float64)
    return (*cols, n, ss, bc)


def _call(tab, hyper=(1.0, 0.1, 0.95, 0.05, 1e-8)):
    L = _capi.lib()
    args = [a.ctypes.data if a is not None else None for a in tab]
    count = len(next(a for a in tab if a is not None))
    return L.xq_adamw_step(*args, count, *hyper, None)


def test_table_capacity_matches_header():
    text = open(os.path.join(ROOT, "include", "xqb200.h")).read()
    assert int(re.search(r"#define XQ_ADAMW_MAX_TENSORS (\d+)", text).group(1)) == _capi.XQ_ADAMW_MAX_TENSORS


def test_c_abi_refuses_bad_arguments_without_gpu():
    """every refusal happens before the first CUDA call, so none of these touches a device"""
    L = _capi.lib()
    assert L.xq_adamw_step(*[None] * 7, 0, 1.0, 0.1, 0.95, 0.05, 1e-8, None) == 0           # n == 0: no-op
    assert L.xq_adamw_step(*[None] * 7, -1, 1.0, 0.1, 0.95, 0.05, 1e-8, None) == ERR_ARG
    tab = _table([4096], [16])
    for k in range(7):                                                                        # NULL arrays with n > 0
        assert _call(tuple(None if j == k else a for j, a in enumerate(tab))) == ERR_ARG
    assert _call(_table([4096], [-1])) == ERR_ARG                                            # negative numel
    for k in range(4):
        quad = tuple(4096 + 64 * j for j in range(4))
        null = tuple(0 if j == k else q for j, q in enumerate(quad))
        odd = tuple(q + 2 if j == k else q for j, q in enumerate(quad))
        assert _call(_table([null], [16])) == ERR_ARG                                        # NULL pointer, non-empty entry
        assert _call(_table([odd], [16])) == ERR_ARG                                         # not 4-byte aligned
    for bad in (float("nan"), float("inf")):
        assert _call(_table([4096], [16], ([bad], [0.5]))) == ERR_ARG                       # non-finite per-tensor scalars
        assert _call(_table([4096], [16], ([-1e-3], [bad]))) == ERR_ARG
        for k in range(5):
            hyper = [1.0, 0.1, 0.95, 0.05, 1e-8]
            hyper[k] = bad
            assert _call(_table([4096], [16]), tuple(hyper)) == ERR_ARG
    assert _call(_table([0, 0], [0, 0])) == 0                                                # only empty entries: nothing to launch


def test_c_abi_validates_every_entry_before_the_first_launch():
    """a bad entry after more than two launches' worth of valid ones is still refused with XQ_ERR_ARG (a launch on these dummy
    pointers would have been attempted first otherwise, and fail with a CUDA error on this host)"""
    m = 2 * _capi.XQ_ADAMW_MAX_TENSORS + 7
    good = [4096 + 64 * i for i in range(m)]
    for bad_ptr, bad_n in ((4097, 16), (4096, -3)):
        assert _call(_table(good + [bad_ptr], [16] * m + [bad_n])) == ERR_ARG
    assert _call(_table(good + [4096], [16] * (m + 1), ([-1e-3] * m + [float("nan")], [0.5] * (m + 1)))) == ERR_ARG


def _params(seed=0):
    torch.manual_seed(seed)
    model = torch.nn.Sequential(torch.nn.Linear(4, 3), torch.nn.LayerNorm(3), torch.nn.Linear(3, 2))
    return model


def _groups(model):
    return [{"params": list(model[0].parameters())},
            {"params": list(model[1].parameters()) + list(model[2].parameters()), "lr": 2e-4, "weight_decay": 5e-4}]


def test_param_groups_and_empty_state_dict_match_torch():
    model = _params()
    kw = dict(lr=3e-5, betas=(0.9, 0.95), weight_decay=5e-5)
    ours, ref = AdamW(_groups(model), **kw), torch.optim.AdamW(_groups(model), **kw)
    assert ours.param_groups == ref.param_groups
    assert ours.state_dict() == ref.state_dict()
    assert ours.defaults == ref.defaults
    ours_default, ref_default = AdamW(model.parameters()), torch.optim.AdamW(model.parameters())
    assert ours_default.state_dict() == ref_default.state_dict()


def test_torch_state_dict_loads_into_ours():
    """a CPU step of torch's own AdamW makes the state the reference checkpoints; ours loads it unchanged"""
    model = _params()
    ref = torch.optim.AdamW(_groups(model), lr=1e-3, betas=(0.9, 0.95), weight_decay=0.0)
    model(torch.randn(5, 4)).square().sum().backward()
    ref.step()
    sd = ref.state_dict()
    ours = AdamW(_groups(model), lr=1e-3, betas=(0.9, 0.95), weight_decay=0.0)
    ours.load_state_dict(sd)
    assert ours.param_groups == ref.param_groups
    got = ours.state_dict()
    assert got["param_groups"] == sd["param_groups"]
    assert got["state"].keys() == sd["state"].keys()
    for k, st in sd["state"].items():
        assert set(got["state"][k]) == {"step", "exp_avg", "exp_avg_sq"}
        for name, v in st.items():
            w = got["state"][k][name]
            assert w.dtype == v.dtype and w.device == v.device and torch.equal(w, v), (k, name)
    assert sd["state"][0]["step"].dtype == torch.float32 and sd["state"][0]["step"].device.type == "cpu"


@pytest.mark.parametrize("kw", [dict(amsgrad=True), dict(maximize=True), dict(capturable=True), dict(differentiable=True),
                                dict(fused=True), dict(foreach=False), dict(lr=torch.tensor(1e-3)),
                                dict(betas=(torch.tensor(0.9), 0.95)), dict(betas=(0.9, torch.tensor(0.95)))])
def test_unsupported_constructor_options_raise(kw):
    with pytest.raises((ValueError, RuntimeError)):
        AdamW(_params().parameters(), **kw)


def test_cpu_params_raise_before_writing():
    model = _params()
    model(torch.randn(5, 4)).square().sum().backward()
    opt = AdamW(model.parameters())
    before = [p.detach().clone() for p in model.parameters()]
    with pytest.raises(_capi.XqError):                                   # no CPU path
        opt.step()
    assert not opt.state
    for b, p in zip(before, model.parameters()):
        assert torch.equal(b, p.detach())
