"""Weight EMA of the tokenizer trainer -- drop-in for utils/ema.py (update_ema :4-14, requires_grad :17-22).

With `ema: true` (every shipped config) xqgan_train.py keeps `ema = deepcopy(vq_model)` (:315-317), initialises it with
`update_ema(ema, vq_model, decay=0)` (:405-406), calls `update_ema(ema, vq_model)` after every optimizer step (:461-462) and
saves `ema.state_dict()` as checkpoint["ema"] (:584-585).  The reference loops over the parameters in Python, two kernels per
tensor; here one call is one launch of csrc/ema_kernel.cu for up to XQ_EMA_MAX_TENSORS tensors (all of a shipped config), with
the same bits:

    from imagefolder_b200.ema import update_ema, requires_grad     # instead of: from utils.ema import ...
"""
from __future__ import annotations

from collections import OrderedDict

import numpy as np
import torch

from . import _capi

__all__ = ["update_ema", "requires_grad"]


@torch.no_grad()
def update_ema(ema_model, model, decay=0.9999):
    """Step the EMA model towards the current model: for every parameter name of `model`,
    ema = ema * decay + (1 - decay) * param, bit-identical to the reference's `mul_(decay).add_(param, alpha=1 - decay)`.

    A complex64 parameter (the RoPE decoder's `freqs_1d`) is averaged through its real view, component by component
    (DESIGN.md section 8 states where that differs from torch's complex mul_ / add_: signed zeros and non-finite values).
    Every pair is checked before anything is launched (same shape and dtype, fp32 or complex64, contiguous CUDA tensors on
    one device), so a refused
    call leaves the EMA model unchanged.  The pointer table is rebuilt on every call: `.to()`, `load_state_dict` or a wrapper
    that rebinds parameters can all move the storage between calls."""
    ema_params = OrderedDict(ema_model.named_parameters())
    model_params = OrderedDict(model.named_parameters())
    pairs = []
    for name, param in model_params.items():
        e = ema_params[name]
        if e.shape != param.shape:
            raise ValueError(f"update_ema: {name}: ema shape {tuple(e.shape)} != model shape {tuple(param.shape)}")
        if e.dtype not in (torch.float32, torch.complex64) or param.dtype != e.dtype:
            raise ValueError(f"update_ema: {name}: fp32 or complex64 tensors of one dtype are required (ema {e.dtype}, "
                             f"model {param.dtype})")
        if e.numel():
            if e.dtype == torch.complex64:
                e, param = torch.view_as_real(e), torch.view_as_real(param)
            pairs.append((name, e, param))
    emas, params, numels = [], [], []
    device = None
    for name, e, param in pairs:
        emas.append(_capi.ptr(e))
        params.append(_capi.ptr(param))
        numels.append(e.numel())
        if device is None:
            device = e.device
        if e.device != device or param.device != device:
            raise ValueError(f"update_ema: {name}: tensors on {e.device} / {param.device}, expected {device}")
    if not emas:
        return
    n = len(emas)
    e_arr = np.array(emas, dtype=np.uint64)
    p_arr = np.array(params, dtype=np.uint64)
    n_arr = np.array(numels, dtype=np.int64)
    L = _capi.lib()
    with torch.cuda.device(device):
        _capi.call("xq_ema_update", -(-n // _capi.XQ_EMA_MAX_TENSORS), L.xq_ema_update, e_arr.ctypes.data, p_arr.ctypes.data,
                   n_arr.ctypes.data, n, float(decay), float(1 - decay), _capi.stream_ptr(device), nbytes=12 * int(n_arr.sum()))
    # the kernel writes through raw pointers: bump the version counters as the reference's in-place ops do, so autograd still
    # refuses a backward through a graph that saved one of these tensors before the update
    torch.autograd.graph.increment_version([e for _, e, _ in pairs])


def requires_grad(model, flag=True):
    """Set requires_grad flag for all parameters in a model."""
    for p in model.parameters():
        p.requires_grad = flag
