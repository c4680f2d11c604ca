"""GPU tests of the gradient-norm clipping (imagefolder_b200/optim.py::clip_grad_norm_, csrc/clip_kernel.cu) against torch's
foreach clip_grad_norm_ as the reference trainer calls it (xqgan_train.py:456-458, 471-473), bit for bit: every comparison is
an int32-view equality against torch run on a copy of the same grads at the same storage offsets."""
import math

import numpy as np
import pytest
import torch

from imagefolder_b200 import _capi
from imagefolder_b200.optim import AdamW, clip_grad_norm_
from test_ema_cpu import build_shipped
from test_gpu_adamw import _disc_backward, vq_backward

pytestmark = pytest.mark.gpu

CHUNK = _capi.XQ_GRAD_NORM_CHUNK
T = _capi.XQ_CLIP_MAX_TENSORS
FLT_MAX = torch.finfo(torch.float32).max


def bits(t):
    return t.detach().contiguous().view(torch.int32)


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


def flat_views(sizes, offsets, seed=0, values=None, pad=5):
    """grads as views into one flat buffer, each at the given float offset past a 16-byte boundary (DDP bucket views)"""
    starts, pos = [], 0
    for n, o in zip(sizes, offsets):
        pos = (pos + 3) // 4 * 4 + o
        starts.append(pos)
        pos += n + pad
    g = torch.Generator(device="cuda").manual_seed(seed)
    buf = torch.randn(pos + 4, generator=g, device="cuda") if values is None else values(pos + 4, g)
    return buf, [buf[s:s + n] for s, n in zip(starts, sizes)], starts


def twin_views(buf, sizes, starts):
    """the same views into a copy of the buffer: the same alignment, so torch takes the same load paths"""
    b2 = buf.clone()
    return b2, [b2[s:s + n] for s, n in zip(starts, sizes)]


def c_norms(grads):
    """xq_grad_norm into a NaN-filled array, so an unwritten entry cannot pass"""
    n = len(grads)
    ptrs = np.array([g.data_ptr() for g in grads], dtype=np.uint64)
    numel = np.array([g.numel() for g in grads], dtype=np.int64)
    L = _capi.lib()
    ws = _capi.workspace(L.xq_grad_norm_workspace_bytes(n, numel.ctypes.data), "cuda")
    norms = torch.full((n,), math.nan, device="cuda")
    _capi.check(L.xq_grad_norm(ptrs.ctypes.data, numel.ctypes.data, n, norms.data_ptr(), ws.data_ptr(), ws.numel(),
                               _capi.stream_ptr()), "xq_grad_norm")
    return norms


def torch_norms(grads):
    return torch.stack(torch._foreach_norm(grads))


def as_params(views):
    ps = []
    for v in views:
        p = torch.nn.Parameter(torch.empty(v.shape, device="cuda"))
        p.grad = v
        ps.append(p)
    return ps


SIZES = [1, 3, 4, 5, 511, 512, 513, CHUNK - 1, CHUNK, CHUNK + 1, 2 * CHUNK - 4, 2 * CHUNK, 2 * CHUNK + 3, 5 * CHUNK + 4,
         10_000_001, 10_000_000]


@pytest.mark.parametrize("offset", [0, 1, 2, 3])
def test_per_tensor_norms(offset):
    sizes = SIZES + [0, 7, 0]
    offsets = [offset if i % 2 == 0 else (offset + i) % 4 for i in range(len(sizes))]
    _, views, _ = flat_views(sizes, offsets, seed=offset)
    got = c_norms(views)
    torch.cuda.synchronize()
    assert same_bits(got, torch_norms(views))
    assert float(got[len(SIZES)]) == 0.0 and float(got[-1]) == 0.0


def test_tables_longer_than_one_launch():
    base = [1, 4, 5, 17, 513, 4096, CHUNK + 1, 0, 1000]
    sizes = [base[i % len(base)] for i in range(2 * T + 57)]
    for i in (T - 1, T, 2 * T + 3):
        sizes[i] = 3 * CHUNK + 1
    buf, views, starts = flat_views(sizes, [i % 4 for i in range(len(sizes))], seed=7)
    buf2, views2 = twin_views(buf, sizes, starts)
    assert same_bits(c_norms(views), torch_norms(views))
    ps = as_params(views)
    n0 = _capi.LAUNCHES[0]
    total = clip_grad_norm_(ps, 0.5)
    assert _capi.LAUNCHES[0] - n0 == 3 * 2 + 3                                # per table: partials, finish, scale
    want = torch.nn.utils.clip_grad_norm_(as_params(views2), 0.5)
    assert same_bits(total, want)
    for a, b in zip(views, views2):
        assert same_bits(a, b)


def _special_values(overflow):
    sp = [0.0, -0.0, 1e-40, -1e-40, 1.4e-45, -1.4e-45, 1.2e-38] + ([1e20, -3e19, FLT_MAX] if overflow else [])

    def values(total, g):
        v = torch.randn(total, generator=g, device="cuda")
        pick = torch.rand(total, generator=g, device="cuda") < 0.05
        spt = torch.tensor(sp, device="cuda")
        v[pick] = spt[torch.randint(0, len(sp), (int(pick.sum()),), generator=g, device="cuda")]
        return v
    return values


@pytest.mark.parametrize("overflow", [False, True])
@pytest.mark.parametrize("extra", [None, math.inf, -math.inf, math.nan])
def test_special_values(overflow, extra):
    """±0 and subnormals everywhere, and with `overflow` values whose squares overflow (norm inf); one tensor also holds
    ±inf or NaN.  The per-tensor norms, the total norm and every grad match torch's, NaN bit patterns included."""
    sizes = [5, 4, 1, 513, CHUNK + 3, 100, 3]
    offs = [1, 0, 3, 2, 0, 1, 0]
    buf, views, starts = flat_views(sizes, offs, seed=3, values=_special_values(overflow))
    if extra is not None:
        views[4][CHUNK + 1] = extra
    buf2, views2 = twin_views(buf, sizes, starts)
    assert same_bits(c_norms(views), torch_norms(views))
    total = clip_grad_norm_(as_params(views), 1.0)
    want = torch.nn.utils.clip_grad_norm_(as_params(views2), 1.0)
    assert same_bits(total, want)
    assert same_bits(buf, buf2)
    assert math.isfinite(float(want)) == (not overflow and extra is None)


def test_all_small_values_clip_exactly():
    """subnormal-only grads: the norm is tiny and the coefficient clamps to 1"""
    sizes, offs = [7, 9], [1, 0]
    buf, views, starts = flat_views(sizes, offs, values=lambda n, g: torch.randn(n, generator=g, device="cuda") * 1e-41)
    buf2, views2 = twin_views(buf, sizes, starts)
    assert same_bits(clip_grad_norm_(as_params(views), 1.0), torch.nn.utils.clip_grad_norm_(as_params(views2), 1.0))
    assert same_bits(buf, buf2)


def _twin_grads(params):
    return [torch.nn.Parameter(p.detach().clone()) for p in params]


def _compare_call(params, max_norm, **kw):
    """our call on `params` against torch's on clones of their grads; params without a grad stay without"""
    ref = _twin_grads(params)
    for p, r in zip(params, ref):
        r.grad = None if p.grad is None else p.grad.clone()
    total = clip_grad_norm_(params, max_norm, **kw)
    want = torch.nn.utils.clip_grad_norm_(ref, max_norm, **kw)
    torch.cuda.synchronize()
    assert same_bits(total, want), (float(total), float(want))
    for i, (p, r) in enumerate(zip(params, ref)):
        assert (p.grad is None) == (r.grad is None), i
        if p.grad is not None:
            assert same_bits(p.grad, r.grad), i
    return float(want)


@pytest.mark.parametrize("max_norm", [1e-3, 1e9])
def test_vq8192_as_shipped(max_norm):
    """all params of VQ-8192 (the frozen teachers' grads are None) with grads of a real bf16 forward / backward"""
    model = build_shipped("VQ-8192").cuda().train()
    vq_backward(model, (torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(0)) * 2 - 1).cuda())
    params = list(model.parameters())
    assert any(p.grad is None for p in params) and sum(p.grad is not None for p in params) == 357
    versions = [p.grad._version for p in params if p.grad is not None]
    total = _compare_call(params, max_norm)
    assert (total > max_norm) == (max_norm < 1)                               # one clips, one does not
    assert [p.grad._version for p in params if p.grad is not None] == [v + 1 for v in versions]


def test_msbr4096():
    model = build_shipped("MSBR10P2-4096").cuda().train()
    params = [p for p in model.parameters() if p.requires_grad]
    g = torch.Generator(device="cuda").manual_seed(2)
    for p in params:
        p.grad = torch.randn(p.shape, generator=g, device="cuda") * 1e-3
    _compare_call(params, 1.0)
    _compare_call(params, 1e-2)


def test_dinodisc_heads():
    import warnings
    from imagefolder_b200.discriminator_dino import DinoDisc
    warnings.filterwarnings("ignore", message=".*RANDOM.*")
    torch.manual_seed(0)
    disc = DinoDisc(device="cuda").cuda().train()
    _disc_backward(disc, (torch.rand(4, 3, 256, 256, generator=torch.Generator().manual_seed(1)) * 2 - 1).cuda())
    params = [p for p in disc.parameters() if p.requires_grad]
    _compare_call(params, 1.0)
    _compare_call(params, 1e-4)


def test_bucket_views():
    """grads as views into one flat buffer, as DDP's gradient_as_bucket_view makes them: every offset, both load paths"""
    sizes = [3, 4096, 1, CHUNK + 5, 768, 12, 2 * CHUNK, 511, 3 * 256 * 16 * 16 + 1]
    offs = [0, 1, 3, 2, 0, 1, 0, 3, 2]
    buf, views, starts = flat_views(sizes, offs, seed=11)
    buf2, views2 = twin_views(buf, sizes, starts)
    for max_norm in (1.0, 1e6):
        total = clip_grad_norm_(as_params(views), max_norm)
        want = torch.nn.utils.clip_grad_norm_(as_params(views2), max_norm)
        assert same_bits(total, want) and same_bits(buf, buf2)


def test_training_sequence_with_grad_scaler():
    """five fp16 steps of GradScaler -> unscale_ -> clip -> AdamW, ours against torch's clip; step 2 overflows and is skipped"""
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(96, 257), torch.nn.GELU(), torch.nn.LayerNorm(257), torch.nn.Linear(257, 33)).cuda()
    ref = torch.nn.Sequential(torch.nn.Linear(96, 257), torch.nn.GELU(), torch.nn.LayerNorm(257), torch.nn.Linear(257, 33)).cuda()
    ref.load_state_dict(net.state_dict())
    arms = []
    for model, clip in ((net, clip_grad_norm_), (ref, torch.nn.utils.clip_grad_norm_)):
        opt = AdamW(model.parameters(), lr=1e-3, betas=(0.9, 0.95), weight_decay=5e-4)
        arms.append((model, clip, opt, torch.amp.GradScaler("cuda", init_scale=2.0 ** 14)))
    g = torch.Generator(device="cuda").manual_seed(4)
    for step in range(5):
        x = torch.randn(64, 96, generator=g, device="cuda")
        totals = []
        for model, clip, opt, scaler in arms:
            opt.zero_grad(set_to_none=True)
            with torch.autocast("cuda", dtype=torch.float16):
                loss = model(x).float().square().mean()
            scaler.scale(loss).backward()
            if step == 2:
                model[0].weight.grad[3, 5] = math.inf
            scaler.unscale_(opt)
            totals.append(clip(model.parameters(), 0.05))
            scaler.step(opt)
            scaler.update()
        torch.cuda.synchronize()
        assert same_bits(totals[0], totals[1]), step
        assert arms[0][3].get_scale() == arms[1][3].get_scale()
        for (n1, p1), (n2, p2) in zip(net.named_parameters(), ref.named_parameters()):
            assert same_bits(p1, p2) and same_bits(p1.grad, p2.grad), (step, n1)
            s1, s2 = arms[0][2].state[p1], arms[1][2].state[p2]
            assert same_bits(s1["exp_avg"], s2["exp_avg"]) and same_bits(s1["exp_avg_sq"], s2["exp_avg_sq"]), (step, n1)
            assert torch.equal(s1["step"], s2["step"]), (step, n1)
    assert float(arms[0][2].state[net[0].weight]["step"]) == 4.0               # the overflowing step was skipped


def test_error_if_nonfinite_leaves_grads():
    for bad in (math.inf, math.nan):
        sizes, offs = [100, 5, CHUNK + 1], [0, 1, 2]
        buf, views, starts = flat_views(sizes, offs, seed=5)
        views[1][2] = bad
        before = buf.clone()
        ps = as_params(views)
        versions = [v._version for v in views]
        with pytest.raises(RuntimeError, match="non-finite"):
            clip_grad_norm_(ps, 1.0, error_if_nonfinite=True)
        torch.cuda.synchronize()
        assert same_bits(buf, before) and [v._version for v in views] == versions
    # finite grads with error_if_nonfinite=True clip as torch does
    buf, views, starts = flat_views([100, 5], [0, 3], seed=6)
    buf2, views2 = twin_views(buf, [100, 5], starts)
    assert same_bits(clip_grad_norm_(as_params(views), 1.0, error_if_nonfinite=True),
                     torch.nn.utils.clip_grad_norm_(as_params(views2), 1.0, error_if_nonfinite=True))
    assert same_bits(buf, buf2)


def test_python_refusals_write_nothing():
    buf, views, _ = flat_views([100, 7, 6], [0, 1, 0], seed=8)
    before = buf.clone()
    cases = []
    ps = as_params(views)
    cases.append((ps, dict(norm_type=1.0), ValueError))
    cases.append((ps, dict(foreach=False), ValueError))
    half = torch.nn.Parameter(torch.zeros(4, device="cuda", dtype=torch.float16))
    half.grad = torch.ones(4, device="cuda", dtype=torch.float16)
    cases.append((ps + [half], {}, ValueError))
    nc = torch.nn.Parameter(torch.zeros(3, 4, device="cuda"))
    nc.grad = torch.ones(4, 3, device="cuda").t()
    cases.append((ps + [nc], {}, ValueError))
    cpu = torch.nn.Parameter(torch.zeros(3))
    cpu.grad = torch.ones(3)
    cases.append((ps + [cpu], {}, _capi.XqError))
    for params, kw, exc in cases:
        with pytest.raises(exc):
            clip_grad_norm_(params, 1e-3, **kw)
        torch.cuda.synchronize()
        assert same_bits(buf, before)
        assert half.grad.eq(1).all() and nc.grad.eq(1).all() and cpu.grad.eq(1).all()


def test_c_abi_refusal_after_a_full_table_writes_nothing():
    m = T + 9
    buf, views, _ = flat_views([5] * m, [i % 4 for i in range(m)], seed=9)
    before = buf.clone()
    ptrs = np.array([v.data_ptr() for v in views] + [views[-1].data_ptr() + 2], dtype=np.uint64)   # the last one misaligned
    numel = np.array([5] * (m + 1), dtype=np.int64)
    L = _capi.lib()
    ws = _capi.workspace(L.xq_grad_norm_workspace_bytes(m + 1, numel.ctypes.data), "cuda")
    norms = torch.full((m + 1,), math.nan, device="cuda")
    coef = torch.tensor(0.5, device="cuda")
    assert L.xq_grad_norm(ptrs.ctypes.data, numel.ctypes.data, m + 1, norms.data_ptr(), ws.data_ptr(), ws.numel(),
                          _capi.stream_ptr()) == -1
    assert L.xq_grad_scale(ptrs.ctypes.data, numel.ctypes.data, m + 1, coef.data_ptr(), _capi.stream_ptr()) == -1
    torch.cuda.synchronize()
    assert torch.isnan(norms).all() and same_bits(buf, before)


def test_streams():
    """the call runs on the current stream, after the work queued there before it, on the default and on a side stream"""
    sizes, offs = [4 * CHUNK + 1, 1000, 4096], [1, 0, 0]
    for side in (False, True):
        buf, views, starts = flat_views(sizes, offs, seed=12)
        buf2, views2 = twin_views(buf, sizes, starts)
        big = torch.randn(4096, 4096, device="cuda")
        torch.cuda.synchronize()
        s = torch.cuda.Stream() if side else torch.cuda.current_stream()
        with torch.cuda.stream(s):
            for _ in range(4):
                big = big @ big / 64.0                                        # keep the stream busy
            buf.mul_(3.0).add_(big[0, 0] * 0)                                 # the grads change after that work
            total = clip_grad_norm_(as_params(views), 1.0)
            buf2.mul_(3.0).add_(big[0, 0] * 0)
            want = torch.nn.utils.clip_grad_norm_(as_params(views2), 1.0)
        s.synchronize()
        assert same_bits(total, want) and same_bits(buf, buf2), side
