"""GPU tests of the AdamW step (imagefolder_b200/optim.py, csrc/adamw_kernel.cu) against torch.optim.AdamW constructed as the
reference does (xqgan_train.py:344-347: no foreach / fused argument, so torch's foreach step), bit for bit."""
import copy
import io
import math

import numpy as np
import pytest
import torch

from imagefolder_b200 import _capi
from imagefolder_b200.optim import AdamW
from test_ema_cpu import build_shipped

pytestmark = pytest.mark.gpu

FLT_MAX = torch.finfo(torch.float32).max
SPECIALS = [0.0, -0.0, math.inf, -math.inf, math.nan, FLT_MAX, -FLT_MAX, 1e-40, -1e-40, 1.4e-45, -1.4e-45,
            torch.finfo(torch.float32).tiny]


def same_bits(a, b):
    return torch.equal(a.detach().contiguous().view(torch.int32), b.detach().contiguous().view(torch.int32))


def same_bits_or_both_nan(a, b):
    a, b = a.detach(), b.detach()
    an, bn = torch.isnan(a), torch.isnan(b)
    return torch.equal(an, bn) and same_bits(torch.where(an, 0.0, a), torch.where(bn, 0.0, b))


def twin(params):
    return [p.detach().clone().requires_grad_(True) for p in params]


def assert_same(ours, ref, ours_params, ref_params, nan_ok=False):
    eq = same_bits_or_both_nan if nan_ok else same_bits
    for i, (p, r) in enumerate(zip(ours_params, ref_params)):
        assert eq(p, r), ("param", i)
        so, sr = ours.state.get(p, {}), ref.state.get(r, {})
        assert so.keys() == sr.keys(), i
        if so:
            assert so["step"].dtype == sr["step"].dtype == torch.float32 and so["step"].device == sr["step"].device
            assert torch.equal(so["step"], sr["step"]), ("step", i)
            assert eq(so["exp_avg"], sr["exp_avg"]), ("exp_avg", i)
            assert eq(so["exp_avg_sq"], sr["exp_avg_sq"]), ("exp_avg_sq", i)


def copy_grads(src, dst):
    for s, d in zip(src, dst):
        d.grad = None if s.grad is None else s.grad.clone()


def reload(opt_cls, params, sd, **kw):
    """a fresh optimizer of `opt_cls` that loads `sd` after a round trip through torch.save, as a checkpoint does"""
    buf = io.BytesIO()
    torch.save(sd, buf)
    buf.seek(0)
    opt = opt_cls(params, **kw)
    opt.load_state_dict(torch.load(buf, map_location="cpu", weights_only=True))
    return opt


def vq_backward(model, x):
    with torch.autocast("cuda", dtype=torch.bfloat16):
        dec, (vq, commit, ent, usages), _, _, _ = model(x, 0, 0.0, 0.0, 100)
        loss = torch.nn.functional.mse_loss(dec.float(), x) + vq + commit
    model.zero_grad(set_to_none=True)
    loss.backward()


def test_vq8192_as_shipped(record_property):
    """trainable params of VQ-8192, grads from a real bf16 forward / backward, lr 3e-5, betas (0.9, 0.95), wd 0; five steps with
    the lr changed between steps, some grads None on some steps, and a state_dict swapped across the two kinds after step 3"""
    model = build_shipped("VQ-8192").cuda().train()
    params = [p for p in model.parameters() if p.requires_grad]
    ref_params, fused_params = twin(params), twin(params)
    kw = dict(lr=3e-5, betas=(0.9, 0.95), weight_decay=0.0)
    ours, ref = AdamW(params, **kw), torch.optim.AdamW(ref_params, **kw)
    fused = torch.optim.AdamW(fused_params, fused=True, **kw)
    g = torch.Generator().manual_seed(0)
    fused_equal = []
    for step in range(5):
        x = (torch.rand(2, 3, 256, 256, generator=g) * 2 - 1).cuda()
        vq_backward(model, x)
        if step in (1, 3):                                             # per-tensor step counts diverge
            for p in params[step::7]:
                p.grad = None
        copy_grads(params, ref_params)
        copy_grads(params, fused_params)
        for o in (ours, ref, fused):
            o.param_groups[0]["lr"] = 3e-5 * (1 + 0.37 * step)
        n0 = _capi.LAUNCHES[0]
        ours.step()
        assert _capi.LAUNCHES[0] - n0 == -(-sum(p.grad is not None for p in params) // _capi.XQ_ADAMW_MAX_TENSORS)
        ref.step()
        fused.step()
        torch.cuda.synchronize()
        assert_same(ours, ref, params, ref_params)
        fused_equal.append(all(same_bits(a, b) for a, b in zip(params, fused_params)))
        if step == 2:
            sd_ours, sd_ref = ours.state_dict(), ref.state_dict()
            ours = reload(AdamW, params, sd_ref, **kw)
            ref = reload(torch.optim.AdamW, ref_params, sd_ours, **kw)
            assert_same(ours, ref, params, ref_params)
    steps = {float(ours.state[p]["step"]) for p in params if ours.state[p]}
    assert {4.0, 5.0} <= steps, steps
    record_property("fused_true_bit_identical_per_step", fused_equal)
    print("torch fused=True bit-identical to the foreach step, per step:", fused_equal)


def _disc_backward(disc, x):
    out = disc(x)
    disc.zero_grad(set_to_none=True)
    torch.relu(1.0 - out).mean().backward()


def test_weight_decay_dinodisc_heads():
    import warnings
    from imagefolder_b200.discriminator_dino import DinoDisc
    warnings.filterwarnings("ignore", message=".*RANDOM.*")
    torch.manual_seed(0)
    disc = DinoDisc(device="cuda").cuda().train()
    params = [p for p in disc.parameters() if p.requires_grad]
    ref_params = twin(params)
    kw = dict(lr=1e-4, betas=(0.9, 0.95), weight_decay=5e-4)
    ours, ref = AdamW(params, **kw), torch.optim.AdamW(ref_params, **kw)
    g = torch.Generator().manual_seed(1)
    for _ in range(3):
        _disc_backward(disc, (torch.rand(4, 3, 256, 256, generator=g) * 2 - 1).cuda())
        copy_grads(params, ref_params)
        ours.step()
        ref.step()
        torch.cuda.synchronize()
        assert_same(ours, ref, params, ref_params)


def test_weight_decay_msbr4096():
    """the trainable params of MSBR10P2-4096 as shipped, with seeded grads of training magnitude"""
    model = build_shipped("MSBR10P2-4096").cuda().train()
    params = [p for p in model.parameters() if p.requires_grad]
    ref_params = twin(params)
    kw = dict(lr=1e-4, betas=(0.9, 0.95), weight_decay=5e-5)
    ours, ref = AdamW(params, **kw), torch.optim.AdamW(ref_params, **kw)
    g = torch.Generator(device="cuda").manual_seed(2)
    for _ in range(2):
        for p in params:
            p.grad = torch.randn(p.shape, generator=g, device="cuda") * 1e-3
        copy_grads(params, ref_params)
        ours.step()
        ref.step()
        torch.cuda.synchronize()
        assert_same(ours, ref, params, ref_params)


# ---- stress: 2 200 tensors in flat buffers with sentinels ---------------------------------------------------------------------
def _sizes():
    base = [1, 2, 3, 4, 5, 6, 7, 15, 16, 17, 16383, 16384, 16385, 64, 100, 1000, 4099]
    sizes = [base[i % len(base)] for i in range(2200)]
    for i in (3, 583, 584, 1167, 1168, 2199):                        # 1 Mi + 3 spread over the four launches
        sizes[i] = (1 << 20) + 3
    return sizes


def _values(total, seed, special_frac):
    g = torch.Generator(device="cuda").manual_seed(seed)
    v = torch.randn(total, generator=g, device="cuda")
    sp = torch.tensor(SPECIALS, device="cuda")
    pick = torch.rand(total, generator=g, device="cuda") < special_frac
    v[pick] = sp[torch.randint(0, len(SPECIALS), (int(pick.sum()),), generator=g, device="cuda")]
    return v


class _Layout:
    """views into flat buffers at chosen float offsets, with sentinels between them"""

    def __init__(self, sizes, offsets, guard=8):
        self.spans, at = [], 0
        for n, o in zip(sizes, offsets):
            at += guard + o
            self.spans.append((at, n))
            at += n
        self.total = at + guard
        self.mask = torch.zeros(self.total, dtype=torch.bool, device="cuda")
        for s, n in self.spans:
            self.mask[s:s + n] = True

    def buffer(self, values):
        return torch.where(self.mask, values, torch.full_like(values, 1234.5))

    def views(self, buf):
        return [buf[s:s + n] for s, n in self.spans]


HYPERS = [(1e-3, (0.9, 0.999), 1e-8, 1e-2),
          (3e-5, (0.9, 0.95), 1e-8, 0.0),
          (0.5, (0.5, 0.0), 1e-3, 5e-4),       # lerp weight 0.5 (the large-weight branch), addcmul value 1
          (2.0, (0.2, 0.3), 0.0, 0.25),        # lerp weight 0.8, eps 0
          (1e-2, (0.0, 0.9), 1e-6, 0.0)]       # lerp weight 1


@pytest.mark.parametrize("hyper", HYPERS, ids=[f"h{i}" for i in range(len(HYPERS))])
def test_stress_table_alignment_specials(hyper):
    lr, betas, eps, wd = hyper
    sizes = _sizes()
    lay = _Layout(sizes, [(i // 3) % 4 for i in range(len(sizes))])
    bufs = {k: lay.buffer(_values(lay.total, seed, frac)) for k, seed, frac in
            (("p", 1, 0.01), ("g", 2, 0.05), ("m", 3, 0.05), ("v", 4, 0.05))}
    bufs["v"] = torch.where(torch.rand(lay.total, device="cuda") < 0.9, bufs["v"].abs(), bufs["v"])
    before = {k: b.clone() for k, b in bufs.items()}
    ref_bufs = {k: b.clone() for k, b in bufs.items()}
    kw = dict(lr=lr, betas=betas, eps=eps, weight_decay=wd)

    def build(b, cls):
        params = [torch.nn.Parameter(v) for v in lay.views(b["p"])]
        for i, (p, gv) in enumerate(zip(params, lay.views(b["g"]))):
            p.grad = None if i % 11 == 5 else gv
        opt = cls(params, **kw)
        for i, (p, m, v) in enumerate(zip(params, lay.views(b["m"]), lay.views(b["v"]))):
            opt.state[p] = {"step": torch.tensor(float(i % 9), dtype=torch.float32), "exp_avg": m, "exp_avg_sq": v}
        return params, opt

    params, ours = build(bufs, AdamW)
    ref_params, ref = build(ref_bufs, torch.optim.AdamW)
    assert any(p.data_ptr() % 16 for p in params) and any(p.data_ptr() % 16 == 0 for p in params)
    n0 = _capi.LAUNCHES[0]
    ours.step()
    assert _capi.LAUNCHES[0] - n0 == 4
    ref.step()
    torch.cuda.synchronize()
    for k in ("p", "m", "v"):
        assert same_bits(bufs[k][~lay.mask], before[k][~lay.mask]), k                        # sentinels
        assert same_bits_or_both_nan(bufs[k], ref_bufs[k]), k
    assert same_bits(bufs["g"], before["g"])
    for i, (p, r) in enumerate(zip(params, ref_params)):
        assert torch.equal(ours.state[p]["step"], ref.state[r]["step"]), i
    skipped = [i for i in range(len(sizes)) if i % 11 == 5]
    s, n = lay.spans[skipped[1]]
    assert same_bits(bufs["p"][s:s + n], before["p"][s:s + n])
    assert not same_bits(bufs["m"][lay.mask], before["m"][lay.mask])


# ---- refusals --------------------------------------------------------------------------------------------------------------------
def test_c_abi_refusal_after_a_launch_worth_writes_nothing():
    m = _capi.XQ_ADAMW_MAX_TENSORS + 9
    bufs = [torch.randn(m * 8, device="cuda") for _ in range(4)]
    before = [b.clone() for b in bufs]
    ptrs = [np.array([b.data_ptr() + 32 * i for i in range(m)] + [b.data_ptr() + 2], dtype=np.uint64) for b in bufs]
    numel = np.full(m + 1, 8, dtype=np.int64)
    ss, bc = np.full(m + 1, -1e-3), np.full(m + 1, 0.5)
    rc = _capi.lib().xq_adamw_step(*[a.ctypes.data for a in ptrs], numel.ctypes.data, ss.ctypes.data, bc.ctypes.data, m + 1,
                                   1.0, 0.1, 0.95, 0.05, 1e-8, _capi.stream_ptr())
    torch.cuda.synchronize()
    assert rc == -1
    for a, b in zip(bufs, before):
        assert same_bits(a, b)


def _small_model(seed=3):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(64, 64), torch.nn.LayerNorm(64), torch.nn.Linear(64, 32)).cuda()


def _snapshot(opt, params):
    return [(p.detach().clone(), {k: v.clone() for k, v in opt.state[p].items()} if p in opt.state else None) for p in params]


def _assert_snapshot(opt, params, snap):
    for p, (pv, st) in zip(params, snap):
        assert same_bits(p, pv.to(p.device))
        if st is None:
            assert p not in opt.state or not opt.state[p]
        else:
            for k, v in st.items():
                assert torch.equal(opt.state[p][k], v), k


def _bad_cases():
    """(what, mutate(opt, params)) -- each breaks the last param of the group or a group option"""
    def group(k, v):
        return lambda opt, ps: opt.param_groups[0].__setitem__(k, v)

    def last_param(make):
        def f(opt, ps):
            p = torch.nn.Parameter(make())
            p.grad = torch.zeros_like(p) if not p.is_sparse else None
            opt.param_groups[0]["params"].append(p)
            ps.append(p)
        return f

    def sparse_grad(opt, ps):
        emb = torch.nn.Embedding(10, 4, sparse=True).cuda()
        emb(torch.tensor([1, 2], device="cuda")).sum().backward()
        opt.param_groups[0]["params"].append(emb.weight)
        ps.append(emb.weight)

    def strided_state(opt, ps):
        p = ps[-2]                                                     # the last Linear's weight
        opt.state[p]["exp_avg"] = torch.zeros(p.shape[::-1], device="cuda").t()

    return [("amsgrad", group("amsgrad", True)), ("maximize", group("maximize", True)),
            ("capturable", group("capturable", True)), ("differentiable", group("differentiable", True)),
            ("fused", group("fused", True)), ("foreach False", group("foreach", False)),
            ("tensor lr", group("lr", torch.tensor(1e-3))), ("tensor beta", group("betas", (torch.tensor(0.9), 0.95))),
            ("fp16 param", last_param(lambda: torch.randn(8, device="cuda", dtype=torch.float16))),
            ("sparse grad", sparse_grad),
            ("cpu param", last_param(lambda: torch.randn(8))),
            ("non-contiguous param", last_param(lambda: torch.randn(8, 6, device="cuda").t())),
            ("non-contiguous state", strided_state)]


@pytest.mark.parametrize("case", range(13))
def test_python_refusals_write_nothing(case):
    what, mutate = _bad_cases()[case]
    model = _small_model()
    params = list(model.parameters())
    opt = AdamW(params, lr=1e-3, weight_decay=1e-2)
    model(torch.randn(8, 64, device="cuda")).square().sum().backward()
    opt.step()                                                         # state exists for the good params
    model(torch.randn(8, 64, device="cuda")).square().sum().backward()
    mutate(opt, params)
    snap = _snapshot(opt, params)
    n0 = _capi.LAUNCHES[0]
    with pytest.raises((ValueError, _capi.XqError)):
        opt.step()
    torch.cuda.synchronize()
    assert _capi.LAUNCHES[0] == n0, what
    _assert_snapshot(opt, params, snap)


def test_mixed_devices_raise():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    model = _small_model()
    params = list(model.parameters())
    p1 = torch.nn.Parameter(torch.randn(8, device="cuda:1"))
    p1.grad = torch.zeros_like(p1)
    model(torch.randn(8, 64, device="cuda")).square().sum().backward()
    opt = AdamW(params + [p1])
    with pytest.raises(ValueError):
        opt.step()
    assert not opt.state


# ---- streams and GradScaler ------------------------------------------------------------------------------------------------------
def test_runs_on_the_current_stream_after_its_earlier_work():
    model = _small_model(5)
    params = list(model.parameters())
    ref_params = twin(params)
    ours, ref = AdamW(params, lr=1e-3), torch.optim.AdamW(ref_params, lr=1e-3)
    grads = [torch.randn_like(p) for p in params]
    for p in params:
        p.grad = torch.zeros_like(p)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(20_000_000)                                # the step must wait for the copies below
        for p, g in zip(params, grads):
            p.grad.copy_(g)
        ours.step()
    s.synchronize()
    for r, g in zip(ref_params, grads):
        r.grad = g.clone()
    ref.step()
    torch.cuda.synchronize()
    assert_same(ours, ref, params, ref_params)
    for p in params:
        assert p._version > 0 and ours.state[p]["exp_avg"]._version == 1 and ours.state[p]["exp_avg_sq"]._version == 1


def test_grad_scaler_skips_inf_steps_and_matches_finite_ones():
    model = _small_model(6)
    ref_model = copy.deepcopy(model)
    ours, ref = AdamW(model.parameters(), lr=1e-3, weight_decay=5e-4), torch.optim.AdamW(ref_model.parameters(), lr=1e-3,
                                                                                            weight_decay=5e-4)
    sc, sc_ref = torch.amp.GradScaler("cuda", enabled=True), torch.amp.GradScaler("cuda", enabled=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    for step in range(4):
        x = torch.randn(16, 64, generator=g, device="cuda")
        for m, o, s in ((model, ours, sc), (ref_model, ref, sc_ref)):
            o.zero_grad(set_to_none=True)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = m(x).float().square().mean()
            s.scale(loss).backward()
            if step == 2:
                m[0].weight.grad[0, 0] = math.inf
        snap = _snapshot(ours, list(model.parameters()))
        for o, s in ((ours, sc), (ref, sc_ref)):
            s.step(o)
            s.update()
        torch.cuda.synchronize()
        if step == 2:
            _assert_snapshot(ours, list(model.parameters()), snap)
        assert sc.get_scale() == sc_ref.get_scale()
        assert_same(ours, ref, list(model.parameters()), list(ref_model.parameters()))
    assert float(ours.state[model[0].weight]["step"]) == 3.0
