"""GPU tests of the weight EMA (imagefolder_b200/ema.py, csrc/ema_kernel.cu) against the reference's own loop
(utils/ema.py:4-14: `ema.mul_(decay).add_(param, alpha=1 - decay)` per parameter), bit for bit."""
import copy
import math
from collections import OrderedDict

import pytest
import torch

from imagefolder_b200 import _capi
from imagefolder_b200.ema import requires_grad, update_ema
from test_ema_cpu import build_shipped

pytestmark = pytest.mark.gpu

FLT_MAX = torch.finfo(torch.float32).max
SPECIALS = [0.0, -0.0, math.inf, -math.inf, math.nan, FLT_MAX, -FLT_MAX, 1e-40, -1e-40, 1.4e-45, -1.4e-45,
            torch.finfo(torch.float32).tiny]


@torch.no_grad()
def reference_update_ema(ema_model, model, decay=0.9999):
    ema_params = OrderedDict(ema_model.named_parameters())
    for name, param in OrderedDict(model.named_parameters()).items():
        ema_params[name].mul_(decay).add_(param.data, alpha=1 - decay)


def same_bits(a, b):
    return torch.equal(a.detach().contiguous().view(torch.int32), b.detach().contiguous().view(torch.int32))


def same_bits_or_both_nan(a, b):
    a, b = a.detach(), b.detach()
    an, bn = torch.isnan(a), torch.isnan(b)
    return torch.equal(an, bn) and same_bits(torch.where(an, 0.0, a), torch.where(bn, 0.0, b))


@torch.no_grad()
def add_noise(model, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    for p in model.parameters():
        p.add_(torch.randn(p.shape, generator=g, device=p.device) * 1e-2)


def test_shipped_parameter_set_bit_identical():
    """VQ-8192 as shipped (531 tensors, frozen DINOv2 teacher included): the decay-0 initialisation and three 0.9999 steps"""
    model = build_shipped("VQ-8192").cuda()
    ema = copy.deepcopy(model)
    requires_grad(ema, False)
    ref = copy.deepcopy(ema)
    names = [n for n, _ in model.named_parameters()]
    assert len(names) == 531
    add_noise(model, 0)
    for rnd, decay in enumerate([0, 0.9999, 0.9999, 0.9999]):
        if rnd:
            add_noise(model, rnd)
        n0 = _capi.LAUNCHES[0]
        update_ema(ema, model, decay)
        assert _capi.LAUNCHES[0] == n0 + 1
        reference_update_ema(ref, model, decay)
        torch.cuda.synchronize()
        e, r = dict(ema.named_parameters()), dict(ref.named_parameters())
        for n in names:
            assert same_bits(e[n], r[n]), (rnd, n)
    m = dict(model.named_parameters())
    assert any(not torch.equal(e[n], m[n]) for n in names)           # the steps did average


def _edge_sizes():
    base = [1, 3, 4, 5, 15, 16, 17, 16383, 16384, 16385, 64, 100, 7, 2, 1000]
    sizes = [base[i % len(base)] for i in range(2500)]
    for i in (3, 1019, 1020, 2044, 2499):                            # 1 Mi + 3 on both sides of each table boundary
        sizes[i] = (1 << 20) + 3
    return sizes


class _Flat(torch.nn.Module):
    """parameters that are views into one flat buffer, each at a chosen float offset, with sentinels in between"""

    def __init__(self, sizes, offsets, values, guard=8):
        super().__init__()
        total = sum(guard + o + n for n, o in zip(sizes, offsets)) + guard
        self.buf = torch.full((total,), 1234.5, device="cuda")
        self.mask = torch.zeros(total, dtype=torch.bool, device="cuda")
        at = 0
        for i, (n, o) in enumerate(zip(sizes, offsets)):
            at += guard + o
            self.buf[at:at + n] = values[at:at + n]
            self.mask[at:at + n] = True
            v = self.buf[at:at + n]
            if n == 16:
                v = v.view(4, 4)
            self.register_parameter(f"p{i}", torch.nn.Parameter(v, requires_grad=False))
            at += n


def _values(total, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    v = torch.randn(total, generator=g, device="cuda")
    sp = torch.tensor(SPECIALS, device="cuda")
    pick = torch.rand(total, generator=g, device="cuda") < 0.05
    v[pick] = sp[torch.randint(0, len(SPECIALS), (int(pick.sum()),), generator=g, device="cuda")]
    v[:len(SPECIALS)] = sp
    return v


@pytest.mark.parametrize("decay", [0, 0.5, 0.9999, 1.0])
def test_table_and_alignment_edges(decay):
    """2500 tensors (three launches), sizes around the 16 Ki-float chunk and the float4 width, storage offsets of 0-3 floats
    (scalar path), special values in both operands; the floats around every tensor must be untouched"""
    sizes = _edge_sizes()
    offsets = [(i // 3) % 4 for i in range(len(sizes))]
    total = sum(8 + o + n for n, o in zip(sizes, offsets)) + 8
    ema = _Flat(sizes, offsets, _values(total, 1))
    model = _Flat(sizes, offsets, _values(total, 2))
    ref = _Flat(sizes, offsets, ema.buf.clone())
    assert any(p.data_ptr() % 16 for p in ema.parameters()) and any(p.data_ptr() % 16 == 0 for p in ema.parameters())
    before = ema.buf.clone()
    n0 = _capi.LAUNCHES[0]
    update_ema(ema, model, decay)
    assert _capi.LAUNCHES[0] == n0 + math.ceil(len(sizes) / _capi.XQ_EMA_MAX_TENSORS) == n0 + 3
    reference_update_ema(ref, model, decay)
    torch.cuda.synchronize()
    assert same_bits(ema.buf[~ema.mask], before[~ema.mask])                 # sentinels
    assert same_bits_or_both_nan(ema.buf[ema.mask], ref.buf[ref.mask])
    if decay == 0.5:
        assert not same_bits(ema.buf[ema.mask], before[ema.mask])


def test_refused_call_writes_nothing():
    """one bad entry among valid ones, last in the iteration order: every ema tensor keeps its bits, nothing is launched"""
    torch.manual_seed(3)
    model = torch.nn.Sequential(*[torch.nn.Linear(64, 64) for _ in range(4)]).cuda()
    cases = []
    bad = copy.deepcopy(model)                                              # non-contiguous ema tensor
    bad[3].weight = torch.nn.Parameter(torch.randn(64, 64, device="cuda").t())
    cases.append((bad, model, _capi.XqError))
    bad = copy.deepcopy(model)                                              # CPU ema tensor
    bad[3].bias = torch.nn.Parameter(torch.randn(64))
    cases.append((bad, model, _capi.XqError))
    src = copy.deepcopy(model)                                              # CPU model tensor
    src[3].bias = torch.nn.Parameter(torch.randn(64))
    cases.append((copy.deepcopy(model), src, _capi.XqError))
    bad = copy.deepcopy(model)                                              # shape mismatch
    bad[3].bias = torch.nn.Parameter(torch.randn(1, 64, device="cuda"))
    cases.append((bad, model, ValueError))
    if torch.cuda.device_count() > 1:
        src = copy.deepcopy(model)
        src[3].bias = torch.nn.Parameter(torch.randn(64, device="cuda:1"))
        cases.append((copy.deepcopy(model), src, ValueError))
    add_noise(model, 4)
    for ema, src, exc in cases:
        before = [p.detach().clone() for p in ema.parameters()]
        n0 = _capi.LAUNCHES[0]
        with pytest.raises(exc):
            update_ema(ema, src, 0.5)
        torch.cuda.synchronize()
        assert _capi.LAUNCHES[0] == n0
        for b, p in zip(before, ema.parameters()):
            assert same_bits(b.to(p.device), p)


def test_runs_on_the_current_stream_after_its_earlier_work():
    torch.manual_seed(5)
    model = torch.nn.Sequential(torch.nn.Linear(512, 2048), torch.nn.Linear(2048, 512)).cuda()
    ema = copy.deepcopy(model)
    ref = copy.deepcopy(model)
    new = [torch.randn_like(p) for p in model.parameters()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(20_000_000)                                       # the update must wait for the copies below
        with torch.no_grad():
            for p, v in zip(model.parameters(), new):
                p.copy_(v)
        update_ema(ema, model, 0.9)
    s.synchronize()
    reference_update_ema(ref, model, 0.9)
    torch.cuda.synchronize()
    for a, b in zip(ema.parameters(), ref.parameters()):
        assert same_bits(a, b)
        assert a._version == 1                                              # the in-place write is visible to autograd


@pytest.mark.parametrize("name", ["VQ-8192", "MSVR10P2-4096"])
def test_ema_copy_in_use(name, tmp_path):
    """the reference's recipe: deepcopy, decay-0 initialisation, then the copy is the model that is evaluated and saved"""
    model = build_shipped(name).cuda()
    ema = copy.deepcopy(model)
    requires_grad(ema, False)
    add_noise(model, 7)
    update_ema(ema, model, decay=0)
    # same flags on both sides: ATen's matmul folds a non-contiguous 3-D input into one mm when the weight requires grad (even
    # under no_grad) and runs a bmm otherwise, and the two round differently -- decoder.to_pixel's nn.Linear takes that path
    requires_grad(model, False)
    model.eval()
    ema.eval()
    g = torch.Generator().manual_seed(11)
    x = (torch.rand(2, 3, 256, 256, generator=g) * 2 - 1).cuda()
    with torch.no_grad():
        rec_m = model.img_to_reconstructed_img(x)
        rec_e = ema.img_to_reconstructed_img(x)
        assert torch.equal(rec_m, rec_e)
        toks_m, toks_e = model.img_to_idxBl(x), ema.img_to_idxBl(x)
        flat = lambda t: [u for v in t for u in (flat(v) if isinstance(v, (list, tuple)) else [v])]
        assert all(torch.equal(a, b) for a, b in zip(flat(toks_m), flat(toks_e)))
        assert torch.equal(ema.decode_tokens(toks_e), model.decode_tokens(toks_m))
    path = tmp_path / "ckpt.pt"
    torch.save({"ema": ema.state_dict()}, path)
    restored = copy.deepcopy(model)
    add_noise(restored, 8)
    restored.load_state_dict(torch.load(path, map_location="cuda")["ema"])
    sd = ema.state_dict()
    assert list(restored.state_dict()) == list(sd)
    for k, v in restored.state_dict().items():
        assert same_bits(v, sd[k]) if v.dtype == torch.float32 else torch.equal(v, sd[k]), k
