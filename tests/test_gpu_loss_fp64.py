"""The LPIPS stage and DiffAug kernels (imagefolder_b200/csrc/loss_kernels.cu) against the fp64 references of
tests/loss_budget.py, with its per-image (LPIPS value) and per-element budgets (calibrated on the CPU by
test_loss_budget_cpu.py), through loss_ops and once through the C ABI:
  * LPIPS: the five VGG stages at 256x256 at batch 128 (bf16 under autocast on `indep` and `sparse`, fp32 on `indep`);
    every input family at a small batch on the stage shapes and on ragged ones (HW not a multiple of 256 / 512, odd HW
    in bf16, which the wrapper sends to the fp32 kernel, C = 3 and C = 130); the near-identical maps next to the CPU
    model's prediction;
  * DiffAug: all seven flag sets at 128 x 3 x 256 x 256 on the `edges` family and on (255, 257), (30, 30), (12, 20)
    with C in {1, 3, 8}; flag sets without colour exactly equal to the reference, cut cells exactly 0; every parameter
    decision within 4 ulps of a bin boundary equal to the reference's;
  * forward, backward (and the per-sample sums) bitwise repeatable.
Each case prints its largest error / budget ratio per output (pytest -s)."""
import contextlib

import numpy as np
import pytest
import torch

import loss_budget as lb

pytestmark = pytest.mark.gpu

STAGES = [(64, 256, 256), (128, 128, 128), (256, 64, 64), (512, 32, 32), (512, 16, 16)]
RAGGED = [(64, 14, 14), (64, 37, 29), (3, 20, 26), (130, 37, 29), (130, 9, 12)]
MEM_GIB = 12.0


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _same_bits(a, b):
    return torch.equal(_bits(a), _bits(b))


# ---- LPIPS -----------------------------------------------------------------------------------------------------------
def _lpips_run(f0, f1, w, g, autocast):
    from imagefolder_b200.loss_ops import lpips_stage
    a, b = f0.detach().requires_grad_(True), f1.detach().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16) if autocast else contextlib.nullcontext():
        val = lpips_stage(a, b, w.view(1, -1, 1, 1))
    g0, g1 = torch.autograd.grad(val, (a, b), g)
    return val.detach(), g0, g1


def _lpips_case(family, B, C, H, W, dtype, seed, autocast=False):
    f0, f1, w, g = lb.lpips_inputs(family, B, C, H, W, dtype, seed, device="cuda")
    val, g0, g1 = _lpips_run(f0, f1, w, g, autocast)
    assert g0.dtype == dtype and g1.dtype == dtype
    again = _lpips_run(f0, f1, w, g, autocast)
    torch.cuda.synchronize()
    assert all(_same_bits(x, y) for x, y in zip((val, g0, g1), again)), "LPIPS stage not bitwise repeatable"
    del again
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    rel = {}
    res = lb.lpips_evaluate(f0, f1, w, g, {"kernel": {"val": val, "g0": g0, "g1": g1}}, chunk_elems=2 ** 24,
                            report=rel)["kernel"]
    peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
    print(f"\nlpips {family:8s} {str(dtype)[6:]:8s} B={B} C={C} {H}x{W}{' autocast' if autocast else ''}: " +
          " ".join(f"{o} {res[o]:.3g}" for o in lb.LP_OUTS) + f"  (val rel. err. {rel['kernel']:.2e}, {peak:.2f} GiB)")
    for o in lb.LP_OUTS:
        assert res[o] <= 1.0, f"{o}: error {res[o]:.3f} of the budget"
    assert peak < MEM_GIB, f"{peak:.2f} GiB of extra device memory for the fp64 reference"
    return res, peak


@pytest.mark.parametrize("family,dtype", [("indep", torch.bfloat16), ("sparse", torch.bfloat16),
                                          ("indep", torch.float32)], ids=["indep-bf16", "sparse-bf16", "indep-fp32"])
def test_lpips_five_vgg_stages_at_batch_128(family, dtype):
    for i, (C, H, W) in enumerate(STAGES):
        _lpips_case(family, 128, C, H, W, dtype, 1000 + 10 * i, autocast=dtype == torch.bfloat16)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("family", lb.LP_FAMILIES)
def test_lpips_every_family_on_stage_and_ragged_shapes(family, dtype):
    for i, (C, H, W) in enumerate(STAGES + RAGGED):
        _lpips_case(family, 2 + i % 3, C, H, W, dtype, 100 * i + lb.LP_FAMILIES.index(family))


def test_lpips_near_identical_maps_next_to_the_model():
    """relative error of the stage value for f1 = relu(f0 + delta n), C = 64, RMS over 16 images of 4x4 pixels (the
    CPU test's setup) and over 4 images at stage 1, kernel next to the rounding model"""
    print("\n   delta   shape            kernel rel. err.   model rel. err.   kernel / budget")
    for shp in [(16, 64, 4, 4), (4, 64, 256, 256)]:
        for delta in (1e-1, 1e-2, 3e-3, 1e-3, 1e-4):
            g = torch.Generator(device="cuda").manual_seed(0)
            f0 = torch.relu(torch.randn(shp, generator=g, device="cuda"))
            f1 = torch.relu(f0 + delta * torch.randn(shp, generator=g, device="cuda"))
            w = torch.rand(64, generator=g, device="cuda") * 0.1
            go = torch.ones(shp[0], device="cuda")
            val, g0, g1 = _lpips_run(f0, f1, w, go, False)
            ref = lb.lpips_reference(f0, f1, w, go)["val"]
            mval = lb.lpips_model(f0, f1, w, go)["val"].cuda() if shp[2] == 4 else None
            res = lb.lpips_evaluate(f0, f1, w, go, {"kernel": {"val": val, "g0": g0, "g1": g1}})["kernel"]

            def rms(v):
                return float((((v.double() - ref) / ref) ** 2).mean().sqrt())
            print(f"   {delta:7.0e}   {str(shp):16s} {rms(val):16.2e}   " +
                  (f"{rms(mval):15.2e}" if mval is not None else f"{'-':>15s}") +
                  "   " + " ".join(f"{o} {res[o]:.3g}" for o in lb.LP_OUTS))
            for o in lb.LP_OUTS:
                assert res[o] <= 1.0, f"delta {delta} {shp}: {o} error {res[o]:.3f} of the budget"


def test_lpips_c_abi_matches_loss_ops():
    from imagefolder_b200 import _capi as C
    L = C.lib()
    for dtype in (torch.bfloat16, torch.float32):
        B, Cc, H, W = 4, 256, 64, 64
        f0, f1, w, g = lb.lpips_inputs("indep", B, Cc, H, W, dtype, 7, device="cuda")
        val, g0, g1 = _lpips_run(f0, f1, w, g, False)
        out = torch.empty(B, device="cuda")
        ws = C.workspace(L.xq_lpips_workspace_bytes(B, H * W), f0.device)
        st = C.stream_ptr(f0.device)
        bf = int(dtype == torch.bfloat16)
        assert L.xq_lpips_layer_forward(C.ptr(f0), C.ptr(f1), bf, C.ptr(w), B, Cc, H * W, lb.EPS, 0, C.ptr(out),
                                        C.ptr(ws), ws.numel(), st) == 0
        c0, c1 = torch.empty_like(f0), torch.empty_like(f1)
        assert L.xq_lpips_layer_backward(C.ptr(f1), C.ptr(f0), bf, C.ptr(w), B, Cc, H * W, lb.EPS, C.ptr(g), C.ptr(c0),
                                         st) == 0
        assert L.xq_lpips_layer_backward(C.ptr(f0), C.ptr(f1), bf, C.ptr(w), B, Cc, H * W, lb.EPS, C.ptr(g), C.ptr(c1),
                                         st) == 0
        torch.cuda.synchronize()
        assert _same_bits(out, val) and _same_bits(c0, g0) and _same_bits(c1, g1)
        res = lb.lpips_evaluate(f0, f1, w, g, {"abi": {"val": out, "g0": c0, "g1": c1}})["abi"]
        print(f"\nlpips C ABI {str(dtype)[6:]}: " + " ".join(f"{o} {res[o]:.3g}" for o in lb.LP_OUTS))
        assert max(res.values()) <= 1.0


# ---- DiffAug ---------------------------------------------------------------------------------------------------------
def _aug_run(x, r01, flags, g):
    from imagefolder_b200.loss_ops import diffaug_apply
    B, C, H, W = x.shape
    ch, cw = lb.cut_size(H, W)
    xs = x.detach().requires_grad_(True)
    y = diffaug_apply(xs, r01, flags, ch, cw)
    (gx,) = torch.autograd.grad(y, xs, g)
    return y.detach(), gx


def _aug_case(B, C, H, W, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand(B, C, H, W, generator=gen, device="cuda") * 2 - 1
    g = torch.randn(B, C, H, W, generator=gen, device="cuda")
    r01 = lb.edges_rand01(B, H, W, seed)
    rd = torch.from_numpy(r01).cuda()
    worst = {}
    for flags in range(1, 8):
        y, gx = _aug_run(x, rd, flags, g)
        y2, gx2 = _aug_run(x, rd, flags, g)
        torch.cuda.synchronize()
        assert _same_bits(y, y2) and _same_bits(gx, gx2), f"flags={flags}: not bitwise repeatable"
        del y2, gx2
        yr, gxr = lb.diffaug_reference(x, g, r01, flags)
        by, bg = lb.diffaug_budget(x, g, r01, flags)
        if flags & 4:
            p = lb.aug_params(r01, flags, H, W, "cuda")
            cut = (lb.cut_mask(p, H, W, "cuda") == 0).expand_as(y)
            assert bool((y[cut] == 0).all()), f"flags={flags}: a cut cell is not 0"
        if not flags & 2:                                   # pure copies (torch.equal: br = 0 turns -0 into +0)
            assert torch.equal(y.double(), yr), f"flags={flags}: forward is not an exact copy"
            assert torch.equal(gx.double(), gxr), f"flags={flags}: backward is not an exact copy"
        ry, rg = lb.ratio(y, yr, by), lb.ratio(gx, gxr, bg)
        worst[flags] = (ry, rg)
        assert ry <= 1.0 and rg <= 1.0, f"flags={flags}: y {ry:.3f} gx {rg:.3f} of the budget"
        del yr, gxr, by, bg
    print(f"\ndiffaug edges B={B} C={C} {H}x{W}: " + " ".join(f"[{f}] y {a:.3g} gx {b:.3g}" for f, (a, b) in worst.items()))


def test_diffaug_every_flag_set_at_training_batch():
    _aug_case(128, 3, 256, 256, 1)


@pytest.mark.parametrize("C", [1, 3, 8])
@pytest.mark.parametrize("H,W", [(255, 257), (30, 30), (12, 20)])
def test_diffaug_every_flag_set_on_odd_shapes(H, W, C):
    _aug_case(25, C, H, W, 10 * H + W + C)


def test_diffaug_c_abi_and_per_sample_sums():
    from imagefolder_b200 import _capi as C
    L = C.lib()
    B, Cc, H, W = 128, 3, 256, 256
    gen = torch.Generator(device="cuda").manual_seed(3)
    x = torch.rand(B, Cc, H, W, generator=gen, device="cuda") * 2 - 1
    g = torch.randn(B, Cc, H, W, generator=gen, device="cuda")
    r01 = lb.edges_rand01(B, H, W, 3)
    rd = torch.from_numpy(r01).cuda()
    ch, cw = lb.cut_size(H, W)
    st = C.stream_ptr(x.device)
    y_ops, gx_ops = _aug_run(x, rd, 7, g)
    outs = []
    for _ in range(2):
        y, gx = torch.empty_like(x), torch.empty_like(x)
        s_f, s_b = torch.empty(B, device="cuda"), torch.empty(B, device="cuda")
        assert L.xq_diffaug_forward(C.ptr(x), C.ptr(rd), B, Cc, H, W, 7, ch, cw, C.ptr(y), C.ptr(s_f), st) == 0
        assert L.xq_diffaug_backward(C.ptr(g), C.ptr(rd), B, Cc, H, W, 7, ch, cw, C.ptr(gx), C.ptr(s_b), st) == 0
        outs.append((y, gx, s_f, s_b))
    torch.cuda.synchronize()
    assert all(_same_bits(a, b) for a, b in zip(*outs)), "C ABI DiffAug not bitwise repeatable"
    y, gx, s_f, s_b = outs[0]
    assert _same_bits(y, y_ops) and _same_bits(gx, gx_ops)
    # the sums: the translated image (forward) and the masked upstream gradient (backward), fp64-accumulated
    p = lb.aug_params(r01, 7, H, W, "cuda")
    want_f = lb.translate(x.double(), p["th"], p["tw"]).sum((1, 2, 3))
    want_b = (g.double() * lb.cut_mask(p, H, W, "cuda")).sum((1, 2, 3))
    for got, want, mag in ((s_f, want_f, x.double().abs().sum((1, 2, 3))), (s_b, want_b, g.double().abs().sum((1, 2, 3)))):
        r = float(((got.double() - want).abs() / (lb.U * want.abs() + 2.0 ** -50 * mag)).max())
        assert r <= 1.0, f"per-sample sum: {r:.3f} of one fp32 rounding"


def _decisions(H, W, r, flags):
    """run the kernel on an image that encodes the decision of `flags` and return (kernel output, reference output)"""
    from imagefolder_b200.loss_ops import diffaug_apply
    B = r.shape[0]
    r01 = np.stack([r] * 7).astype(np.float32)
    ch, cw = lb.cut_size(H, W)
    if flags == 1:                                          # x[h, w] = h W + w + 1: the output names its source pixel
        x = (torch.arange(H * W, device="cuda", dtype=torch.float32) + 1).view(1, 1, H, W).expand(B, 1, H, W)
    else:                                                   # all ones: the zeros are the cutout
        x = torch.ones(B, 1, H, W, device="cuda")
    x = x.contiguous()
    y = diffaug_apply(x, torch.from_numpy(r01).cuda(), flags, ch, cw)
    yr, _ = lb.diffaug_reference(x, torch.zeros_like(x), r01, flags)
    return y, yr, lb.aug_params(r01, flags, H, W, "cuda")


@pytest.mark.parametrize("H,W", [(256, 256), (30, 30), (255, 257)])
def test_diffaug_parameter_decisions_at_every_bin_boundary(H, W):
    dh, dw = round(H * 0.125), round(W * 0.125)
    ch, cw = lb.cut_size(H, W)
    # translation: th, tw from the source coordinate the centre output pixel reads
    r = np.union1d(lb.boundary_r(2 * dh + 1), lb.boundary_r(2 * dw + 1))
    nt = len(r)
    y, yr, p = _decisions(H, W, r, 1)
    src = y[:, 0, H // 2, W // 2].long() - 1
    assert torch.equal(src // W - H // 2, p["th"]) and torch.equal(src % W - W // 2, p["tw"])
    assert torch.equal(y.double(), yr)
    # cutout offsets: the zero pattern of an all-ones image
    r = np.union1d(lb.boundary_r(H + 1 - ch % 2), lb.boundary_r(W + 1 - cw % 2))
    y, yr, p = _decisions(H, W, r, 4)
    assert torch.equal(y == 0, yr == 0), "cutout rectangles differ from the reference's"
    print(f"\ndiffaug decisions {H}x{W}: {nt} translation and {len(r)} cutout offsets equal")
