"""The fp64 references, budgets, rounding model and mutants of tests/loss_budget.py, on the CPU:
  * the references reproduce the reference's own outputs in tests/golden/loss_stack.npz;
  * the rounding model of the kernels stays within half of every budget on every input family, and so does the control
    (the exact values rounded once to the output type);
  * every named mutant exceeds its budget on the family built for it;
  * the model reproduces the near-identical-maps estimate of the LPIPS value's relative error (printed with -s)."""
import numpy as np
import pytest
import torch

import loss_budget as lb
from conftest import load_golden

LP_SHAPES = [(2, 64, 16, 20), (2, 130, 6, 10), (3, 3, 9, 7)]
AUG_SHAPES = [(25, 3, 30, 30), (25, 1, 12, 20), (9, 8, 17, 23)]


def test_references_reproduce_the_reference_goldens():
    g = load_golden("loss_stack")
    for li in range(3):
        f0, f1, w, go = (torch.from_numpy(g[f"lp{li}_{k}"]) for k in ("f0", "f1", "w", "g"))
        r = lb.lpips_reference(f0, f1, w, go)
        np.testing.assert_allclose(r["val"].numpy(), g[f"lp{li}_val"], rtol=2e-5, atol=1e-7)
        np.testing.assert_allclose(r["g1"].numpy(), g[f"lp{li}_gf1"], rtol=2e-4, atol=1e-7)
    for ci in g["aug_cases"]:
        f3 = [int(f) for f in g[f"aug{ci}_flags"]]
        flags = f3[0] | (f3[1] << 1) | (f3[2] << 2)
        x, gy = torch.from_numpy(g[f"aug{ci}_x"]), torch.from_numpy(g[f"aug{ci}_g"])
        y, gx = lb.diffaug_reference(x, gy, g[f"aug{ci}_rand01"], flags)
        np.testing.assert_allclose(y.numpy(), g[f"aug{ci}_y"], rtol=1e-5, atol=2e-6)
        np.testing.assert_allclose(gx.numpy(), g[f"aug{ci}_gx"], rtol=1e-5, atol=2e-6)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("family", lb.LP_FAMILIES)
def test_lpips_model_and_control_within_half_budget(family, dtype):
    for i, shp in enumerate(LP_SHAPES):
        f0, f1, w, g = lb.lpips_inputs(family, *shp, dtype, 10 * i + lb.LP_FAMILIES.index(family))
        bf16 = dtype == torch.bfloat16 and (shp[2] * shp[3]) % 2 == 0
        res = lb.lpips_evaluate(f0, f1, w, g, {"model": lb.lpips_model(f0, f1, w, g),
                                               "control": lambda sl, ref: lb.lpips_control(sl, ref, bf16)})
        for name, d in res.items():
            for o, r in d.items():
                assert r <= 0.5, f"{name} {o} at {shp}: {r:.3f} of the budget"


@pytest.mark.parametrize("mutant", lb.LP_MUTANTS)
def test_lpips_mutant_exceeds_budget(mutant):
    family, dtype, shp = lb.LP_MUTANT_CASE[mutant]
    f0, f1, w, g = lb.lpips_inputs(family, *shp, dtype, 5)
    res = lb.lpips_evaluate(f0, f1, w, g, {mutant: lb.lpips_model(f0, f1, w, g, mutant=mutant)})[mutant]
    assert max(res.values()) > 1.0, f"mutant {mutant} passes the budget on {family}: {res}"


@pytest.mark.parametrize("shape", AUG_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_diffaug_model_control_and_mutants(shape):
    B, C, H, W = shape
    gen = torch.Generator().manual_seed(B + C + H)
    x = torch.rand(shape, generator=gen) * 2 - 1
    g = torch.randn(shape, generator=gen)
    r01 = lb.edges_rand01(B, H, W, H * W)
    for flags in range(1, 8):
        y, gx = lb.diffaug_reference(x, g, r01, flags)
        by, bg = lb.diffaug_budget(x, g, r01, flags)
        my, mg = lb.diffaug_model(x, g, r01, flags)
        for name, a, b in (("model", my, mg), ("control", y.float(), gx.float())):
            ry, rg = lb.ratio(a, y, by), lb.ratio(b, gx, bg)
            assert ry <= 0.5 and rg <= 0.5, f"{name} flags={flags}: y {ry:.3f} gx {rg:.3f} of the budget"
        for mutant, need in lb.AUG_MUTANT_FLAGS.items():
            if flags & need == need:
                a, b = lb.diffaug_model(x, g, r01, flags, mutant=mutant)
                assert max(lb.ratio(a, y, by), lb.ratio(b, gx, bg)) > 1.0, f"mutant {mutant} passes with flags={flags}"


def test_edges_family_covers_every_edge_case():
    for (H, W) in [(256, 256), (30, 30), (12, 20), (255, 257)]:
        r01 = lb.edges_rand01(25, H, W, 0)
        p = lb.aug_params(r01, 7, H, W)
        dh, dw = round(H * 0.125), round(W * 0.125)
        assert {(int(a), int(b)) for a, b in zip(p["th"], p["tw"])} == \
            {(a, b) for a in (-dh, -1, 0, 1, dh) for b in (-dw, -1, 0, 1, dw)}
        ch, cw = p["ch"], p["cw"]
        top, bottom = p["oh"] - ch // 2 < 0, p["oh"] - ch // 2 + ch > H
        left, right = p["ow"] - cw // 2 < 0, p["ow"] - cw // 2 + cw > W
        for vh in (top, bottom, ~top & ~bottom):
            for vw in (left, right, ~left & ~right):
                assert bool((vh & vw).any())
        if ch % 2 == 0:
            assert int(p["oh"].max()) == H                   # an even cutout centred one past the last row
        assert float(p["sat"].min()) == 0 and float(p["sat"].max()) > 1.99
        assert float(p["con"].min()) == 0.5 and float(p["con"].max()) > 1.49
        assert float(p["br"].min()) == -0.5 and float(p["br"].max()) > 0.4999


def test_cutout_clamping_equals_dropping_out_of_range_cells():
    """Why the cutout mutant moves the rectangle instead of dropping its out-of-range cells: for every offset the
    reference can draw (oh in [0, H + 1 - ch % 2)), the clamped index grid zeroes exactly the in-range cells of the
    rectangle, so dropping the out-of-range cells is not a different result."""
    for H in range(1, 40):
        for ch in range(1, 2 * H + 2):
            for oh in range(H + 1 - ch % 2):
                cells = np.arange(ch) + oh - ch // 2
                clamped = set(np.clip(cells, 0, H - 1).tolist())
                dropped = set(cells[(cells >= 0) & (cells < H)].tolist())
                assert clamped == dropped, (H, ch, oh)


def test_near_identical_maps_relative_error_of_the_value():
    """The model's relative error of the stage value for f1 = relu(f0 + delta n), C = 64 (RMS over 16 images of 4x4
    pixels), next to the estimate it must reproduce within 3x; it grows as delta^-2.  The model stays inside the
    budget, which carries this as its absolute floor."""
    estimate = {1e-2: 4e-5, 3e-3: 5e-4, 1e-3: 1.3e-2, 1e-4: 0.9}
    got = {}
    print("\n   delta   model rel. err.   estimate   model / budget")
    for delta, want in estimate.items():
        g = torch.Generator().manual_seed(0)
        f0 = torch.relu(torch.randn(16, 64, 4, 4, generator=g))
        f1 = torch.relu(f0 + delta * torch.randn(16, 64, 4, 4, generator=g))
        w = torch.rand(64, generator=g) * 0.1
        go = torch.ones(16)
        m = lb.lpips_model(f0, f1, w, go)
        ref = lb.lpips_reference(f0, f1, w, go)
        rel = float((((m["val"].double() - ref["val"]) / ref["val"]) ** 2).mean().sqrt())
        r = lb.lpips_evaluate(f0, f1, w, go, {"model": m})["model"]["val"]
        print(f"   {delta:7.0e}   {rel:15.2e}   {want:8.1e}   {r:.3f}")
        got[delta] = rel
        assert want / 3 <= rel <= want * 3, f"delta {delta}: {rel:.2e}, estimate {want:.1e}"
        assert r <= 0.5
    assert got[1e-4] / got[1e-2] > 1e3
