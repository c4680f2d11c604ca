"""The attention budgets (tests/attn_budget.py) checked on the CPU, before any kernel is measured against them:
  * an exact model of the kernels' rounding sequence stays within half of every budget, on every input family, in
    bf16 and f16, at every length class of the kernels (ragged query tiles, 1-4 trailing keys, multi-block rows);
  * each named mutant (a plausible kernel bug, in fp64) exceeds the budget on the family built for it, and the
    control (delta from the fp64 O) does not;
  * the max-normalised criterion of test_gpu_attn.py accepts a leaked padding key on Gaussian inputs: the gap these
    budgets close."""
import pytest
import torch

import attn_budget as ab

NS = [1, 2, 63, 64, 65, 127, 128, 129, 130, 131, 132, 133, 191, 192, 193, 257, 385, 513, 514]
DTYPES = [torch.bfloat16, torch.float16]


def _seed(family, N, dtype):
    return 1000 * ab.FAMILIES.index(family) + N + (7 if dtype == torch.float16 else 0)


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f16"])
@pytest.mark.parametrize("family", ab.FAMILIES)
def test_emulated_kernel_within_half_budget(family, dtype):
    worst = {}
    for N in NS:
        qkv, g = ab.make_inputs(family, 1, N, 2, dtype, _seed(family, N, dtype))
        res = ab.evaluate(qkv, g, 2, {"emulated": ab.emulated, "control": ab.control})
        for name, d in res.items():
            for out, ratio in d.items():
                assert ratio <= (0.5 if name == "emulated" else 1.0), f"{name} {out} N={N}: {ratio:.3f} of the budget"
                worst[name, out] = max(worst.get((name, out), 0.0), ratio)
    print(f"\n{family} {dtype}: " + "  ".join(f"{n}.{o} {r:.3f}" for (n, o), r in sorted(worst.items())))


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f16"])
@pytest.mark.parametrize("mutant", sorted(ab.MUTANTS))
def test_mutant_rejected_on_its_family(mutant, dtype):
    family, applies = ab.MUTANT_FAMILY[mutant]
    lows = []
    for N in NS:
        if not applies(N):
            continue
        qkv, g = ab.make_inputs(family, 1, N, 2, dtype, _seed(family, N, dtype))
        res = ab.evaluate(qkv, g, 2, {mutant: ab.MUTANTS[mutant]})[mutant]
        worst = max(res.values())
        assert worst > 1.0, f"{mutant} passes the budget on {family} at N={N} ({worst:.3f})"
        lows.append((worst, N))
    assert lows
    print(f"\n{mutant} on {family} {dtype}: smallest max error/budget {min(lows)[0]:.3g} (N={min(lows)[1]})")


def test_ktail_matches_the_backward_launch_rule():
    # attn_bwd_ktail: N mod 128 in 1..4 with N > 128 goes to the prep kernel
    assert [N for N in range(1, 700) if ab.ktail(N)] == [n for b in (128, 256, 384, 512, 640) for n in range(b + 1, b + 5)]


def test_neg_family_makes_a_padding_key_dominant():
    qkv, g = ab.make_inputs("neg", 1, 513, 2, torch.bfloat16, 3)
    q, k, _ = ab.pairs(qkv, 2)
    s = (q.double() @ k.double().mT) * ab.SCALE
    assert s.max().item() <= -12.0
    # the weight a zero-filled key (score 0) would take from every row
    assert (1.0 / (1.0 + s.exp().sum(-1))).min().item() > 0.99


@pytest.mark.parametrize("family", ["max_last", "max_first"])
def test_max_families_put_the_row_maximum_in_the_chosen_block(family):
    N = 385
    qkv, g = ab.make_inputs(family, 2, N, 2, torch.float16, 5)
    q, k, _ = ab.pairs(qkv, 2)
    s = (q.double() @ k.double().mT) * ab.SCALE
    top = s.topk(2, -1)
    assert (top.values[..., 0] - top.values[..., 1]).min().item() >= 20.0
    blk = top.indices[..., 0] // ab.BK
    assert (blk == ((N - 1) // ab.BK if family == "max_last" else 0)).all()


def test_tail_family_moves_weight_to_the_trailing_keys():
    N = 513
    qkv, g = ab.make_inputs("tail", 1, N, 2, torch.bfloat16, 9)
    q, k, v = ab.pairs(qkv, 2)
    r = ab.reference(q.double(), k.double(), v.double(), ab.heads(g, 2).double())
    w = r["P"][..., N - ab.ktail(N):].sum(-1)
    assert w[:, ::2].mean().item() > 0.5                 # captured queries put most of their weight on the trailing key
    # and those keys carry O(1) of the dK / dQ gradient
    assert r["dK"][:, -1].abs().max().item() > 0.5 * r["dK"].abs().max().item()


def test_max_normalised_criterion_accepts_a_leaked_padding_key():
    """test_gpu_attn.py's forward check (8e-3 of max |O|) on its own Gaussian inputs at B = 2, N = 513, H = 3 cannot see
    one zero-filled key let into the softmax; the per-element budget on the `neg` family does (above)."""
    torch.manual_seed(0)
    for amp in (1.0, 2.5):
        qkv = (torch.randn(2, 513, 3 * 3 * 64) * amp).to(torch.bfloat16)
        g = torch.randn(2, 513, 3 * 64).to(torch.bfloat16)
        q, k, v = (t.double() for t in ab.pairs(qkv, 3))
        dO = ab.heads(g, 3).double()
        ref = ab.reference(q, k, v, dO)
        ctx = ab.Ctx(slice(None), q, k, v, dO, ref, qkv.dtype)
        leak = ab.mut_leaked_key(ctx)
        err = (leak["O"] - ref["O"]).abs().max().item()
        assert 0 < err <= 8e-3 * max(1.0, ref["O"].abs().max().item())
