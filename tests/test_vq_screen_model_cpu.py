"""The CPU model of the tensor-core VQ search's screening (tests/vq_screen_model.py) on the adversarial families:
with the kernel's constants it returns the oracle's index on every family; each family reaches the branch it was
built for on a stated share of its rows; and each safeguard, turned off, gives a wrong index on its family."""
import numpy as np
import pytest

import vq_screen_model as m

N = 512
# (family, V, C): the shapes the GPU tests use for the tensor-core path
SHAPES = [("F1", 300, 32), ("F1", 1000, 32), ("F1", 4096, 64), ("F2", 1000, 32), ("F2", 4096, 64),
          ("F3", 4096, 32), ("F3", 8192, 64), ("F4", 300, 32), ("F4", 4096, 64), ("F5", 300, 64), ("F5", 4096, 32),
          ("F6", 5, 32), ("F6", 33, 32), ("F6", 129, 64), ("F6", 300, 32), ("F6", 1000, 64), ("F7", 33, 32),
          ("F7", 1000, 32), ("F7", 4096, 64)]

_cache = {}


def _case(fam, V, C):
    key = (fam, V, C)
    if key not in _cache:
        z, E = m.FAMILIES[fam](V, C, N)
        _cache[key] = (z, E, m.oracle_idx(z, E))
    return _cache[key]


@pytest.mark.parametrize("fam,V,C", SHAPES)
@pytest.mark.parametrize("design", ["flag", "fold"])
def test_model_with_kernel_constants_returns_oracle_index(fam, V, C, design):
    """'flag' is the kernel (unit-norm scores, full scan after the degenerate-codebook flag); 'fold' scores every code
    with dot - ee/2 instead and is exact on its own."""
    z, E, ref = _case(fam, V, C)
    kw = {} if design == "flag" else dict(fold_ee=True, ee_flag=False)
    idx = m.screen(z, E, **kw)[0]
    np.testing.assert_array_equal(idx, ref)


# share of rows on the branch each family targets (the observed shares are higher; see the builders' docstrings)
@pytest.mark.parametrize("fam,V,C,what,share", [
    ("F1", 300, 32, "overflow", 1.0), ("F1", 4096, 64, "overflow", 1.0),     # the degenerate-codebook flag
    ("F2", 1000, 32, "overflow", 0.99), ("F2", 4096, 64, "overflow", 0.99),
    ("F3", 4096, 32, "compacted", 0.3), ("F3", 4096, 32, "overflow", 0.3),
    ("F4", 300, 32, "multi", 0.99), ("F4", 4096, 64, "multi", 0.99),
    ("F5", 300, 64, "rescored", 0.99), ("F5", 4096, 32, "rescored", 0.99),
])
def test_family_reaches_its_branch(fam, V, C, what, share):
    z, E, _ = _case(fam, V, C)
    _, path, compacted, multi = m.screen(z, E)
    got = {"rescored": path == m.RESCORED, "overflow": path == m.OVERFLOW, "compacted": compacted, "multi": multi}[what]
    assert float(got.mean()) >= share, f"{fam}: {what} on {float(got.mean()):.3f} of the rows"


def test_zero_codes_win_rows_whose_best_dot_is_below_half():
    """F1's premise: the oracle picks a zero / tiny code for a large share of the rows at small V."""
    z, E, ref = _case("F1", 300, 32)
    special = np.nonzero(np.linalg.norm(E, axis=1) < 1e-12)[0]
    assert float(np.isin(ref, special).mean()) > 0.3


# each mutant with the family it must fail on (index differs from the oracle's on at least `min_bad` rows)
@pytest.mark.parametrize("fam,V,C,kw,min_bad", [
    # neither the flag nor the fold: the kernel before this check
    ("F1", 300, 32, dict(ee_flag=False), 50), ("F1", 1000, 32, dict(ee_flag=False), 50),
    ("F1", 4096, 64, dict(ee_flag=False), 50),
    ("F6", 33, 32, dict(mask_padding=False), 50), ("F6", 129, 64, dict(mask_padding=False), 50),
    ("F6", 300, 32, dict(mask_padding=False), 50),
    ("F2", 1000, 32, dict(honour_overflow=False), 50), ("F2", 4096, 64, dict(honour_overflow=False), 50),
    ("F3", 4096, 32, dict(honour_overflow=False), 50),
    ("F4", 300, 32, dict(check_multi=False), 100), ("F4", 4096, 64, dict(check_multi=False), 100),
    # F5's reversal is ~0.96e-3 (see f5_worst_truncation), so W = 0.8e-3 drops the true argmin
    ("F5", 300, 64, dict(W=0.8e-3), 100), ("F5", 4096, 32, dict(W=0.8e-3), 100),
])
def test_mutant_fails_on_its_family(fam, V, C, kw, min_bad):
    z, E, ref = _case(fam, V, C)
    bad = int((m.screen(z, E, **kw)[0] != ref).sum())
    assert bad >= min_bad, f"mutant {kw} on {fam}: only {bad} wrong rows"


def test_fold_alone_handles_zero_codes_and_padding():
    """The alternative design: with s = dot - ee/2 neither the flag nor the padding mask is needed on F1 / F6, and
    F1 rows reach the rescoring on their own (the zero and tiny codes sit at 0 and 31 of one group)."""
    for fam, V, C in (("F1", 300, 32), ("F1", 4096, 64), ("F6", 33, 32), ("F6", 300, 32)):
        z, E, ref = _case(fam, V, C)
        idx, path, _, _ = m.screen(z, E, fold_ee=True, ee_flag=False, mask_padding=False)
        np.testing.assert_array_equal(idx, ref)
        if fam == "F1":
            assert float((path == m.RESCORED).mean()) > 0.2


def test_reversal_designs_are_exact_and_reversed():
    """F4 / F5 designs: z, A, B normalise to themselves; TF32 ranks A above B while B has the larger true dot."""
    rng = np.random.default_rng(0)
    for C in (32, 64):
        for _ in range(8):
            z, A, B = m._reversal_design(rng, C)
            X = np.stack([z, A, B])
            np.testing.assert_array_equal(m.normalise(X), X)
            t = m.tf32(X).astype(np.float64)
            true_gap = float(z.astype(np.float64) @ B - z.astype(np.float64) @ A)
            rev = float(t[0] @ t[1] - t[0] @ t[2])
            assert 0 < true_gap < 2.0 ** -9
            assert rev - true_gap > 0.9e-3
