"""wgmma attention kernels (vit_ops.attn_tc_forward / attn_tc_backward) against the fp64 reference, element by element,
with the per-element budgets of tests/attn_budget.py (calibrated on the CPU by test_attn_budget_cpu.py), in bf16 and f16:
  * every length class of the kernels (ragged query tiles, the prep kernel's 1-4 trailing keys, multi-block rows) on every
    constructed input family, with the named mutants evaluated on the same inputs and rejected where they apply;
  * the training shapes (B, N, H) = (128, 513, 12), (128, 499, 12), (128, 379, 12), (64, 769, 12) on Gaussian and `neg`
    inputs, and a backward of many waves with N mod 128 = 1;
  * O, L2, dK and dV bitwise repeatable (one writer per element, fixed summation order); dQ and the qkv-bias gradient,
    which go through fp32 atomics, against the budget only.
Each case prints its largest error / budget ratio per output (pytest -s)."""
import pytest
import torch

import attn_budget as ab

pytestmark = pytest.mark.gpu

NS = [1, 2, 63, 64, 65, 127, 128, 129, 130, 131, 132, 133, 191, 192, 193, 257, 385, 513, 514]
DTYPES = [torch.bfloat16, torch.float16]
TRAIN = [(128, 513, 12), (128, 499, 12), (128, 379, 12), (64, 769, 12)]


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _check(family, B, N, H, dtype, seed, mutants=True):
    from imagefolder_b200 import vit_ops
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    qkv, g = ab.make_inputs(family, B, N, H, dtype, seed, device="cuda")
    out, lse2 = vit_ops.attn_tc_forward(qkv, H)
    dqkv, db = vit_ops.attn_tc_backward(qkv, out, lse2, g, H, want_bias_grad=True)
    out2, lse22 = vit_ops.attn_tc_forward(qkv, H)
    dqkv2 = vit_ops.attn_tc_backward(qkv, out, lse2, g, H)
    torch.cuda.synchronize()
    assert torch.equal(_bits(out), _bits(out2)) and torch.equal(_bits(lse2), _bits(lse22)), "forward not repeatable"
    d1, d2 = dqkv.view(B, N, 3, -1), dqkv2.view(B, N, 3, -1)
    assert torch.equal(_bits(d1[:, :, 1:]), _bits(d2[:, :, 1:])), "dK / dV not repeatable"
    del out2, lse22, dqkv2, d1, d2

    kout = ab.kernel_outputs(out, lse2, dqkv, H)
    cands = {"kernel": lambda c: {k: t[c.sl] for k, t in kout.items()}}
    if mutants:
        cands["control"] = ab.control
        for name, fn in ab.MUTANTS.items():
            fam, applies = ab.MUTANT_FAMILY[name]
            if fam == family and applies(N):
                cands[name] = fn
    res, cs_ref, cs_bud = ab.evaluate(qkv, g, H, cands, colsums=True)
    # qkv-bias gradient: fp32 column sums of the rounded packed gradient, against the reference's column sums
    absum = dqkv.double().abs().sum((0, 1)).view(3, H, 64)
    tol = cs_bud + (B * N + 64) * 2.0 ** -23 * absum
    bias_ratio = ((db.double().view(3, H, 64) - cs_ref).abs() / tol).nan_to_num(nan=float("inf")).max().item()
    peak_gib = (torch.cuda.max_memory_allocated() - base) / 2 ** 30

    k = res.pop("kernel")
    print(f"\n{family:9s} {str(dtype)[6:]:8s} B={B} N={N} H={H}: kernel " +
          " ".join(f"{o} {k[o]:.3f}" for o in ab.OUTS) + f" bias {bias_ratio:.3f}" + f" ({peak_gib:.2f} GiB)" +
          "".join(f" | {n} {max(d.values()):.3g}" for n, d in res.items() if d))
    for o in ab.OUTS:
        assert k[o] <= 1.0, f"{o}: error {k[o]:.3f} of the budget"
    assert bias_ratio <= 1.0, f"qkv-bias gradient: error {bias_ratio:.3f} of the budget"
    assert peak_gib < 8.0, f"{peak_gib:.2f} GiB of device memory"
    if mutants:
        assert max(res["control"].values()) <= 1.0, "the control mutant exceeds the budget"
        for name, d in res.items():
            if name != "control":
                assert max(d.values()) > 1.0, f"mutant {name} passes the budget on {family}"


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f16"])
@pytest.mark.parametrize("family", ab.FAMILIES)
@pytest.mark.parametrize("N", NS)
def test_attention_every_length_class_within_fp64_budget(N, family, dtype):
    _check(family, 2, N, 3, dtype, 100 * N + ab.FAMILIES.index(family) + (50 if dtype == torch.float16 else 0))


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f16"])
@pytest.mark.parametrize("family", ["gauss1", "neg"])
@pytest.mark.parametrize("B,N,H", TRAIN)
def test_attention_training_shapes_within_fp64_budget(B, N, H, family, dtype):
    _check(family, B, N, H, dtype, 7 * N + (1 if family == "neg" else 0), mutants=False)


@pytest.mark.parametrize("family", ["gauss2.5", "tail"])
def test_attention_many_wave_backward_with_one_trailing_key(family):
    # 385 = 3 x 128 + 1: three tensor-core key blocks per (batch, head) -> 3 x 192 CTAs over 132 SMs, plus the prep
    # kernel's trailing key; the dQ atomics of one (batch, head) come from CTAs of different waves
    _check(family, 16, 385, 12, torch.bfloat16, 11, mutants=family == "tail")
