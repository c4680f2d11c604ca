"""Inputs of the 680-token multi-scale goldens (tests/golden/make_ms680_golden.py).

The codebook, Phi weights, feature map, output gradient and `dropout` are drawn from a seeded CPU generator, so the golden
files hold only the seed and the reference's outputs.  f_hat at every scale is stored on a stride-3 grid and the
idxBl_to_var_input rows at stride 4 (FHAT_SUB, VAR_SUB), which keeps each file a few hundred KB."""
import numpy as np
import torch

PN680 = [1, 2, 3, 4, 5, 6, 8, 10, 13, 16]
FHAT_SUB = (slice(None), slice(None), slice(None, None, 3), slice(None, None, 3))
VAR_SUB = (slice(None), slice(None, None, 4))


def ms680_inputs(seed, V=4096, C=32, B=2, K=4):
    """-> dict of float32 / int64 numpy arrays: E [V,C], phi_w [K,C,C,3,3], phi_b [K,C], f and g_out [B,C,16,16],
    dropout [B] (scale counts 3..10)"""
    g = torch.Generator().manual_seed(int(seed))
    H = PN680[-1]
    E = torch.randn(V, C, generator=g) * 0.5
    phi_w = torch.randn(K, C, C, 3, 3, generator=g) * 0.06
    phi_b = torch.randn(K, C, generator=g) * 0.1
    f = torch.randn(B, C, H, H, generator=g)
    g_out = torch.randn(B, C, H, H, generator=g)
    dropout = torch.randint(3, len(PN680) + 1, (B,), generator=g)
    return dict(E=E.numpy(), phi_w=phi_w.numpy(), phi_b=phi_b.numpy(), f=f.numpy(), g_out=g_out.numpy(),
                dropout=dropout.numpy().astype(np.int64))


def load680(name):
    """a 680-token golden with its inputs regenerated from the stored seed; gE made dense"""
    from conftest import load_golden
    g = load_golden(name)
    g.update(ms680_inputs(int(g["seed"]), int(g["V"]), int(g["C"]), int(g["B"]), int(g["K"])))
    gE = np.zeros_like(g["E"])
    gE[g["gE_rows"]] = g["gE_vals"]
    g["gE"] = gE
    return g
