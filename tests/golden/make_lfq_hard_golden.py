"""Golden vectors of LFQ(soft_entropy=False) made by RUNNING THE REFERENCE'S OWN MODULE (CPU, fp32).

    XQ_REFERENCE=<checkout of the reference> python tests/golden/make_lfq_hard_golden.py   # writes tests/golden/lfq_hard_*.npz

The reference materialises the [B, HW, 1, 2^C] logits of entropy_loss (lookup_free_quantize.py:220-229), so only small C
is run here.  The import recipe and stubs are make_golden.py's.  lfq_hard_b1.npz records what the reference does at
batch size 1 (the exception it raises).
"""
import os
import sys

import numpy as np
import torch

OUT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, OUT)
import make_golden as mg  # noqa: E402

MS = [1, 1, 2, 3, 3, 4, 5, 6, 8, 11]


def case_lfq_hard(LFQ, name, C, B, patch_nums, using_znorm=True, codebook_drop=0.5, seed=3, entropy_weight=0.1,
                  scale=1.0, w_sample=1.0, w_batch=1.0):
    torch.manual_seed(seed)
    H = patch_nums[-1]
    q = LFQ(2 ** C, C, using_znorm=using_znorm, v_patch_nums=patch_nums, num_latent_tokens=H * H, share_quant_resi=4,
            codebook_drop=codebook_drop, scale=scale, entropy_weight=entropy_weight, sample_minimization_weight=w_sample,
            batch_maximization_weight=w_batch, soft_entropy=False).train()
    phis = list(q.quant_resi.qresi_ls)
    f = torch.randn(B, C, H, H, requires_grad=True)
    SN = len(patch_nums)
    dropout = torch.randint(3, SN + 1, (B,))
    out, usages, vq, commit, ent = q(f, ret_usages=True, dropout=dropout)
    g_out = torch.randn_like(out)
    loss = (out * g_out).sum() + 1.3 * vq + 0.7 * commit + 1.1 * ent
    loss.backward()
    idx_list = q.f_to_idxBl_or_fhat(f.detach(), to_fhat=False, v_patch_nums=patch_nums)
    fhat_list = q.f_to_idxBl_or_fhat(f.detach(), to_fhat=True, v_patch_nums=patch_nums)
    d = dict(f=mg.npy(f), phi_w=np.stack([mg.npy(p.weight) for p in phis]), phi_b=np.stack([mg.npy(p.bias) for p in phis]),
             patch_nums=np.array(patch_nums), dropout=mg.npy(dropout), codebook_drop=codebook_drop,
             using_znorm=using_znorm, out=mg.npy(out), vq=mg.npy(vq), commit=mg.npy(commit), entropy=mg.npy(ent),
             usages=np.array(usages), g_out=mg.npy(g_out), w_vq=1.3, w_commit=0.7, w_ent=1.1, gf=mg.npy(f.grad),
             gphi_w=np.stack([mg.npy(p.weight.grad) if p.weight.grad is not None else np.zeros_like(mg.npy(p.weight))
                              for p in phis]),
             gphi_b=np.stack([mg.npy(p.bias.grad) if p.bias.grad is not None else np.zeros_like(mg.npy(p.bias))
                              for p in phis]),
             fhat_last=mg.npy(fhat_list[-1]), entropy_weight=entropy_weight, scale=scale, scaler=mg.npy(q.scaler),
             w_sample=w_sample, w_batch=w_batch, ema=mg.npy(q.ema_vocab_hit_SV))
    for si, ix in enumerate(idx_list):
        d[f"idx{si}"] = mg.npy(ix)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(name, "vq", float(vq), "commit", float(commit), "ent", float(ent), "dropout", mg.npy(dropout).tolist())


def case_b1(LFQ, name="lfq_hard_b1"):
    q = LFQ(2 ** 4, 4, using_znorm=True, v_patch_nums=[1, 2, 3], num_latent_tokens=9, codebook_drop=0.5,
            soft_entropy=False).train()
    torch.manual_seed(0)
    f = torch.randn(1, 4, 3, 3)
    try:
        q(f, ret_usages=True, dropout=torch.tensor([2]))
        err, is_runtime = "", False
    except Exception as e:         # what the reference raises is the recorded result
        err, is_runtime = type(e).__name__, isinstance(e, RuntimeError)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), error=np.array(err), is_runtime_error=is_runtime)
    print(name, "raises", err or "nothing", "(RuntimeError subclass)" if is_runtime else "")


def main():
    if not os.path.isdir(mg.REF):
        raise SystemExit("set XQ_REFERENCE to a checkout of the reference (lxa9867/ImageFolder)")
    _, _, LFQ, _ = mg.import_reference()
    case_lfq_hard(LFQ, "lfq_hard_c4", 4, 4, [1, 2, 3, 5], using_znorm=True, codebook_drop=0.75, seed=41)
    case_lfq_hard(LFQ, "lfq_hard_c5_nonorm", 5, 3, [1, 2, 3, 5], using_znorm=False, codebook_drop=0.67, seed=42,
                  scale=0.8, w_sample=0.6, w_batch=1.4)
    case_lfq_hard(LFQ, "lfq_hard_c6", 6, 4, MS, using_znorm=True, codebook_drop=0.5, seed=43)
    case_lfq_hard(LFQ, "lfq_hard_c8", 8, 3, MS, using_znorm=True, codebook_drop=0.34, seed=44, scale=1.2)
    case_b1(LFQ)


if __name__ == "__main__":
    main()
