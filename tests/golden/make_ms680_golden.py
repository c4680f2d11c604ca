"""Golden vectors of VAR's default 680-token pyramid, made by RUNNING THE REFERENCE'S OWN MODULES (CPU, fp32).

    XQ_REFERENCE=<checkout of the reference> python tests/golden/make_ms680_golden.py

v_patch_nums = [1, 2, 3, 4, 5, 6, 8, 10, 13, 16] (1 + 4 + ... + 256 = 680 tokens per image) is the default of the
reference's xqgan_train.py and of VAR's own trainer.  Writes
  msvr680_znorm.npz   VectorQuantizer2, C = 32, V = 4096, using_znorm, share_quant_resi = 4, codebook_drop = 0.5
  msvr680_l2.npz      VAR's quantizer: the L2 metric (using_znorm = False), share_quant_resi = 4, no codebook drop
  varhelp680.npz      embed_to_fhat and the get_next_autoregressive_input chain at this pyramid, C = 32
The quantizer cases draw their inputs with tests/ms680_inputs.py and store only the seed and the reference's outputs.
Seeds are screened as make_golden.case_vq2 screens them: the first seed whose smallest top-2 margin, as the oracle
measures it, is above 1e-5.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import make_golden as mg  # noqa: E402
from ms680_inputs import FHAT_SUB, PN680, VAR_SUB, ms680_inputs  # noqa: E402
from oracle import xq_oracle as xo  # noqa: E402


def case_msvr680(VQ2, name, V=4096, C=32, B=2, using_znorm=True, share=4, codebook_drop=0.5, seed=680):
    while True:
        x = ms680_inputs(seed, V, C, B, share)
        fw = xo.vq2_forward(x["f"], x["E"], x["phi_w"], x["phi_b"], PN680, using_znorm=using_znorm)
        if min(float(m.min()) for m in fw["margins"]) > 1e-5:
            break
        seed += 1000
    H = PN680[-1]
    q = VQ2(V, C, using_znorm=using_znorm, v_patch_nums=PN680, num_latent_tokens=H * H, share_quant_resi=share,
            codebook_drop=codebook_drop).train()
    q.embedding.weight.data = torch.from_numpy(x["E"]).clone()
    phis = list(q.quant_resi.qresi_ls)
    for k, p in enumerate(phis):
        p.weight.data = torch.from_numpy(x["phi_w"][k]).clone()
        p.bias.data = torch.from_numpy(x["phi_b"][k]).clone()
    f = torch.from_numpy(x["f"]).clone().requires_grad_(True)
    SN = len(PN680)
    out, usages, vq, commit, _ = q(f, ret_usages=True, dropout=torch.from_numpy(x["dropout"]))
    ((out * torch.from_numpy(x["g_out"])).sum() + 1.3 * vq + 0.7 * commit).backward()
    idx_list = q.f_to_idxBl_or_fhat(f.detach(), to_fhat=False, v_patch_nums=PN680)
    fhat_list = q.f_to_idxBl_or_fhat(f.detach(), to_fhat=True, v_patch_nums=PN680)
    var_in = q.idxBl_to_var_input(idx_list)
    gE_rows, gE_vals = mg.sparse_rows(mg.npy(q.embedding.weight.grad))
    zeros = lambda p: np.zeros_like(mg.npy(p))
    d = dict(seed=seed, V=V, C=C, B=B, K=share, patch_nums=np.array(PN680), codebook_drop=codebook_drop,
             using_znorm=using_znorm, share=share, steps=1,
             out=mg.npy(out), vq=mg.npy(vq), commit=mg.npy(commit), usages=np.array([float(u) for u in usages]),
             ema=mg.npy(q.ema_vocab_hit_SV), w_vq=1.3, w_commit=0.7, gf=mg.npy(f.grad),
             gE_rows=gE_rows, gE_vals=gE_vals,
             gphi_w=np.stack([mg.npy(p.weight.grad) if p.weight.grad is not None else zeros(p.weight) for p in phis]),
             gphi_b=np.stack([mg.npy(p.bias.grad) if p.bias.grad is not None else zeros(p.bias) for p in phis]),
             var_input_sub=np.ascontiguousarray(mg.npy(var_in)[VAR_SUB]))
    for si in range(SN):
        d[f"idx{si}"] = mg.npy(idx_list[si])
        d[f"fhat_sub{si}"] = np.ascontiguousarray(mg.npy(fhat_list[si])[FHAT_SUB])
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **d)
    print(name, "seed", seed, "vq", float(vq), "commit", float(commit), "tokens per image",
          sum(int(t.shape[1]) for t in idx_list))


def main():
    if not os.path.isdir(mg.REF):
        raise SystemExit("set XQ_REFERENCE to a checkout of the reference (lxa9867/ImageFolder)")
    VQ, VQ2, LFQ, _ = mg.import_reference()
    case_msvr680(VQ2, "msvr680_znorm")
    case_msvr680(VQ2, "msvr680_l2", using_znorm=False, codebook_drop=0.0, seed=681)
    mg.OUT = HERE
    mg.case_var_helpers(VQ2, "varhelp680", 32, 1, PN680, args=(4096, 32), seed=14)


if __name__ == "__main__":
    main()
