"""Generate golden vectors by RUNNING THE REFERENCE'S OWN MODULES (CPU, fp32).

    python tests/golden/make_golden.py            # writes tests/golden/*.npz

Needs a checkout of the reference, named by the XQ_REFERENCE environment variable (the tests only
read the committed .npz / .json files).  The reference ships no tests or golden
vectors (SURVEY.md section 4), so these files are what pins the oracle -- and through it the
CUDA path -- to the reference's behaviour.  Recipe: SURVEY.md section 8c (stub timm / peft /
webdataset, 1-rank gloo group).
"""
import os
import sys
import types

import numpy as np
import torch
import torch.distributed as tdist

REF = os.environ.get("XQ_REFERENCE", "")    # a checkout of lxa9867/ImageFolder (the reference)
OUT = os.path.dirname(os.path.abspath(__file__))


class _Stub(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)

        def deco(*a, **k):
            if len(a) == 1 and callable(a[0]) and not k:
                return a[0]
            return lambda f: f
        return deco


def import_reference():
    sys.path.insert(0, REF)
    for m in ["timm", "timm.models", "timm.layers", "timm.data", "timm.models._builder", "timm.models._features",
              "timm.models._manipulate", "timm.models._registry", "peft", "webdataset", "timm.layers.helpers",
              "timm.models.layers"]:
        sys.modules[m] = _Stub(m)
    if not tdist.is_initialized():
        tdist.init_process_group("gloo", init_method="tcp://127.0.0.1:29533", rank=0, world_size=1)
    from tokenizer.tokenizer_image.quant import VectorQuantizer2
    from tokenizer.tokenizer_image.lookup_free_quantize import LFQ
    from tokenizer.tokenizer_image.latent_perturbation import add_perturbation
    from tokenizer.tokenizer_image.xqgan_model import VectorQuantizer
    return VectorQuantizer, VectorQuantizer2, LFQ, add_perturbation


def npy(t):
    return t.detach().cpu().numpy()


def sparse_rows(g):
    rows = np.nonzero(np.abs(g).sum(axis=1))[0]
    return rows.astype(np.int64), g[rows]


def case_vq(VQ, name, V, C, B, hw, codebook_norm=True, seed=0, randn_codebook=False, steps=1):
    torch.manual_seed(seed)
    q = VQ(V, C, 0.25, codebook_norm).train()
    if randn_codebook:
        q.embedding.weight.data = torch.randn(V, C) * 0.3
    E0 = npy(q.embedding.weight).copy()
    z = torch.randn(B, C, hw, hw, requires_grad=True)
    for _ in range(steps):
        out, usages, vq, commit, _ = q(z, ret_usages=True)
    g_out = torch.randn_like(out)
    loss = (out * g_out).sum() + 1.7 * vq + 0.9 * commit
    loss.backward()
    idx = q.f_to_idxBl_or_fhat(z.detach(), to_fhat=False, v_patch_nums=None)[0]
    fhat = q.f_to_idxBl_or_fhat(z.detach(), to_fhat=True, v_patch_nums=None)[0]
    gr, gv = sparse_rows(npy(q.embedding.weight.grad))
    np.savez_compressed(os.path.join(OUT, name + ".npz"), z=npy(z), E=E0, out=npy(out), vq=npy(vq), commit=npy(commit),
                        usage=np.float64(usages[0]), ema=npy(q.ema_vocab_hit_SV), idx=npy(idx), fhat=npy(fhat),
                        g_out=npy(g_out), w_vq=1.7, w_commit=0.9, gz=npy(z.grad), gE_rows=gr, gE_vals=gv,
                        codebook_norm=codebook_norm, beta=0.25, steps=steps)
    print(name, "vq", float(vq), "commit", float(commit), "usage", usages)


def case_perturb(VQ, add_perturbation, name, V, C, B, hw, alpha, beta, delta, seed=1, codebook_norm=True):
    torch.manual_seed(seed)
    q = VQ(V, C, 0.25, codebook_norm).train()
    q.embedding.weight.data = torch.randn(V, C) * 0.3
    z = torch.randn(B, C, hw, hw, requires_grad=True)
    zq, _, vq, commit, _ = q(z, ret_usages=True)
    zq_leaf = zq.detach().clone().requires_grad_(True)
    N = B * hw * hw
    torch.manual_seed(seed + 100)
    u = torch.rand(N)
    j = torch.randint(0, delta, (N,))
    torch.manual_seed(seed + 100)
    out = add_perturbation(z, zq_leaf, C, codebook_norm, q.embedding, alpha, beta, delta)
    g = torch.randn_like(out)
    gz, gzq = torch.autograd.grad((out * g).sum(), [z, zq_leaf])
    np.savez_compressed(os.path.join(OUT, name + ".npz"), z=npy(z), zq=npy(zq_leaf), E=npy(q.embedding.weight),
                        rand_u=npy(u), rand_j=npy(j), out=npy(out), g=npy(g), gz=npy(gz), gzq=npy(gzq),
                        alpha=alpha, beta=beta, delta=delta, codebook_norm=codebook_norm)
    print(name, "changed samples", int(B * beta))


def case_vq2(VQ2, name, V, C, B, patch_nums, using_znorm=True, codebook_drop=0.5, seed=2, share=4, steps=1):
    # Index equality is only well-defined away from fp32 near-ties (a flipped index at scale k
    # changes the residual of every later scale).  Pick the first seed whose smallest top-2
    # margin, as measured by the oracle, is > 1e-5; the chosen seed is stored in the file.
    sys.path.insert(0, os.path.dirname(os.path.dirname(OUT)))
    from oracle import xq_oracle as xo
    while True:
        torch.manual_seed(seed)
        H = patch_nums[-1]
        q = VQ2(V, C, using_znorm=using_znorm, v_patch_nums=patch_nums, num_latent_tokens=H * H,
                share_quant_resi=share, codebook_drop=codebook_drop)
        q.embedding.weight.data = torch.randn(V, C) * 0.5
        phis = list(q.quant_resi.qresi_ls) if share > 1 else [q.quant_resi.qresi]
        f = torch.randn(B, C, H, H)
        fw = xo.vq2_forward(npy(f), npy(q.embedding.weight), np.stack([npy(p.weight) for p in phis]),
                            np.stack([npy(p.bias) for p in phis]), patch_nums, using_znorm=using_znorm)
        if min(float(m.min()) for m in fw["margins"]) > 1e-5:
            break
        seed += 1000
    torch.manual_seed(seed)
    H = patch_nums[-1]
    q = VQ2(V, C, using_znorm=using_znorm, v_patch_nums=patch_nums, num_latent_tokens=H * H,
            share_quant_resi=share, codebook_drop=codebook_drop).train()
    q.embedding.weight.data = torch.randn(V, C) * 0.5
    K = len(q.quant_resi.qresi_ls) if share > 1 else 1
    phis = list(q.quant_resi.qresi_ls) if share > 1 else [q.quant_resi.qresi]
    f = torch.randn(B, C, H, H, requires_grad=True)
    SN = len(patch_nums)
    dropout = torch.randint(3, SN + 1, (B,))
    for _ in range(steps):
        out, usages, vq, commit, _ = q(f, ret_usages=True, dropout=dropout)
    g_out = torch.randn_like(out)
    loss = (out * g_out).sum() + 1.3 * vq + 0.7 * commit
    loss.backward()
    idx_list = q.f_to_idxBl_or_fhat(f.detach(), to_fhat=False, v_patch_nums=patch_nums)
    fhat_list = q.f_to_idxBl_or_fhat(f.detach(), to_fhat=True, v_patch_nums=patch_nums)
    var_in = q.idxBl_to_var_input(idx_list)
    d = dict(f=npy(f), E=npy(q.embedding.weight), phi_w=np.stack([npy(p.weight) for p in phis]),
             phi_b=np.stack([npy(p.bias) for p in phis]), patch_nums=np.array(patch_nums), dropout=npy(dropout),
             codebook_drop=codebook_drop, using_znorm=using_znorm, out=npy(out), vq=npy(vq), commit=npy(commit),
             usages=np.array(usages), ema=npy(q.ema_vocab_hit_SV), g_out=npy(g_out), w_vq=1.3, w_commit=0.7,
             gf=npy(f.grad), gE=npy(q.embedding.weight.grad),
             gphi_w=np.stack([npy(p.weight.grad) if p.weight.grad is not None else np.zeros_like(npy(p.weight)) for p in phis]),
             gphi_b=np.stack([npy(p.bias.grad) if p.bias.grad is not None else np.zeros_like(npy(p.bias)) for p in phis]),
             fhat_last=npy(fhat_list[-1]), fhat_mid=npy(fhat_list[SN // 2]), var_input=npy(var_in), steps=steps,
             share=share, seed=seed)
    for si, ix in enumerate(idx_list):
        d[f"idx{si}"] = npy(ix)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(name, "vq", float(vq), "commit", float(commit))


def case_lfq(LFQ, name, C, B, patch_nums, using_znorm=True, codebook_drop=0.5, seed=3, entropy_weight=0.1, scale=1.0):
    torch.manual_seed(seed)
    H = patch_nums[-1]
    q = LFQ(2 ** C, C, using_znorm=using_znorm, v_patch_nums=patch_nums, num_latent_tokens=H * H,
            share_quant_resi=4, codebook_drop=codebook_drop, scale=scale, entropy_weight=entropy_weight).train()
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
    d = dict(f=npy(f), phi_w=np.stack([npy(p.weight) for p in phis]), phi_b=np.stack([npy(p.bias) for p in phis]),
             patch_nums=np.array(patch_nums), dropout=npy(dropout), codebook_drop=codebook_drop,
             using_znorm=using_znorm, out=npy(out), vq=npy(vq), commit=npy(commit), entropy=npy(ent),
             usages=np.array(usages), g_out=npy(g_out), w_vq=1.3, w_commit=0.7, w_ent=1.1, gf=npy(f.grad),
             gphi_w=np.stack([npy(p.weight.grad) if p.weight.grad is not None else np.zeros_like(npy(p.weight)) for p in phis]),
             gphi_b=np.stack([npy(p.bias.grad) if p.bias.grad is not None else np.zeros_like(npy(p.bias)) for p in phis]),
             fhat_last=npy(fhat_list[-1]), entropy_weight=entropy_weight, scale=scale, scaler=npy(q.scaler))
    if 2 ** C <= 4096:
        d["ema"] = npy(q.ema_vocab_hit_SV)
    for si, ix in enumerate(idx_list):
        d[f"idx{si}"] = npy(ix)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(name, "vq", float(vq), "commit", float(commit), "ent", float(ent))


def case_var_helpers(Q, name, C, B, patch_nums, seed=11, share=4, **qkw):
    """feature-map helpers of the VAR side (quant.py:148-180, 247-258; lookup_free_quantize.py:311-343, 404-415):
    embed_to_fhat(all_to_max_scale=True, last_one=False/True) and the get_next_autoregressive_input chain."""
    torch.manual_seed(seed)
    H = patch_nums[-1]
    SN = len(patch_nums)
    q = Q(*qkw.pop("args"), v_patch_nums=patch_nums, num_latent_tokens=H * H, share_quant_resi=share, **qkw).eval()
    phis = list(q.quant_resi.qresi_ls) if share > 1 else [q.quant_resi.qresi]
    for p in phis:                      # non-trivial Phi weights
        p.weight.data.normal_(0, 0.2)
        p.bias.data.normal_(0, 0.1)
    hs = [torch.randn(B, C, pn, pn) for pn in patch_nums]
    with torch.no_grad():
        fh_list = q.embed_to_fhat([h.clone() for h in hs], all_to_max_scale=True, last_one=False)
        fh_last = q.embed_to_fhat([h.clone() for h in hs], all_to_max_scale=True, last_one=True)
        f_hat = torch.zeros(B, C, H, H)
        nexts = []
        for si in range(SN):
            f_hat, nxt = q.get_next_autoregressive_input(si, SN, f_hat, hs[si].clone())
            nexts.append(nxt.clone())
    d = dict(patch_nums=np.array(patch_nums), phi_w=np.stack([npy(p.weight) for p in phis]),
             phi_b=np.stack([npy(p.bias) for p in phis]), share=share, fh_last=npy(fh_last), ar_f_hat=npy(f_hat))
    for si in range(SN):
        d[f"h{si}"] = npy(hs[si])
        d[f"fh{si}"] = npy(fh_list[si])
        d[f"next{si}"] = npy(nexts[si])
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(name, "fhat abs max", float(fh_last.abs().max()))


def import_loss_reference():
    """row f-1: the reference's loss stack.  wandb is absent here and the LPIPS / DINO checkpoints cannot be downloaded:
    wandb is stubbed, and only code paths that need no pretrained weights are run."""
    sys.path.insert(0, REF)
    for m in ["wandb", "timm", "timm.models", "timm.layers", "peft", "webdataset"]:
        sys.modules.setdefault(m, _Stub(m))
    if not tdist.is_initialized():
        tdist.init_process_group("gloo", init_method="tcp://127.0.0.1:29533", rank=0, world_size=1)
    from tokenizer.tokenizer_image import diffaug, lpips, vq_loss, discriminator_dino
    return diffaug, lpips, vq_loss, discriminator_dino


def case_loss_stack():
    diffaug, lpips, vq_loss, ddino = import_loss_reference()
    d = {}
    # ---- DiffAug.aug (diffaug.py:45-118) for every flag combination that the three Bernoulli draws can produce;
    # the CPU generator decides the flags (torch.rand(3) <= prob) and the parameters (torch.rand(7,B,1,1))
    cases = []
    for ci, (seed, prob, B, C, H, W) in enumerate([(0, 1.0, 3, 3, 32, 32), (1, 1.0, 2, 3, 40, 24), (2, 0.5, 4, 3, 16, 16),
                                                   (5, 0.5, 2, 3, 20, 20), (7, 0.34, 3, 3, 16, 16), (9, 0.0, 2, 3, 8, 8),
                                                   (11, 0.6, 2, 1, 12, 12), (13, 0.5, 2, 3, 16, 16), (0, 0.5, 3, 3, 24, 24),
                                                   (1, 0.5, 2, 3, 16, 20), (4, 0.5, 3, 3, 10, 10), (16, 0.5, 2, 3, 16, 16),
                                                   (4, 0.5, 2, 3, 5, 5)]):
        aug = diffaug.DiffAug(prob=prob, cutout=0.2)
        torch.manual_seed(100 + seed)
        x = torch.randn(B, C, H, W, requires_grad=True)
        torch.manual_seed(seed)                 # the draws of aug() start here
        y = aug.aug(x, 0)
        g = torch.randn_like(y)
        if y.requires_grad:
            (gx,) = torch.autograd.grad(y, x, g)
        else:
            gx = g.clone()
        # replay the generator to record what was drawn
        torch.manual_seed(seed)
        flags3 = (torch.rand(3) <= abs(prob)) if abs(prob) >= 1e-6 else torch.zeros(3, dtype=torch.bool)
        rand01 = torch.rand(7, B, 1, 1) if bool(flags3.any()) else torch.zeros(7, B, 1, 1)
        d[f"aug{ci}_x"], d[f"aug{ci}_y"], d[f"aug{ci}_g"], d[f"aug{ci}_gx"] = npy(x), npy(y), npy(g), npy(gx)
        d[f"aug{ci}_flags"] = npy(flags3).astype(np.int64)
        d[f"aug{ci}_rand01"] = npy(rand01).reshape(7, B)
        d[f"aug{ci}_meta"] = np.array([seed, B, C, H, W], dtype=np.int64)
        d[f"aug{ci}_prob"] = np.float64(prob)
        cases.append(ci)
    d["aug_cases"] = np.array(cases)
    # ---- LPIPS stage arithmetic (lpips.py:79-90, 152-159) on synthetic post-ReLU features with the reference's functions
    torch.manual_seed(3)
    for li, (B, C, H, W) in enumerate([(2, 64, 8, 8), (3, 128, 5, 7), (2, 512, 3, 3)]):
        f0 = torch.relu(torch.randn(B, C, H, W))
        f1 = (f0 + 0.3 * torch.randn(B, C, H, W)).relu().requires_grad_(True)
        lin = lpips.NetLinLayer(C, use_dropout=True).eval()
        lin.model[1].weight.data.uniform_(0, 0.2)
        diff = (lpips.normalize_tensor(f0) - lpips.normalize_tensor(f1)) ** 2
        val = lpips.spatial_average(lin.model(diff), keepdim=True)
        g = torch.randn_like(val)
        (gf1,) = torch.autograd.grad(val, f1, g)
        d[f"lp{li}_f0"], d[f"lp{li}_f1"], d[f"lp{li}_w"] = npy(f0), npy(f1), npy(lin.model[1].weight).reshape(-1)
        d[f"lp{li}_val"], d[f"lp{li}_g"], d[f"lp{li}_gf1"] = npy(val).reshape(-1), npy(g).reshape(-1), npy(gf1)
    sl = lpips.ScalingLayer()
    xin = torch.rand(2, 3, 4, 4) * 2 - 1
    d["scal_x"], d["scal_y"] = npy(xin), npy(sl(xin))
    # state-dict key names of the reference LPIPS (built without downloads: torchvision weights / ckpt loading patched out)
    import torchvision
    orig_vgg = torchvision.models.vgg16
    lpips.models.vgg16 = lambda pretrained=False, **k: orig_vgg(weights=None)
    lpips.LPIPS.load_from_pretrained = lambda self, name="vgg_lpips": None
    ref_lp = lpips.LPIPS().eval()
    d["lpips_keys"] = np.array(sorted(ref_lp.state_dict().keys()))
    d["lpips_shapes"] = np.array([str(tuple(v.shape)) for k, v in sorted(ref_lp.state_dict().items())])
    # ---- GAN loss functions and schedules (vq_loss.py:18-77)
    torch.manual_seed(4)
    lr, lf = torch.randn(5, 7) * 2, torch.randn(5, 7) * 2
    d["gan_lr"], d["gan_lf"] = npy(lr), npy(lf)
    d["hinge_d"] = npy(vq_loss.hinge_d_loss(lr, lf))
    d["vanilla_d"] = npy(vq_loss.vanilla_d_loss(lr, lf))
    d["nonsat_d"] = npy(vq_loss.non_saturating_d_loss(lr, lf))
    d["hinge_g"] = npy(vq_loss.hinge_gen_loss(lf))
    d["nonsat_g"] = npy(vq_loss.non_saturating_gen_loss(lf))
    ema = vq_loss.LeCAM_EMA()
    ema.update(lr, lf)
    ema.update(lr * 0.5, lf + 1)
    d["lecam_ema"] = np.array([ema.logits_real_ema, ema.logits_fake_ema])
    d["lecam_reg"] = npy(vq_loss.lecam_reg(lr, lf, ema))
    d["adopt"] = np.array([vq_loss.adopt_weight(0.5, s, threshold=10, value=0.0) for s in (0, 9, 10, 11)])
    d["anneal"] = np.array([vq_loss.anneal_weight(1.0, s, threshold=10, initial_value=0.3, final_value=0.1, anneal_steps=20)
                            for s in (0, 10, 15, 30, 31, 100)])
    # ---- DinoDisc pieces that need no checkpoint: BatchNormLocal, one head, the frozen ViT with random weights
    torch.manual_seed(6)
    bn = ddino.BatchNormLocal(6, virtual_bs=4)
    bn.weight.data.uniform_(0.5, 1.5)
    bn.bias.data.normal_()
    xb = torch.randn(8, 6, 9)
    d["bnl_x"], d["bnl_w"], d["bnl_b"], d["bnl_y"] = npy(xb), npy(bn.weight), npy(bn.bias), npy(bn(xb))
    vit = ddino.FrozenDINOSmallNoDrop(depth=3, key_depths=(0, 2), embed_dim=48, num_heads=3)
    for p_ in vit.parameters():
        p_.data.normal_(0, 0.05)
    img = torch.rand(2, 3, 224, 224) * 2 - 1
    acts = vit(img)
    d["dino_keys"] = np.array(sorted(vit.state_dict().keys()))
    for k, v in vit.state_dict().items():
        d["dinow_" + k] = npy(v)
    d["dino_img"] = npy(img)[:, :, ::8, ::8].copy()       # the test rebuilds the image by nearest upsampling x8
    img_up = torch.from_numpy(d["dino_img"]).repeat_interleave(8, 2).repeat_interleave(8, 3)
    acts = vit(img_up)
    for i, a in enumerate(acts):
        d[f"dino_act{i}"] = npy(a)
    head = torch.nn.Sequential(
        ddino.make_block(48, kernel_size=1, norm_type="bn", norm_eps=1e-6, using_spec_norm=True),
        ddino.ResidualBlock(ddino.make_block(48, kernel_size=9, norm_type="bn", norm_eps=1e-6, using_spec_norm=True)),
        ddino.SpectralConv1d(48, 1, kernel_size=1, padding=0)).eval()
    d["head_keys"] = np.array(sorted(head.state_dict().keys()))
    for k, v in head.state_dict().items():
        d["headw_" + k] = npy(v)
    d["head_y"] = npy(head(acts[0]))
    from tokenizer.tokenizer_image.discriminator_patchgan import NLayerDiscriminator
    pg = NLayerDiscriminator(input_nc=3, n_layers=3, ndf=16)
    d["patchgan_keys"] = np.array(sorted(pg.state_dict().keys()))
    d["patchgan_shapes"] = np.array([str(tuple(v.shape)) for k, v in sorted(pg.state_dict().items())])
    from tokenizer.tokenizer_image.discriminator_stylegan import Discriminator as SGD
    sg = SGD(input_nc=3, image_size=32)
    d["stylegan_keys"] = np.array(sorted(sg.state_dict().keys()))
    d["stylegan_shapes"] = np.array([str(tuple(v.shape)) for k, v in sorted(sg.state_dict().items())])
    np.savez_compressed(os.path.join(OUT, "loss_stack.npz"), **d)
    print("loss_stack: aug cases", len(cases), "lpips keys", len(d["lpips_keys"]), "dino acts", len(acts))


# ---------------------------------------------------------------------------------------------------------------------
# round 2: BASELINE-shaped cases (configs #2 / #3) and an UNSCREENED multi-scale case.  Inputs and weights come from
# tests/golden/vit_det_init.py (name-seeded / CPU-generator tensors), so the files hold only the reference's OUTPUTS.
# ---------------------------------------------------------------------------------------------------------------------
def det_inputs(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g)


def case_vq_big(VQ, name, V, C, B=4, hw=16, seed=21):
    from vit_det_init import apply_det_init
    q = VQ(V, C, 0.25, True).train()
    apply_det_init(q)                                  # embedding.weight <- name-seeded randn / sqrt(C)
    z = det_inputs((B, C, hw, hw), seed).requires_grad_(True)
    out, usages, vq, commit, _ = q(z, ret_usages=True)
    g_out = det_inputs(tuple(out.shape), seed + 1)
    ((out * g_out).sum() + 1.7 * vq + 0.9 * commit).backward()
    idx = q.f_to_idxBl_or_fhat(z.detach(), to_fhat=False, v_patch_nums=None)[0]
    gr, gv = sparse_rows(npy(q.embedding.weight.grad))
    np.savez_compressed(os.path.join(OUT, name + ".npz"), V=V, C=C, B=B, hw=hw, seed=seed, idx=npy(idx).astype(np.int32),
                        out_sub=npy(out)[:, :, ::2, ::2], out_sum=np.float64(out.double().sum()), vq=npy(vq), commit=npy(commit),
                        usage=np.float64(usages[0]), gz_sub=npy(z.grad)[:, :, ::2, ::2], gz_abs=np.float64(z.grad.double().abs().sum()),
                        gE_rows=gr.astype(np.int32), gE_vals=gv, w_vq=1.7, w_commit=0.9, beta=0.25)
    print(name, "vq", float(vq), "commit", float(commit), "usage", usages, "distinct codes", len(np.unique(npy(idx))))


def case_vq2_unscreened(VQ2, name, V=4096, C=32, B=6, patch_nums=(1, 1, 2, 3, 3, 4, 5, 6, 8, 11), seed=31):
    """no seed screening (make_golden.case_vq2 skips seeds with fp32 near-ties): the test COUNTS index mismatches against
    these reference indices and requires each first divergence to be a near-tie (top-2 margin < 1e-5)."""
    from vit_det_init import apply_det_init
    patch_nums = list(patch_nums)
    H = patch_nums[-1]
    q = VQ2(V, C, using_znorm=True, v_patch_nums=patch_nums, num_latent_tokens=H * H, share_quant_resi=4,
            codebook_drop=0.0).eval()
    apply_det_init(q)
    f = det_inputs((B, C, H, H), seed)
    with torch.no_grad():
        idx_list = q.f_to_idxBl_or_fhat(f, to_fhat=False, v_patch_nums=patch_nums)
        fhat = q.f_to_idxBl_or_fhat(f, to_fhat=True, v_patch_nums=patch_nums)[-1]
    d = dict(V=V, C=C, B=B, patch_nums=np.array(patch_nums), seed=seed, fhat_sub=npy(fhat)[:, :, ::2, ::2])
    for si, ix in enumerate(idx_list):
        d[f"idx{si}"] = npy(ix).astype(np.int32)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(name, "tokens", sum(int(i.numel()) for i in idx_list))


def main_round2():
    VQ, VQ2, LFQ, add_perturbation = import_reference()
    sys.path.insert(0, OUT)
    case_vq_big(VQ, "vq8192_c32", 8192, 32)            # BASELINE config #2 codebook
    case_vq_big(VQ, "vq16384_c32", 16384, 32, seed=23)  # BASELINE config #3 codebook
    case_vq2_unscreened(VQ2, "msvr_unscreened")


def write_config_golden():
    """reference_configs.json: the values of the reference's configs/*.yaml that config.SHIPPED_CONFIGS restates"""
    import glob
    import json

    import yaml
    sys.path.insert(0, os.path.dirname(os.path.dirname(OUT)))
    from imagefolder_b200 import config as xcfg
    out = {}
    for f in sorted(glob.glob(os.path.join(REF, "configs", "*.yaml"))):
        y = yaml.safe_load(open(f))
        name = os.path.basename(f)[:-5]
        out[name] = {k: y[k] for k in xcfg.SHIPPED_CONFIGS.get(name, y) if k in y}
    with open(os.path.join(OUT, "reference_configs.json"), "w") as fh:
        fh.write("{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(v, sort_keys=True)}" for k, v in sorted(out.items())) + "\n}\n")


def main():
    if not os.path.isdir(REF):
        raise SystemExit("set XQ_REFERENCE to a checkout of the reference (lxa9867/ImageFolder)")
    if "--configs-only" in sys.argv:
        write_config_golden()
        return
    if "--round2-only" in sys.argv:
        main_round2()
        return
    if "--loss-only" in sys.argv:
        case_loss_stack()
        return
    VQ, VQ2, LFQ, add_perturbation = import_reference()
    if "--var-helpers-only" in sys.argv:
        case_var_helpers(VQ2, "varhelp_msvr", 16, 3, [1, 1, 2, 3, 3, 4, 5, 6, 8, 11], args=(256, 16))
        case_var_helpers(VQ2, "varhelp_shared1", 8, 2, [1, 2, 4, 7], share=1, args=(128, 8), seed=12)
        case_var_helpers(LFQ, "varhelp_lfq", 10, 2, [1, 2, 3, 5], args=(2 ** 10, 10), seed=13)
        return
    MS = [1, 1, 2, 3, 3, 4, 5, 6, 8, 11]
    # BASELINE config #1: VQ-4096 (C=64) on one 256x256 image -> 16x16 tokens. Reference init codebook.
    case_vq(VQ, "vq4096_b1", 4096, 64, 1, 16)
    case_vq(VQ, "vq512_randn", 512, 32, 3, 8, randn_codebook=True, steps=3)
    case_vq(VQ, "vq300_nonorm", 300, 24, 2, 5, codebook_norm=False, randn_codebook=True)
    case_perturb(VQ, add_perturbation, "perturb_a07", 512, 32, 4, 8, alpha=0.7, beta=0.5, delta=20)
    case_perturb(VQ, add_perturbation, "perturb_a0", 256, 16, 2, 4, alpha=0.0, beta=0.0, delta=100)
    case_vq2(VQ2, "msvr_small", 256, 16, 4, MS, steps=2)
    case_vq2(VQ2, "msvr_4096", 4096, 32, 2, MS, codebook_drop=0.5)
    case_vq2(VQ2, "msvr_l2", 200, 12, 3, [1, 2, 3, 5], using_znorm=False, codebook_drop=0.34)
    case_vq2(VQ2, "msvr_shared1", 128, 8, 2, [1, 2, 4, 7], share=1, codebook_drop=0.0)
    case_lfq(LFQ, "msbr_small", 8, 4, MS)
    case_lfq(LFQ, "msbr_14", 14, 3, MS, codebook_drop=0.34)
    case_lfq(LFQ, "lfq_nonorm", 6, 4, [1, 2, 3, 5], using_znorm=False, scale=0.8)
    case_cnn()
    case_var_helpers(VQ2, "varhelp_msvr", 16, 3, [1, 1, 2, 3, 3, 4, 5, 6, 8, 11], args=(256, 16))
    case_var_helpers(VQ2, "varhelp_shared1", 8, 2, [1, 2, 4, 7], share=1, args=(128, 8), seed=12)
    case_var_helpers(LFQ, "varhelp_lfq", 10, 2, [1, 2, 3, 5], args=(2 ** 10, 10), seed=13)
    case_loss_stack()


def case_cnn(name="cnn_small", seed=5):
    """reference CNN Encoder / Decoder (xqgan_model.py:454-584), tiny widths, fp32 CPU."""
    from tokenizer.tokenizer_image.xqgan_model import Decoder, Encoder
    torch.manual_seed(seed)
    enc = Encoder(ch=32, ch_mult=(1, 2), num_res_blocks=1, z_channels=8).eval()
    dec = Decoder(ch=32, ch_mult=(1, 2), num_res_blocks=1, z_channels=8).eval()
    x = torch.randn(2, 3, 16, 16)
    z = torch.randn(2, 8, 8, 8)
    with torch.no_grad():
        h, y = enc(x), dec(z)
    d = dict(x=npy(x), z=npy(z), h=npy(h), y=npy(y))
    for k, v in enc.state_dict().items():
        d["enc." + k] = npy(v)
    for k, v in dec.state_dict().items():
        d["dec." + k] = npy(v)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(name, h.shape, y.shape)

if __name__ == "__main__":
    main()
