"""LFQ forward + backward at the MSBR10P2 branch shapes: soft entropy vs full-softmax entropy vs the reference's op sequence.

    python tools/bench_lfq_entropy.py [--shapes 16384 4096] [--iters 20] [--warmup 3] [--rounds 3]

One product-quantizer branch of MSBR10P2-16384 (C = 14) and MSBR10P2-4096 (C = 12): B = 128 images, 11 x 11 latents, the 10
scales 1,1,2,3,3,4,5,6,8,11, using_znorm, codebook_drop 0.1.  Three arms run the same training-mode forward + backward of
(f_hat, vq, commit, entropy):
  soft     LFQ(soft_entropy=True)   (libxqb200, mode XQ_MS_BSQ)
  hard     LFQ(soft_entropy=False)  (libxqb200, mode XQ_MS_BSQ_HARD: closed-form 2^C-code softmax entropy)
  torch    an eager restatement of the reference's LFQ.forward with soft_entropy=False (lookup_free_quantize.py:149-250):
           per scale area pool, sign codes, bicubic up, Phi, masked f_hat, and entropy_loss on the explicit
           [B, HW, 1, 2^C] logits; autograd backward
Time: CUDA events around --iters calls, the arms alternated --rounds times; the median round is reported.  Peak memory:
torch.cuda.max_memory_allocated over one call.  An arm that runs out of memory is reported as "OOM".  The card's name,
power limit and clocks are read in the same process.  Prints one JSON line.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PN = [1, 1, 2, 3, 3, 4, 5, 6, 8, 11]


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return dict(zip(q.split(","), [s.strip() for s in out[0].split(",")])) if out else {}
    except (OSError, subprocess.SubprocessError):
        return {"error": "nvidia-smi unavailable"}


def torch_lfq(q, f, dropout):
    """the reference's training-mode forward, soft_entropy=False, restated with torch ops (q supplies the weights)."""
    B, C, H, W = f.shape
    SN = len(q.v_patch_nums)
    fn = F.normalize(f, dim=1) if q.using_znorm else f
    f_no_grad = fn.detach()
    f_rest = f_no_grad.clone()
    f_hat = torch.zeros_like(f_rest)
    nq = torch.full((B,), float(SN + 1), device=f.device)
    nd = int(B * q.codebook_drop)
    nq[:nd] = dropout[:nd].to(f.device).float()
    bits = (torch.arange(2 ** C, device=f.device)[:, None] >> torch.arange(C, device=f.device)) & 1
    codebook = bits.float() * 2 - 1
    weights = 2 ** torch.arange(C, device=f.device)
    mods = q.quant_resi.modules_list()
    vq = commit = ent = 0.0
    for si, pn in enumerate(q.v_patch_nums):
        s = q.scaler[si].float()
        rest = F.interpolate(f_rest, size=(pn, pn), mode="area") if si != SN - 1 else f_rest
        idx = ((rest > 0).long() * weights[:, None, None]).sum(1)                       # [B, pn, pn]
        code = torch.where(((idx[..., None] >> torch.arange(C, device=f.device)) & 1) != 0, s, -s).permute(0, 3, 1, 2)
        h = F.interpolate(code, size=(H, W), mode="bicubic") if si != SN - 1 else code
        if mods:
            phi = mods[q._phi_map(SN)[si]]
            r = abs(q.quant_resi_ratio)
            h = h * (1 - r) + F.conv2d(h, phi.weight, phi.bias, padding=1) * r
        x = (fn - f_hat.detach()).permute(0, 2, 3, 1).reshape(B, H * W, 1, C)
        mask = (si < nq).float()
        f_hat = f_hat + h * mask[:, None, None, None]
        f_rest = f_rest - h
        ratio = mask.sum() / B
        logits = 2 * torch.einsum("bnid,jd->bnij", x, codebook * s)
        probs = torch.softmax(logits / 0.01, -1)
        log_probs = torch.log_softmax(logits / 0.01 + 1e-5, -1)
        mw = mask[:, None, None, None] / mask.sum()
        avg = (probs * mw).sum(0).reshape(-1, 2 ** C).mean(0)
        hc = -(avg * torch.log(avg + 1e-5)).sum()
        hs = ((-(probs * log_probs).sum(-1)) * mw[..., 0]).sum(0).mean()
        ent = ent + (q.sample_minimization_weight * hs - q.batch_maximization_weight * hc) * (q.entropy_weight / ratio)
        vq = vq + F.mse_loss(f_hat, f_no_grad, reduction="none").mul(mask[:, None, None, None]).mean() / ratio
        commit = commit + F.mse_loss(f_hat.detach(), fn, reduction="none").mul(mask[:, None, None, None]).mean() * (q.beta / ratio)
    out = (f_hat.detach() - f_no_grad) + fn
    return out, vq / SN, commit / SN, ent / SN


def make_arm(kind, C, seed=0):
    from imagefolder_b200 import LFQ
    torch.manual_seed(seed)
    q = LFQ(2 ** C, C, using_znorm=True, v_patch_nums=PN, num_latent_tokens=121, codebook_drop=0.1, entropy_weight=0.1,
            soft_entropy=(kind == "soft")).cuda().train()
    g = torch.Generator().manual_seed(seed + 1)
    f = torch.randn(128, C, 11, 11, generator=g).cuda().requires_grad_(True)
    dropout = torch.randint(3, len(PN) + 1, (128,), generator=g)

    def step():
        if kind == "torch":
            out, vq, commit, ent = torch_lfq(q, f, dropout)
        else:
            out, _, vq, commit, ent = q(f, dropout=dropout)
        (out.sum() + vq + commit + ent).backward()
        f.grad = None
    return step


def time_arm(step, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        step()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", type=int, default=[16384, 4096])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lfq_entropy needs a CUDA device")
    res = {"gpu": gpu_info(), "shapes": {}}
    for V in args.shapes:
        C = V.bit_length() - 1
        arms, row = {}, {}
        for kind in ("soft", "hard", "torch"):
            try:
                step = make_arm(kind, C)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                step()
                torch.cuda.synchronize()
                row[kind] = {"peak_mem_mb": round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)}
                for _ in range(args.warmup):
                    step()
                arms[kind] = step
            except torch.cuda.OutOfMemoryError:
                row[kind] = {"ms": "OOM", "peak_mem_mb": "OOM"}
                torch.cuda.empty_cache()
        times = {k: [] for k in arms}
        for _ in range(args.rounds):
            for kind, step in arms.items():
                if times[kind] is None:
                    continue
                try:
                    times[kind].append(time_arm(step, args.iters))
                except torch.cuda.OutOfMemoryError:
                    times[kind] = None
                    row[kind] = {"ms": "OOM", "peak_mem_mb": "OOM"}
                    torch.cuda.empty_cache()
        for kind, t in times.items():
            if t:
                row[kind]["ms"] = round(statistics.median(t), 3)
                row[kind]["ms_rounds"] = [round(x, 3) for x in t]
        res["shapes"][f"MSBR10P2-{V} branch (B=128, C={C}, 11x11, 10 scales)"] = row
    res["note"] = "forward + backward of (f_hat, vq, commit, entropy); ms = median over rounds of the mean of --iters calls"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
