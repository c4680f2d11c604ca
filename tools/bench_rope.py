"""RoPE decoder timings: the q / k rotation kernels per call, and a whole decoder training step with and without RoPE.

Per call (B = 128, N = 513, H = 12, L = 256, bf16): xq_vit_rope_fwd / xq_vit_rope_bwd against the reference's op sequence
(vision_transformer.py:246-259: the two apply_rotary_emb calls on the q / k slices, written back into the qkv tensor; its
backward is autograd's).  Decoder step (ViT-B, --batch latents of 256 tokens, bf16 autocast, forward + backward):
DINOv2Decoder(use_rope=True) against use_rope=False on the same fused kernels.  Arms alternate in windows of --calls /
--window launches (CUDA events around each window) for --rounds rounds; medians are reported.  The GPU's name, power limit
and clocks are read in the same run.  Prints one JSON object; --out also writes it to a file.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm,temperature.gpu"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable: {e}"


def timed(fn, n):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


def alternate(arms, n, rounds):
    for fn in arms.values():          # warm-up
        fn()
    torch.cuda.synchronize()
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            res[k].append(timed(fn, n))
    return {k: statistics.median(v) for k, v in res.items()}


def per_call(args):
    from imagefolder_b200 import vit_ops
    from imagefolder_b200.dino_enc.vision_transformer import apply_rotary_emb, compute_mixed_cis, init_t_xy
    B, N, H, P, L = 128, 513, 12, 1, 256
    qkv = torch.randn(B, N, 3 * H * 64, device="cuda").bfloat16()
    g = torch.randn_like(qkv)
    freqs = torch.randn(2, H * 32, device="cuda") * 0.3
    f1 = torch.randn(L, 32, 2, device="cuda")
    t_x, t_y = (t.cuda() for t in init_t_xy(16, 16))
    rot = vit_ops.rope_forward(qkv, freqs, f1, H, P)
    fr = freqs.clone().requires_grad_()
    f1c = torch.view_as_complex(f1).clone().requires_grad_()

    def ref_forward(x):
        q5 = x.view(B, N, 3, H, 64).permute(2, 0, 3, 1, 4)
        q, k = q5[0], q5[1]
        cis = compute_mixed_cis(fr, t_x, t_y, H)
        q[:, :, P:-L], k[:, :, P:-L] = apply_rotary_emb(q[:, :, P:-L], k[:, :, P:-L], cis)
        q[:, :, -L:], k[:, :, -L:] = apply_rotary_emb(q[:, :, -L:], k[:, :, -L:], f1c)
        return x

    def ref_fwd():
        with torch.no_grad():
            ref_forward(qkv.clone())

    def ref_fwd_bwd():
        x = qkv.clone().requires_grad_()
        y = ref_forward(x * 1)
        torch.autograd.backward(y, g)

    ours = alternate({"ours_fwd": lambda: vit_ops.rope_forward(qkv, freqs, f1, H, P),
                      "ours_bwd": lambda: vit_ops.rope_backward(qkv, g, freqs, f1, H, P),
                      "ref_fwd": ref_fwd, "ref_fwd_bwd": ref_fwd_bwd}, args.calls, args.rounds)
    nbytes = qkv.numel() * 2
    ours["ours_fwd_GBps"] = 2 * nbytes / ours["ours_fwd"] / 1e6
    ours["ours_bwd_GBps"] = 3 * nbytes / ours["ours_bwd"] / 1e6
    del rot
    return ours


def decoder_step(args):
    from imagefolder_b200.dino_enc.dinov2 import DINOv2Decoder
    kw = dict(model_name="vit_base_patch14_dinov2.lvd142m", model_kwargs=dict(img_size=256, patch_size=16, drop_path_rate=0.0),
              pretrained=False, tuning_method="full", num_latent_tokens=256, to_pixel="linear")
    decs = {}
    for rope in (False, True):
        torch.manual_seed(0)
        decs["rope" if rope else "no_rope"] = DINOv2Decoder(use_rope=rope, **kw).cuda().train()
    z = torch.randn(args.batch, 256, 768, device="cuda")

    def step(dec):
        def run():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                out = dec(z)
            out.float().square().mean().backward()
        return run

    res = alternate({k: step(d) for k, d in decs.items()}, args.window, args.rounds)
    res["rope_minus_no_rope_per_layer"] = (res["rope"] - res["no_rope"]) / 12
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--window", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rope.py measures the GPU kernels: no CUDA device")
    res = {"gpu_before": gpu_state(), "per_call_ms": per_call(args), "decoder_step_ms": decoder_step(args),
           "batch": args.batch, "gpu_after": gpu_state()}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
