"""Time the frozen guide teachers on the module path and on the frozen fused path (vit_ops.frozen_forward).

  python tools/bench_teacher.py [--batch 128] [--rounds 5] [--iters 10] [--steps 3] [--out DIR]

Prints the card (name, power limit, max SM clock) and one JSON line per measurement:
  - the three teacher calls of a training step at B = 128, 256 x 256, bf16 autocast -- DINOv2 ViT-B `forward` (the class
    token, semantic guide with guide_type_1 'class'), DINOv2 ViT-B `forward_features`, CLIP ViT-B `forward_features`
    (detail guide) -- each as the median of `rounds` alternating windows of `iters` calls per path, CUDA events, after a
    warm-up of both paths; with the peak-memory increase of one call over what was allocated before it;
  - the VQ-8192 training step with `semantic_guide: dinov2` and the MSBR10P2-16384 step with both teachers
    (guide_type_2 'patch'), fused teachers against module teachers, alternating windows of `steps` steps.
Teacher weights are random (timing only).  The module path is forced by switching the routing test off.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import warnings

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception as e:
        out = f"nvidia-smi unavailable ({e!r})"
    return {"card": out, "torch_name": torch.cuda.get_device_name(0)}


class module_path:
    """context manager: the teachers run their module path (the routing test answers no)"""

    def __enter__(self):
        from imagefolder_b200.dino_enc import vision_transformer as vt
        self.vt, self.saved = vt, vt.frozen_path_ok
        vt.frozen_path_ok = lambda vit, x: False

    def __exit__(self, *exc):
        self.vt.frozen_path_ok = self.saved


def frozen(name):
    from imagefolder_b200.dino_enc.vision_transformer import create_model
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = create_model(name, pretrained=True, img_size=256, patch_size=16, drop_path_rate=0.0)
    m.eval()
    for p in m.parameters():
        p.requires_grad = False
    return m.cuda()


def time_window(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def peak_increase(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del out
    return peak


def compare(fused_fn, module_fn, rounds, iters, warm=2):
    for _ in range(warm):
        fused_fn()
        with module_path():
            module_fn()
    torch.cuda.synchronize()
    tf, tm = [], []
    for _ in range(rounds):
        tf.append(time_window(fused_fn, iters))
        with module_path():
            tm.append(time_window(module_fn, iters))
    return statistics.median(tf), statistics.median(tm), tf, tm


def teacher_calls(args):
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.rand(args.batch, 3, 256, 256, device="cuda", generator=g) * 2 - 1
    dino, clip = frozen("vit_base_patch14_dinov2.lvd142m"), frozen("vit_base_patch16_clip_224.openai")
    calls = [("dinov2_vitb_forward_cls", lambda: dino(x)), ("dinov2_vitb_forward_features", lambda: dino.forward_features(x)),
             ("clip_vitb_forward_features", lambda: clip.forward_features(x))]
    rows = []
    for name, fn in calls:
        with torch.autocast("cuda", dtype=torch.bfloat16), torch.no_grad():
            f_ms, m_ms, tf, tm = compare(fn, fn, args.rounds, args.iters)
            mem_f = peak_increase(fn)
            with module_path():
                mem_m = peak_increase(fn)
        rows.append({"call": name, "batch": args.batch, "fused_ms": round(f_ms, 3), "module_ms": round(m_ms, 3),
                     "speedup": round(m_ms / f_ms, 3), "fused_windows_ms": [round(t, 3) for t in tf],
                     "module_windows_ms": [round(t, 3) for t in tm], "fused_peak_MB": round(mem_f / 2 ** 20, 1),
                     "module_peak_MB": round(mem_m / 2 ** 20, 1)})
        print(json.dumps(rows[-1]), flush=True)
    del dino, clip
    torch.cuda.empty_cache()
    return rows


def train_step(workload, guides, batch):
    from imagefolder_b200 import config as xcfg
    cfg = dict(xcfg.SHIPPED_CONFIGS[workload])
    cfg.update(guides)
    a = xcfg.parse_args([])
    for k, v in cfg.items():
        setattr(a, k, v)
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model = xcfg.build_vq_model(a).cuda()
    model.train()
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=3e-5, betas=(0.9, 0.95),
                            weight_decay=0.0, fused=True)
    alpha, beta, delta = xcfg.perturbation_schedule(a, 0)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand(batch, 3, 256, 256, device="cuda", generator=g) * 2 - 1

    def step():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            dec, (vq, commit, ent, _), sem, det, dep = model(x, 0, alpha, beta, delta)
            loss = F.mse_loss(dec.float(), x) + vq + commit + ent + dep
            for t in (sem, det):
                if t is not None:
                    loss = loss + t
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
    return model, step


def train_steps(args):
    rows = []
    for workload, guides in [("VQ-8192", dict(semantic_guide="dinov2", detail_guide="none")),
                             ("MSBR10P2-16384", dict(semantic_guide="dinov2", detail_guide="clip", guide_type_2="patch"))]:
        model, step = train_step(workload, guides, args.batch)
        f_ms, m_ms, tf, tm = compare(step, step, args.rounds, args.steps)
        rows.append({"step": workload, "guides": guides, "batch": args.batch, "fused_teacher_ms": round(f_ms, 2),
                     "module_teacher_ms": round(m_ms, 2), "speedup": round(m_ms / f_ms, 3),
                     "fused_windows_ms": [round(t, 2) for t in tf], "module_windows_ms": [round(t, 2) for t in tm]})
        print(json.dumps(rows[-1]), flush=True)
        del model, step
        torch.cuda.empty_cache()
    return rows


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--batch", type=int, default=128)
    p.add_argument("--rounds", type=int, default=5, help="alternating windows per path")
    p.add_argument("--iters", type=int, default=10, help="teacher calls per window")
    p.add_argument("--steps", type=int, default=3, help="training steps per window")
    p.add_argument("--skip-steps", action="store_true", help="time the teacher calls only")
    p.add_argument("--out", type=str, default=None, help="also write the results as JSON to DIR/bench_teacher.json")
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_teacher.py needs a CUDA device")
    import imagefolder_b200  # noqa: F401
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    info = card()
    print(json.dumps(info), flush=True)
    res = {"card": info, "calls": teacher_calls(args)}
    if not args.skip_steps:
        res["steps"] = train_steps(args)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_teacher.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
