"""Multi-scale quantizers on the 286-token (1 -> 11) and 680-token (1 -> 16) pyramids: per-call kernel time, the PQ-2
training step, and the 1 -> 11 backward against another build of libxqb200 (e.g. the previous commit's).

    python tools/bench_ms_pyramid.py [--baseline-lib path/to/libxqb200.so] [--windows 7] [--iters 10]

Prints one JSON object.  Reads the card's name, power limit and max SM clock in the same run.
  calls     xq_ms_forward / xq_ms_backward of one training step of VectorQuantizer2 at B = 128, C = 32 (znorm,
            share_quant_resi = 4, codebook_drop = 0.1), V = 4096 and 16384, both pyramids: CUDA events around each C
            call (imagefolder_b200._capi.TIMING); the four shapes alternate window by window; per shape the median over
            windows of each window's median call.
  step      images/s of the bf16 training step (forward, loss, backward, fused AdamW) of the PQ-2 MSVR10P2-4096 model
            (ViT-B encoder and decoder, no guide teachers) at B = 128 on both pyramids, and of the same model driven
            the reference's eager way (oracle/eager_ref.EagerTokenizer) on the 680-token pyramid.
  baseline  with --baseline-lib: the 1 -> 11 step at V = 4096 run through both libraries on the same inputs (outputs,
            indices, losses and gradients bitwise equal, the codebook gradient up to fp32 atomic order), then the two
            libraries' xq_ms_backward alternated window by window.
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

PN286 = [1, 1, 2, 3, 3, 4, 5, 6, 8, 11]
PN680 = [1, 2, 3, 4, 5, 6, 8, 10, 13, 16]


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # the numbers below still stand; say what could not be read
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unread ({e})", "max_sm_clock": "unread"}


def quantizer(V, pn, seed=0):
    from imagefolder_b200 import VectorQuantizer2
    g = torch.Generator().manual_seed(seed)
    q = VectorQuantizer2(V, 32, using_znorm=True, v_patch_nums=pn, num_latent_tokens=pn[-1] ** 2, share_quant_resi=4,
                         codebook_drop=0.1)
    with torch.no_grad():
        q.embedding.weight.copy_(torch.randn(V, 32, generator=g) * 0.5)
        for m in q.quant_resi.modules_list():
            m.weight.copy_(torch.randn(m.weight.shape, generator=g) * 0.06)
            m.bias.copy_(torch.randn(32, generator=g) * 0.1)
    f = torch.randn(128, 32, pn[-1], pn[-1], generator=g)
    dropout = torch.randint(1, len(pn) + 1, (128,), generator=g)
    g_out = torch.randn(f.shape, generator=g) / f.numel()
    return q.cuda().train(), f.cuda(), dropout, g_out.cuda()


def quant_step(q, f, dropout, g_out):
    """one training step of the quantizer alone -> everything it computes"""
    for m in [q.embedding] + q.quant_resi.modules_list():
        for p in m.parameters():
            p.grad = None
    ft = f.clone().requires_grad_(True)
    out, _, vq, commit, _ = q(ft, dropout=dropout)
    ((out * g_out).sum() + 1.3 * vq + 0.7 * commit).backward()
    mods = q.quant_resi.modules_list()
    return dict(out=out.detach(), vq=vq.detach(), commit=commit.detach(), idx=torch.cat([t.reshape(-1) for t in q.last_idx_Bl]),
                fhat=torch.stack(q.f_to_idxBl_or_fhat(f, to_fhat=True)), f_grad=ft.grad,
                phi_w_grad=torch.stack([m.weight.grad for m in mods]), phi_b_grad=torch.stack([m.bias.grad for m in mods]),
                E_grad=q.embedding.weight.grad.clone())


def timed_calls(arm, iters):
    """`iters` quantizer steps of one arm -> {entry: [ms per call]}"""
    from imagefolder_b200 import _capi
    _capi.TIMING = {}
    for _ in range(iters):
        quant_step(*arm)
    torch.cuda.synchronize()
    t, _capi.TIMING = _capi.TIMING, None
    return {k: [s.elapsed_time(e) for s, e, _, _ in v] for k, v in t.items() if k in ("xq_ms_forward", "xq_ms_backward")}


def alternate(arms, windows, iters, before=None):
    """arms: {label: quantizer arm}; window by window every arm in turn -> {label: {entry: median of window medians}}"""
    meds = {k: {} for k in arms}
    for w in range(windows + 1):
        for label, arm in arms.items():
            if before:
                before(label)
            r = timed_calls(arm, iters)
            if w == 0:
                continue           # warm-up window
            for entry, ts in r.items():
                meds[label].setdefault(entry, []).append(statistics.median(ts))
    return {k: {e: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v), "windows": len(v)}
                for e, v in d.items()} for k, d in meds.items()}


def training_step(pn, impl, B=128):
    import torch.nn.functional as F
    from imagefolder_b200 import config as xcfg
    cfg = dict(xcfg.SHIPPED_CONFIGS["MSVR10P2-4096"])
    cfg.update(semantic_guide="none", detail_guide="none", v_patch_nums=pn, num_latent_tokens=pn[-1] ** 2)
    args = xcfg.parse_args([])
    for k, v in cfg.items():
        setattr(args, k, v)
    torch.manual_seed(0)
    model = xcfg.build_vq_model(args).cuda().train()
    net = model
    if impl == "eager":
        from oracle.eager_ref import EagerTokenizer
        net = EagerTokenizer(model)
    opt = torch.optim.AdamW(model.parameters(), lr=3e-5, betas=(0.9, 0.95), weight_decay=0.0, fused=True)
    x = torch.rand(B, 3, 256, 256, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1)) * 2 - 1

    def step():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            dec, (vq, commit, ent, _), _, _, _ = net(x, 0, 0.0, 0.0, 100)
            loss = F.mse_loss(dec.float(), x) + vq + commit + ent
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        return loss
    return model, step


def images_per_s(pn, impl, steps, warmup, B=128):
    import gc
    model, step = training_step(pn, impl, B)
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    r = {"img_s": B * steps / (ms * 1e-3), "ms_per_step": ms / steps, "steps": steps, "warmup": warmup,
         "loss_finite": bool(torch.isfinite(loss))}
    del model, step
    gc.collect()
    torch.cuda.empty_cache()
    return r


def load_lib(path):
    """a second libxqb200 with the binding's argument types, without replacing the loaded one"""
    from imagefolder_b200 import _capi
    saved = (_capi.LIB_PATH, _capi._lib)
    try:
        _capi.LIB_PATH, _capi._lib = os.path.abspath(path), None
        return _capi.lib()
    finally:
        _capi.LIB_PATH, _capi._lib = saved


def compare_libs(arm, libs):
    from imagefolder_b200 import _capi
    res = {}
    for label, L in libs.items():
        _capi._lib = L
        res[label] = quant_step(*arm)
    _capi._lib = libs["this"]
    a, b = res["this"], res["baseline"]
    same = {k: bool(torch.equal(a[k], b[k])) for k in a if k != "E_grad"}
    d = (a["E_grad"] - b["E_grad"]).abs().max().item()
    same["E_grad_max_abs_diff"] = d
    same["E_grad_max_abs"] = b["E_grad"].abs().max().item()
    return same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-lib", default=None, help="another libxqb200.so to compare the 1 -> 11 backward with")
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--skip-step", action="store_true", help="per-call times only")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from imagefolder_b200 import _capi
    res = {"gpu": gpu_info(), "B": 128, "C": 32}
    arms = {f"{tok}_V{V}": quantizer(V, pn) for tok, pn in (("286", PN286), ("680", PN680)) for V in (4096, 16384)}
    res["calls"] = alternate(arms, a.windows, a.iters)
    if a.baseline_lib:
        libs = {"this": _capi.lib(), "baseline": load_lib(a.baseline_lib)}
        arm = arms["286_V4096"]
        res["baseline_outputs_equal"] = compare_libs(arm, libs)

        def use(label):
            _capi._lib = libs[label]
        res["baseline_backward_286_V4096"] = alternate({"this": arm, "baseline": arm}, a.windows, a.iters, before=use)
        _capi._lib = libs["this"]
    del arms
    torch.cuda.empty_cache()
    if not a.skip_step:
        res["step"] = {"286_ours": images_per_s(PN286, "ours", a.steps, a.warmup),
                       "680_ours": images_per_s(PN680, "ours", a.steps, a.warmup),
                       "680_eager": images_per_s(PN680, "eager", max(2, a.steps // 2), 1)}
    res["gpu_after"] = gpu_info()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
