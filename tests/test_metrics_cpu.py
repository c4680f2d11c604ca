"""CPU checks of the reconstruction metrics (imagefolder_b200/evaluate.py::psnr_ssim / reconstruction_metrics,
csrc/metric_kernels.cu, oracle/metric_oracle.py): the kernel's moment-filter scheme against scipy's uniform_filter, the uint8
conversion, closed-form values, C-ABI refusals before any CUDA call, and the world_size-2 aggregation."""
import math
import os
import re
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from imagefolder_b200 import _capi
from imagefolder_b200.evaluate import to_uint8_nhwc
from oracle import metric_oracle as mo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_ARG, ERR_WORKSPACE = -1, -2


def test_moment_filter_scheme_matches_scipy_uniform_filter():
    """per-axis fp64 `sum / 7` rounded to fp32 == scipy.ndimage.uniform_filter(., 7) on the interior, bit for bit, over 100
    planes: 20 pairs of a quantised reconstruction r and a uniform ground truth g, and their products r*r, g*g, r*g"""
    rng = np.random.default_rng(0)
    mismatches = total = 0
    for _ in range(20):
        r = mo.restored(rng.uniform(-1, 1, (256, 256)).astype(np.float32))
        g = mo.ground_truth(rng.uniform(-1, 1, (256, 256)).astype(np.float32))
        for plane in (r, g, r * r, g * g, r * g):
            a = mo.uniform7(plane)[3:-3, 3:-3]
            b = mo.scipy_uniform(plane)[3:-3, 3:-3]
            mismatches += int(np.count_nonzero(a.view(np.int32) != b.view(np.int32)))
            total += a.size
    print(f"moment filter: {mismatches} mismatches in {total} interior values")
    assert mismatches == 0


def test_ssim_with_scipy_filter_equals_ssim_with_kernel_scheme():
    rng = np.random.default_rng(1)
    r = mo.restored(rng.uniform(-1, 1, (40, 53)).astype(np.float32))
    g = mo.ground_truth(np.clip(rng.normal(0, 0.5, (40, 53)), -1, 1).astype(np.float32))
    assert mo.ssim_channel(r, g) == mo.ssim_channel(r, g, filt=mo.scipy_uniform)


def test_uint8_conversion_equals_to_uint8_nhwc_at_every_threshold():
    """s at (k - 128) / 127.5 and one fp32 ulp either side, for every k: where 127.5 * s + 128 crosses an integer"""
    base = np.array([(k - 128) / 127.5 for k in range(0, 257)], dtype=np.float32)
    s = np.concatenate([base, np.nextafter(base, np.float32(-2)), np.nextafter(base, np.float32(2)),
                        np.array([-1.0, 1.0, -1.5, 1.5, 0.0], np.float32)])
    want = to_uint8_nhwc(torch.from_numpy(s).view(1, 1, 1, -1)).view(-1).numpy()
    got = mo.to_uint8(s)
    assert np.array_equal(got, want)
    assert len(np.unique(got)) == 256
    np.testing.assert_array_equal(mo.restored(s), got.astype(np.float32) / np.float32(255))


def test_identical_images_give_ssim_one_and_psnr_inf():
    rng = np.random.default_rng(2)
    p = rng.uniform(0, 1, (3, 19, 23)).astype(np.float32)
    assert all(mo.ssim_channel(p[c], p[c]) == 1.0 for c in range(3))
    assert mo.psnr_image(p, p) == math.inf
    # through the whole conversion: s = x = +-1 gives r = g in {0, 1}
    x = np.where(rng.uniform(size=(2, 3, 16, 12)) < 0.5, -1.0, 1.0).astype(np.float32)
    psnr, ssim = mo.psnr_ssim(x, x)
    assert np.all(psnr == math.inf) and np.all(ssim == 1.0)


def test_constant_offset_has_closed_form_psnr():
    g = (np.arange(3 * 16 * 16, dtype=np.float32) % 128 / np.float32(256)).reshape(3, 16, 16)
    for d in (0.25, 0.125, 2.0 ** -10):
        assert math.isclose(mo.psnr_image(g + np.float32(d), g), 10 * math.log10(1 / (d * d)), rel_tol=1e-14)
    # r = 1 (s = 1 -> 255), g = 0.75 (x = 0.5): mse = 1/16
    psnr, _ = mo.psnr_ssim(np.ones((1, 3, 8, 8), np.float32), np.full((1, 3, 8, 8), 0.5, np.float32))
    assert math.isclose(psnr[0], 10 * math.log10(16.0), rel_tol=1e-14)


def test_seven_by_seven_image_is_one_window():
    """a 7x7 image has one interior pixel, whose window is the whole image: SSIM is the textbook formula with the image
    means, the ddof=1 variances and covariance, computed here independently in fp64"""
    rng = np.random.default_rng(3)
    for _ in range(5):
        r = mo.restored(rng.uniform(-1, 1, (7, 7)).astype(np.float32)).astype(np.float64)
        g = mo.ground_truth(rng.uniform(-1, 1, (7, 7)).astype(np.float32)).astype(np.float64)
        mx, my = r.mean(), g.mean()
        vx, vy = r.var(ddof=1), g.var(ddof=1)
        cxy = ((r - mx) * (g - my)).sum() / 48
        c1, c2 = (0.01 * 2.0) ** 2, (0.03 * 2.0) ** 2
        want = (2 * mx * my + c1) * (2 * cxy + c2) / ((mx * mx + my * my + c1) * (vx + vy + c2))
        assert abs(mo.ssim_channel(r.astype(np.float32), g.astype(np.float32)) - want) < 1e-6


def test_strip_rows_match_header():
    text = open(os.path.join(ROOT, "include", "xqb200.h")).read()
    assert int(re.search(r"#define XQ_METRIC_STRIP_ROWS (\d+)", text).group(1)) == _capi.XQ_METRIC_STRIP_ROWS


def test_workspace_bytes():
    L = _capi.lib()
    S = _capi.XQ_METRIC_STRIP_ROWS
    assert L.xq_recon_psnr_ssim_workspace_bytes(2, 3, 64, 64) == 2 * 3 * (64 // S) * 16
    assert L.xq_recon_psnr_ssim_workspace_bytes(1, 1, 7, 7) == 16
    assert L.xq_recon_psnr_ssim_workspace_bytes(1, 1, 7, 1019) == 3 * 16          # three column tiles
    for bad in ((0, 3, 8, 8), (1, 0, 8, 8), (1, 3, 6, 8), (1, 3, 8, 6)):
        assert L.xq_recon_psnr_ssim_workspace_bytes(*bad) == 0


@pytest.mark.skipif(torch.cuda.is_available(), reason="dummy device pointers must never reach a real GPU")
def test_c_abi_refuses_bad_arguments_without_gpu():
    """every refusal happens before the first CUDA call, so none of these touches a device"""
    L = _capi.lib()
    R, X, P, S, WS = 1 << 20, 2 << 20, 3 << 20, 4 << 20, 5 << 20               # aligned dummy pointers

    def call(rec=R, bf16=0, x=X, B=2, C=3, H=16, W=16, psnr=P, ssim=S, ws=WS, ws_bytes=1 << 20):
        return L.xq_recon_psnr_ssim(rec, bf16, x, B, C, H, W, psnr, ssim, ws, ws_bytes, None)

    for kw in (dict(rec=None), dict(x=None), dict(psnr=None), dict(ssim=None), dict(ws=None),
               dict(H=6), dict(W=6), dict(H=0), dict(B=0), dict(C=0), dict(B=-1), dict(C=-2),
               dict(bf16=2), dict(bf16=-1), dict(rec=R + 2), dict(rec=R + 1, bf16=1), dict(x=X + 2),
               dict(psnr=P + 4), dict(ssim=S + 4), dict(ws=WS + 8), dict(B=1 << 30, C=1 << 30)):
        assert call(**kw) == ERR_ARG, kw
    assert call(ws_bytes=L.xq_recon_psnr_ssim_workspace_bytes(2, 3, 16, 16) - 1) == ERR_WORKSPACE
    assert call(ws_bytes=0) == ERR_WORKSPACE


def test_python_wrapper_refuses_before_any_launch():
    from imagefolder_b200.evaluate import psnr_ssim
    x = torch.zeros(2, 3, 16, 16)
    with pytest.raises(_capi.XqError):                                             # no CPU path
        psnr_ssim(x.clone(), x)
    with pytest.raises(ValueError, match="shape"):
        psnr_ssim(x[:1], x)
    with pytest.raises(ValueError, match="fp32 or bf16"):
        psnr_ssim(x.half(), x)
    with pytest.raises(ValueError, match="fp32 or bf16"):
        psnr_ssim(x, x.double())


# ---- world_size-2 aggregation, with the kernel replaced by the oracle so that it runs without a GPU ----

def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class _Halver(torch.nn.Module):
    """stands in for VQModel: the loop only needs img_to_reconstructed_img"""

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1))

    def img_to_reconstructed_img(self, x):
        return (x * 0.5).clamp(-1, 1)


def _rank_batches(rank):
    g = torch.Generator().manual_seed(200 + rank)
    return [(torch.rand(3, 3, 9, 11, generator=g) * 2 - 1, None) for _ in range(2)]


def _oracle_psnr_ssim(rec, x):
    p, s = mo.psnr_ssim(rec.float().numpy(), x.numpy())
    return torch.from_numpy(p), torch.from_numpy(s)


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from imagefolder_b200 import evaluate
        evaluate.psnr_ssim = _oracle_psnr_ssim
        m = _Halver().train()
        res = evaluate.reconstruction_metrics(m, _rank_batches(rank), device="cpu")
        assert m.training
        q.put((rank, res.psnr, res.ssim, res.psnr_per_image.tolist(), res.ssim_per_image.tolist(), res.count))
    finally:
        dist.destroy_process_group()


def test_world2_aggregation_is_rank_major():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=180)
        assert p.exitcode == 0
    got = dict((v[0], v[1:]) for v in (q.get(timeout=5) for _ in range(2)))
    assert got[0] == got[1]                                                       # every rank returns the same result
    psnr, ssim, psnr_all, ssim_all, count = got[0]
    # the reference: each rank's per-image list in loader order, all_gather_object, chain (rank-major), sum / len
    want_p, want_s = [], []
    for r in range(2):
        for x, _ in _rank_batches(r):
            p, s = mo.psnr_ssim((x * 0.5).clamp(-1, 1).numpy(), x.numpy())
            want_p += p.tolist()
            want_s += s.tolist()
    assert count == 12 and psnr_all == want_p and ssim_all == want_s
    assert psnr == sum(want_p) / len(want_p) and ssim == sum(want_s) / len(want_s)
