"""GPU tests of the reconstruction metrics (csrc/metric_kernels.cu, imagefolder_b200/evaluate.py::psnr_ssim /
reconstruction_metrics) against the host restatement of the reference's scikit-image calls (oracle/metric_oracle.py)."""
import math

import numpy as np
import pytest
import torch

from imagefolder_b200 import _capi
from imagefolder_b200.evaluate import psnr_ssim, reconstruction_metrics
from oracle import metric_oracle as mo
from test_model_cpu import small_model

pytestmark = pytest.mark.gpu

S = _capi.XQ_METRIC_STRIP_ROWS
SHAPES = [(1, 3, 7, 7), (2, 3, 8, 9), (3, 3, 37, 53), (5, 1, 64, 64), (128, 3, 256, 256), (2, 3, 512, 512)]
# heights at each strip boundary +-1, widths at each column-tile boundary +-1 (tiles of 512 input columns, 506 output columns)
BOUNDARY = ([(2, 3, h, 21) for h in (S - 1, S, S + 1, 2 * S - 1, 2 * S, 2 * S + 1, 3 * S + 1)]
            + [(1, 2, 11, w) for w in (511, 512, 513, 1017, 1018, 1019, 1524, 1525)])
PSNR_RTOL, SSIM_ATOL = 1e-9, 1e-6


def make_inputs(shape, seed):
    """x uniform in [-1, 1]; rec = clamp(x + noise), with a quarter of its values moved onto the uint8 truncation thresholds
    (k - 128) / 127.5 and one ulp either side, and a few at exactly -1 and 1"""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(shape, generator=g) * 2 - 1
    rec = (x + 0.15 * torch.randn(shape, generator=g)).clamp(-1, 1)
    k = torch.randint(0, 257, shape, generator=g)
    thr = torch.from_numpy(((k.numpy() - 128) / 127.5).astype(np.float32))
    step = torch.randint(-1, 2, shape, generator=g)
    thr = torch.where(step < 0, torch.nextafter(thr, torch.tensor(-2.0)),
                      torch.where(step > 0, torch.nextafter(thr, torch.tensor(2.0)), thr)).clamp(-1, 1)
    rec = torch.where(torch.rand(shape, generator=g) < 0.25, thr, rec)
    rec = torch.where(torch.rand(shape, generator=g) < 0.01, torch.sign(rec), rec)
    return rec, x


def check(rec, x, label):
    """kernel vs oracle; rec may be bf16 (the oracle gets its fp32 widening)"""
    p, s = psnr_ssim(rec.cuda(), x.cuda())
    wp, ws = mo.psnr_ssim(rec.float().numpy(), x.numpy())
    p, s = p.cpu().numpy(), s.cpu().numpy()
    assert p.dtype == np.float64 and s.dtype == np.float64 and p.shape == (x.shape[0],)
    finite = np.isfinite(wp)
    assert np.array_equal(np.isfinite(p), finite) and np.array_equal(p[~finite], wp[~finite])
    rel = float(np.max(np.abs(p[finite] - wp[finite]) / np.abs(wp[finite]), initial=0.0))
    ssim_err = float(np.max(np.abs(s - ws)))
    print(f"{label}: max PSNR rel err {rel:.3e}, max SSIM abs err {ssim_err:.3e}")
    assert rel <= PSNR_RTOL and ssim_err <= SSIM_ATOL


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("shape", SHAPES + BOUNDARY, ids=lambda s: "x".join(map(str, s)))
def test_matches_oracle(shape, dtype):
    rec, x = make_inputs(shape, seed=sum(shape))
    check(rec.to(dtype), x, f"{tuple(shape)} {dtype}")


def test_identical_images_and_constant_offset():
    g = torch.Generator().manual_seed(5)
    x = torch.where(torch.rand(3, 3, 40, 33, generator=g) < 0.5, -1.0, 1.0)
    p, s = psnr_ssim(x.cuda(), x.cuda())                       # r = g in {0, 1}
    assert torch.all(p == math.inf) and torch.all(s == 1.0)
    p, s = psnr_ssim(torch.ones(2, 3, 9, 8, device="cuda"), torch.full((2, 3, 9, 8), 0.5, device="cuda"))   # r = 1, g = 0.75
    assert torch.allclose(p, torch.full_like(p, 10 * math.log10(16.0)), rtol=1e-12, atol=0)
    _, ws = mo.psnr_ssim(np.ones((1, 3, 9, 8), np.float32), np.full((1, 3, 9, 8), 0.5, np.float32))
    assert torch.all(s.cpu() == float(ws[0]))


def test_outputs_written_deterministic_and_stream_ordered():
    rec, x = make_inputs((6, 3, 70, 1030), seed=7)
    rec, x = rec.cuda(), x.cuda()
    L = _capi.lib()
    B, C, H, W = x.shape
    nbytes = L.xq_recon_psnr_ssim_workspace_bytes(B, C, H, W)
    ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device="cuda")                  # NaN-patterned workspace
    runs = []
    side = torch.cuda.Stream()
    for stream in (torch.cuda.current_stream(), side, side):
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            p = torch.full((B,), math.nan, dtype=torch.float64, device="cuda")
            s = torch.full((B,), math.nan, dtype=torch.float64, device="cuda")
            rc = L.xq_recon_psnr_ssim(rec.data_ptr(), 0, x.data_ptr(), B, C, H, W, p.data_ptr(), s.data_ptr(), ws.data_ptr(),
                                      nbytes, stream.cuda_stream)
            assert rc == 0
        torch.cuda.current_stream().wait_stream(stream)
        assert not torch.isnan(p).any() and not torch.isnan(s).any()
        runs.append((p.clone(), s.clone()))
    for p, s in runs[1:]:
        assert torch.equal(p.view(torch.int64), runs[0][0].view(torch.int64))
        assert torch.equal(s.view(torch.int64), runs[0][1].view(torch.int64))
    check(rec.cpu(), x.cpu(), "6x3x70x1030")


def test_refused_call_writes_nothing():
    rec, x = make_inputs((2, 3, 16, 16), seed=9)
    rec, x = rec.cuda(), x.cuda()
    L = _capi.lib()
    p = torch.full((2,), math.nan, dtype=torch.float64, device="cuda")
    s = torch.full((2,), math.nan, dtype=torch.float64, device="cuda")
    nbytes = L.xq_recon_psnr_ssim_workspace_bytes(2, 3, 16, 16)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    assert L.xq_recon_psnr_ssim(rec.data_ptr(), 0, x.data_ptr(), 2, 3, 16, 16, p.data_ptr(), s.data_ptr(), ws.data_ptr(),
                                nbytes - 1, st) == -2
    assert L.xq_recon_psnr_ssim(rec.data_ptr(), 0, x.data_ptr(), 2, 3, 16, 6, p.data_ptr(), s.data_ptr(), ws.data_ptr(),
                                nbytes, st) == -1
    assert L.xq_recon_psnr_ssim(rec.data_ptr(), 2, x.data_ptr(), 2, 3, 16, 16, p.data_ptr(), s.data_ptr(), ws.data_ptr(),
                                nbytes, st) == -1
    with pytest.raises(ValueError):
        psnr_ssim(rec.half(), x)
    torch.cuda.synchronize()
    assert torch.isnan(p).all() and torch.isnan(s).all()


def test_reconstruction_metrics_end_to_end():
    """reconstruction_metrics on a small random-weight VQModel == the oracle applied to img_to_reconstructed_img of the same
    batches; eval mode only for the loop"""
    model, _ = small_model("MSVR10P2-4096")
    model = model.cuda().train()
    g = torch.Generator().manual_seed(11)
    batches = [(torch.rand(2, 3, 256, 256, generator=g) * 2 - 1, torch.zeros(2)) for _ in range(2)]
    res = reconstruction_metrics(model, batches)
    assert model.training and res.count == 4
    model.eval()
    wp, ws = [], []
    with torch.no_grad():
        for x, _ in batches:
            rec = model.img_to_reconstructed_img(x.cuda()).float().cpu().numpy()
            p, s = mo.psnr_ssim(rec, x.numpy())
            wp += p.tolist()
            ws += s.tolist()
    wp, ws = np.array(wp), np.array(ws)
    print(f"end to end: PSNR {res.psnr:.6f} (oracle {wp.mean():.6f}), SSIM {res.ssim:.8f} (oracle {ws.mean():.8f})")
    np.testing.assert_allclose(res.psnr_per_image, wp, rtol=PSNR_RTOL, atol=0)
    np.testing.assert_allclose(res.ssim_per_image, ws, rtol=0, atol=SSIM_ATOL)
    assert res.psnr == sum(res.psnr_per_image.tolist()) / 4 and res.ssim == sum(res.ssim_per_image.tolist()) / 4
    assert abs(res.psnr - wp.mean()) <= PSNR_RTOL * abs(wp.mean()) and abs(res.ssim - ws.mean()) <= SSIM_ATOL
