"""ViT encoder / decoder parity against goldens produced by the REFERENCE's own modules
(tests/golden/make_vit_golden.py: dino_enc/dinov2.py + the vendored dino_enc/vision_transformer.py + VQModel.encode /
decode; only timm's PatchEmbed / Mlp / DropPath / resample_abs_pos_embed are stand-ins there).

CPU (fp32, tolerance 1e-3 relative as the north star states -- observed ~1e-5): the product's modules and the oracle
restatement (oracle/vit_ref.py) both have to reproduce the reference's numbers from the same name-seeded weights.
GPU: the fused bf16 path (libxqb200 glue + wgmma attention) against the same goldens at bf16 tolerance."""
import ast
import os
import sys

import numpy as np
import pytest
import torch

from imagefolder_b200 import config as xcfg

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from vit_det_init import apply_det_init, golden_inputs  # noqa: E402

CASES = ["vit_vq", "vit_vp2", "vit_ms", "vit_relpos"]


def load_case(name):
    g = np.load(os.path.join(HERE, "golden", name + ".npz"))
    cfg = ast.literal_eval(str(g["cfg_json"]))
    return g, cfg


def build_ours(cfg):
    args = xcfg.parse_args([])
    for k, v in cfg.items():
        setattr(args, k, v)
    torch.manual_seed(0)
    model = xcfg.build_vq_model(args).eval()
    apply_det_init(model)
    return model


def check(g, tok, h, dec, rtol, atol):
    np.testing.assert_allclose(tok[:, ::4], g["tok_sub"], rtol=rtol, atol=atol)
    assert tuple(h.shape) == tuple(g["h_shape"])
    np.testing.assert_allclose(h.reshape(h.shape[0], h.shape[1], -1)[:, :, ::4], g["h_sub"], rtol=rtol, atol=atol)
    np.testing.assert_allclose(dec[:, :, ::4, ::4], g["dec_sub"], rtol=rtol, atol=atol)
    # full-tensor sums catch anything the subsampling skipped
    assert abs(float(tok.astype(np.float64).sum()) - float(g["tok_sum"])) <= atol * tok.size * 0.05 + rtol * float(g["tok_abs"])
    assert abs(float(dec.astype(np.float64).sum()) - float(g["dec_sum"])) <= atol * dec.size * 0.05 + rtol * float(g["dec_abs"])


@pytest.mark.parametrize("name", CASES)
def test_product_vit_matches_reference_golden_cpu(name):
    g, cfg = load_case(name)
    model = build_ours(cfg)
    x, q = golden_inputs(int(g["q_shape"][1]), int(g["q_shape"][2]))
    assert abs(float(x.double().sum()) - float(g["x_sum"])) < 1e-6 and abs(float(q.double().sum()) - float(g["q_sum"])) < 1e-6
    with torch.no_grad():
        tok = model.encoder(x)
        h = model.encode(x)
        dec = model.decode(q)
    check(g, tok.numpy(), h.numpy(), dec.numpy(), rtol=1e-3, atol=1e-4)
    assert int(g["enc_S"]) == {"vit_vq": 513, "vit_vp2": 769, "vit_ms": 499, "vit_relpos": 513}[name]


@pytest.mark.parametrize("name", CASES)
def test_oracle_vit_matches_reference_golden(name):
    from oracle import vit_ref
    g, cfg = load_case(name)
    model = build_ours(cfg)          # only as a container of the name-seeded state_dict
    ref = vit_ref.RefTokenizer(model.state_dict(), vit_ref.cfg_from_model_args(model.config, num_heads=6))
    x, q = golden_inputs(int(g["q_shape"][1]), int(g["q_shape"][2]))
    with torch.no_grad():
        h = ref.encode(x)
        dec = ref.decode(q)
    np.testing.assert_allclose(h.numpy().reshape(h.shape[0], h.shape[1], -1)[:, :, ::4], g["h_sub"], rtol=1e-3, atol=1e-4)
    np.testing.assert_allclose(dec.numpy()[:, :, ::4, ::4], g["dec_sub"], rtol=1e-3, atol=1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_fused_cuda_vit_matches_reference_golden(name):
    """bf16 autocast through the fused path (residual+LN / GELU glue kernels, wgmma attention, library GEMMs).
    Tolerance: bf16 GEMM operands over 12 blocks -> a few 1e-2 absolute on O(1) activations."""
    g, cfg = load_case(name)
    model = build_ours(cfg).cuda()
    x, q = golden_inputs(int(g["q_shape"][1]), int(g["q_shape"][2]))
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        tok = model.encoder(x.cuda()).float().cpu().numpy()
        h = model.encode(x.cuda()).float().cpu().numpy()
        dec = model.decode(q.cuda()).float().cpu().numpy()
    for got, want in ((tok[:, ::4], g["tok_sub"]), (h.reshape(h.shape[0], h.shape[1], -1)[:, :, ::4], g["h_sub"]),
                      (dec[:, :, ::4, ::4], g["dec_sub"])):
        err = np.abs(got - want)
        assert err.max() < 0.15 and err.mean() < 0.02, (err.max(), err.mean())
    # fp32 on the GPU (module path, library kernels): the 1e-3 bar
    with torch.no_grad():
        tok32 = model.encoder(x.cuda()).cpu().numpy()
        dec32 = model.decode(q.cuda()).cpu().numpy()
    np.testing.assert_allclose(tok32[:, ::4], g["tok_sub"], rtol=1e-3, atol=1e-3)
    np.testing.assert_allclose(dec32[:, :, ::4, ::4], g["dec_sub"], rtol=1e-3, atol=1e-3)
