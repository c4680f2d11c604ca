"""CPU checks of the image-transform path (csrc/img_kernels.cu, imagefolder_b200/data.py, oracle/aug_oracle.py):
the numpy restatement of Pillow's resize is bit-exact against PIL, the oracle reproduces the reference-generated golden
(tests/golden/make_aug_golden.py), the host plans reproduce the reference's draws and sizes, collate packing round-trips, and
the new C-ABI entry points refuse bad arguments before anything is launched."""
import ctypes
import random

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import aug_oracle as ao


def golden_cases():
    g = load_golden("aug_crops")
    for i in range(len(g["seed"])):
        h, w = (int(v) for v in g["hw"][i])
        S = int(g["S"][i])
        crop = g["crops_u8"][g["crop_off"][i]:g["crop_off"][i + 1]].reshape(S, S, 3)
        yield g, i, h, w, S, crop


def golden_plan_row(g, i):
    h, w = (int(v) for v in g["hw"][i])
    S = int(g["S"][i])
    s, cy, cx, f = (int(v) for v in g["draws"][i])
    rh, rw = (int(v) for v in g["rs_hw"][i])
    if not g["train"][i]:
        cy, cx = (rh - S) // 2, (rw - S) // 2
    return np.array([h, w, int(g["levels"][i]), rh, rw, cy, cx, f], np.int32)


def test_golden_covers_every_halving_depth():
    g = load_golden("aug_crops")
    assert set(g["levels"].tolist()) == {0, 1, 2, 3, 4}
    assert set(g["draws"][:, 3].tolist()) == {0, 1}


@pytest.mark.parametrize("use_pil", [False, True])
def test_oracle_reproduces_reference_golden(use_pil):
    if use_pil:
        pytest.importorskip("PIL")
    for g, i, h, w, S, crop in golden_cases():
        img = ao.synth_image(int(g["seed"][i]), h, w)
        got = ao.crop_u8(img, golden_plan_row(g, i), S, use_pil=use_pil)
        assert np.array_equal(got, crop), f"golden case {i} ({h}x{w}, S={S})"


def test_plans_reproduce_reference_draws_and_sizes():
    from imagefolder_b200 import data
    g = load_golden("aug_crops")
    for gi, seed in enumerate(g["group_seed"].tolist()):
        idx = np.nonzero(g["group"] == gi)[0]
        sizes = [tuple(int(v) for v in g["hw"][i]) for i in idx]
        S = int(g["S"][idx[0]])
        random.seed(seed)
        torch.manual_seed(seed)
        if g["train"][idx[0]]:
            plan = data.plan_random_crop(sizes, S)
        else:
            plan = data.plan_center_crop(sizes, S)
        for r, i in zip(plan, idx):
            assert np.array_equal(r, golden_plan_row(g, i)), (gi, i, r)
            if g["train"][i]:
                s = int(g["draws"][i][0])
                assert min(r[3], r[4]) == s                      # the BICUBIC short side is the drawn s


def test_resample_matches_pil_bit_for_bit():
    Image = pytest.importorskip("PIL.Image")
    sizes = [(1, 1), (2, 3), (7, 5), (31, 17), (129, 77), (257, 300), (375, 500), (511, 1023)]
    outs = [(1, 1), (3, 2), (16, 13), (128, 64), (255, 341), (300, 400), (700, 900), (64, 1000)]
    for h, w in sizes:
        img = ao.synth_image(h * 7 + w, h, w)
        for oh, ow in outs + [(max(1, h // 2), max(1, w // 2)), (h, w), (h, max(1, w - 1)), (h + 1, w)]:
            for kind, pk in ((ao.BOX, Image.BOX), (ao.BICUBIC, Image.BICUBIC)):
                ref = np.asarray(Image.fromarray(img).resize((ow, oh), resample=pk))
                assert np.array_equal(ao.resample(img, (oh, ow), kind), ref), (h, w, oh, ow, kind)


def test_to_tensor_normalize_matches_torchvision():
    T = pytest.importorskip("torchvision.transforms")
    u = np.arange(256, dtype=np.uint8).reshape(16, 16, 1).repeat(3, 2)
    ref = T.Normalize(mean=[0.5] * 3, std=[0.5] * 3, inplace=True)(T.ToTensor()(u))
    assert torch.equal(torch.from_numpy(ao.to_tensor_normalize(u)), ref)


def test_collate_packs_and_round_trips():
    from imagefolder_b200 import data
    imgs = [ao.synth_image(k, h, w) for k, (h, w) in enumerate([(5, 7), (1, 1), (64, 33), (3, 300)])]
    batch = [((a, data.plan_center_crop([a.shape[:2]], 1)[0]), k) for k, a in enumerate(imgs)]
    packed, offs, plan, labels = data.collate(batch)
    assert packed.dtype == torch.uint8 and packed.numel() == sum(a.size for a in imgs)
    assert offs.tolist() == [0, 105, 108, 108 + 64 * 33 * 3]
    assert plan.shape == (4, 8) and plan.dtype == torch.int32 and labels.tolist() == [0, 1, 2, 3]
    for a, b in zip(imgs, data.unpack(packed, offs, plan)):
        assert np.array_equal(a, b)
    with pytest.raises(ValueError):
        data.collate([((np.zeros((4, 4), np.uint8), plan[0].numpy()), 0)])


def test_gpu_decode_draws_like_the_reference_transform():
    """GpuDecode consumes random / torch draws exactly like random_crop_arr + RandomHorizontalFlip, one image after another."""
    Image = pytest.importorskip("PIL.Image")
    from imagefolder_b200 import data
    g = load_golden("aug_crops")
    idx = [i for i in range(len(g["seed"])) if g["group"][i] == 8]           # the five-image training group
    random.seed(int(g["group_seed"][8]))
    torch.manual_seed(int(g["group_seed"][8]))
    t = data.GpuDecode(int(g["S"][idx[0]]), train=True)
    for i in idx:
        h, w = (int(v) for v in g["hw"][i])
        arr, row = t(Image.fromarray(ao.synth_image(int(g["seed"][i]), h, w)))
        assert arr.shape == (h, w, 3) and np.array_equal(row, golden_plan_row(g, i))


def test_image_entry_points_validate_arguments_without_gpu():
    """xq_img_* (csrc/img_kernels.cu): invalid plans are refused by the host-side layout query, NULL pointers and bad sizes by
    the launchers, all before any CUDA call."""
    from imagefolder_b200 import _capi, data
    L = _capi.lib()
    plan = np.ascontiguousarray(np.concatenate([data.plan_center_crop([(375, 500), (1100, 1500)], 256),
                                                data.plan_center_crop([(100, 90)], 256)]))
    off = np.zeros(3, np.int64)
    n = L.xq_img_workspace_bytes(plan.ctypes.data, 3, 256, off.ctypes.data)
    a1 = (1100 // 2) * (1500 // 2) * 3
    assert plan[1, 2] == 2 and n == a1 + (1100 // 4) * (1500 // 4) * 3
    assert off.tolist() == [0, 0, n]                                              # image 1 holds both buffers
    assert L.xq_img_workspace_bytes(plan.ctypes.data, 1, 256, None) == 16           # no halving: minimum size
    assert L.xq_img_workspace_bytes(None, 3, 256, None) == 0
    assert L.xq_img_workspace_bytes(plan.ctypes.data, 3, 0, None) == 0
    assert L.xq_img_workspace_bytes(plan.ctypes.data, 3, 257, None) == 0           # rs < S
    for col, v in ((5, -1), (6, 500), (7, 2), (2, -1), (2, 12), (0, 0)):
        bad = plan.copy()
        bad[0, col] = v
        assert L.xq_img_workspace_bytes(bad.ctypes.data, 3, 256, None) == 0, (col, v)
    bad = plan.copy()
    bad[1, 2] = 0                                                                   # 1100 -> 256 in one BICUBIC: 39 taps
    assert L.xq_img_workspace_bytes(bad.ctypes.data, 3, 256, None) == 0
    one = ctypes.c_void_p(4096)
    assert L.xq_img_box_halve(None, 16, one, one, 1, 256, 1, 8, 8, one, 16, None) == -1
    assert L.xq_img_box_halve(one, 16, one, one, 1, 256, 0, 8, 8, one, 16, None) == -1     # level 0
    assert L.xq_img_box_halve(one, 16, one, one, 1, 256, 1, 8, 8, None, 16, None) == -1    # no workspace
    assert L.xq_img_box_halve(one, 16, one, one, 0, 256, 1, 8, 8, one, 16, None) == -1     # B = 0
    assert L.xq_img_resize_crop_normalize(one, 16, one, one, 1, 256, None, 0, None, None) == -1
    assert L.xq_img_resize_crop_normalize(one, 16, None, one, 1, 256, None, 0, one, None) == -1
    assert L.xq_img_resize_crop_normalize(one, 16, one, one, 1, 8192, None, 0, one, None) == -1  # S > XQ_IMG_MAX_SIZE
    with pytest.raises(ValueError):
        data.gpu_transform(torch.zeros(16, dtype=torch.uint8), [0], plan[:1] * 0, 256)
