"""GPU image transforms (csrc/img_kernels.cu through imagefolder_b200.data) bit-exact against the CPU oracle
(oracle/aug_oracle.py, itself pinned to Pillow and to the reference-generated golden by tests/test_aug_cpu.py).

Every call writes into an output that is NaN-filled beforehand and followed by a guard image, so an unwritten pixel fails
torch.equal and a write past the batch changes the guard.  Plans are built with the same size arithmetic as the reference
(data._halve) and choose s / crop / flip explicitly where a case needs it."""
import random

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import aug_oracle as ao

pytestmark = pytest.mark.gpu


def run(imgs, plan, S):
    from imagefolder_b200 import data
    batch = [((a, p), 0) for a, p in zip(imgs, plan)]
    packed, offs, plan_t, _ = data.collate(batch)
    src = packed.cuda()
    full = torch.full((len(imgs) + 1, 3, S, S), float("nan"), device="cuda")
    full[-1].fill_(7.0)
    out = data.gpu_transform(src, offs, plan_t, S, out=full[:-1])
    torch.cuda.synchronize()
    assert out.data_ptr() == full.data_ptr()
    assert bool((full[-1] == 7.0).all()), "write past the batch"
    return full[:-1].cpu()


def check(imgs, plan, S):
    got = run(imgs, plan, S)
    for k, (a, p) in enumerate(zip(imgs, plan)):
        ref = torch.from_numpy(ao.apply_plan(a, p, S))
        assert torch.equal(got[k], ref), f"image {k}: {a.shape[:2]} plan {list(p)}, " \
                                         f"{int((got[k] != ref).sum())} values differ"


def row(h, w, S, s, cy="mid", cx="mid", flip=0):
    from imagefolder_b200 import data
    levels, rh, rw = data._halve(h, w, s)
    pick = lambda v, n: {"min": 0, "max": n - S, "mid": (n - S) // 2}[v] if isinstance(v, str) else v
    return np.array([h, w, levels, rh, rw, pick(cy, rh), pick(cx, rw), flip], np.int32)


def img(h, w, seed=0):
    return ao.synth_image(seed * 7919 + h * 31 + w, h, w)


@pytest.mark.parametrize("short", [255, 256, 257, 511, 512, 513, 1023, 1024, 1025, 2047, 2048, 2049, 4095, 4096, 4097])
def test_every_halving_depth_single_image(short):
    """short sides around 256 * 2^k: depths 0..4 at s = 256 (center crop) and s = 320 (largest random short side)"""
    S = 256
    for k, (h, w) in enumerate([(short, short * 4 // 3 + 1), (short * 4 // 3 + 1, short)]):   # landscape, portrait
        plans = ((256, "mid", "mid", 0), (320, "max", "min", 1), (289, "min", "max", k))
        if short > 1100:                          # the oracle takes seconds per image at these sides: fewer plans
            plans = () if (k and short > 3000) else plans[:1] if k else plans[:2]
        for s, cy, cx, flip in plans:
            p = row(h, w, S, s, cy, cx, flip)
            check([img(h, w, k)], [p], S)


def test_depths_reach_four():
    from imagefolder_b200 import data
    assert data._halve(4097, 5463, 256)[0] == 4 and data._halve(4095, 5461, 256)[0] == 3 and data._halve(255, 300, 256)[0] == 0


@pytest.mark.parametrize("h,w", [(320, 451), (451, 320), (256, 301), (301, 256), (256, 256), (640, 977)])
def test_copy_path_short_side_equals_target(h, w):
    """the BICUBIC resize to the same size is a copy in Pillow; with one halving first (640 -> 320) as well"""
    S = 256
    for s in (256, 320):
        for flip in (0, 1):
            p = row(h, w, S, s, "max", "max", flip)
            if min(h, w) >> p[2] == s:
                assert (p[3], p[4]) == (h >> p[2], w >> p[2])
            check([img(h, w)], [p], S)


@pytest.mark.parametrize("h,w", [(100, 150), (1, 1), (37, 255), (255, 17), (200, 201)])
def test_upscale(h, w):
    S = 256
    check([img(h, w)], [row(h, w, S, 256, "min", "max", 1), row(h, w, S, 320, "max", "min", 0)], S)


def test_rounding_half_sizes():
    """long sides where (side * scale) lands exactly on .5, so Python's round() (half to even) picks the resized size"""
    S, found = 256, 0
    for short in (384, 400, 480, 300):
        for s in range(256, 321):
            scale = s / short
            for w in range(short + 1, 2 * short):
                if short < 2 * s and (w * scale) % 1.0 == 0.5:
                    p = row(short, w, S, s, "max", "max", 1)
                    check([img(short, w)], [p], S)
                    found += 1
                    break
            if found >= 6:
                return
    assert found >= 3


def test_reference_golden_on_gpu():
    """the stored reference crops directly: GPU output = ToTensor + Normalize of what random_crop_arr / center_crop_arr made"""
    from test_aug_cpu import golden_cases, golden_plan_row
    for g, i, h, w, S, crop in golden_cases():
        got = run([ao.synth_image(int(g["seed"][i]), h, w)], [golden_plan_row(g, i)], S)
        assert torch.equal(got[0], torch.from_numpy(ao.to_tensor_normalize(crop))), f"golden case {i}"


def test_batch_of_128_mixed_sizes():
    """one batch with every depth, both orientations, odd sides, upscales and copies: many CTAs per launch, and the halving
    levels run only on the images that need them"""
    from imagefolder_b200 import data
    rng = np.random.default_rng(5)
    sizes = [(int(a), int(b)) for a, b in rng.integers(200, 1300, size=(116, 2))]
    # short side 5121 >= 16 * 320: four halvings whatever s is drawn; 2600 >= 8 * 320 (and < 16 * 256): three
    sizes += [(5121, 5200), (2600, 3001), (3001, 2600), (1030, 1031), (513, 700), (700, 513), (256, 333), (333, 256),
              (120, 90), (1, 1), (321, 320), (640, 641)]
    assert len(sizes) == 128
    random.seed(3)
    torch.manual_seed(3)
    plan = data.plan_random_crop(sizes, 256)
    assert set(plan[:, 2].tolist()) >= {0, 1, 2, 3, 4} and set(plan[:, 7].tolist()) == {0, 1}
    check([img(h, w, 1) for h, w in sizes], plan, 256)
    check([img(h, w, 2) for h, w in sizes[:64]], data.plan_center_crop(sizes[:64], 256), 256)


def test_small_crop_sizes():
    """S other than 256: fewer columns than threads, a partial last strip (S % 16 != 0)"""
    for S in (1, 24, 100):
        imgs = [img(h, w) for h, w in [(40, 90), (500, 375), (S, S)]]
        random.seed(S)
        torch.manual_seed(S)
        from imagefolder_b200 import data
        check(imgs, data.plan_random_crop([a.shape[:2] for a in imgs], S), S)


class _Synth(torch.utils.data.Dataset):
    """PIL images of mixed sizes, like ImageFolder's pil_loader output."""

    def __init__(self, transform):
        self.sizes = [(375, 500), (500, 333), (600, 800), (256, 300), (1200, 900), (90, 120), (480, 640), (331, 499)] * 2
        self.transform = transform

    def __len__(self):
        return len(self.sizes)

    def __getitem__(self, i):
        from PIL import Image
        h, w = self.sizes[i]
        return self.transform(Image.fromarray(ao.synth_image(i, h, w))), i


def _reference_style_transform(image_size):
    """random_crop_arr (dataset/augmentation.py:29-50) + RandomHorizontalFlip + ToTensor + Normalize written out the reference's
    way, with the oracle's Pillow restatement in place of Image.resize."""
    def f(pil_image):
        import math
        a = np.asarray(pil_image)
        s = random.randrange(math.ceil(image_size / 1.0), math.ceil(image_size / 0.8) + 1)
        while min(a.shape[:2]) >= 2 * s:
            a = ao.resample(a, (a.shape[0] // 2, a.shape[1] // 2), ao.BOX)
        scale = s / min(a.shape[:2])
        a = ao.resample(a, (round(a.shape[0] * scale), round(a.shape[1] * scale)), ao.BICUBIC)
        cy = random.randrange(a.shape[0] - image_size + 1)
        cx = random.randrange(a.shape[1] - image_size + 1)
        a = a[cy:cy + image_size, cx:cx + image_size]
        if torch.rand(1) < 0.5:
            a = a[:, ::-1]
        return torch.from_numpy(ao.to_tensor_normalize(np.ascontiguousarray(a)))
    return f


def test_two_worker_loader_matches_reference_style_loader():
    from torch.utils.data import DataLoader
    from imagefolder_b200 import data
    S = 256
    mk = lambda ds, **k: DataLoader(ds, batch_size=4, num_workers=2, generator=torch.Generator().manual_seed(1234), **k)
    gpu = data.GpuTransformLoader(mk(_Synth(data.GpuDecode(S)), collate_fn=data.collate, pin_memory=True), "cuda", S)
    ref = mk(_Synth(_reference_style_transform(S)))
    n = 0
    for (x, y), (xr, yr) in zip(gpu, ref):
        assert x.is_cuda and x.shape == (4, 3, S, S)
        assert torch.equal(y, yr)
        assert torch.equal(x.cpu(), xr), f"batch {n}"
        n += 1
    assert n == len(gpu) == 4
