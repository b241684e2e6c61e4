"""GPU: the pre-training augmentation kernels (mmae_augment_batch, MMAE_GPU_AUGMENT) against tests/augment_oracle.py.

1. 512 seeded samples at S = 224 and 64 (images around 500 x 375 and the golden fixtures' sizes: large downscales,
   upscales of a few pixels, very thin crops, the identity size), both flips, both mean / std choices: every rgb, depth
   and semseg tensor equals the oracle bitwise.
2. End to end: a DataLoader with 2 workers over a seeded image-folder tree (PNG files), once with the reference's transform
   (the stand-in utils package under tests/augment_standin) and once with the switch's crop-only dataset and loader: the
   batches are bitwise equal, the targets identical, and the switch's batches live on the GPU."""
import os
import random
import sys

import numpy as np
import pytest
import torch

import augment_oracle as AO
from multimae_b200 import data as D

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STANDIN = os.path.join(ROOT, "tests", "augment_standin")
FIXTURE_SIZES = [(375, 500), (500, 375), (480, 360), (300, 420), (256, 192), (40, 30), (24, 32), (17, 21), (64, 64),
                 (64, 80), (3, 200), (200, 2), (20, 300), (400, 12), (1, 50), (90, 7)]


class _Args:
    def __init__(self, input_size, default_norm, hflip=0.5, data_path="", domains=("rgb", "depth", "semseg")):
        self.input_size, self.hflip, self.imagenet_default_mean_and_std = input_size, hflip, default_norm
        self.data_path, self.all_domains = data_path, list(domains)


@pytest.mark.parametrize("S", [224, 64])
def test_kernels_equal_oracle_bitwise(S):
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(S)
    sizes = FIXTURE_SIZES + [(int(rng.integers(300, 520)), int(rng.integers(300, 520))) for _ in range(48)]
    checked = 0
    for b0 in range(0, 256, 32):
        default_norm = (b0 // 32) % 2 == 1
        t = D.CropOnlyTransform(_Args(S, default_norm))
        samples, expected = [], []
        for n in range(b0, b0 + 32):
            h, w = sizes[n % len(sizes)]
            imgs = AO.make_images(10_000 * S + n % len(sizes), h, w,
                                  tasks=("rgb", "depth", "semseg") if n % 3 else ("semseg", "rgb", "depth"))
            random.seed(n)
            torch.manual_seed(n)
            crops = t(dict(imgs))
            draws = (crops.flip,) + _draws(n, imgs)
            assert draws[3:] == (crops.h, crops.w)
            samples.append((crops, n))
            expected.append(AO.augment(imgs, draws, S, t.mean, t.std))
        by_order = {}
        for s, e in zip(samples, expected):                      # one batch per task order
            by_order.setdefault(tuple(s[0].arrays), []).append((s, e))
        for group in by_order.values():
            packed, target = t.collate([s for s, _ in group])
            out = packed.to_device(dev)
            torch.cuda.synchronize()
            for k, (_, e) in enumerate(group):
                for task, ref in e.items():
                    got = out[task][k].cpu()
                    assert got.dtype == ref.dtype and got.shape == ref.shape, task
                    assert torch.equal(got, ref), (S, b0, k, task, (got != ref).sum().item())
                checked += 1
    assert checked == 256


def _draws(n, imgs):
    """(i, j, h, w) the reference draws for seed n: random.random() first, then get_params of the first task."""
    random.seed(n)
    torch.manual_seed(n)
    random.random()
    first = next(iter(imgs.values()))
    return D.random_resized_crop_params(first.height, first.width)


def _write_tree(root, rng):
    for c in ("class_a", "class_b"):
        for n in range(10):
            h, w = int(rng.integers(150, 420)), int(rng.integers(150, 420))
            imgs = AO.make_images(int(rng.integers(1 << 30)), h, w)
            for task, img in imgs.items():
                os.makedirs(os.path.join(root, task, c), exist_ok=True)
                img.save(os.path.join(root, task, c, "img%02d.png" % n))


def _worker_init(worker_id):
    random.seed(1234 + worker_id)
    torch.manual_seed(1234 + worker_id)
    np.random.seed(1234 + worker_id)


def test_dataloader_end_to_end_bitwise(tmp_path):
    from torch.utils.data import DataLoader
    _write_tree(str(tmp_path), np.random.default_rng(0))
    sys.path.insert(0, STANDIN)
    try:
        import utils.datasets as ud
        args = _Args(96, True, data_path=str(tmp_path))

        def batches(dataset, loader_cls):
            loader = loader_cls(dataset, batch_size=6, shuffle=True, num_workers=2, worker_init_fn=_worker_init,
                                generator=torch.Generator().manual_seed(7), drop_last=True, pin_memory=True)
            return [(x, y) for x, y in loader]
        ref_ds = ud.build_multimae_pretraining_dataset(args)
        gpu_ds = D.build_gpu_augment_dataset(args, ud.build_multimae_pretraining_dataset)
        assert isinstance(gpu_ds.transform, D.CropOnlyTransform)
        ref = batches(ref_ds, DataLoader)
        got = batches(gpu_ds, D._AugmentingDataLoader)
        assert len(ref) == len(got) == 3
        for (rx, ry), (gx, gy) in zip(ref, got):
            assert torch.equal(ry, gy.cpu())
            assert list(rx) == list(gx) == ["rgb", "depth", "semseg"]
            for task in rx:
                assert gx[task].is_cuda and gx[task].dtype == rx[task].dtype
                assert torch.equal(gx[task].cpu(), rx[task]), task
    finally:
        sys.path.remove(STANDIN)
        for m in [m for m in sys.modules if m == "utils" or m.startswith("utils.")]:
            del sys.modules[m]
