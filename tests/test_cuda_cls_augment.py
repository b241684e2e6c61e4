"""GPU: the classification fine-tuning augmentation kernels (mmae_cls_augment_batch, MMAE_GPU_AUGMENT) against
tests/cls_augment_oracle.py.

1. Every op kind forced (both filters, the transposes, identity) at S = 224 and 40, with 1, 2 and 3 RandAugment layers,
   on crops of many sizes, both flips and both resize filters: the fp32 batch equals the oracle bitwise.
2. The golden fixtures (recorded from the live reference) reproduced on the GPU, train and eval; batches drawn with
   magnitudes above 10 (mmax), where the LUT ops' levels leave their range, equal the oracle.
3. End to end: DataLoaders with 2 workers over a seeded JPEG image folder, built through the switch's rebinding of
   build_transform on the stand-in of the reference's utils.datasets (tests/cls_augment_standin), against the stand-in's
   CPU transform: the batches are bitwise equal, the targets identical, and the switch's batches live on the GPU."""
import functools
import os
import random
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from PIL import Image

import cls_augment_oracle as O
from helpers import load_fixture
from multimae_b200 import data as D

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STANDIN = os.path.join(ROOT, "tests", "cls_augment_standin")
GOLDEN = os.path.join(ROOT, "tests", "golden")
FILL = (124, 116, 104)
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def _forced_ops(rng, k, S):
    """The k-th op of a cycle through every kind and argument shape."""
    f = float(rng.choice([0.1, 0.46, 1.0, 1.37, 1.9]))
    filt = D.FILTER_BILINEAR if (k // 17) % 2 == 0 else D.FILTER_BICUBIC
    ops = [D.ClsOp(D.OP_IDENTITY), D.ClsOp(D.OP_INVERT), D.ClsOp(D.OP_POSTERIZE, int(rng.integers(0, 5))),
           D.ClsOp(D.OP_SOLARIZE, int(rng.integers(0, 257))), D.ClsOp(D.OP_SOLARIZE_ADD, int(rng.integers(0, 111))),
           D.ClsOp(D.OP_AUTOCONTRAST), D.ClsOp(D.OP_EQUALIZE), D.ClsOp(D.OP_COLOR, factor=f),
           D.ClsOp(D.OP_CONTRAST, factor=f), D.ClsOp(D.OP_BRIGHTNESS, factor=f), D.ClsOp(D.OP_SHARPNESS, factor=f),
           D.ClsOp(D.OP_AFFINE, matrix=D._rotate_matrix(float(rng.uniform(-30, 30)) % 360.0, S, S), filt=filt),
           D.ClsOp(D.OP_AFFINE, matrix=(1., float(rng.uniform(-.3, .3)), 0., 0., 1., 0.), filt=filt),
           D.ClsOp(D.OP_AFFINE, matrix=(1., 0., 0., float(rng.uniform(-.3, .3)), 1., 0.), filt=filt),
           D.ClsOp(D.OP_AFFINE, matrix=(1., 0., float(rng.uniform(-.45, .45)) * S, 0., 1., 0.), filt=filt),
           D.ClsOp(D.OP_TRANSPOSE, [90, 180, 270][k % 3]),
           D.ClsOp(D.OP_AFFINE, matrix=(1., 0., 0., 0., 1., float(rng.uniform(-.45, .45)) * S), filt=filt)]
    return ops[k % len(ops)]


@pytest.mark.parametrize("S", [224, 40])
@pytest.mark.parametrize("layers", [1, 2, 3])
def test_kernels_equal_oracle_bitwise(S, layers):
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(S * 10 + layers)
    B = 40
    samples = []
    for b in range(B):
        h, w = int(rng.integers(3, 500)), int(rng.integers(3, 500))
        if b % 8 == 0:
            h, w = S, S
        crop = O.make_image(int(rng.integers(1 << 30)), h, w, flat=(9, 99, 199) if b % 13 == 5 else None)
        ops = [_forced_ops(rng, b * layers + l, S) for l in range(layers)]
        samples.append(D.ClsSample(crop, D.FILTER_BICUBIC if b % 3 else D.FILTER_BILINEAR, b % 2 == 1, ops))
    packed = D.pack_cls_batch(samples, S, MEAN, STD, FILL)
    out = packed.to_device(dev)
    torch.cuda.synchronize()
    assert out.shape == (B, 3, S, S) and out.dtype == torch.float32
    for b, s in enumerate(samples):
        ref = O.train_sample(s, S, MEAN, STD, FILL)
        got = out[b].cpu()
        assert torch.equal(got, ref), (b, [o.kind for o in s.ops], (got != ref).sum().item())


def test_fixtures_reproduced_on_gpu():
    dev = torch.device("cuda:0")
    fx = load_fixture(GOLDEN, "cls_augment.pt")
    S = fx["input_size"]
    groups = {}
    for c in fx["cases"]:
        args = SimpleNamespace(input_size=S, imagenet_default_mean_and_std=c["default_norm"], aa=c.get("aa"),
                               train_interpolation=c.get("interp"), crop_pct=224 / 256)
        t = D.ClsTrainTransform(args) if c["train"] else D.ClsEvalTransform(args)
        random.seed(c["seed"])
        np.random.seed(c["seed"])
        torch.manual_seed(c["seed"])
        rec = t(Image.fromarray(O.make_image(c["seed"], *c["size"])))
        groups.setdefault((c["train"], c.get("aa"), c.get("interp"), c["default_norm"]), (t, []))[1].append((rec, c))
    n = 0
    for t, items in groups.values():
        packed, _ = t.collate([(rec, 0) for rec, _ in items])
        out = packed.to_device(dev)
        torch.cuda.synchronize()
        for k, (_, c) in enumerate(items):
            assert torch.equal(out[k].cpu(), c["out"]), c["seed"]
            n += 1
    assert n == len(fx["cases"]) == 68


@pytest.mark.parametrize("aa", ["rand-m15-mmax30-mstd3-n2-inc1", "rand-m15-mmax30-mstd3-n2", "rand-m30-mmax30-n3"])
def test_high_magnitude_batches_equal_oracle(aa):
    """Magnitudes above 10 (mmax): a batch of 128 drawn by the workers, with LUT ops whose levels left their range,
    plus every LUT op forced at magnitudes 15 and 30."""
    dev = torch.device("cuda:0")
    S = 64
    t = D.ClsTrainTransform(SimpleNamespace(input_size=S, imagenet_default_mean_and_std=False, aa=aa,
                                            train_interpolation="random"))
    rng = np.random.default_rng(3)
    random.seed(1)
    np.random.seed(1)
    torch.manual_seed(1)
    recs = [t(Image.fromarray(O.make_image(int(rng.integers(1 << 30)), int(rng.integers(40, 200)),
                                           int(rng.integers(40, 200))))) for _ in range(128)]
    names = ["Posterize", "PosterizeIncreasing", "Solarize", "SolarizeIncreasing", "SolarizeAdd"]
    for k, (name, m) in enumerate((n, m) for n in names for m in (15.0, 30.0)):
        recs[k].ops[0] = t.ra.level_op(name, m, S)
    packed, _ = t.collate([(r, 0) for r in recs])
    out = packed.to_device(dev)
    torch.cuda.synchronize()
    for b, r in enumerate(recs):
        ref = O.train_sample(r, S, t.mean, t.std, t.fill)
        assert torch.equal(out[b].cpu(), ref), (b, r.ops)


def _write_tree(root, rng):
    for c in ("class_a", "class_b"):
        os.makedirs(os.path.join(root, c), exist_ok=True)
        for n in range(10):
            h, w = int(rng.integers(150, 420)), int(rng.integers(150, 420))
            Image.fromarray(O.make_image(int(rng.integers(1 << 30)), h, w)).save(
                os.path.join(root, c, "img%02d.jpg" % n), quality=90)


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
        stock = ud.build_transform

        def batches(loader_cls, is_train):
            args = SimpleNamespace(input_size=96, imagenet_default_mean_and_std=True, aa="rand-m9-mstd0.5-inc1",
                                   train_interpolation="random", reprob=0.0, crop_pct=None, data_path=str(tmp_path),
                                   eval_data_path=str(tmp_path), nb_classes=2)
            ds, _ = ud.build_dataset(is_train, args)
            loader = loader_cls(ds, batch_size=6, shuffle=True, num_workers=2, worker_init_fn=_worker_init,
                                generator=torch.Generator().manual_seed(7), drop_last=True, pin_memory=True)
            return ds, [(x, y) for x, y in loader]
        for is_train in (True, False):
            ud.build_transform = stock
            _, ref = batches(DataLoader, is_train)
            ud.build_transform = functools.partial(D.build_gpu_cls_transform, stock=stock)
            ds, got = batches(D._AugmentingDataLoader, is_train)
            assert isinstance(ds.transform, D.ClsTrainTransform if is_train else D.ClsEvalTransform)
            assert len(ref) == len(got) == 3
            for (rx, ry), (gx, gy) in zip(ref, got):
                assert torch.equal(ry, gy.cpu())
                assert gx.is_cuda and gx.dtype == rx.dtype and gx.shape == rx.shape
                assert torch.equal(gx.cpu(), rx), is_train
    finally:
        sys.path.remove(STANDIN)
        for m in [m for m in sys.modules if m == "utils" or m.startswith("utils.")]:
            del sys.modules[m]
