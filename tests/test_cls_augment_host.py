"""CPU: the classification fine-tuning augmentation of MMAE_GPU_AUGMENT (multimae_b200.data: ClsTrainTransform,
ClsEvalTransform, pack_cls_batch, build_gpu_cls_transform) and its oracle (tests/cls_augment_oracle.py).

1. The oracle equals the installed Pillow bitwise, op by op, called as the reference calls it: random images of several
   sizes (224 and odd sizes), magnitudes 0, 9 and 10 with negated levels, both filters, flat and single-colour images, and
   the angles that take Image.rotate's shortcuts.
2. The golden fixtures (recorded from the live reference by tests/golden/make_golden_cls_augment.py): the workers leave
   Python's, NumPy's and torch's generators in the reference's state after every sample, and the oracle applied to the
   workers' records gives the reference's tensors bitwise, train and eval, both normalisations.
3. The fallbacks keep the reference transform and print one line."""
import hashlib
import os
import random
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from PIL import Image, ImageEnhance, ImageOps

import cls_augment_oracle as O
from helpers import load_fixture
from multimae_b200 import data as D

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FILL = (124, 116, 104)
IMAGES = [(224, 224, None), (37, 53, None), (64, 64, None), (9, 9, None), (31, 31, None), (50, 50, (7, 200, 33)),
          (40, 40, (0, 0, 0))]


def _image(k):
    h, w, flat = IMAGES[k]
    a = O.make_image(100 + k, h, w, flat)
    if flat is None and k == 4:                       # few distinct levels: Equalize / AutoContrast corner cases
        a = (a // 85 * 85).astype(np.uint8)
    return a


def _eq(got, ref):
    ref = np.asarray(ref)
    assert got.shape == ref.shape and np.array_equal(got, ref), int((got != ref).sum())


@pytest.mark.parametrize("k", range(len(IMAGES)))
@pytest.mark.parametrize("filt", [D.FILTER_BILINEAR, D.FILTER_BICUBIC])
def test_resize_equals_pillow(k, filt):
    a = _image(k)
    for S in (224, 48, 31):
        _eq(O.resize(a, S, filt), Image.fromarray(a).resize((S, S), filt))


@pytest.mark.parametrize("k", range(len(IMAGES)))
def test_lut_and_blend_ops_equal_pillow(k):
    a = _image(k)
    img = Image.fromarray(a)
    _eq(O.apply_op(a, D.ClsOp(D.OP_AUTOCONTRAST), FILL), ImageOps.autocontrast(img))
    _eq(O.apply_op(a, D.ClsOp(D.OP_EQUALIZE), FILL), ImageOps.equalize(img))
    _eq(O.apply_op(a, D.ClsOp(D.OP_INVERT), FILL), ImageOps.invert(img))
    for bits in range(0, 8):
        _eq(O.apply_op(a, D.ClsOp(D.OP_POSTERIZE, bits), FILL), ImageOps.posterize(img, bits))
    for m in (0, 9, 10):
        t = int(m / 10 * 256)
        for thresh in (t, 256 - t):
            _eq(O.apply_op(a, D.ClsOp(D.OP_SOLARIZE, thresh), FILL), ImageOps.solarize(img, thresh))
        add = int(m / 10 * 110)
        lut = [min(255, i + add) if i < 128 else i for i in range(256)]
        _eq(O.apply_op(a, D.ClsOp(D.OP_SOLARIZE_ADD, add), FILL), img.point(lut * 3))
    factors = {(m / 10) * 1.8 + 0.1 for m in (0, 9, 10)} | {max(0.1, 1.0 + s * (m / 10) * .9) for m in (0, 9, 10)
                                                           for s in (1, -1)} | {0.37, 1.0}
    for f in sorted(factors):
        _eq(O.apply_op(a, D.ClsOp(D.OP_COLOR, factor=f), FILL), ImageEnhance.Color(img).enhance(f))
        _eq(O.apply_op(a, D.ClsOp(D.OP_CONTRAST, factor=f), FILL), ImageEnhance.Contrast(img).enhance(f))
        _eq(O.apply_op(a, D.ClsOp(D.OP_BRIGHTNESS, factor=f), FILL), ImageEnhance.Brightness(img).enhance(f))
        _eq(O.apply_op(a, D.ClsOp(D.OP_SHARPNESS, factor=f), FILL), ImageEnhance.Sharpness(img).enhance(f))


def _rotate_op(degrees, size, filt):
    angle = degrees % 360.0
    if angle == 0:
        return D.ClsOp(D.OP_IDENTITY)
    if angle in (90, 180, 270):
        return D.ClsOp(D.OP_TRANSPOSE, int(angle))
    return D.ClsOp(D.OP_AFFINE, matrix=D._rotate_matrix(angle, size, size), filt=filt)


@pytest.mark.parametrize("k", [0, 2, 3, 4, 5])
@pytest.mark.parametrize("filt", [D.FILTER_BILINEAR, D.FILTER_BICUBIC])
def test_geometric_ops_equal_pillow(k, filt):
    a = _image(k)
    img = Image.fromarray(a)
    S = a.shape[0]
    for m in (0, 9, 10):
        for sign in (1, -1):
            deg = sign * (m / 10) * 30.
            _eq(O.apply_op(a, _rotate_op(deg, S, filt), FILL), img.rotate(deg, resample=filt, fillcolor=FILL))
            f = sign * (m / 10) * 0.3
            _eq(O.apply_op(a, D.ClsOp(D.OP_AFFINE, matrix=(1., f, 0., 0., 1., 0.), filt=filt), FILL),
                img.transform(img.size, Image.AFFINE, (1, f, 0, 0, 1, 0), resample=filt, fillcolor=FILL))
            _eq(O.apply_op(a, D.ClsOp(D.OP_AFFINE, matrix=(1., 0., 0., f, 1., 0.), filt=filt), FILL),
                img.transform(img.size, Image.AFFINE, (1, 0, 0, f, 1, 0), resample=filt, fillcolor=FILL))
            p = sign * (m / 10) * 0.45
            _eq(O.apply_op(a, D.ClsOp(D.OP_AFFINE, matrix=(1., 0., p * S, 0., 1., 0.), filt=filt), FILL),
                img.transform(img.size, Image.AFFINE, (1, 0, p * S, 0, 1, 0), resample=filt, fillcolor=FILL))
            _eq(O.apply_op(a, D.ClsOp(D.OP_AFFINE, matrix=(1., 0., 0., 0., 1., p * S), filt=filt), FILL),
                img.transform(img.size, Image.AFFINE, (1, 0, 0, 0, 1, p * S), resample=filt, fillcolor=FILL))
    for deg in (90, 180, 270, -90, 360, 0.0, 45.0, 1e-9):            # the shortcuts, and near them
        _eq(O.apply_op(a, _rotate_op(deg, S, filt), FILL), img.rotate(deg, resample=filt, fillcolor=FILL))


def _digest():
    h = hashlib.sha256(repr(random.getstate()).encode())
    st = np.random.get_state()
    h.update(st[1].tobytes() + repr(st[2:]).encode())
    h.update(torch.get_rng_state().numpy().tobytes())
    return h.hexdigest()


def _args(c, size):
    return SimpleNamespace(input_size=size, imagenet_default_mean_and_std=c["default_norm"], color_jitter=0.4,
                           aa=c.get("aa"), train_interpolation=c.get("interp"), reprob=0.0, crop_pct=None)


def test_fixtures_reproduced():
    fx = load_fixture(GOLDEN, "cls_augment.pt")
    S = fx["input_size"]
    assert len(fx["cases"]) == 68
    clamped = 0
    for c in fx["cases"]:
        args = _args(c, S)
        img = Image.fromarray(O.make_image(c["seed"], *c["size"]))
        if c["train"]:
            t = D.ClsTrainTransform(args)
            random.seed(c["seed"])
            np.random.seed(c["seed"])
            torch.manual_seed(c["seed"])
            rec = t(img)
            assert _digest() == c["rng"], c["seed"]
            clamped += sum(_clamped(op) for op in rec.ops)
            got = O.train_sample(rec, S, t.mean, t.std, t.fill)
            assert torch.equal(O.pil_train_sample(rec, S, t.mean, t.std, t.fill), c["out"])
        else:
            args.crop_pct = 224 / 256
            t = D.ClsEvalTransform(args)
            got = O.eval_sample(t(img), S, t.mean, t.std)
            assert torch.equal(O.pil_eval_sample(img, t.resize, S, t.mean, t.std), c["out"])
        assert torch.equal(got, c["out"]), (c["seed"], c.get("aa"), (got != c["out"]).sum().item())
    assert clamped >= 3                       # the mmax configs draw LUT ops whose level left its range


def _clamped(op):
    return (op.kind == D.OP_POSTERIZE and op.iarg == 0) or (op.kind == D.OP_SOLARIZE and op.iarg in (0, 256)) or \
        (op.kind == D.OP_SOLARIZE_ADD and op.iarg == 255)


def _in_kernel_range(op):
    """The argument ranges mmae_cls_augment_batch accepts."""
    return {D.OP_POSTERIZE: 0 <= op.iarg <= 8, D.OP_SOLARIZE: 0 <= op.iarg <= 256, D.OP_SOLARIZE_ADD: 0 <= op.iarg <= 255,
            D.OP_TRANSPOSE: op.iarg in (90, 180, 270)}.get(op.kind, True)


@pytest.mark.parametrize("m", [10.5, 15.0, 23.3, 24.0, 30.0, 100.0])
def test_high_magnitude_lut_ops_equal_pillow(m):
    """Magnitudes above 10 (mmax): the clamped records give what the reference's level arguments give in Pillow."""
    a = _image(0)
    img = Image.fromarray(a)
    ra = D.RandAugmentDraws("rand-m9-mmax100", FILL, D.FILTER_BICUBIC)
    level = m / 10
    bits = int(level * 4)
    t = int(level * 256)
    add = int(level * 110)
    refs = {"Posterize": img if bits >= 8 else ImageOps.posterize(img, bits),
            "PosterizeIncreasing": ImageOps.posterize(img, 4 - bits),
            "Solarize": ImageOps.solarize(img, t), "SolarizeIncreasing": ImageOps.solarize(img, 256 - t),
            "SolarizeAdd": img.point([min(255, i + add) if i < 128 else i for i in range(256)] * 3)}
    for name, ref in refs.items():
        op = ra.level_op(name, m, 224)
        assert _in_kernel_range(op), (name, m, op)
        _eq(O.apply_op(a, op, FILL), ref)


@pytest.mark.parametrize("aa", ["rand-m15-mmax30-mstd3-n2-inc1", "rand-m15-mmax30-mstd3-n2", "rand-m30-mmax30-n3"])
def test_records_stay_in_kernel_ranges(aa):
    t = D.ClsTrainTransform(SimpleNamespace(input_size=48, imagenet_default_mean_and_std=True, aa=aa,
                                            train_interpolation="random"))
    img = Image.fromarray(O.make_image(0, 40, 40))
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)
    ops = [op for _ in range(2000) for op in t(img).ops]
    assert all(_in_kernel_range(op) for op in ops)
    assert any(_clamped(op) for op in ops)


def test_draws_follow_the_config():
    args = SimpleNamespace(input_size=224, imagenet_default_mean_and_std=True, aa="rand-m9-mstd0.5-inc1",
                           train_interpolation="bicubic")
    t = D.ClsTrainTransform(args)
    assert t.ra.num_layers == 2 and t.ra.magnitude == 9 and t.ra.mstd == 0.5 and t.fill == FILL
    assert "PosterizeIncreasing" in t.ra.names and "SolarizeIncreasing" in t.ra.names
    t = D.ClsTrainTransform(SimpleNamespace(input_size=224, imagenet_default_mean_and_std=False,
                                            aa="rand-m10-n3-w0-mmax20", train_interpolation="random"))
    assert t.ra.num_layers == 3 and t.ra.mmax == 20 and t.filter is None and t.fill == (128, 128, 128)
    assert abs(float(np.sum(t.ra.weights)) - 1.0) < 1e-12


def test_pack_layout():
    rng = np.random.default_rng(0)
    samples = [D.ClsSample(O.make_image(k, 30 + k, 40 - k), D.FILTER_BICUBIC if k % 2 else D.FILTER_BILINEAR, k % 2 == 0,
                           [D.ClsOp(D.OP_SOLARIZE, 100 + k), D.ClsOp(D.OP_AFFINE, matrix=rng.random(6), filt=3)])
               for k in range(3)]
    p = D.pack_cls_batch(samples, 32, (0.5,) * 3, (0.5,) * 3, FILL)
    buf = p.buffer.numpy()
    desc = buf[:3 * D.DESC_FIELDS * 4].view(np.int32).reshape(3, D.DESC_FIELDS)
    ops = buf[p.ops_offset * 16:p.ops_offset * 16 + 3 * 2 * 72].view(D.OP_DTYPE).reshape(3, 2)
    for k, s in enumerate(samples):
        h, w = s.crop.shape[:2]
        assert list(desc[k, [0, 2, 3, 4]]) == [0, h, w, int(s.flip)]
        np.testing.assert_array_equal(buf[desc[k, 1] * 16:desc[k, 1] * 16 + h * w * 3], s.crop.reshape(-1))
        col = buf[desc[k, 5] * 16:].view(np.int32)
        assert list(col[:4]) == [w, 32, col[2], D.TABLE_BICUBIC if s.filter == D.FILTER_BICUBIC else D.TABLE_BILINEAR]
        assert ops[k, 0]["kind"] == D.OP_SOLARIZE and ops[k, 0]["iarg"] == 100 + k
        np.testing.assert_array_equal(ops[k, 1]["m"], s.ops[1].matrix)
    assert p.inter_bytes >= sum(s.crop.shape[0] * 32 * 3 for s in samples)


@pytest.mark.parametrize("train,change,expect", [
    (True, dict(reprob=0.25), "--reprob 0.25 > 0 (RandomErasing)"),
    (True, dict(aa=""), "--aa is empty (ColorJitter)"),
    (True, dict(aa=None), "--aa is empty (ColorJitter)"),
    (True, dict(aa="v0"), "--aa v0 is not RandAugment"),
    (True, dict(aa="augmix-m5"), "--aa augmix-m5 is not RandAugment"),
    (True, dict(input_size=32), "input_size 32 <= 32 (RandomCrop with padding)"),
    (False, dict(input_size=32), "input_size 32 <= 32 (RandomCrop with padding)"),
    (True, dict(train_interpolation="lanczos"), "--train_interpolation lanczos"),
])
def test_fallbacks_print_one_line(train, change, expect, capsys, monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    args = SimpleNamespace(input_size=224, imagenet_default_mean_and_std=True, aa="rand-m9-mstd0.5-inc1",
                           train_interpolation="bicubic", reprob=0.0, crop_pct=None)
    for k, v in change.items():
        setattr(args, k, v)
    stock = object()
    assert D.build_gpu_cls_transform(train, args, lambda is_train, a: stock) is stock
    out = capsys.readouterr().out.splitlines()
    assert out == ["MMAE_GPU_AUGMENT: %s; keeping the reference %s transform" % (expect, "train" if train else "eval")]


def test_no_cuda_falls_back(capsys, monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    args = SimpleNamespace(input_size=224, imagenet_default_mean_and_std=True, aa="rand-m9-mstd0.5-inc1",
                           train_interpolation="bicubic", reprob=0.0, crop_pct=None)
    assert D.build_gpu_cls_transform(False, args, lambda is_train, a: "stock") == "stock"
    assert capsys.readouterr().out == "MMAE_GPU_AUGMENT: CUDA is not available; keeping the reference eval transform\n"


def test_switch_builds_gpu_transforms(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    args = SimpleNamespace(input_size=224, imagenet_default_mean_and_std=True, aa="rand-m9-mstd0.5-inc1",
                           train_interpolation="bicubic", reprob=0.0, crop_pct=None)
    assert isinstance(D.build_gpu_cls_transform(True, args, None), D.ClsTrainTransform)
    ev = D.build_gpu_cls_transform(False, args, None)
    assert isinstance(ev, D.ClsEvalTransform) and ev.resize == 256 and args.crop_pct == 224 / 256
    assert ev.transforms == [ev]
