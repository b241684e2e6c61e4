"""CPU: the GPU pre-training augmentation (MMAE_GPU_AUGMENT, multimae_b200.data + mmae_augment_batch) without a GPU.

1. tests/augment_oracle.py reproduces the reference's DataAugmentationForMultiMAE outputs of tests/golden/augment.*.pt
   bitwise from the stored draws, and the crop-only transform makes those draws from the stored seeds.
2. The host's resampling tables, evaluated with numpy integer / double arithmetic in the order the kernels use, equal
   Pillow's resize bitwise: BICUBIC for 'RGB' and 'I;16', NEAREST for 'P', on several hundred random size pairs.
3. Packing: descriptor table, table and crop offsets, scratch layout.
4. The overlay switch: the rebinding, each fallback line and the ValueError of a depth image that is not 'I;16'.
5. mmae_augment_batch refuses bad arguments before any launch."""
import ctypes
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch
from PIL import Image

import augment_oracle as AO
from helpers import load_fixture
from multimae_b200 import _lib as L
from multimae_b200 import data as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STANDIN = os.path.join(ROOT, "tests", "augment_standin")


@pytest.fixture(scope="module")
def fx(golden_dir):
    return load_fixture(golden_dir, "augment.pt")


class _Args:
    def __init__(self, input_size=64, hflip=0.5, default_norm=False, domains=("rgb", "depth", "semseg"), data_path=""):
        self.input_size, self.hflip, self.imagenet_default_mean_and_std = input_size, hflip, default_norm
        self.all_domains, self.data_path = list(domains), data_path


def _norm(default):
    return (AO.DEFAULT_MEAN, AO.DEFAULT_STD) if default else (AO.INCEPTION_MEAN, AO.INCEPTION_STD)


def test_oracle_reproduces_reference_fixtures(fx):
    assert len(fx["cases"]) >= 30
    for c in fx["cases"]:
        imgs = AO.make_images(c["seed"], *c["size"])
        out = AO.augment(imgs, c["draws"], fx["input_size"], *_norm(c["default_norm"]))
        for task in ("rgb", "depth", "semseg"):
            assert out[task].dtype == c[task].dtype and torch.equal(out[task], c[task]), (c["seed"], c["size"], task)


def test_crop_only_transform_makes_the_reference_draws(fx):
    for c in fx["cases"]:
        imgs = AO.make_images(c["seed"], *c["size"])
        random.seed(c["seed"])
        torch.manual_seed(c["seed"])
        crops = D.CropOnlyTransform(_Args(fx["input_size"], fx["hflip"], c["default_norm"]))(imgs)
        flip, i, j, h, w = c["draws"]
        assert (crops.flip, crops.h, crops.w) == (flip, h, w), c["seed"]
        assert list(crops.arrays) == ["rgb", "depth", "semseg"]
        for task, img in imgs.items():
            np.testing.assert_array_equal(crops.arrays[task], np.asarray(img)[i:i + h, j:j + w])
        assert crops.arrays["depth"].dtype == np.uint16


def test_draws_and_rng_streams_match_torchvision():
    transforms = pytest.importorskip("torchvision.transforms")
    img = Image.new("RGB", (9, 7))
    for seed in range(200):
        h, w = [(7, 9), (375, 500), (2, 300), (300, 3), (64, 64)][seed % 5]
        torch.manual_seed(seed)
        ref = transforms.RandomResizedCrop.get_params(img.resize((w, h)), scale=(0.2, 1.0), ratio=(0.75, 1.3333))
        ref_state = torch.get_rng_state()
        torch.manual_seed(seed)
        assert D.random_resized_crop_params(h, w) == tuple(ref), seed
        assert torch.equal(torch.get_rng_state(), ref_state), seed


# ---- 2. tables against Pillow --------------------------------------------------------------------------------------
def _pass8(a, bounds, fixed):
    """One bicubic pass over axis 1 of uint8 a [rows, n_in, C]: the kernels' int32 fixed-point sum and clip."""
    out = np.empty((a.shape[0], len(bounds)) + a.shape[2:], np.int64)
    for o, (lo, cnt) in enumerate(bounds):
        ss = np.full((a.shape[0],) + a.shape[2:], 1 << 21, np.int64)
        for k in range(cnt):
            ss += a[:, lo + k].astype(np.int64) * int(fixed[o, k])
        assert np.all(np.abs(ss) < 2 ** 31)
        out[:, o] = np.clip(ss >> 22, 0, 255)
    return out


def _pass16(a, bounds, w):
    """One bicubic pass over axis 1 of uint16 a [rows, n_in]: the kernels' double sum, rounding and byte-wise clip."""
    out = np.empty((a.shape[0], len(bounds)), np.int64)
    for o, (lo, cnt) in enumerate(bounds):
        ss = np.zeros(a.shape[0])
        for k in range(cnt):
            ss = ss + a[:, lo + k].astype(np.float64) * w[o, k]
        si = np.where(ss >= 0, ss + 0.5, ss - 0.5).astype(np.int64)
        lo8 = np.clip(np.fmod(si, 256), 0, 255)
        hi8 = np.clip(si >> 8, 0, 255)
        out[:, o] = lo8 | (hi8 << 8)
    return out


def _resize_tables(a, S, sixteen):
    h, w = a.shape[:2]
    bw, ww = D.bicubic_coeffs(w, S)
    bh, wh = D.bicubic_coeffs(h, S)
    if sixteen:
        tmp = _pass16(a, bw, ww)
        return _pass16(tmp.T, bh, wh).T
    tmp = _pass8(a, bw, D.fixed_point_coeffs(ww))
    return _pass8(tmp.transpose(1, 0, 2), bh, D.fixed_point_coeffs(wh)).transpose(1, 0, 2)


def test_tables_equal_pillow_on_random_size_pairs():
    rng = np.random.default_rng(7)
    pairs = 0
    for n in range(300):
        h, w = (int(v) for v in rng.integers(1, 160, 2))
        S = int(rng.integers(1, 130))
        saturated = n % 3 == 0      # 0 / max pixels: bicubic overshoot on both sides
        img8 = (rng.integers(0, 2, (h, w, 3)) * 255 if saturated else rng.integers(0, 256, (h, w, 3))).astype(np.uint8)
        ref8 = np.asarray(Image.fromarray(img8, "RGB").resize((S, S)))
        np.testing.assert_array_equal(_resize_tables(img8, S, False), ref8, err_msg=str((h, w, S)))
        img16 = (rng.integers(0, 2, (h, w)) * 65535 if saturated else rng.integers(0, 65536, (h, w))).astype(np.uint16)
        pil16 = Image.frombuffer("I;16", (w, h), img16.astype("<u2").tobytes(), "raw", "I;16", 0, 1)
        ref16 = np.asarray(pil16.resize((S, S)))
        np.testing.assert_array_equal(_resize_tables(img16, S, True), ref16, err_msg=str((h, w, S)))
        lab = rng.integers(0, 256, (h, w)).astype(np.uint8)
        refp = np.asarray(Image.frombytes("P", (w, h), lab.tobytes()).resize((S, S)))
        np.testing.assert_array_equal(lab[D.nearest_map(h, S)][:, D.nearest_map(w, S)], refp, err_msg=str((h, w, S)))
        pairs += 1
    assert pairs == 300


def test_fixed_point_rounds_half_away_from_zero():
    w = np.array([0.5 / 2 ** 22, -0.5 / 2 ** 22, 1.0, -0.25, 1.5 / 2 ** 22])
    np.testing.assert_array_equal(D.fixed_point_coeffs(w), [1, -1, 1 << 22, -(1 << 20), 2])


# ---- 3. packing ----------------------------------------------------------------------------------------------------
def test_pack_layout():
    rng = np.random.default_rng(3)
    S = 64
    crops = []
    for b, (h, w) in enumerate([(30, 50), (30, 50), (100, 7)]):
        arrays = {"depth": rng.integers(0, 65536, (h, w)).astype(np.uint16),
                  "rgb": rng.integers(0, 256, (h, w, 3)).astype(np.uint8),
                  "semseg": rng.integers(0, 40, (h, w)).astype(np.uint8)}
        crops.append(D.Crops(arrays, b == 1, h, w))
    pb = D.pack_batch(crops, S, AO.DEFAULT_MEAN, AO.DEFAULT_STD)
    assert pb.tasks == ["depth", "rgb", "semseg"] and pb.batch == 3 and pb.size == S
    buf = pb.buffer.numpy()
    assert buf.size % 16 == 0
    desc = buf[:3 * 3 * D.DESC_FIELDS * 4].view(np.int32).reshape(3, 3, D.DESC_FIELDS)

    def table(off16):
        return buf[off16 * 16:].view(np.int32)
    m4 = table(pb.map4)
    assert list(m4[:4]) == [S, S // 4, 0, D.TABLE_NEAREST]
    np.testing.assert_array_equal(m4[4:4 + S // 4], D.nearest_map(S, S // 4))
    scratch_ends = []
    for b, c in enumerate(crops):
        for t, task in enumerate(pb.tasks):
            d = desc[b, t]
            kind = D.AUGMENT_KINDS[task]
            assert list(d[:5]) == [kind, d[1], c.h, c.w, int(c.flip)]
            a = c.arrays[task]
            np.testing.assert_array_equal(buf[d[1] * 16:d[1] * 16 + a.nbytes], a.reshape(-1).view(np.uint8))
            for off, n_in in ((d[5], c.w), (d[6], c.h)):
                tab = table(off)
                if kind == 2:
                    assert list(tab[:4]) == [n_in, S, 0, D.TABLE_NEAREST]
                    np.testing.assert_array_equal(tab[4:4 + S], D.nearest_map(n_in, S))
                else:
                    bounds, w = D.bicubic_coeffs(n_in, S)
                    k = w.shape[1]
                    assert list(tab[:4]) == [n_in, S, k, D.TABLE_BICUBIC]
                    np.testing.assert_array_equal(tab[4:4 + 2 * S], bounds.reshape(-1))
                    np.testing.assert_array_equal(tab[4 + 2 * S:4 + 2 * S + S * k], D.fixed_point_coeffs(w).reshape(-1))
                    dbl = ((16 + 8 * S + 4 * S * k + 7) // 8) * 8
                    np.testing.assert_array_equal(buf[off * 16 + dbl:off * 16 + dbl + 8 * S * k].view(np.float64),
                                                  w.reshape(-1))
            if kind != 2:
                scratch_ends.append((d[7] * 16, d[7] * 16 + c.h * S * a.itemsize * (3 if kind == 0 else 1)))
    scratch_ends.sort()
    for (s0, e0), (s1, _) in zip(scratch_ends, scratch_ends[1:]):
        assert e0 <= s1
    assert scratch_ends[-1][1] <= pb.scratch_bytes
    # same size pairs share one table: crops 0 and 1 have the same size
    assert desc[0, 1, 5] == desc[1, 1, 5] and desc[0, 1, 6] == desc[1, 1, 6]


def test_collate_and_pinning_keep_targets():
    t = D.CropOnlyTransform(_Args())
    imgs = AO.make_images(5, 40, 60)
    samples = [(t(dict(imgs)), k) for k in (3, 1)]
    packed, target = t.collate(samples)
    assert isinstance(packed, D.PackedBatch) and target.dtype == torch.int64 and target.tolist() == [3, 1]


# ---- 4. overlay switch ---------------------------------------------------------------------------------------------
def _run(env_extra, body):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([STANDIN, os.path.join(ROOT, "tests"), ROOT]), **env_extra)
    env.pop("MMAE_DEVICE_FEED", None)
    code = "import sys\nimport torch.utils.data as tud\nfrom multimae_b200 import data as D\n" + body
    return subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)


def test_switch_off_changes_nothing():
    r = _run({"MMAE_GPU_AUGMENT": "0"}, "import utils.datasets as ud\nstock = ud.build_multimae_pretraining_dataset\n"
             "stock_dl = tud.DataLoader\nprint(D.install())\n"
             "assert ud.build_multimae_pretraining_dataset is stock and tud.DataLoader is stock_dl\n")
    assert r.returncode == 0, r.stderr
    assert r.stdout.strip() == "[]" and "MMAE_GPU_AUGMENT" not in r.stdout


def test_switch_rebinds_builder_and_loader():
    r = _run({"MMAE_GPU_AUGMENT": "1"}, "import utils.datasets as ud\nprint(D.install())\n"
             "assert ud.build_multimae_pretraining_dataset.keywords['stock'].__module__ == 'utils.datasets'\n"
             "assert tud.DataLoader is D._AugmentingDataLoader\n")
    assert r.returncode == 0, r.stderr
    assert r.stdout.strip() == "['gpu_augment']"


def test_synthetic_data_wins():
    r = _run({"MMAE_GPU_AUGMENT": "1", "MMAE_SYNTHETIC_DATA": "16"}, "print(D.install())\n")
    assert r.returncode == 0, r.stderr
    lines = r.stdout.strip().splitlines()
    assert lines[0].startswith("MMAE_GPU_AUGMENT:") and "MMAE_SYNTHETIC_DATA" in lines[0]
    assert lines[1] == "['synthetic']"


def test_fallback_lines(monkeypatch, capsys):
    sys.path.insert(0, STANDIN)
    try:
        import utils.datasets as ud  # the stand-in
        stock_calls = []

        def stock(args):
            stock_calls.append(args)
            return "stock"
        monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
        assert D.build_gpu_augment_dataset(_Args(domains=("rgb", "normal")), stock) == "stock"
        out = capsys.readouterr().out.strip().splitlines()
        assert len(out) == 1 and out[0].startswith("MMAE_GPU_AUGMENT:") and "normal" in out[0]
        monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
        assert D.build_gpu_augment_dataset(_Args(), stock) == "stock"
        out = capsys.readouterr().out.strip().splitlines()
        assert len(out) == 1 and out[0].startswith("MMAE_GPU_AUGMENT:") and "CUDA" in out[0]
        assert len(stock_calls) == 2
        assert ud.__file__.startswith(STANDIN)
    finally:
        sys.path.remove(STANDIN)
        for m in [m for m in sys.modules if m == "utils" or m.startswith("utils.")]:
            del sys.modules[m]


def test_depth_that_is_not_16_bit_is_refused():
    imgs = AO.make_images(1, 30, 40)
    imgs["depth"] = imgs["depth"].convert("I")
    with pytest.raises(ValueError, match=r"MMAE_GPU_AUGMENT.*'I'"):
        D.CropOnlyTransform(_Args())(imgs)


# ---- 5. C ABI ------------------------------------------------------------------------------------------------------
def test_entry_point_validates_before_any_launch():
    lib = L.lib()
    S = 64
    crops = [D.Crops({"rgb": np.zeros((20, 30, 3), np.uint8), "depth": np.zeros((20, 30), np.uint16),
                      "semseg": np.zeros((20, 30), np.uint8)}, False, 20, 30)]
    pb = D.pack_batch(crops, S, AO.DEFAULT_MEAN, AO.DEFAULT_STD)
    good = pb.buffer.clone()
    base = 1 << 20                 # fake, 16-byte aligned device addresses: nothing is launched

    def call(buf=None, nbytes=None, batch=1, T=3, kinds=(0, 1, 2), size=S, map4=None, scratch=base, sbytes=None,
             outs=(base, base, base), mean=AO.DEFAULT_MEAN, std=AO.DEFAULT_STD, dev=base):
        buf = good if buf is None else buf
        return lib.mmae_augment_batch(buf.data_ptr(), dev, buf.numel() if nbytes is None else nbytes, batch, T,
                                      (ctypes.c_int * len(kinds))(*kinds), size, pb.map4 if map4 is None else map4,
                                      scratch, pb.scratch_bytes if sbytes is None else sbytes,
                                      (ctypes.c_void_p * len(outs))(*outs), (ctypes.c_float * 3)(*mean),
                                      (ctypes.c_float * 3)(*std), None)

    def patched(byte_off, value):
        b = good.clone()
        b.numpy()[byte_off:byte_off + 4].view(np.int32)[0] = value
        return b
    d0 = 0
    rgb_desc = good.numpy()[:96].view(np.int32).reshape(3, 8)
    before = lib.mmae_launch_count()
    cases = [
        (dict(batch=0), "bad batch"),
        (dict(T=9, kinds=(0,) * 9, outs=(base,) * 9), "task count"),
        (dict(size=2), "output size"),
        (dict(dev=base + 4), "16-byte aligned"),
        (dict(nbytes=64), "cannot hold"),
        (dict(kinds=(0, 1, 3)), "bad kind"),
        (dict(kinds=(1, 0, 2)), "kind"),
        (dict(outs=(base, 0, base)), "output pointer"),
        (dict(std=(0.5, 0.0, 0.5)), "mean / std"),
        (dict(map4=rgb_desc[0, 5]), "table at"),
        (dict(sbytes=16), "scratch"),
        (dict(scratch=0), "bad scratch"),
        (dict(buf=patched(d0 + 8, 0)), "bad crop"),
        (dict(buf=patched(d0 + 16, 2)), "flip"),
        (dict(buf=patched(d0 + 4, (good.numel() // 16))), "crop outside"),
        (dict(buf=patched(d0 + 12, 31)), "expected"),
        (dict(buf=patched(rgb_desc[0, 5] * 16 + 16, 29)), "taps"),
        (dict(buf=patched(rgb_desc[2, 5] * 16 + 16, 30)), "nearest index"),
        (dict(buf=patched(rgb_desc[0, 5] * 16 + 8, 10 ** 6)), "tap count"),
    ]
    for kw, msg in cases:
        rc = call(**kw)
        assert rc == 1, kw
        assert msg in lib.mmae_last_error().decode(), (kw, lib.mmae_last_error())
    assert lib.mmae_launch_count() == before
