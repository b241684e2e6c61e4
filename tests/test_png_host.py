"""CPU: the worker half of the GPU PNG decode (multimae_b200/png.py, data.load_pretrain_image, pack_batch) and its NumPy
oracle (tests/png_oracle.py).

1. The oracle equals Image.open(f) + the reference's convert bitwise on PNGs written here: every task's stored forms,
   sizes 1x1 to 4100 wide, filter types 0-4 alone and mixed, zlib levels 0-9 and every strategy, IDAT in 1 to 10
   chunks; and on PNGs Pillow writes.
2. The parser hands every other file to Pillow: interlaced, tRNS, 1 / 2 / 4-bit, 16-bit RGB, alpha, APNG, bad CRCs,
   JPEG and non-image files, and stored forms a task's conversion does not copy.
3. The loader under MMAE_GPU_JPEG makes the same draws as without it and leaves Python's, NumPy's and torch's generators
   in the same state after every sample; the packed batch carries each stream and its rectangle."""
import io
import os
import random
import struct
import sys
import zlib

import numpy as np
import pytest
import torch
from PIL import Image

import augment_oracle as AO
import png_oracle as O
from multimae_b200 import data as D
from multimae_b200 import png as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STANDIN = os.path.join(ROOT, "tests", "augment_standin")


def _pillow(data, task):
    return np.asarray(D._load_with_pillow(io.BytesIO(data), task))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_equals_pillow(seed):
    for name, task, data in O.corpus(seed):
        src = P.parse(data, task)
        assert src is not None, name
        ref = _pillow(data, task)
        got = O.decode(src, task)
        assert got.dtype == ref.dtype and np.array_equal(got, ref), name


@pytest.mark.parametrize("level", range(10))
@pytest.mark.parametrize("strategy", O.STRATEGIES)
def test_levels_and_strategies(level, strategy):
    rng = np.random.default_rng(level * 7 + strategy)
    w, h = 61, 23
    rows = O.samples(rng, 8, 2, h, w)
    for filters in ([0] * h, [1] * h, [2] * h, [3] * h, [4] * h, [int(f) for f in rng.integers(0, 5, h)]):
        data = O.encode(rows, w, h, 8, 2, filters, level=level, strategy=strategy, chunks=1 + level)
        src = P.parse(data, "rgb")
        assert np.array_equal(O.decode(src, "rgb"), _pillow(data, "rgb"))


def test_pillow_written_files():
    rng = np.random.default_rng(5)
    imgs = AO.make_images(11, 37, 53)                          # the forms the pre-training folders hold
    imgs["semseg"].putpalette(list(range(256)) * 3)           # Pillow writes a short palette with fewer bits
    for task, img in imgs.items():
        f = io.BytesIO()
        img.save(f, format="PNG")
        data = f.getvalue()
        src = P.parse(data, task)
        assert src is not None and src.mode == img.mode, task
        assert np.array_equal(O.decode(src, task), _pillow(data, task)), task
    for mode in ("L", "P", "RGB"):
        f = io.BytesIO()
        Image.fromarray(rng.integers(0, 256, (20, 30, 3), dtype=np.uint8)).convert(mode).save(f, format="PNG",
                                                                                               optimize=True)
        assert np.array_equal(O.decode(P.parse(f.getvalue(), "rgb"), "rgb"), _pillow(f.getvalue(), "rgb"))


def test_semseg_conversion_is_an_identity_for_l_and_p():
    """Image.convert('P') keeps a palette image's indices and maps gray level g to index g: the kernels copy both."""
    rng = np.random.default_rng(1)
    a = rng.integers(0, 256, (9, 13), dtype=np.uint8)
    for mode in ("L", "P"):
        img = Image.fromarray(a, "L") if mode == "L" else Image.fromarray(a, "P")
        assert np.array_equal(np.asarray(img.convert("P")), a)


def _one(w=9, h=5, depth=8, ctype=2, **kw):
    rng = np.random.default_rng(0)
    rows = rng.integers(0, 256, (h, w * {(8, 0): 1, (16, 0): 2, (8, 2): 3, (8, 3): 1, (16, 2): 6, (8, 6): 4,
                                          (8, 4): 2}.get((depth, ctype), 1)), dtype=np.uint8)
    return O.encode(rows, w, h, depth, ctype, **kw)


def _low_bit(depth, ctype=0):
    """A 1 / 2 / 4-bit image as Pillow writes it."""
    a = np.random.default_rng(depth).integers(0, 1 << depth, (6, 11), dtype=np.uint8)
    f = io.BytesIO()
    Image.fromarray(a, "P").save(f, format="PNG", bits=depth)
    return f.getvalue()


def test_parser_decisions():
    ok = _one()
    assert P.parse(ok, "rgb") is not None
    assert P.parse(ok, "depth") is None and P.parse(ok, "semseg") is None       # RGB -> 'P' is not a copy
    assert P.parse(_one(depth=16, ctype=0), "depth") is not None
    assert P.parse(_one(depth=16, ctype=0), "rgb") is None
    assert P.parse(_one(ctype=0), "depth") is None                                # 'L' depth: the transform refuses it
    assert P.parse(_one(ctype=0), "semseg_coco") is not None
    refused = {
        "interlaced": _one(interlace=1),
        "tRNS": _one(extra=[(b"tRNS", b"\0\1\0\2\0\3")]),
        "16-bit RGB": _one(depth=16, ctype=2),
        "RGBA": _one(ctype=6),
        "gray + alpha": _one(ctype=4),
        "APNG": _one(extra=[(b"acTL", struct.pack(">II", 1, 0))]),
        "iCCP": _one(extra=[(b"iCCP", b"x\0\0" + zlib.compress(b"profile"))]),
        "JPEG": _jpeg(),
        "text": b"hello world, not an image",
    }
    for depth in (1, 2, 4):
        refused["%d-bit" % depth] = _low_bit(depth)
    bad_crc = bytearray(ok)
    bad_crc[8 + 8 + 13] ^= 1                                                      # IHDR's CRC
    refused["bad IHDR CRC"] = bytes(bad_crc)
    for name, data in refused.items():
        assert P.parse(data, "rgb") is None, name
    # Pillow checks the CRCs of the chunks before the image data only
    idat = ok.index(b"IDAT")
    length = struct.unpack_from(">I", ok, idat - 4)[0]
    late = bytearray(ok)
    late[idat + 4 + length] ^= 1
    assert P.parse(bytes(late), "rgb") is not None
    assert np.array_equal(_pillow(bytes(late), "rgb"), _pillow(ok, "rgb"))
    harmless = _one(extra=[(b"gAMA", struct.pack(">I", 45455)), (b"pHYs", struct.pack(">IIB", 1, 1, 0))])
    assert P.parse(harmless, "rgb") is not None


def _jpeg():
    f = io.BytesIO()
    Image.new("RGB", (8, 8), (10, 20, 30)).save(f, format="JPEG")
    return f.getvalue()


def _write_tree(root, rng, n=6):
    """rgb as JPEG or PNG (RGB, L or P), depth as 16-bit PNG, semseg as 'P' or 'L' PNG; mixed sizes."""
    for k in range(n):
        h, w = int(rng.integers(40, 120)), int(rng.integers(40, 120))
        imgs = AO.make_images(int(rng.integers(1 << 30)), h, w)
        imgs["semseg"].putpalette(list(range(256)) * 3)       # 8-bit: Pillow writes a short palette with fewer bits
        rgb = imgs["rgb"].convert(("RGB", "L", "P")[k % 3]) if k % 4 else imgs["rgb"]
        for task, img, ext in (("rgb", rgb, ".jpg" if k % 4 == 0 else ".png"), ("depth", imgs["depth"], ".png"),
                               ("semseg", imgs["semseg"] if k % 2 else imgs["semseg"].convert("L"), ".png")):
            os.makedirs(os.path.join(root, task, "c"), exist_ok=True)
            img.save(os.path.join(root, task, "c", "img%02d%s" % (k, ext)))


class _Args:
    def __init__(self, data_path, input_size=64):
        self.input_size, self.hflip, self.imagenet_default_mean_and_std = input_size, 0.5, True
        self.data_path, self.all_domains = data_path, ["rgb", "depth", "semseg"]


def _states():
    return random.getstate(), np.random.get_state()[1].tobytes(), torch.get_rng_state()


def test_loader_makes_the_same_draws_and_packs_the_tables_in_the_host_part(tmp_path):
    _write_tree(str(tmp_path), np.random.default_rng(0))
    sys.path.insert(0, STANDIN)
    try:
        import utils.datasets as ud
        args = _Args(str(tmp_path))
        folder = ud.MultiTaskImageFolder(args.data_path, args.all_domains, transform=D.CropOnlyTransform(args))
        comp = D.CompressedMultiTaskImages(folder)
        assert len(comp) == len(folder) == 6 and comp.transform is folder.transform
        kinds = set()
        samples = []
        for i in range(len(folder)):
            for seed in range(3):
                random.seed(seed)
                np.random.seed(seed)
                torch.manual_seed(seed)
                ref, ry = folder[i]
                after = _states()
                random.seed(seed)
                np.random.seed(seed)
                torch.manual_seed(seed)
                got, gy = comp[i]
                assert _states()[0] == after[0] and _states()[1] == after[1]
                assert torch.equal(_states()[2], after[2])
                assert ry == gy and (ref.flip, ref.h, ref.w) == (got.flip, got.h, got.w)
                for task, a in ref.arrays.items():
                    g = got.arrays[task]
                    assert isinstance(g, tuple), (i, task)       # every file of this tree is one the kernels decode
                    src, (y, x, h, w) = g
                    kinds.add(type(src).__name__)
                    full = O.decode(src, task) if isinstance(src, P.PngSource) else _pillow(src.data, "rgb")
                    assert np.array_equal(full[y:y + h, x:x + w], a), (i, task)
            samples.append((got, gy))
        assert kinds == {"JpegSource", "PngSource"}
        packed, target = folder.transform.collate(samples)
        assert packed.jpeg is not None and packed.png is not None and packed.device_bytes > packed.buffer.numel()
        buf = packed.buffer.numpy()
        pdesc = buf[packed.png[0] * 16:].view(np.int32)[:packed.png[1] * D.PNG_FIELDS].reshape(-1, D.PNG_FIELDS)
        desc = buf[:len(samples) * 3 * D.DESC_FIELDS * 4].view(np.int32).reshape(len(samples), 3, D.DESC_FIELDS)
        k = 0
        for b, (c, _) in enumerate(samples):
            for t, task in enumerate(packed.tasks):
                src, rect = c.arrays[task]
                assert desc[b, t, 1] * 16 >= packed.buffer.numel()               # the crop lies in the device tail
                if isinstance(src, P.PngSource):
                    d = pdesc[k]
                    assert list(d[:5]) == [src.width, src.height, src.depth, src.ctype, D.AUGMENT_KINDS[task]]
                    assert bytes(buf[d[5] * 16:d[5] * 16 + d[6]]) == src.stream
                    assert tuple(d[8:12]) == rect and d[12] == desc[b, t, 1]
                    assert packed.png_files[k][:3] == (src.path, task, d[12] * 16)
                    k += 1
        assert k == packed.png[1]
        assert int(desc[..., 5:7].max()) * 16 < packed.buffer.numel()         # the tables lie in the host part
    finally:
        sys.path.remove(STANDIN)
        for m in [m for m in sys.modules if m == "utils" or m.startswith("utils.")]:
            del sys.modules[m]


def test_fallback_files_load_as_the_reference_loads_them(tmp_path):
    path = str(tmp_path / "x.png")
    Image.fromarray(np.zeros((6, 10, 4), np.uint8)).save(path)                  # RGBA
    got = D.load_pretrain_image(path, "rgb")
    assert isinstance(got, Image.Image) and got.mode == "RGB"
    bad = str(tmp_path / "bad.png")
    with open(bad, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\nnot really")
    with pytest.raises(Exception) as ref:
        D._load_with_pillow(bad, "rgb")
    with pytest.raises(type(ref.value)):
        D.load_pretrain_image(bad, "rgb")
