"""GPU: the parallel entropy decode of mmae_jpeg_decode_batch (restart intervals of at least jpeg.PARALLEL_MIN_BYTES,
one CTA each) against the installed Pillow, bitwise, on the whole image and on crops touching each edge.

Each test also reads the subsequence records the decode leaves in its scratch, to check which path every interval the
rectangle needs took: clean intervals the parallel decode, corrupt ones (a code longer than 16 bits, data truncated
before EOI) the sequential kernel.  The corpus is generated from seeds with Pillow: grayscale, 4:4:4, 4:2:2, 4:2:0,
qualities 10 to 100, optimized tables, one MCU up to 4000 x 3000, restart markers, periodic content (slow to
synchronise), a stuffed FF 00 pair on a subsequence boundary, and bit flips.  Corrupt files equal Pillow only where
libjpeg-turbo runs its x86-64 SIMD IDCT, so they are left out elsewhere."""
import io
import os
import random
import sys

import numpy as np
import pytest
import torch
from PIL import Image

import jpeg_oracle as O
from multimae_b200 import data as D
from multimae_b200 import jpeg as J
from multimae_b200 import kernels as K

pytestmark = pytest.mark.gpu

MEAN, STD, FILL = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225), (124, 116, 104)


def _pillow(data):
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def _rects(H, W, rng):
    """The whole image, a strip along each edge and an inner rectangle."""
    h, w = max(1, H // 3), max(1, W // 3)
    i, j = int(rng.integers(0, H - h + 1)), int(rng.integers(0, W - w + 1))
    return [(0, 0, H, W), (0, 0, h, W), (H - h, 0, h, W), (0, 0, H, w), (0, W - w, H, w), (i, j, h, w)]


def _intervals(src, rect):
    """[(interval, parallel)] of the restart intervals the rectangle needs: whether the kernels try it in parallel."""
    mpr, mcu0, mcu1, bpm, _ = J.geometry(src.width, src.height, src.ncomp, src.hmax, src.vmax, *rect)
    total = mpr * -(-src.height // (8 * src.vmax))
    ri = src.restart or total
    out = []
    for k, (a, b) in enumerate(src.intervals):
        first, last = k * ri, min(k * ri + ri, total)
        if first < min(mcu1 * mpr, last) and last > mcu0 * mpr:
            out.append((k, J.parallel_interval(int(b - a))))
    return out


def _decode(items, dev):
    """items: [(bytes, rect)] -> ([decoded rectangle], [[interval, path]] per item: path 'parallel', 'fallback' or
    'sequential')."""
    samples = [D.ClsSample(None, D.FILTER_BICUBIC, False, [], jpeg=(J.parse(data), rect)) for data, rect in items]
    p = D.pack_cls_batch(samples, 32, MEAN, STD, FILL)
    host = p.buffer
    devbuf = torch.zeros(p.device_bytes, dtype=torch.uint8, device=dev)
    devbuf[:host.numel()].copy_(host)
    off, n, coef_blocks, plane_bytes = p.jpeg
    scratch = K.jpeg_decode_batch(host, devbuf, *p.jpeg).cpu().numpy()
    got = devbuf.cpu().numpy()
    buf = host.numpy()
    desc = buf[:len(samples) * D.DESC_FIELDS * 4].view(np.int32).reshape(-1, D.DESC_FIELDS)
    jd = buf[off * 16:off * 16 + n * D.JPEG_FIELDS * 4].view(np.int32).reshape(n, D.JPEG_FIELDS)
    records = scratch[K.jpeg_scratch_bytes(coef_blocks, plane_bytes):].view(np.int32).reshape(-1, 12)
    outs, paths = [], []
    for b, s in enumerate(samples):
        h, w = s.shape
        outs.append(got[desc[b, 1] * 16:desc[b, 1] * 16 + h * w * 3].reshape(h, w, 3))
        src, rect = s.jpeg
        row = []
        for k, par in _intervals(src, rect):
            if not par:
                row.append((k, "sequential"))
                continue
            fallback = records[jd[b, 24] + src.intervals[k][0] // J.SLOT_BYTES + k, 11]
            assert fallback in (0, 1)
            row.append((k, "fallback" if fallback else "parallel"))
        paths.append(row)
    return outs, paths


def _check(files, dev, seed, expect):
    """Decode every file in `files` ([(name, bytes)]) at _rects; each rectangle equals Pillow's and every interval
    the kernels try in parallel takes the path `expect(name)` ('parallel' or 'fallback', None: either)."""
    rng = np.random.default_rng(seed)
    items, refs, names = [], [], []
    for name, data in files:
        assert J.parse(data) is not None, name
        full = _pillow(data)
        for r in _rects(*full.shape[:2], rng):
            items.append((data, r))
            refs.append(full[r[0]:r[0] + r[2], r[1]:r[1] + r[3]])
            names.append(name)
    outs, paths = _decode(items, dev)
    tried = 0
    for name, (data, r), got, ref, row in zip(names, items, outs, refs, paths):
        assert np.array_equal(got, ref), (name, r)
        want = expect(name)
        for k, path in row:
            tried += path != "sequential"
            assert want is None or path in ("sequential", want), (name, r, k, path)
    return tried


def _image(seed, w, h, gray=False, noise=30.0):
    rng = np.random.default_rng(seed)
    x = np.linspace(0, 255, w)[None, :, None] * np.ones((h, 1, 1 if gray else 3))
    a = np.clip(x + rng.normal(0, noise, x.shape), 0, 255).astype(np.uint8)
    return a[..., 0] if gray else a


def test_clean_files_take_the_parallel_decode():
    dev = torch.device("cuda:0")
    files = [("1x1", O.encode(_image(0, 1, 1))), ("8x8 gray", O.encode(_image(1, 8, 8, True), quality=95))]
    for q in (10, 30, 50, 75, 90, 100):
        for ss in (0, 1, 2):
            w, h = (1300, 950 + ss * 7) if q == 10 else (600 + q, 450 + ss * 7)   # 16 KiB of data or more
            files.append(("q%d ss%d" % (q, ss), O.encode(_image(q + ss, w, h), quality=q, subsampling=ss)))
        files.append(("q%d gray" % q, O.encode(_image(q, 833, 571, True), quality=q)))
    for ss in (1, 2):
        files.append(("optimize ss%d" % ss, O.encode(_image(5 + ss, 640, 480), quality=90, subsampling=ss,
                                                      optimize=True)))
    files.append(("optimize gray", O.encode(_image(9, 640, 480, True), quality=85, optimize=True)))
    for name, data in files[2:]:
        assert all(J.parallel_interval(int(b - a)) for a, b in J.parse(data).intervals), name
    tried = _check(files, dev, 0, lambda name: "parallel")
    assert tried >= 100


def test_large_images_span_hundreds_of_subsequences():
    dev = torch.device("cuda:0")
    files = [("4000x3000 ss2", O.encode(_image(11, 4000, 3000, noise=12.0), quality=85, subsampling=2)),
             ("4001x3001 gray", O.encode(_image(12, 4001, 3001, True, noise=8.0), quality=75)),
             ("1500x1100 ss0", O.encode(_image(13, 1500, 1100), quality=95, subsampling=0))]
    for _, data in files:
        src = J.parse(data)
        assert src.restart == 0 and (src.scan[1] - src.scan[0]) // J.SUB_BYTES >= 4 * 256
    _check(files, dev, 1, lambda name: "parallel")


def test_restart_markers():
    dev = torch.device("cuda:0")
    a, g = _image(21, 900, 700), _image(22, 900, 700, True)
    files = []
    for ss in (0, 1, 2):
        for kw in (dict(restart_marker_rows=1), dict(restart_marker_rows=5), dict(restart_marker_blocks=7),
                   dict(restart_marker_blocks=300)):
            files.append(("ss%d %s" % (ss, kw), O.encode(a, quality=92, subsampling=ss, **kw)))
    files.append(("gray rows 3", O.encode(g, quality=90, restart_marker_rows=3)))
    straddle = 0
    for _, data in files:
        src = J.parse(data)
        assert src.restart > 0
        straddle += sum(J.parallel_interval(int(b - a)) and (b - a) % J.SUB_BYTES != 0 for a, b in src.intervals)
    assert straddle >= 10
    assert _check(files, dev, 2, lambda name: "parallel") >= 50


def test_periodic_content_synchronises_slowly():
    """Periodic streams: a decoder started at a guessed state may stay out of phase for many subsequences."""
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(3)
    tile = rng.integers(0, 256, (16, 16, 3), dtype=np.uint8)
    files = [("flat gray", O.encode(np.full((1200, 1600), 77, np.uint8), quality=90)),
             ("flat rgb ss2", O.encode(np.full((1200, 1600, 3), (10, 200, 90), np.uint8), quality=50, subsampling=2)),
             ("tiled ss2", O.encode(np.tile(tile, (75, 100, 1)), quality=90, subsampling=2)),
             ("tiled ss0", O.encode(np.tile(tile, (40, 60, 1)), quality=75, subsampling=0)),
             ("stripes gray", O.encode(np.tile((np.arange(1600) % 8 * 32).astype(np.uint8), (1200, 1)), quality=95))]
    _check(files, dev, 4, lambda name: "parallel")


def _ff00_on_boundary():
    """A file one of whose subsequence boundaries falls on the zero of a stuffed FF 00 pair."""
    for seed in range(50):
        data = O.encode(_image(100 + seed, 700, 500), quality=95, subsampling=seed % 3)
        src = J.parse(data)
        seg = data[src.scan[0]:src.scan[1]]
        if any(seg[r - 1] == 0xFF for r in range(J.SUB_BYTES, len(seg), J.SUB_BYTES)):
            return data
    raise AssertionError("no seed puts an FF 00 pair on a subsequence boundary")


def test_stuffed_pair_on_a_subsequence_boundary():
    dev = torch.device("cuda:0")
    data = _ff00_on_boundary()
    _check([("ff00", data)], dev, 5, lambda name: "parallel")


def _long_code(seed):
    """A file (standard Huffman tables) with 48 one-bits inside its entropy-coded data: every code that starts in them
    is longer than 16 bits."""
    data = O.encode(_image(200 + seed, 300, 220), quality=90, subsampling=seed % 3)
    s, e = J.parse(data).scan
    p = s + (e - s) * (seed % 5 + 2) // 8
    while data[p - 1] == 0xFF:
        p += 1
    return data[:p] + b"\xff\x00" * 6 + data[p:]


def _truncated(seed):
    data = O.encode(_image(300 + seed, 320, 240), quality=85, subsampling=seed % 3)
    s, e = J.parse(data).scan
    p = s + (e - s) * (seed % 4 + 3) // 8
    while data[p - 1] == 0xFF:
        p += 1
    return data[:p] + b"\xff\xd9"


def _flipped(seed, count):
    rng = np.random.default_rng(seed)
    out = []
    for t in range(count):
        d = bytearray(O.encode(_image(seed * 1000 + t, 260, 200, gray=t % 5 == 4), quality=(30, 75, 90, 100)[t % 4],
                               **({} if t % 5 == 4 else {"subsampling": t % 3}),
                               **({"restart_marker_rows": 4} if t % 3 == 0 else {})))
        s, e = J.parse(bytes(d)).scan
        for _ in range(1 + t % 6):
            d[int(rng.integers(s, e))] ^= 1 << int(rng.integers(8))
        if J.parse(bytes(d)) is not None:
            out.append(("flip %d" % t, bytes(d)))
    return out


def _decodable(files):
    out = []
    for name, data in files:
        try:
            _pillow(data)
        except OSError:
            continue
        out.append((name, data))
    return out


@pytest.mark.skipif(not O.X86_64, reason="corrupt data decodes as Pillow only with libjpeg-turbo's x86-64 IDCT")
def test_corrupt_files_fall_back_in_a_mixed_batch():
    dev = torch.device("cuda:0")
    corrupt = _decodable([("long %d" % k, _long_code(k)) for k in range(6)] +
                         [("truncated %d" % k, _truncated(k)) for k in range(6)])
    assert len(corrupt) >= 8
    flips = _decodable(_flipped(7, 40))
    assert len(flips) >= 20
    clean = [("clean %d" % k, O.encode(_image(400 + k, 300, 220), quality=90, subsampling=k % 3)) for k in range(6)]
    files = corrupt + flips + clean

    def expect(name):
        return "parallel" if name.startswith("clean") else None if name.startswith("flip") else "fallback"
    rng = np.random.default_rng(6)
    items, refs, names = [], [], []
    for name, data in files:
        full = _pillow(data)
        for r in _rects(*full.shape[:2], rng)[:1 if name.startswith("flip") else 6]:
            items.append((data, r))
            refs.append(full[r[0]:r[0] + r[2], r[1]:r[1] + r[3]])
            names.append(name)
    outs, paths = _decode(items, dev)
    seen = set()
    for name, (data, r), got, ref, row in zip(names, items, outs, refs, paths):
        assert np.array_equal(got, ref), (name, r)
        for k, path in row:
            seen.add(path)
            if expect(name) == "parallel":
                assert path == "parallel", (name, r, k)
        if r[2:] == _pillow(data).shape[:2] and expect(name) == "fallback":
            assert any(path == "fallback" for _, path in row), name   # the whole image meets the corrupt data
    assert {"parallel", "fallback"} <= seen


def test_two_runs_are_bitwise_equal():
    dev = torch.device("cuda:0")
    files = [("a", O.encode(_image(500, 800, 600), quality=90, subsampling=2)),
             ("b", O.encode(np.tile(np.random.default_rng(1).integers(0, 256, (8, 24, 3), dtype=np.uint8),
                                    (80, 30, 1)), quality=80)),
             ("c", O.encode(_image(501, 640, 480), quality=90, restart_marker_rows=2))]
    if O.X86_64:
        files.append(("d", _long_code(1)))
    items = [(data, (0, 0) + _pillow(data).shape[:2]) for _, data in files]
    a, pa = _decode(items, dev)
    b, pb = _decode(items, dev)
    assert pa == pb
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def _worker_init(worker_id):
    random.seed(1234 + worker_id)
    torch.manual_seed(1234 + worker_id)
    np.random.seed(1234 + worker_id)


def test_cls_dataloader_mixes_parallel_fallback_and_pillow_samples(tmp_path):
    """As test_cuda_jpeg's end-to-end test, over JPEGs large enough for the parallel decode, corrupt ones and files
    Pillow decodes on the worker (progressive, PNG)."""
    from torch.utils.data import DataLoader

    import test_cuda_jpeg as TJ
    rng = np.random.default_rng(8)
    for c in ("class_a", "class_b"):
        os.makedirs(os.path.join(tmp_path, c))
        for n in range(10):
            h, w = int(rng.integers(200, 500)), int(rng.integers(200, 500))
            a = _image(int(rng.integers(1 << 30)), w, h)
            path = os.path.join(tmp_path, c, "img%02d" % n)
            if n == 8:
                Image.fromarray(a).save(path + ".png")
                continue
            data = O.encode(a, quality=90, subsampling=2 if n == 9 else n % 3, progressive=n == 9,
                            **({"restart_marker_rows": 6} if n == 3 else {}))
            if n in (4, 5) and O.X86_64:
                s, e = J.parse(data).scan
                p = s + (e - s) // 2
                while data[p - 1] == 0xFF:
                    p += 1
                data = data[:p] + b"\xff\x00" * 6 + data[p:]
            with open(path + ".jpg", "wb") as f:
                f.write(data)
    sys.path.insert(0, TJ.STANDIN)
    try:
        import utils.datasets as ud
        stock_transform, stock_dataset = ud.build_transform, ud.build_dataset

        def args():
            return TJ.SimpleNamespace(input_size=96, imagenet_default_mean_and_std=True, aa="rand-m9-mstd0.5-inc1",
                                      train_interpolation="random", reprob=0.0, crop_pct=None,
                                      data_path=str(tmp_path), eval_data_path=str(tmp_path), nb_classes=2)
        for is_train in (True, False):
            ud.build_transform = stock_transform
            ref_ds, _ = stock_dataset(is_train, args())
            ud.build_transform = TJ.functools.partial(D.build_gpu_cls_transform, stock=stock_transform)
            gpu_ds, _ = D.build_gpu_cls_dataset(is_train, args(), stock_dataset)
            assert sum(isinstance(gpu_ds.loader(p), J.JpegSource) for p, _ in gpu_ds.samples) == 16
            batches = []
            for ds, cls in ((ref_ds, DataLoader), (gpu_ds, D._AugmentingDataLoader)):
                loader = cls(ds, batch_size=10, shuffle=True, num_workers=2, worker_init_fn=_worker_init,
                             generator=torch.Generator().manual_seed(7), drop_last=True, pin_memory=True)
                batches.append([(x, y) for x, y in loader])
            assert len(batches[0]) == len(batches[1]) == 2
            for (rx, ry), (gx, gy) in zip(*batches):
                assert gx.is_cuda and torch.equal(ry, gy.cpu())
                assert torch.equal(gx.cpu(), rx), is_train
    finally:
        sys.path.remove(TJ.STANDIN)
        for m in [m for m in sys.modules if m == "utils" or m.startswith("utils.")]:
            del sys.modules[m]


def test_pretrain_dataloader_mixes_parallel_fallback_and_pillow_samples(tmp_path):
    """As test_cuda_png's end-to-end test, with rgb JPEGs large enough for the parallel decode, corrupt ones and
    progressive ones (decoded by Pillow on the worker)."""
    import gc

    import test_png_host as H
    gc.collect()
    rng = np.random.default_rng(9)
    for k in range(16):
        h, w = int(rng.integers(200, 330)), int(rng.integers(200, 330))
        imgs = H.AO.make_images(int(rng.integers(1 << 30)), h, w)
        imgs["semseg"].putpalette(list(range(256)) * 3)
        rgb = np.asarray(imgs["rgb"].convert("RGB")).astype(np.float64)
        rgb = np.clip(rgb + np.random.default_rng(k).normal(0, 25, rgb.shape), 0, 255).astype(np.uint8)
        data = O.encode(rgb, quality=90, subsampling=2 if k % 8 == 7 else k % 3, progressive=k % 8 == 7)
        if k % 8 == 3 and O.X86_64:
            s, e = J.parse(data).scan
            p = s + (e - s) // 3
            while data[p - 1] == 0xFF:
                p += 1
            data = data[:p] + b"\xff\x00" * 6 + data[p:]
        for task in ("rgb", "depth", "semseg"):
            os.makedirs(os.path.join(tmp_path, task, "c"), exist_ok=True)
        with open(os.path.join(tmp_path, "rgb", "c", "img%02d.jpg" % k), "wb") as f:
            f.write(data)
        imgs["depth"].save(os.path.join(tmp_path, "depth", "c", "img%02d.png" % k))
        imgs["semseg"].save(os.path.join(tmp_path, "semseg", "c", "img%02d.png" % k))
    sys.path.insert(0, H.STANDIN)
    try:
        import utils.datasets as ud
        args = H._Args(str(tmp_path), input_size=96)

        def batches(dataset):
            loader = D._AugmentingDataLoader(dataset, batch_size=8, shuffle=True, num_workers=2,
                                             worker_init_fn=_worker_init, generator=torch.Generator().manual_seed(7),
                                             drop_last=True, pin_memory=True)
            return [(x, y) for x, y in loader]
        plain = D.build_gpu_augment_dataset(args, ud.build_multimae_pretraining_dataset)
        comp = D.build_gpu_augment_dataset(args, ud.build_multimae_pretraining_dataset, compressed=True)
        assert isinstance(comp, D.CompressedMultiTaskImages)
        ref, got = batches(plain), batches(comp)
        assert len(ref) == len(got) == 2
        for (rx, ry), (gx, gy) in zip(ref, got):
            assert torch.equal(ry.cpu(), gy.cpu())
            for task in rx:
                assert gx[task].is_cuda and torch.equal(gx[task], rx[task]), task
    finally:
        sys.path.remove(H.STANDIN)
        for m in [m for m in sys.modules if m == "utils" or m.startswith("utils.")]:
            del sys.modules[m]
