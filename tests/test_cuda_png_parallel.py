"""GPU: the parallel inflate of mmae_png_decode_batch (slices searched for block starts, the chain confirmed, blocks
expanded with window markers, markers resolved) against Pillow, tests/png_oracle.py and the block walker
(tests/deflate_walker.py).

1. Pillow-written depth, rgb and semseg PNGs, a depth map's rows at every zlib level and strategy, chains with stored
   and fixed-Huffman blocks in the middle, a stored block hiding a valid dynamic header before a slice's true block
   start, a 4000 x 3000 16-bit depth map and streams just under and over the size threshold: every rectangle (the
   whole image and crops touching each edge) equals Pillow and the oracle bitwise.  The records left in the scratch
   show the path of each stream, and a stream decoded in parallel has the walker's block chain.
2. Corrupt streams get the sequential kernel's status words and the loader raises what Pillow raises.
3. A mixed batch decodes bitwise the same twice; a DataLoader mixing parallel, fallback and Pillow-decoded samples
   yields the batches of the MMAE_GPU_AUGMENT dataset bitwise."""
import gc
import io
import os
import struct
import sys
import zlib

import numpy as np
import pytest
import torch
from PIL import Image

import augment_oracle as AO
import deflate_walker as W
import png_oracle as O
import test_png_host as H
from multimae_b200 import data as D
from multimae_b200 import kernels as K
from multimae_b200 import png as P

pytestmark = pytest.mark.gpu

PNG_SHORT, PNG_DISTANCE, PNG_SIZE, PNG_CHECK = 4, 3, 5, 6


def _pillow_png(img):
    f = io.BytesIO()
    img.save(f, "PNG")
    return f.getvalue()


def _decode(items, dev):
    """items: [(PngSource, task, rect)] of one task -> (status list, [rectangle],
    {id(src): (path, walked, blocks, slice records)})."""
    crops = [D.Crops({task: (src, rect)}, False, rect[2], rect[3]) for src, task, rect in items]
    pb = D.pack_batch(crops, 64, (0.5,) * 3, (0.5,) * 3)
    buf = torch.zeros(pb.device_bytes, dtype=torch.uint8, device=dev)
    buf[:pb.buffer.numel()].copy_(pb.buffer)
    scratch = torch.empty(max(pb.png[2], 16), dtype=torch.uint8, device=dev)
    status = K.png_decode_batch(pb.buffer, buf, *pb.png, scratch=scratch).cpu().tolist()
    out = []
    for (src, task, (i, j, h, w)), (_, _, off, _) in zip(items, pb.png_files):
        kind = D.AUGMENT_KINDS[task]
        n = h * w * (3 if kind == 0 else 2 if kind == 1 else 1)
        a = buf[off:off + n].cpu().numpy()
        out.append(a.view(np.uint16).reshape(h, w) if kind == 1 else a.reshape((h, w, 3) if kind == 0 else (h, w)))
    pd = pb.buffer.numpy()[pb.png[0] * 16:].view(np.int32)[:pb.png[1] * D.PNG_FIELDS].reshape(-1, D.PNG_FIELDS)
    sc = scratch.cpu().numpy()
    records = {}
    for d, (src, _, _) in zip(pd, items):
        if not d[14]:
            records[id(src)] = (0, 0, [], [])
            continue
        area = sc[d[14] * 16:].view(np.int32)
        nb = int(area[1])
        ns = P.slices(int(d[6]))
        first = (P.STREAM_RECORD_BYTES + ns * P.SLICE_RECORD_BYTES) // 4
        blocks = [tuple(int(v) for v in area[first + 4 * k:first + 4 * k + 4]) for k in range(nb)]
        s0 = P.STREAM_RECORD_BYTES // 4
        slices = [tuple(int(v) for v in area[s0 + 4 * k:s0 + 4 * k + 4]) for k in range(ns)]
        records[id(src)] = (int(area[0]), int(area[2]), blocks, slices)
    return status, out, records


def _rects(H_, W_, rng):
    h, w = max(1, H_ // 3), max(1, W_ // 3)
    return [(0, 0, H_, W_), (0, int(rng.integers(0, W_ - w + 1)), h, w), (H_ - h, int(rng.integers(0, W_ - w + 1)), h, w),
            (int(rng.integers(0, H_ - h + 1)), 0, h, w), (int(rng.integers(0, H_ - h + 1)), W_ - w, h, w)]


def _depth_rows(seed, h, w):
    """Big-endian rows (uint8 [h, 2w]) of a make_images depth map."""
    a = np.asarray(AO.make_images(seed, h, w, tasks=("depth",))["depth"]).astype(">u2")
    return a.view(np.uint8).reshape(h, 2 * w)


def _decoy_png(seed=3):
    """(file bytes, bit position of the decoy) of a 16-bit depth PNG whose stream holds, in the payload of a stored
    block, a whole dynamic block starting in the same slice as the next true block and after that slice's first
    byte."""
    h, w = 120, 2000
    pitch = 2 * w + 1
    raw = bytearray(O.filter_rows(_depth_rows(seed, h, w), 2, [0] * h))
    dec = W.decoy(seed)
    inner, _, _ = W.inflate_blocks(b"\x78\x9c" + dec + b"\x03\x00" + bytes(4))   # then a final empty fixed block
    assert inner[0][4] == 2 and not inner[0][5]                               # a non-final dynamic block
    a = 5 * pitch + 1
    c = zlib.compressobj(6, zlib.DEFLATED, -15, 9, zlib.Z_DEFAULT_STRATEGY)
    p0 = 2 + len(c.compress(bytes(raw[:a])) + c.flush(zlib.Z_SYNC_FLUSH)) + 5   # the stored payload's first byte
    s = (p0 // P.SLICE_BYTES + 1) * P.SLICE_BYTES                           # the slice that holds the decoy
    for f in range(s + 64 - p0, s + 4000 - p0):                           # zeros, then the decoy inside one row
        at = a + f
        if at % pitch >= 1 and at % pitch + len(dec) <= pitch:
            break
    raw[a:a + f + len(dec)] = bytes(f) + dec
    raw = bytes(raw)
    stream, got = W.chain([("deflate", raw[:a], 6, zlib.Z_DEFAULT_STRATEGY), ("stored", raw[a:a + f + len(dec)]),
                           ("deflate", raw[a + f + len(dec):], 6, zlib.Z_DEFAULT_STRATEGY)])
    assert got == raw and stream[p0 + f:p0 + f + len(dec)] == dec
    assert 8 * (p0 + f) not in [b[0] for b in W.inflate_blocks(stream)[0]]    # not a true block start
    return _png(w, h, 16, 0, stream), 8 * (p0 + f)


def _png(w, h, depth, ctype, stream):
    import struct
    out = P.SIGNATURE + O.chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ctype, 0, 0, 0))
    return out + O.chunk(b"IDAT", stream) + O.chunk(b"IEND", b"")


def _corpus():
    """[(name, task, file bytes, path expected or None)]."""
    out = []
    imgs = AO.make_images(11, 350, 450)
    imgs["semseg"].putpalette(list(range(256)) * 3)       # 8-bit: Pillow writes a short palette with fewer bits
    out.append(("pillow depth", "depth", _pillow_png(imgs["depth"]), P.PATH_PARALLEL))
    out.append(("pillow rgb", "rgb", _pillow_png(imgs["rgb"]), None))
    out.append(("pillow gray", "rgb", _pillow_png(imgs["rgb"].convert("L")), None))
    out.append(("pillow semseg", "semseg", _pillow_png(imgs["semseg"]), None))
    noisy = Image.frombytes("P", (450, 350), np.random.default_rng(4).integers(0, 40, 450 * 350, np.uint8).tobytes())
    noisy.putpalette(list(range(256)) * 3)
    out.append(("pillow noisy semseg", "semseg", _pillow_png(noisy), None))
    for seed in (12, 13):
        out.append(("pillow depth %d" % seed, "depth", _pillow_png(AO.make_images(seed, 350, 450)["depth"]),
                    P.PATH_PARALLEL))
    rows = _depth_rows(21, 350, 450)
    for level in range(10):
        for strategy in O.STRATEGIES:
            data = O.encode(rows, 450, 350, 16, 0, level=level, strategy=strategy, chunks=1 + level % 4)
            out.append(("level %d strategy %d" % (level, strategy), "depth", data, None))
    raw = O.filter_rows(rows, 2, [k % 5 for k in range(350)])
    n = len(raw)
    stream, _ = W.chain([("deflate", raw[:n // 4], 6, zlib.Z_DEFAULT_STRATEGY), ("stored", raw[n // 4:n // 4 + 30000]),
                         ("deflate", raw[n // 4 + 30000:n // 2], 6, zlib.Z_FIXED),
                         ("deflate", raw[n // 2:], 9, zlib.Z_DEFAULT_STRATEGY)])
    out.append(("stored and fixed in the middle", "depth", _png(450, 350, 16, 0, stream), P.PATH_PARALLEL))
    out.append(("decoy header", "depth", _decoy_png()[0], P.PATH_PARALLEL))
    # just under and just over the threshold: noise rows cut to the size whose stream lands next to it
    rng = np.random.default_rng(8)
    for want, name in ((P.PARALLEL_MIN_BYTES - 1, "under"), (P.PARALLEL_MIN_BYTES, "at"),
                       (P.PARALLEL_MIN_BYTES + 700, "over")):
        w = 128
        body = rng.integers(0, 256, (400, w)).astype(np.uint8)
        raw = O.filter_rows(body, 1, [0] * 400)
        for h in range(400, 0, -1):
            s = zlib.compress(raw[:h * (w + 1)], 0)
            if len(s) <= want:
                break
        s = zlib.compress(raw[:h * (w + 1)], 0)
        pad = want - len(s)               # make the length exact: extra bytes after the Adler-32 are ignored
        out.append(("%s the threshold" % name, "semseg", _png(w, h, 8, 0, s + bytes(pad)), None))
    return out


def _check(items, dev, expect):
    """Decode items [(name, task, data, src, full, rects)] of one task; returns the records by name."""
    flat = [(src, task, r) for name, task, data, src, full, rects in items for r in rects]
    status, got, records = _decode(flat, dev)
    k = 0
    out = {}
    for name, task, data, src, full, rects in items:
        for (i, j, h, w) in rects:
            assert status[k] == 0, (name, status[k])
            assert np.array_equal(got[k], full[i:i + h, j:j + w]), (name, (i, j, h, w))
            k += 1
        path, walked, blocks, _ = records[id(src)]
        out[name] = records[id(src)]
        if P.parallel_stream(len(src.stream)):
            assert path in (P.PATH_PARALLEL, P.PATH_WALK, P.PATH_BOUND), (name, path)
            if expect.get(name):
                assert path == expect[name], (name, path, walked)
            if path == P.PATH_PARALLEL:
                ref, _, _ = W.inflate_blocks(src.stream)
                assert blocks == [b[:4] for b in ref], name
        else:
            assert path == 0, name
    return out


def test_parallel_inflate_equals_pillow_and_the_walker():
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    by_task, expect, sizes = {}, {}, {}
    for name, task, data, path in _corpus():
        src = P.parse(data, task)
        assert src is not None, name
        full = H._pillow(data, task)
        assert np.array_equal(O.decode(src, task), full), name
        by_task.setdefault(task, []).append((name, task, data, src, full, _rects(src.height, src.width, rng)))
        expect[name], sizes[name] = path, len(src.stream)
    records = {}
    for task, items in by_task.items():
        records.update(_check(items, dev, expect))
    assert records["under the threshold"][0] == 0 and sizes["under the threshold"] == P.PARALLEL_MIN_BYTES - 1
    assert records["at the threshold"][0] != 0 and records["over the threshold"][0] != 0
    parallel = sum(r[0] == P.PATH_PARALLEL for r in records.values())
    assert parallel >= 20, {k: v[:2] for k, v in records.items()}


def test_decoy_header_is_the_slice_record_and_the_walk_decodes_past_it():
    dev = torch.device("cuda:0")
    data, bit = _decoy_png()
    src = P.parse(data, "depth")
    status, got, records = _decode([(src, "depth", (0, 0, src.height, src.width))], dev)
    path, walked, blocks, slices = records[id(src)]
    assert status == [0] and np.array_equal(got[0], H._pillow(data, "depth"))
    rec = slices[bit // (8 * P.SLICE_BYTES)]
    assert rec[0] == bit and rec[3] & 1                # the slice's first candidate is the decoy, and it decodes
    ref, _, _ = W.inflate_blocks(src.stream)
    assert path == P.PATH_PARALLEL and blocks == [b[:4] for b in ref]
    after = [b for b in ref if b[0] > bit][0]          # the true block after the decoy, in the same slice
    assert after[0] // (8 * P.SLICE_BYTES) == bit // (8 * P.SLICE_BYTES)
    # walked: the empty stored block of the first piece's flush, the stored block holding the decoy, and that block
    assert walked >= 3 and not any(r[0] == after[0] for r in slices)


def test_large_depth_map_has_hundreds_of_blocks():
    dev = torch.device("cuda:0")
    h, w = 3000, 4000
    yy, xx = np.mgrid[0:h, 0:w]
    rng = np.random.default_rng(1)
    a = 32768 + 20000 * np.sin(xx / 300.0) * np.cos(yy / 200.0) + rng.normal(0, 600, (h, w))
    img = Image.frombuffer("I;16", (w, h), np.clip(a, 0, 65535).astype("<u2").tobytes(), "raw", "I;16", 0, 1)
    data = _pillow_png(img)
    src = P.parse(data, "depth")
    full = H._pillow(data, "depth")
    rects = _rects(h, w, np.random.default_rng(2))
    records = _check([("large", "depth", data, src, full, rects)], dev, {"large": P.PATH_PARALLEL})
    assert len(records["large"][2]) >= 200


def _long_depth(seed=5, h=200, w=300):
    rows = _depth_rows(seed, h, w)
    raw = O.filter_rows(rows, 2, [1] * h)
    return w, h, raw, zlib.compress(raw, 6)


def _far_prefix():
    """A non-final fixed block whose first symbol copies 3 bytes from distance 1, then an empty stored block."""
    from test_cuda_png import _bits, _rev
    return _bits([(0, 1), (1, 2), (_rev(1, 7), 7), (0, 5), (0, 7), (0, 1), (0, 2)]) + b"\x00\x00\xff\xff"


def _corrupt():
    """[(name, file bytes, status the sequential kernel writes or None for any non-zero)] of a stream over the
    threshold."""
    w, h, raw, s = _long_depth()
    assert P.parallel_stream(len(s))
    out = [("truncated", _png(w, h, 16, 0, s[:len(s) // 2]), None),
           ("no adler", _png(w, h, 16, 0, s[:-4]), PNG_SHORT)]
    rng = np.random.default_rng(6)
    for k in range(4):
        b = bytearray(s)
        b[int(rng.integers(len(s) // 8, len(s) - 8))] ^= 1 << int(rng.integers(0, 8))
        out.append(("bit flip %d" % k, _png(w, h, 16, 0, bytes(b)), None))
    b = bytearray(s)
    b[-1] ^= 1
    out.append(("bad adler", _png(w, h, 16, 0, bytes(b)), PNG_CHECK))
    # 3 bytes copied from before the first byte, then the rows after their first 3 bytes: the chain's length and the
    # Adler-32 of the bytes a copy from nothing would give (zeros) both hold, so only the marker check refuses it
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    far = b"\x78\x9c" + _far_prefix() + c.compress(raw[3:]) + c.flush() + struct.pack(">I", zlib.adler32(
        bytes(3) + raw[3:]))
    out.append(("distance too far", _png(w, h, 16, 0, far), PNG_DISTANCE))
    out.append(("trailing data", _png(w, h, 16, 0, s + b"trailing bytes"), 0))
    long_raw = raw + bytes(np.random.default_rng(7).integers(0, 256, 9000, np.uint8))
    out.append(("over-long", _png(w, h, 16, 0, zlib.compress(long_raw, 6)), PNG_SIZE))
    return out


_REFUSED_BY_RESOLVE = ("distance too far", "bad adler")   # clean chains of the right length: resolve refuses them


def test_corrupt_streams_take_the_sequential_status_and_raise_what_pillow_raises(tmp_path):
    dev = torch.device("cuda:0")
    w, h, raw, s = _long_depth()
    good = tmp_path / "good.png"
    good.write_bytes(_png(w, h, 16, 0, s))
    for n, (name, data, want) in enumerate(_corrupt()):
        path = tmp_path / ("bad%02d.png" % n)
        path.write_bytes(data)
        src = P.parse(data, "depth")
        assert src is not None and P.parallel_stream(len(src.stream)), name
        status, _, records = _decode([(src, "depth", (0, 0, h, w))], dev)
        state = records[id(src)][0]
        if name in _REFUSED_BY_RESOLVE:
            assert state == P.PATH_RESOLVE, (name, state)
        if want == 0:
            assert status[0] == 0 and state == P.PATH_PARALLEL, (name, status, state)
        else:
            assert state != P.PATH_PARALLEL, name                # the stream went to the sequential kernel
            assert status[0] != 0 and (want is None or status[0] == want), (name, status[0])
        try:
            ref = H._pillow(data, "depth")
            err = None
        except Exception as e:  # noqa: BLE001
            err = e
        crops = [D.Crops({"depth": (P.parse(good.read_bytes(), "depth", str(good)), (0, 0, h, w))}, False, h, w),
                 D.Crops({"depth": (P.parse(data, "depth", str(path)), (0, 0, h, w))}, False, h, w)]
        pb = D.pack_batch(crops, 32, (0.5,) * 3, (0.5,) * 3)
        if err is not None:
            with pytest.raises(type(err)) as got:
                pb.to_device(dev)
            assert str(path) in str(got.value), name
            continue
        out = pb.to_device(dev)["depth"]
        plain = [D.Crops({"depth": H._pillow(good.read_bytes(), "depth")}, False, h, w),
                 D.Crops({"depth": ref}, False, h, w)]
        want_out = D.pack_batch(plain, 32, (0.5,) * 3, (0.5,) * 3).to_device(dev)["depth"]
        assert torch.equal(out, want_out), name


def test_mixed_batch_is_deterministic():
    dev = torch.device("cuda:0")
    items = []
    for seed in range(6):
        data = _pillow_png(AO.make_images(30 + seed, 350, 450, tasks=("depth",))["depth"])
        items.append(P.parse(data, "depth"))
    items.append(P.parse(_png(300, 200, 16, 0, zlib.compress(_long_depth()[2], 6, )), "depth"))
    items.append(P.parse(_png(300, 200, 16, 0, _long_depth()[3][:-9] + bytes(5)), "depth"))       # corrupt
    items.append(P.parse(_pillow_png(AO.make_images(40, 60, 50, tasks=("depth",))["depth"]), "depth"))  # short
    fixed = O.encode(_depth_rows(41, 350, 450), 450, 350, 16, 0, strategy=zlib.Z_FIXED)
    items.append(P.parse(fixed, "depth"))
    flat = [(s, "depth", (0, 0, s.height, s.width)) for s in items]
    s1, g1, r1 = _decode(flat, dev)
    s2, g2, r2 = _decode(flat, dev)
    assert s1 == s2 and s1[-3] != 0 and s1.count(0) == len(items) - 1
    assert all(np.array_equal(a, b) for a, b in zip(g1, g2))
    assert [r1[id(s)][:2] for s in items] == [r2[id(s)][:2] for s in items]
    paths = {r1[id(s)][0] for s in items}
    assert P.PATH_PARALLEL in paths and 0 in paths and paths - {0, P.PATH_PARALLEL}


def _worker_init(worker_id):
    import random
    random.seed(1234 + worker_id)
    torch.manual_seed(1234 + worker_id)
    np.random.seed(1234 + worker_id)


def _write_tree(root):
    """rgb: Pillow PNGs and an RGBA PNG (decoded by Pillow on the worker); depth: Pillow-written maps over the
    threshold (parallel) and maps in many short blocks (more than the walk takes: sequential fallback); semseg."""
    for k in range(16):
        imgs = AO.make_images(100 + k, 300 + 3 * k, 400 - 2 * k)
        imgs["semseg"].putpalette(list(range(256)) * 3)
        rgb = imgs["rgb"].convert("RGBA") if k % 5 == 0 else imgs["rgb"]
        if k % 3 == 0:                    # a sync flush every 1000 bytes: many short blocks in each slice
            img = imgs["depth"]
            raw = O.filter_rows(np.asarray(img).astype(">u2").view(np.uint8).reshape(img.height, -1), 2,
                                [0] * img.height)
            c = zlib.compressobj(6)
            s = b"".join(c.compress(raw[i:i + 1000]) + c.flush(zlib.Z_SYNC_FLUSH) for i in range(0, len(raw), 1000))
            depth = _png(img.width, img.height, 16, 0, s + c.flush())
        else:
            depth = _pillow_png(imgs["depth"])
        for task, data in (("rgb", _pillow_png(rgb)), ("depth", depth), ("semseg", _pillow_png(imgs["semseg"]))):
            os.makedirs(os.path.join(root, task, "c"), exist_ok=True)
            with open(os.path.join(root, task, "c", "img%02d.png" % k), "wb") as f:
                f.write(data)


def test_dataloader_mixes_parallel_fallback_and_pillow_samples(tmp_path):
    dev = torch.device("cuda:0")
    gc.collect()
    _write_tree(str(tmp_path))
    kinds = set()
    for k in range(16):
        for task in ("rgb", "depth"):
            with open(os.path.join(str(tmp_path), task, "c", "img%02d.png" % k), "rb") as f:
                src = P.parse(f.read(), task)
            if src is None:
                kinds.add("pillow")
            elif task == "depth":
                _, _, records = _decode([(src, "depth", (0, 0, 4, 4))], dev)
                kinds.add(records[id(src)][0])
    assert kinds >= {"pillow", P.PATH_PARALLEL, P.PATH_BOUND}, kinds
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
