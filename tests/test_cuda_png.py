"""GPU: the PNG decode kernels (mmae_png_decode_batch, MMAE_GPU_JPEG) against tests/png_oracle.py, and the pre-training
loader that uses them.

1. Every PNG of the host tests' corpus (three seeds), whole and at random rectangles, decodes bitwise as the oracle, and
   the oracle equals Pillow (tests/test_png_host.py).
2. A DataLoader with 2 workers over a seeded folder tree (rgb JPEG and PNG, 16-bit depth PNG, semseg PNG, mixed sizes)
   yields, with the compressed dataset, the same batches bitwise as the MMAE_GPU_AUGMENT dataset.
3. Seeded corruption (a flipped bit in a dynamic Huffman header, a distance beyond the data decoded so far, a truncated
   stream, a bad Adler-32, a filter type above 4): the kernels flag the stream, and the batch raises what Pillow raises,
   naming the file, or, where Pillow decodes the file anyway, carries Pillow's image."""
import gc
import sys
import zlib

import numpy as np
import pytest
import torch

import png_oracle as O
import test_png_host as H
from multimae_b200 import data as D
from multimae_b200 import kernels as K
from multimae_b200 import png as P

pytestmark = pytest.mark.gpu


def _decode(items, dev):
    """items: [(PngSource, task, rect)] of one task -> (status list, [decoded rectangle])."""
    crops = [D.Crops({task: (src, rect)}, False, rect[2], rect[3]) for src, task, rect in items]
    pb = D.pack_batch(crops, 64, (0.5,) * 3, (0.5,) * 3)
    buf = torch.zeros(pb.device_bytes, dtype=torch.uint8, device=dev)
    buf[:pb.buffer.numel()].copy_(pb.buffer)
    status = K.png_decode_batch(pb.buffer, buf, *pb.png).cpu().tolist()
    out = []
    for (src, task, (i, j, h, w)), (_, _, off, _) in zip(items, pb.png_files):
        kind = D.AUGMENT_KINDS[task]
        n = h * w * (3 if kind == 0 else 2 if kind == 1 else 1)
        a = buf[off:off + n].cpu().numpy()
        out.append(a.view(np.uint16).reshape(h, w) if kind == 1 else a.reshape((h, w, 3) if kind == 0 else (h, w)))
    return status, out


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_kernels_equal_oracle_bitwise(seed):
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(seed)
    by_task = {}
    for name, task, data in O.corpus(seed):
        src = P.parse(data, task)
        full = O.decode(src, task)
        H_, W_ = src.height, src.width
        rects = [(0, 0, H_, W_)]
        for _ in range(3):
            h, w = int(rng.integers(1, H_ + 1)), int(rng.integers(1, W_ + 1))
            rects.append((int(rng.integers(0, H_ - h + 1)), int(rng.integers(0, W_ - w + 1)), h, w))
        for r in rects:
            by_task.setdefault(task, []).append((src, task, r, full, name))
    checked = 0
    for task, items in by_task.items():
        status, got = _decode([(s, t, r) for s, t, r, _, _ in items], dev)
        for st, g, (src, _, (i, j, h, w), full, name) in zip(status, got, items):
            assert st == 0, (name, st)
            assert np.array_equal(g, full[i:i + h, j:j + w]), (name, (i, j, h, w))
            checked += 1
    assert checked == 4 * 30


def _bits(pairs):
    """LSB-first packing of (value, bit count) pairs into bytes."""
    acc = n = 0
    out = bytearray()
    for v, k in pairs:
        acc |= v << n
        n += k
        while n >= 8:
            out.append(acc & 255)
            acc >>= 8
            n -= 8
    if n:
        out.append(acc)
    return bytes(out)


def _rev(code, k):
    return int(format(code, "0%db" % k)[::-1], 2)


def _png_with_stream(w, h, stream, depth=8, ctype=0):
    import struct
    out = P.SIGNATURE + O.chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ctype, 0, 0, 0))
    return out + O.chunk(b"IDAT", stream) + O.chunk(b"IEND", b"")


def _corrupt(rng):
    """[(name, task, file bytes)] of seeded corruptions of valid PNGs."""
    w, h = 40, 30
    rows = O.samples(rng, 8, 0, h, w)
    raw = O.filter_rows(rows, 1, [int(f) for f in rng.integers(0, 5, h)])
    stream = zlib.compress(raw, 9)
    out = []
    for k in range(6):                                           # a flipped bit in the dynamic block's header
        s = bytearray(stream)
        s[2 + k // 3] ^= 1 << int(rng.integers(3, 8))
        out.append(("header bit %d" % k, _png_with_stream(w, h, bytes(s))))
    # a fixed block whose first symbol is a match of length 3 at distance 1, before any byte is decoded
    far = b"\x78\x01" + _bits([(1, 1), (1, 2), (_rev(1, 7), 7), (0, 5), (0, 7)])
    out.append(("distance too far", _png_with_stream(w, h, far)))
    out.append(("truncated", _png_with_stream(w, h, stream[:len(stream) // 2])))
    bad_check = bytearray(stream)
    bad_check[-1] ^= 1
    out.append(("bad adler", _png_with_stream(w, h, bytes(bad_check))))
    out.append(("no adler", _png_with_stream(w, h, stream[:-4])))                 # Pillow decodes this one
    bad_filter = bytearray(raw)
    bad_filter[(w + 1) * 7] = 9
    out.append(("filter type 9", _png_with_stream(w, h, zlib.compress(bytes(bad_filter)))))
    return out


def test_corrupt_streams_raise_what_pillow_raises(tmp_path):
    dev = torch.device("cuda:0")
    good = tmp_path / "good.png"
    good.write_bytes(_png_with_stream(40, 30, zlib.compress(O.filter_rows(O.samples(np.random.default_rng(9), 8, 0, 30,
                                                                                      40), 1, [0] * 30))))
    for n, (name, data) in enumerate(_corrupt(np.random.default_rng(3))):
        path = tmp_path / ("bad%02d.png" % n)
        path.write_bytes(data)
        src = P.parse(data, "rgb")
        assert src is not None, name
        status, _ = _decode([(src, "rgb", (0, 0, 30, 40))], dev)
        assert status[0] != 0, name
        try:
            ref = H._pillow(data, "rgb")
            err = None
        except Exception as e:  # noqa: BLE001
            err = e
        crops = [D.Crops({"rgb": (P.parse(good.read_bytes(), "rgb", str(good)), (0, 0, 30, 40))}, False, 30, 40),
                 D.Crops({"rgb": (P.parse(data, "rgb", str(path)), (0, 0, 30, 40))}, False, 30, 40)]
        pb = D.pack_batch(crops, 32, (0.5,) * 3, (0.5,) * 3)
        if err is not None:
            with pytest.raises(type(err)) as got:
                pb.to_device(dev)
            assert str(path) in str(got.value), name
            continue
        out = pb.to_device(dev)["rgb"]
        plain = [D.Crops({"rgb": H._pillow(good.read_bytes(), "rgb")}, False, 30, 40),
                 D.Crops({"rgb": ref}, False, 30, 40)]
        want = D.pack_batch(plain, 32, (0.5,) * 3, (0.5,) * 3).to_device(dev)["rgb"]
        assert torch.equal(out, want), name


def _worker_init(worker_id):
    import random
    random.seed(1234 + worker_id)
    torch.manual_seed(1234 + worker_id)
    np.random.seed(1234 + worker_id)


def test_dataloader_end_to_end_bitwise(tmp_path):
    gc.collect()            # forked workers must not inherit (and free) garbage that holds CUDA tensors
    H._write_tree(str(tmp_path), np.random.default_rng(1), n=24)
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
        assert len(ref) == len(got) == 3
        for (rx, ry), (gx, gy) in zip(ref, got):
            assert torch.equal(ry.cpu(), gy.cpu())
            assert list(rx) == list(gx) == ["rgb", "depth", "semseg"]
            for task in rx:
                assert gx[task].is_cuda and torch.equal(gx[task], rx[task]), task
    finally:
        sys.path.remove(H.STANDIN)
        for m in [m for m in sys.modules if m == "utils" or m.startswith("utils.")]:
            del sys.modules[m]
