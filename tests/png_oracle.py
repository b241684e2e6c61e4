"""NumPy restatement of the PNG decode the kernels make (csrc/png.cu), and a seeded corpus of PNGs built here.

decode(src) = zlib.decompress of the joined IDAT stream, PNG's unfilter (filter types 0-4, byte-wise), then the
expansion of the task's conversion: uint8 RGB [h, w, 3] for rgb (gray replicated, palette looked up in the
zero-padded palette), uint16 [h, w] for depth (big-endian samples), uint8 [h, w] indices for semseg.  The tests hold it
to Image.open(f) + the reference's convert bitwise, and hold the kernels to it.

The corpus writes PNGs by hand (signature, IHDR, PLTE, IDAT chunks with CRCs, IEND), so that every filter type, mixed
filters, IDAT split into one or many chunks and every zlib level and strategy can be chosen."""
import struct
import zlib

import numpy as np

from multimae_b200 import png as P

BPP = {(8, 0): 1, (16, 0): 2, (8, 2): 3, (8, 3): 1}
FORMS = {"rgb": [(8, 0), (8, 2), (8, 3)], "depth": [(16, 0)], "semseg": [(8, 3), (8, 0)]}
STRATEGIES = (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED)


def chunk(cid, body):
    return struct.pack(">I", len(body)) + cid + body + struct.pack(">I", zlib.crc32(cid + body))


def paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filter_rows(rows, bpp, filters):
    """PNG filter each row of uint8 [h, row bytes] with the type filters[r]: the raw stream bytes."""
    h, n = rows.shape
    out = np.zeros((h, n + 1), np.uint8)
    prior = np.zeros(n, np.int32)
    for r in range(h):
        cur = rows[r].astype(np.int32)
        a = np.concatenate([np.zeros(bpp, np.int32), cur[:-bpp]])
        c = np.concatenate([np.zeros(bpp, np.int32), prior[:-bpp]])
        f = filters[r]
        pred = [0, a, prior, (a + prior) >> 1, paeth(a, prior, c)][f]
        out[r, 0] = f
        out[r, 1:] = (cur - pred) & 255
        prior = cur
    return out.tobytes()


def unfilter(raw, h, n, bpp):
    """The inverse, as the kernels do it: uint8 [h, n] (raises ValueError for a filter type above 4)."""
    data = np.frombuffer(raw, np.uint8).reshape(h, n + 1)
    out = np.zeros((h, n), np.uint8)
    prior = np.zeros(n, np.int32)
    for r in range(h):
        f, cur = int(data[r, 0]), data[r, 1:].astype(np.int32)
        if f > 4:
            raise ValueError("filter type %d" % f)
        if f in (0, 2):
            row = (cur + (prior if f == 2 else 0)) & 255
        else:
            row = np.zeros(n, np.int32)
            for x in range(n):
                a = row[x - bpp] if x >= bpp else 0
                b = prior[x]
                c = prior[x - bpp] if x >= bpp else 0
                pred = a if f == 1 else (a + b) >> 1 if f == 3 else int(paeth(a, b, c))
                row[x] = (cur[x] + pred) & 255
        out[r] = row
        prior = row
    return out


def decode(src, task):
    """The decoded image of PngSource `src` as the task's conversion leaves it."""
    bpp = BPP[src.depth, src.ctype]
    rows = unfilter(zlib.decompress(src.stream), src.height, src.width * bpp, bpp)
    if task == "depth":
        pairs = rows.reshape(src.height, src.width, 2).astype(np.uint16)
        return pairs[..., 0] << 8 | pairs[..., 1]
    if task != "rgb":
        return rows
    if src.ctype == 2:
        return rows.reshape(src.height, src.width, 3)
    if src.ctype == 0:
        return np.repeat(rows[..., None], 3, axis=2)
    return np.frombuffer(src.palette, np.uint8).reshape(256, 3)[rows]


def samples(rng, depth, ctype, h, w):
    """Random pixel rows of a form: smooth ramps plus noise, so that every filter and match length occurs."""
    bpp = BPP[depth, ctype]
    n = w * bpp
    base = (np.arange(n)[None, :] + 3 * np.arange(h)[:, None]) % 256
    noise = rng.integers(0, 256, (h, n))
    mix = rng.random((h, 1)) < 0.5
    rows = np.where(mix, base, noise).astype(np.uint8)
    if ctype == 3:
        rows = (rows.astype(np.int32) % int(rng.integers(1, 257))).astype(np.uint8)   # some beyond a short palette
    return rows


def encode(rows, w, h, depth, ctype, filters=None, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, chunks=1,
           palette_entries=None, extra=(), interlace=0, rng=None):
    bpp = BPP.get((depth, ctype), 1)
    filters = [0] * h if filters is None else filters
    raw = filter_rows(rows, bpp, filters)
    c = zlib.compressobj(level, zlib.DEFLATED, 15, 9, strategy)
    stream = c.compress(raw) + c.flush()
    out = P.SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ctype, 0, 0, interlace))
    for cid, body in extra:
        out += chunk(cid, body)
    if ctype == 3:
        k = palette_entries or 256
        pal = (rng or np.random.default_rng(0)).integers(0, 256, 3 * k).astype(np.uint8).tobytes()
        out += chunk(b"PLTE", pal)
    cuts = np.linspace(0, len(stream), chunks + 1).astype(int)
    for a, b in zip(cuts[:-1], cuts[1:]):
        out += chunk(b"IDAT", stream[a:b])
    return out + chunk(b"IEND", b"")


def corpus(seed, sizes=((1, 1), (7, 3), (33, 17), (120, 90), (4100, 2))):
    """[(name, task, bytes)]: every task's forms at each size, with rotating filters, levels, strategies and chunking."""
    rng = np.random.default_rng(seed)
    out = []
    k = 0
    for w, h in sizes:
        for task, forms in FORMS.items():
            for depth, ctype in forms:
                rows = samples(rng, depth, ctype, h, w)
                filters = [int(f) for f in rng.integers(0, 5, h)] if k % 3 else [k % 5] * h
                data = encode(rows, w, h, depth, ctype, filters, level=k % 10, strategy=STRATEGIES[k % 5],
                              chunks=1 + (k % 4) * 3, palette_entries=int(rng.integers(1, 257)), rng=rng)
                out.append(("%s_%dx%d_%d_%d_%d" % (task, w, h, depth, ctype, k), task, data))
                k += 1
    return out
