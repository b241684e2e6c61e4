"""CPU: the pieces of the parallel PNG inflate that need no GPU.

1. The pure-Python block walker (tests/deflate_walker.py), the oracle for the block chains the kernels confirm, equals
   zlib.decompress on the PNG corpus and on every zlib level and strategy, and its blocks tile the stream and the
   output.
2. The chain builder puts stored and fixed-Huffman blocks where it is asked to, and hides a decoy dynamic header.
3. pack_batch reserves the records of each stream the parallel inflate takes (descriptor field 14, after every image's
   rows) and its first unit (field 15), and the fallback descriptors; the size threshold and the constants match
   csrc/png.cu."""
import os
import re
import zlib

import numpy as np
import pytest

import deflate_walker as W
import png_oracle as O
from multimae_b200 import data as D
from multimae_b200 import png as P

CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "multimae_b200", "csrc", "png.cu")


def _check_tiling(stream, blocks, raw):
    assert blocks[0][0] == 16
    for a, b in zip(blocks, blocks[1:]):
        assert a[1] == b[0] and a[2] + a[3] == b[2] and not a[5]
    assert blocks[-1][5] and blocks[-1][2] + blocks[-1][3] == len(raw)
    assert (blocks[-1][1] + 7) // 8 + 4 <= len(stream)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_walker_equals_zlib_on_the_png_corpus(seed):
    for name, task, data in O.corpus(seed):
        src = P.parse(data, task)
        blocks, raw, check = W.inflate_blocks(src.stream)
        assert raw == zlib.decompress(src.stream), name
        assert check == zlib.adler32(raw), name
        _check_tiling(src.stream, blocks, raw)


def test_walker_equals_zlib_at_every_level_and_strategy():
    rng = np.random.default_rng(5)
    rows = O.samples(rng, 16, 0, 60, 700)
    raw = O.filter_rows(rows, 2, [int(f) for f in rng.integers(0, 5, 60)])
    types = set()
    for level in range(10):
        for strategy in O.STRATEGIES:
            c = zlib.compressobj(level, zlib.DEFLATED, 15, 9, strategy)
            stream = c.compress(raw) + c.flush()
            blocks, got, _ = W.inflate_blocks(stream)
            assert got == raw, (level, strategy)
            _check_tiling(stream, blocks, raw)
            types |= {b[4] for b in blocks}
            if level == 0:
                assert {b[4] for b in blocks} == {0}
            if strategy == zlib.Z_FIXED and level:
                assert {b[4] for b in blocks} == {1}
    assert types == {0, 1, 2}


def test_walker_refuses_what_zlib_refuses():
    stream = zlib.compress(bytes(range(256)) * 40, 9)
    for bad in (stream[:len(stream) // 2], stream[:2] + bytes([stream[2] | 0b110]) + stream[3:]):
        with pytest.raises((ValueError, IndexError)):
            W.inflate_blocks(bad)
        with pytest.raises(zlib.error):
            zlib.decompress(bad)


def test_chain_places_stored_fixed_and_decoy_blocks():
    rng = np.random.default_rng(2)
    a = bytes(rng.integers(0, 8, 50000).astype(np.uint8))
    dec = W.decoy(1)
    stream, raw = W.chain([("deflate", a, 6, zlib.Z_DEFAULT_STRATEGY), ("stored", bytes(20000) + dec),
                           ("deflate", a[:9000], 6, zlib.Z_FIXED), ("deflate", a, 9, zlib.Z_DEFAULT_STRATEGY)])
    blocks, got, check = W.inflate_blocks(stream)
    assert got == raw == zlib.decompress(stream) and check == zlib.adler32(raw)
    types = [b[4] for b in blocks]
    assert 1 in types and types.index(1) < len(types) - 1
    stored = [b for b in blocks if b[4] == 0 and b[3] == 20000 + len(dec)][0]
    hidden = (stored[0] + 3 + 7) // 8 * 8 + 32 + 8 * 20000          # the decoy's header, inside the stored payload
    inner, _, _ = W.inflate_blocks(b"\x78\x9c" + dec + b"\x03\x00" + bytes(4))
    assert inner[0][4] == 2 and hidden not in [b[0] for b in blocks]
    assert stream[hidden // 8:hidden // 8 + len(dec)] == dec


def _src(nbytes, w=40, h=30, depth=8, ctype=0):
    return P.PngSource("x.png", w, h, depth, ctype, bytes(nbytes), None)


def test_pack_batch_reserves_the_parallel_records():
    assert not P.parallel_stream(P.PARALLEL_MIN_BYTES - 1) and P.parallel_stream(P.PARALLEL_MIN_BYTES)
    assert P.parallel_stream(P.PARALLEL_MAX_BYTES - 1) and not P.parallel_stream(P.PARALLEL_MAX_BYTES)
    sizes = [100, P.PARALLEL_MIN_BYTES, P.PARALLEL_MIN_BYTES - 1, 200000, 5, P.PARALLEL_MIN_BYTES + 1]
    srcs = [_src(n, 300 + k, 200, 16, 0) for k, n in enumerate(sizes)]
    crops = [D.Crops({"depth": (s, (0, 0, 8, 8))}, False, 8, 8) for s in srcs]
    pb = D.pack_batch(crops, 32, (0.5,) * 3, (0.5,) * 3)
    off, n, scratch = pb.png
    buf = pb.buffer.numpy()
    pd = buf[off * 16:].view(np.int32)[:n * D.PNG_FIELDS].reshape(n, D.PNG_FIELDS)
    rows = 0
    for d, s in zip(pd, srcs):
        assert d[13] * 16 == rows
        rows += -(-(s.height * (1 + 2 * s.width)) // 16) * 16
    end, units = rows, 0
    for d, s, nb in zip(pd, srcs, sizes):
        assert d[15] == units
        if P.parallel_stream(nb):
            assert d[14] * 16 == end
            end += P.record_bytes(nb, s.height * (1 + 2 * s.width))
            units += P.slices(nb) + P.MAX_WALKED
        else:
            assert d[14] == 0
    assert [bool(d[14]) for d in pd] == [False, True, False, True, False, True]
    assert P.slices(200000) == 13 and P.record_bytes(200000, 100) == 64 + 13 * 16 + 21 * 16 + 208
    assert scratch == end + n * P.FALLBACK_DESC_BYTES
    # a batch of short streams only: no records, no fallback descriptors, fields 14 and 15 zero
    pb = D.pack_batch(crops[:1] + crops[2:3], 32, (0.5,) * 3, (0.5,) * 3)
    off, n, scratch = pb.png
    pd = pb.buffer.numpy()[off * 16:].view(np.int32)[:n * D.PNG_FIELDS].reshape(n, D.PNG_FIELDS)
    assert not pd[:, 14:].any() and scratch == sum(-(-(s.height * (1 + 2 * s.width)) // 16) * 16
                                                   for s in (srcs[0], srcs[2]))


def test_constants_match_the_kernels():
    src = open(CU).read()

    def const(name):
        return int(eval(re.search(r"\b%s = ([^,;]+)[,;]" % name, src).group(1)))
    assert const("PNG_SLICE_BYTES") == P.SLICE_BYTES
    assert const("PNG_PARALLEL_MIN_BYTES") == P.PARALLEL_MIN_BYTES
    assert const("PNG_PARALLEL_MAX_BYTES") == P.PARALLEL_MAX_BYTES
    assert const("PNG_MAX_WALKED") == P.MAX_WALKED
    assert const("PNG_STREAM_RECORD") == P.STREAM_RECORD_BYTES
    assert const("PNG_SLICE_RECORD") == P.SLICE_RECORD_BYTES
    assert const("PNG_BLOCK_RECORD") == P.BLOCK_RECORD_BYTES
    states = re.search(r"enum \{ PAR_OK = 1, PAR_WALK = 2, PAR_BOUND = 3, PAR_EXPAND = 4, PAR_RESOLVE = 5 \}", src)
    assert states and (P.PATH_PARALLEL, P.PATH_WALK, P.PATH_BOUND, P.PATH_EXPAND, P.PATH_RESOLVE) == (1, 2, 3, 4, 5)
