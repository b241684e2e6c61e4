"""The worker half of decoding classification JPEGs on the GPU (MMAE_GPU_AUGMENT): the marker parser, the Huffman tables
as the kernels read them (csrc/jpeg.cu) and the block geometry of a pixel rectangle.

`parse(data)` accepts what the kernels decode bitwise as libjpeg-turbo (Pillow's decoder) does: one interleaved scan of
an 8-bit baseline or extended-sequential Huffman JPEG with 1 component, or 3 YCbCr components whose luma is sampled 1x1,
2x1 or 2x2 and whose chroma is sampled 1x1, restart markers in sequence, ended by EOI.  For anything else it returns None
and the caller decodes with Pillow.  libjpeg's choices that decide the colour space are restated: JFIF implies YCbCr; an
Adobe APP14 transform flag 0 means RGB; without either, component ids 'R', 'G', 'B' mean RGB.  Files Pillow refuses to
open are returned as None too, so that Pillow raises for them: a side above libjpeg-turbo's 65500, or more than twice
PIL.Image.MAX_IMAGE_PIXELS pixels (DecompressionBombError).

The kernels restate libjpeg-turbo's x86-64 arithmetic; on other hosts (aarch64 runs its NEON IDCT) the decode equals
Pillow's on valid files, and on corrupt ones only where the two IDCTs agree.
"""
import functools
import re

import numpy as np
from PIL import Image

# jpeg_natural_order: zigzag index -> natural (row-major) index
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                   7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                   39, 46, 53, 60, 61, 54, 47, 55, 62, 63], np.int32)
LOOKAHEAD = 9                  # bits resolved by one lookup in the kernels' Huffman tables
TABLE_BYTES = 4 * (512 + 18 + 18) + 256
_SAMPLINGS = ((1, 1), (2, 1), (2, 2))
MAX_SIDE = 65500               # libjpeg-turbo's JPEG_MAX_DIMENSION
SUB_BYTES = 512                # bytes of entropy-coded data per subsequence of the parallel decode (csrc/jpeg.cu)
SLOT_BYTES = 256               # bytes of entropy-coded data per subsequence record reserved in the decode's scratch
PARALLEL_MIN_BYTES = 16384     # shorter restart intervals are decoded by one thread
PARALLEL_MAX_BYTES = 1 << 28   # so are longer ones (bit positions in int32)
SUB_RECORD_BYTES = 48          # one subsequence's record in the decode's scratch
_MARKER = re.compile(rb"\xff[^\x00]")


class JpegSource:
    """A JPEG the kernels decode: the file bytes, the frame, the tables of each component and the byte range of each
    restart interval of the entropy-coded segment.  `size` is (width, height), as PIL.Image.size."""

    def __init__(self, data, width, height, hmax, vmax, restart, scan, intervals, quant, tables):
        self.data, self.width, self.height, self.hmax, self.vmax = data, width, height, hmax, vmax
        self.restart, self.scan, self.intervals, self.quant, self.tables = restart, scan, intervals, quant, tables

    @property
    def size(self):
        return self.width, self.height

    @property
    def ncomp(self):
        return len(self.tables)


def _check_huffman(bits, vals, is_dc):
    """libjpeg's jpeg_make_d_derived_tbl checks: no code may be all ones, DC symbols are at most 15."""
    code = 0
    for l in range(1, 17):
        code += bits[l - 1]
        if code >= 1 << l:
            return False
        code <<= 1
    return not (is_dc and any(v > 15 for v in vals))


def parse(data):
    """A JpegSource for `data` (bytes), or None when the kernels do not decode it."""
    n = len(data)
    if n < 4 or data[0] != 0xFF or data[1] != 0xD8:
        return None
    pos, jfif, adobe, restart, frame = 2, False, None, 0, None
    quant, huff = {}, {}
    while True:
        if pos >= n or data[pos] != 0xFF:
            return None
        while pos < n and data[pos] == 0xFF:
            pos += 1
        if pos + 2 >= n:
            return None
        m = data[pos]
        if m == 0x01 or 0xD0 <= m <= 0xD9:
            return None
        length = (data[pos + 1] << 8) | data[pos + 2]
        seg = data[pos + 3:pos + 1 + length]
        if length < 2 or len(seg) != length - 2:
            return None
        pos += 1 + length
        if m == 0xE0 and len(seg) >= 14 and seg[:5] == b"JFIF\0":
            jfif = True
        elif m == 0xEE and len(seg) >= 12 and seg[:5] == b"Adobe":
            adobe = seg[11]
        elif m == 0xDB:
            k = 0
            while k < len(seg):
                pq, tq = seg[k] >> 4, seg[k] & 15
                size = 128 if pq else 64
                if pq > 1 or tq > 3 or k + 1 + size > len(seg):
                    return None
                q = np.frombuffer(seg, np.dtype(">u2") if pq else np.uint8, 64, k + 1).astype(np.int32)
                table = np.zeros(64, np.int32)
                table[ZIGZAG] = q
                quant[tq] = table
                k += 1 + size
        elif m == 0xC4:
            k = 0
            while k < len(seg):
                if k + 17 > len(seg):
                    return None
                tc, th, bits = seg[k] >> 4, seg[k] & 15, seg[k + 1:k + 17]
                count = sum(bits)
                if tc > 1 or th > 3 or count > 256 or k + 17 + count > len(seg):
                    return None
                huff[tc, th] = bytes(bits) + bytes(seg[k + 17:k + 17 + count])
                k += 17 + count
        elif m == 0xDD:
            if len(seg) < 2:
                return None
            restart = (seg[0] << 8) | seg[1]
        elif m in (0xC0, 0xC1):
            if frame is not None or len(seg) < 6 or seg[0] != 8:
                return None
            h, w, nc = (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if h == 0 or w == 0 or nc not in (1, 3) or len(seg) < 6 + 3 * nc or max(h, w) > MAX_SIDE:
                return None
            if Image.MAX_IMAGE_PIXELS is not None and w * h > 2 * Image.MAX_IMAGE_PIXELS:
                return None                      # Image.open raises DecompressionBombError
            frame = (w, h, [(seg[6 + 3 * c], seg[7 + 3 * c] >> 4, seg[7 + 3 * c] & 15, seg[8 + 3 * c]) for c in range(nc)])
        elif 0xC2 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            return None                          # progressive, lossless, hierarchical or arithmetic-coded
        elif m == 0xDA:
            break
    if frame is None:
        return None
    w, h, comps = frame
    nc = len(comps)
    if len(seg) != 4 + 2 * nc or seg[0] != nc or seg[-3:] != b"\x00\x3f\x00":
        return None                              # not one scan over every component in frame order
    if nc == 1:
        if comps[0][1:3] != (1, 1):
            return None
        hmax = vmax = 1
    else:
        if (comps[0][1], comps[0][2]) not in _SAMPLINGS or any(c[1:3] != (1, 1) for c in comps[1:]):
            return None
        hmax, vmax = comps[0][1], comps[0][2]
        ids = tuple(c[0] for c in comps)
        if not jfif and (adobe == 0 or (adobe is None and ids == (82, 71, 66))):
            return None                          # RGB, not YCbCr
    tables = []
    for c in range(nc):
        if seg[1 + 2 * c] != comps[c][0] or comps[c][3] not in quant:
            return None
        td, ta = seg[2 + 2 * c] >> 4, seg[2 + 2 * c] & 15
        dc, ac = huff.get((0, td)), huff.get((1, ta))
        if dc is None or ac is None or not _check_huffman(dc[:16], dc[16:], True) or \
                not _check_huffman(ac[:16], ac[16:], False):
            return None
        tables.append((dc, ac))
    start = pos
    mcus = -(-w // (8 * hmax)) * -(-h // (8 * vmax))
    nint = -(-mcus // restart) if restart else 1
    bounds = [start]
    for mk in _MARKER.finditer(data, start):
        x = data[mk.start() + 1]
        if x == 0xD9:
            if len(bounds) != 2 * nint - 1:
                return None
            bounds.append(mk.start())
            intervals = np.array(bounds, np.int32).reshape(-1, 2) - start
            return JpegSource(data, w, h, hmax, vmax, restart, (start, mk.start()), intervals,
                              np.stack([quant[c[3]] for c in comps]), tables)
        expect = 0xD0 + ((len(bounds) - 1) // 2) % 8
        if not restart or x != expect or len(bounds) >= 2 * nint - 1:
            return None                          # a marker other than the next restart marker inside the scan
        bounds += [mk.start(), mk.start() + 2]
    return None                                  # no EOI


@functools.lru_cache(maxsize=256)
def huffman_table_bytes(table):
    """One Huffman table (16 code-length counts then the symbols) as the kernels read it: int32 lookup[512] of the
    next 9 bits (length << 8 | symbol, 0 for longer codes), int32 maxcode[18] (-1 where no code has that length, 17 a
    sentinel), int32 valoffset[18], uint8 symbols[256]."""
    bits, vals = table[:16], table[16:]
    lookup = np.zeros(1 << LOOKAHEAD, np.int32)
    maxcode = np.full(18, -1, np.int32)
    valoffset = np.zeros(18, np.int32)
    code = p = 0
    for l in range(1, 17):
        if bits[l - 1]:
            valoffset[l] = p - code
            for _ in range(bits[l - 1]):
                if l <= LOOKAHEAD:
                    lookup[code << (LOOKAHEAD - l):(code + 1) << (LOOKAHEAD - l)] = (l << 8) | vals[p]
                code += 1
                p += 1
            maxcode[l] = code - 1
        code <<= 1
    maxcode[17] = 0xFFFFF
    symbols = np.zeros(256, np.uint8)
    symbols[:len(vals)] = np.frombuffer(vals, np.uint8)
    return np.concatenate([lookup, maxcode, valoffset]).view(np.uint8).tobytes() + symbols.tobytes()


def _window(lo, hi, sub, extent):
    """Sample range of a component that outputs [lo, hi] need: the same range, or for a component subsampled 2:1 the
    samples under it with the fancy upsampler's neighbours, inside the component's `extent` samples."""
    if not sub:
        return lo, hi
    return max((lo >> 1) - 1, 0), min((hi >> 1) + 1, extent - 1)


def geometry(width, height, ncomp, hmax, vmax, y0, x0, rh, rw):
    """The blocks that decoding the rectangle [y0, y0 + rh) x [x0, x0 + rw) needs, as csrc/jpeg.cu's jpeg_geometry
    computes them: (MCUs per row, first MCU row, end MCU row, blocks per MCU, [(first block row, end block row,
    first block column, end block column)] per component)."""
    mpr = -(-width // (8 * hmax))
    bpm = 1 if ncomp == 1 else hmax * vmax + 2
    wins, mcu0, mcu1 = [], None, 0
    for c in range(ncomp):
        hs, vs = (hmax, vmax) if c == 0 else (1, 1)
        r0, r1 = _window(y0, y0 + rh - 1, vs < vmax, -(-height * vs // vmax))
        c0, c1 = _window(x0, x0 + rw - 1, hs < hmax, -(-width * hs // hmax))
        win = (r0 >> 3, (r1 >> 3) + 1, c0 >> 3, (c1 >> 3) + 1)
        wins.append(win)
        mcu0 = win[0] // vs if mcu0 is None else min(mcu0, win[0] // vs)
        mcu1 = max(mcu1, (win[1] - 1) // vs + 1)
    return mpr, mcu0, mcu1, bpm, wins


def parallel_interval(nbytes):
    """Whether the kernels decode a restart interval of `nbytes` bytes of entropy-coded data in parallel (one CTA,
    subsequences of SUB_BYTES) rather than with one thread; csrc/jpeg.cu's jpeg_parallel_interval.  Corrupt data in
    such an interval still sends it to the one-thread decode."""
    return PARALLEL_MIN_BYTES <= nbytes < PARALLEL_MAX_BYTES


def subsequence_slots(data_bytes, nint):
    """Subsequence records an image of `data_bytes` bytes of entropy-coded data in `nint` restart intervals reserves in
    the decode's scratch: interval k's start at (its first byte) // SLOT_BYTES + k."""
    return data_bytes // SLOT_BYTES + nint


def subsequences(segment):
    """The subsequences the parallel decode cuts one restart interval's bytes into, as the kernel computes them:
    [(first byte, its index with the stuffed zero bytes removed)], one per SUB_BYTES, moved one byte on where it would
    start on the zero of an FF 00 pair."""
    seg = np.frombuffer(segment, np.uint8)
    n = len(seg)
    starts = [r + 1 if 0 < r < n and seg[r - 1] == 0xFF else r for r in range(0, n, SUB_BYTES)]
    ff = np.concatenate([[0], np.cumsum(seg == 0xFF)])
    return [(r, r - int(ff[r])) for r in starts]
