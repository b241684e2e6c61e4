"""The worker half of decoding pre-training PNGs on the GPU (MMAE_GPU_JPEG): the chunk parser (csrc/png.cu decodes).

`parse(data, task)` accepts what the kernels decode bitwise as Pillow does: a non-interlaced PNG without tRNS whose
stored form the task's conversion maps by a copy or a table,
  rgb     8-bit gray ('L', replicated), 8-bit RGB ('RGB') or 8-bit palette ('P', looked up): Image.convert('RGB');
  depth   16-bit gray ('I;16'), used as stored;
  semseg  8-bit palette ('P') or 8-bit gray ('L'): Image.convert('P') keeps the index, and turns a gray level into the
          same index of a gray palette (both are an identity mapping of the stored samples).
For anything else it returns None and the caller decodes with Pillow: Adam7 interlacing, 1 / 2 / 4-bit samples, 16-bit
RGB, alpha, tRNS, APNG, other stored forms, files Pillow refuses to open (bad signature, IHDR fields, CRCs of the
chunks before the image data, which are the ones Pillow checks; a decompression bomb) and chunk layouts it treats in
ways not restated here.  The image data is checked on the GPU: a stream the kernels do not decode exactly as zlib and
Pillow do is decoded by Pillow after all (multimae_b200/data.py).
"""
import re
import struct
import zlib

from PIL import Image

SIGNATURE = b"\x89PNG\r\n\x1a\n"
# the parallel inflate (csrc/png.cu)
SLICE_BYTES = 16384            # compressed bytes per slice: one warp searches each for a block start
PARALLEL_MIN_BYTES = 32768     # shorter streams are inflated by one warp
PARALLEL_MAX_BYTES = 1 << 28   # so are longer ones (bit positions in int32)
MAX_WALKED = 8                 # blocks per stream that no slice found, decoded while confirming the chain
STREAM_RECORD_BYTES = 64       # int32 {state, blocks, blocks walked, Adler-32 in the stream, inflated bytes, ...}
SLICE_RECORD_BYTES = 16        # int32 {start bit or -1, end bit or -1, inflated bytes, ok | final << 1}
BLOCK_RECORD_BYTES = 16        # int32 {start bit, end bit, output offset, inflated bytes}
FALLBACK_DESC_BYTES = 64       # per image: its descriptor as the fallback inflate reads it
# stream record states: the parallel decode wrote the rows, or the stream went to the one-warp inflate because
# the walk met a block or a stream end it refuses, found more than MAX_WALKED blocks without a slice record, a block's
# second decode disagreed with its first, or a copy reached before the first byte / the Adler-32 differed
PATH_PARALLEL, PATH_WALK, PATH_BOUND, PATH_EXPAND, PATH_RESOLVE = 1, 2, 3, 4, 5
_CID = re.compile(rb"\w\w\w\w")                # Pillow's is_cid
_MODES = {(8, 0): "L", (16, 0): "I;16", (8, 2): "RGB", (8, 3): "P"}
_DECODED = {"rgb": ("L", "RGB", "P"), "depth": ("I;16",), "semseg": ("P", "L")}
# chunks before the image data whose Pillow handler cannot fail at these lengths (others with a handler fall back)
_HARMLESS = {b"gAMA": 4, b"sRGB": 1, b"pHYs": 9, b"cHRM": 32}
_HANDLED = {b"IHDR", b"PLTE", b"IDAT", b"IEND", b"tRNS", b"iCCP", b"tEXt", b"zTXt", b"iTXt", b"eXIf", b"acTL", b"fcTL",
            b"fdAT", b"sRGB", b"gAMA", b"cHRM", b"pHYs", b"bKGD", b"sBIT", b"tIME", b"hIST", b"sPLT", b"cICP", b"mDCv",
            b"cLLi"}


class PngSource:
    """A PNG the kernels decode: the file's path (for Pillow to decode it after all when the stream is not one the
    kernels decode exactly), the header fields, the joined zlib stream and, for a palette image, its colours padded to
    256 entries with zeros as Pillow's conversion reads them.  `size` is (width, height) and `mode` the PIL mode."""

    def __init__(self, path, width, height, depth, ctype, stream, palette):
        self.path, self.width, self.height, self.depth, self.ctype = path, width, height, depth, ctype
        self.stream, self.palette = stream, palette

    @property
    def size(self):
        return self.width, self.height

    @property
    def mode(self):
        return _MODES[self.depth, self.ctype]


def is_png(data):
    return data[:8] == SIGNATURE


def parallel_stream(nbytes):
    """Whether mmae_png_decode_batch tries the parallel inflate on a zlib stream of `nbytes` (csrc/png.cu's
    png_parallel); a stream it does not decode exactly is inflated by one warp after all."""
    return PARALLEL_MIN_BYTES <= nbytes < PARALLEL_MAX_BYTES


def slices(nbytes):
    return -(-nbytes // SLICE_BYTES)


def units(nbytes):
    """Warps per parallel stream in the search and expand launches: one per slice, and room for MAX_WALKED blocks."""
    return slices(nbytes) + MAX_WALKED


def record_bytes(nbytes, raw):
    """Scratch of one parallel stream of `nbytes` inflating to `raw` bytes: its stream record, slice records, block
    records, and a uint16 plane of the inflated bytes (0-255 a byte, 256 + j byte j of the 32 KiB before the block)."""
    return (STREAM_RECORD_BYTES + slices(nbytes) * SLICE_RECORD_BYTES + units(nbytes) * BLOCK_RECORD_BYTES
            + (2 * raw + 15) // 16 * 16)


def parse(data, task, path=None):
    """A PngSource for the file bytes `data` loaded for `task`, or None when the kernels do not decode it."""
    if task not in _DECODED and "semseg" not in task or not is_png(data):
        return None
    want = _DECODED["semseg" if "semseg" in task else task]
    n, pos = len(data), 8
    header, palette, idat = None, None, []
    while True:
        if pos + 8 > n:
            return None
        length, cid = struct.unpack_from(">I", data, pos)[0], data[pos + 4:pos + 8]
        body = pos + 8
        if not _CID.match(cid) or body + length + 4 > n:
            return None
        if cid == b"IDAT":
            break
        chunk = data[body:body + length]
        if struct.unpack_from(">I", data, body + length)[0] != zlib.crc32(cid + chunk):
            return None                          # Pillow raises SyntaxError
        if header is None:
            if cid != b"IHDR" or length != 13:
                return None
            w, h, depth, ctype, comp, filt, interlace = struct.unpack(">IIBBBBB", chunk)
            mode = _MODES.get((depth, ctype))
            if mode not in want or w == 0 or h == 0 or comp or filt or interlace:
                return None
            if Image.MAX_IMAGE_PIXELS is not None and w * h > 2 * Image.MAX_IMAGE_PIXELS:
                return None                      # Image.open raises DecompressionBombError
            header = (w, h, depth, ctype)
        elif cid == b"PLTE":
            if palette is not None or length == 0 or length % 3 or length > 768:
                return None
            palette = chunk + bytes(768 - length)
        elif cid in _HANDLED and _HARMLESS.get(cid) != length:
            return None
        pos = body + length + 4
    if header is None or (header[3] == 3 and palette is None):
        return None
    while pos + 8 <= n and data[pos + 4:pos + 8] == b"IDAT":
        length = struct.unpack_from(">I", data, pos)[0]
        if pos + 8 + length > n:
            return None
        idat.append(data[pos + 8:pos + 8 + length])
        pos += 12 + length
    if data[pos + 4:pos + 8] in (b"fdAT", b"DDAT"):
        return None                              # Pillow reads these as more image data
    w, h, depth, ctype = header
    return PngSource(path, w, h, depth, ctype, b"".join(idat), palette if ctype == 3 else None)
