"""Pure-Python deflate block walker: the oracle for the block chain the parallel inflate (csrc/png.cu) confirms, and
builders of zlib streams whose chains are chosen block by block.

inflate_blocks(stream) inflates a zlib stream (RFC 1950 / 1951) and lists its blocks: (start bit, end bit, output
offset, output bytes, block type, final), bit positions counted from the stream's first byte, LSB first, as the kernels
count them.  It is held to zlib.decompress by tests/test_png_parallel_host.py."""
import struct
import zlib

LEN_BASE = (3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195,
            227, 258)
LEN_EXTRA = (0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0)
DIST_BASE = (1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
             4097, 6145, 8193, 12289, 16385, 24577)
DIST_EXTRA = (0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13)
CL_ORDER = (16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)


def _table(lens):
    """A lookup of 2**max bits (LSB first) -> symbol << 4 | length, -1 where no code matches."""
    top = max(lens) or 1
    table = [-1] * (1 << top)
    code = 0
    for length in range(1, top + 1):
        for sym, n in enumerate(lens):
            if n == length:
                rev = int(format(code, "0%db" % length)[::-1], 2)
                for fill in range(rev, 1 << top, 1 << length):
                    table[fill] = sym << 4 | length
                code += 1
        code <<= 1
    return table, (1 << top) - 1


_FIXED = None


def _fixed():
    global _FIXED
    if _FIXED is None:
        _FIXED = (_table([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8), _table([5] * 30))
    return _FIXED


def inflate_blocks(stream):
    """([(start bit, end bit, output offset, output bytes, type, final)], inflated bytes, Adler-32 in the stream) of
    zlib stream `stream`; raises ValueError where it is not one."""
    data = bytes(stream)
    nbits = 8 * len(data)

    def peek(pos, k=4):
        return int.from_bytes(data[pos >> 3:(pos >> 3) + k], "little") >> (pos & 7)

    if len(data) < 2 or (data[0] * 256 + data[1]) % 31 or data[0] & 15 != 8 or data[1] & 32:
        raise ValueError("zlib header")
    out, blocks, pos = bytearray(), [], 16
    while True:
        start, o0 = pos, len(out)
        v = peek(pos)
        final, typ = v & 1, v >> 1 & 3
        pos += 3
        if typ == 0:
            pos = (pos + 7) & ~7
            n, nn = struct.unpack_from("<HH", data, pos >> 3)
            if n != nn ^ 0xFFFF:
                raise ValueError("stored length")
            b = (pos >> 3) + 4
            out += data[b:b + n]
            pos += 32 + 8 * n
        elif typ == 3:
            raise ValueError("block type 3")
        else:
            if typ == 1:
                (lt, lm), (dt, dm) = _fixed()
            else:
                v = peek(pos)
                nlen, ndist, ncode = (v & 31) + 257, (v >> 5 & 31) + 1, (v >> 10 & 15) + 4
                pos += 14
                cl = [0] * 19
                for k in range(ncode):
                    cl[CL_ORDER[k]] = peek(pos) & 7
                    pos += 3
                ct, cm = _table(cl)
                lens = []
                while len(lens) < nlen + ndist:
                    e = ct[peek(pos) & cm]
                    if e < 0:
                        raise ValueError("code length code")
                    pos += e & 15
                    sym = e >> 4
                    if sym < 16:
                        lens.append(sym)
                        continue
                    if sym == 16:
                        rep, val = 3 + (peek(pos) & 3), lens[-1]
                        pos += 2
                    elif sym == 17:
                        rep, val = 3 + (peek(pos) & 7), 0
                        pos += 3
                    else:
                        rep, val = 11 + (peek(pos) & 127), 0
                        pos += 7
                    lens += [val] * rep
                (lt, lm), (dt, dm) = _table(lens[:nlen]), _table(lens[nlen:nlen + ndist])
            while True:
                e = lt[peek(pos) & lm]
                if e < 0:
                    raise ValueError("literal / length code")
                pos += e & 15
                sym = e >> 4
                if sym < 256:
                    out.append(sym)
                    continue
                if sym == 256:
                    break
                i = sym - 257
                v = peek(pos, 8)
                n = LEN_BASE[i] + (v & ((1 << LEN_EXTRA[i]) - 1))
                v >>= LEN_EXTRA[i]
                e = dt[v & dm]
                if e < 0:
                    raise ValueError("distance code")
                ds = e >> 4
                v >>= e & 15
                d = DIST_BASE[ds] + (v & ((1 << DIST_EXTRA[ds]) - 1))
                pos += LEN_EXTRA[i] + (e & 15) + DIST_EXTRA[ds]
                if d > len(out):
                    raise ValueError("distance too far back")
                if d >= n:
                    out += out[len(out) - d:len(out) - d + n]
                else:
                    chunk = bytes(out[len(out) - d:])
                    out += (chunk * (n // d + 1))[:n]
        if pos > nbits:
            raise ValueError("truncated")
        blocks.append((start, pos, o0, len(out) - o0, typ, final))
        if final:
            break
    b = (pos + 7) >> 3
    if b + 4 > len(data):
        raise ValueError("no Adler-32")
    return blocks, bytes(out), struct.unpack_from(">I", data, b)[0]


def chain(pieces):
    """A zlib stream made of byte-aligned pieces, in order: ("deflate", bytes, level, strategy) a fresh deflate of the
    bytes (its own blocks, then an empty stored block from the sync flush), ("stored", bytes) one stored block.  The
    last piece's last block is final.  Returns (stream, inflated bytes)."""
    body, raw = b"", b""
    for k, piece in enumerate(pieces):
        last = k == len(pieces) - 1
        if piece[0] == "stored":
            data = piece[1]
            body += bytes([1 if last else 0]) + struct.pack("<HH", len(data), len(data) ^ 0xFFFF) + data
        else:
            _, data, level, strategy = piece
            c = zlib.compressobj(level, zlib.DEFLATED, -15, 9, strategy)
            body += c.compress(data) + c.flush(zlib.Z_FINISH if last else zlib.Z_SYNC_FLUSH)
        raw += piece[1]
    return b"\x78\x9c" + body + struct.pack(">I", zlib.adler32(raw)), raw


def decoy(seed=0, n=600):
    """The raw deflate of `n` seeded bytes in one non-final dynamic block, byte-aligned: a valid block header to hide in
    the payload of a stored block."""
    import numpy as np
    rng = np.random.default_rng(seed)
    data = bytes((rng.integers(0, 16, n) * 7 % 256).astype(np.uint8))
    c = zlib.compressobj(9, zlib.DEFLATED, -15, 9, zlib.Z_DEFAULT_STRATEGY)
    return c.compress(data) + c.flush(zlib.Z_SYNC_FLUSH)
