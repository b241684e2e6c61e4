// Pre-training PNG decode on the GPU (MMAE_GPU_JPEG): the pixel rectangle each sample's crop needs, decoded bitwise as
// Pillow decodes Image.open(f) (then convert('RGB') for rgb, convert('P') for semseg) for non-interlaced 8-bit gray,
// 8-bit RGB, 8-bit palette and 16-bit gray PNGs.
//
// The workers parse the chunks (multimae_b200/png.py) and pack, per sample, the IDAT payloads joined into one zlib
// stream and the palette; the decoded rectangle is written to a device-only tail of the same buffer, where
// mmae_augment_batch's descriptor points.  Two kernels for the whole batch:
//   1. png_inflate_kernel: one warp per stream.  Inflate is sequential, so every lane runs the same decode (the same
//      loads, no divergence); a literal is stored by lane 0 and a match is copied by the lanes in runs of up to 32
//      bytes.  Stored, fixed- and dynamic-Huffman blocks; the tables of each block are built in shared memory (lane 0
//      counts and lists the codes, the lanes fill a 9-bit lookup; longer codes take zlib's canonical walk).  Every check zlib's inflate makes is made, and the stream
//      must end as a well-formed stream ends: the last block's end code exactly at the image's last byte, then a
//      matching Adler-32.  Anything else sets a non-zero status word, and the host decodes that sample with Pillow,
//      which raises what it raises or gives the image it gives (multimae_b200/data.py).
//   2. png_unfilter_kernel: one block per image.  Every row's filter type is checked (Pillow refuses types above 4),
//      then one warp undoes filters 0-4 with PNG's byte-wise arithmetic up to the rectangle's last row (Sub, Average
//      and Paeth run along the row, one lane per byte of a pixel, through shared-memory tiles), and the block expands
//      the rectangle: uint8 RGB (gray replicated, palette looked up), uint16 depth (big-endian samples), uint8 semseg
//      indices.
//
// Streams of 32 KiB and more are inflated in parallel within the stream, in the manner of pugz (Kerbiriou & Chikhi,
// "Parallel decompression of gzip-compressed files and random access to DNA sequences", 2019) and rapidgzip (Knespel &
// Brunst, "Rapidgzip: Parallel Decompression and Seeking in Gzip Files Using Cache Prefetching", HPDC 2023).  zlib at
// its default level writes a chain of dynamic-Huffman blocks with bit-aligned boundaries (a 450 x 350 depth map: about
// 10), and each can be decoded once its start is known:
//   1. png_search_kernel, one warp per 16 KiB slice of compressed bytes: the lanes test consecutive bit positions from
//      the slice's start for a dynamic block header that passes every check zlib makes on one (dynamic_header_at), and
//      the warp decodes the first such block to its end, storing nothing: its start, end, length and whether it decoded
//      cleanly.  Slice 0 decodes its block from bit 16, whatever its type.
//   2. png_walk_kernel, one warp per stream: the chain from bit 16.  A block whose start a slice found is confirmed;
//      any other (stored and fixed blocks, a second block in a slice, a slice whose first candidate was false) is
//      decoded here, up to PNG_MAX_WALKED of them.  Then the stream's end: the rows' length, the Adler-32 after it.
//   3. png_expand_kernel, one warp per confirmed block: the block again from its start, into a uint16 plane at its
//      output offset; a byte copied from before the block's first byte is written as 256 + its place in the 32 KiB
//      window before the block, and copies carry these markers as they carry bytes.
//   4. png_resolve_kernel, one warp per stream: the blocks in order, markers replaced by the bytes of the blocks before
//      (final by then), a marker before the stream's first byte refused; then the Adler-32.
//   5. png_inflate_kernel, unchanged, on copies of the descriptors: every stream below the size or where a step above
//      refused anything (its status words are the sequential decode's, whatever the parallel one met), while the
//      streams decoded in parallel stop at once; png_merge_kernel then writes their status 0.
// Seven launches, no host synchronisation.  The search, walk, expand and resolve kernels run one warp per block under
// the same 32-register cap as png_inflate_kernel (1,024 registers, what an SM beside a 384-thread, 168-register GEMM CTA
// has left): search 5.5 KB of shared memory and 40 bytes of spill stores, walk 3.5 KB and 28 bytes, expand 3.5 KB,
// resolve none (-Xptxas -v).  png_merge_kernel's 128-thread blocks (10 registers; 2,048 with the per-warp allocation)
// do not fit there, but each writes 128 status words and ends within microseconds.
#include <climits>

#include "common.cuh"
#include "internal.h"

namespace mmae {
namespace {

constexpr int PD = 16;   // int32 fields of one image's descriptor
enum { PD_W, PD_H, PD_DEPTH, PD_CTYPE, PD_KIND, PD_DATA, PD_BYTES, PD_PALETTE, PD_Y0, PD_X0, PD_RH, PD_RW, PD_OUT,
       PD_RAW, PD_PAR, PD_UNIT };
enum { PNG_OK = 0, PNG_HEADER = 1, PNG_BROKEN = 2, PNG_DISTANCE = 3, PNG_SHORT = 4, PNG_SIZE = 5, PNG_CHECK = 6,
       PNG_FILTER = 7 };
// The inflate kernel is latency-bound (one sequential stream per warp) and its blocks can hold an SM for milliseconds
// beside a training step on another stream: one warp per block and at most 32 registers a thread (1,024 a block, what an
// SM running a 384-thread, 168-register GEMM CTA has left), 3.5 KB of shared memory.
constexpr int PNG_INFLATE_THREADS = 32, PNG_INFLATE_REGS = 32;
constexpr int PNG_UNFILTER_THREADS = 128;
constexpr int PNG_TILE = 960;          // bytes of a row per shared-memory tile: a multiple of every pixel size (1, 2, 3)
constexpr int PNG_LOOK = 9;            // bits resolved by one table lookup
constexpr int64_t PNG_MAX_RAW = INT_MAX;
// The parallel inflate (multimae_b200/png.py restates these): streams of PNG_PARALLEL_MIN_BYTES to
// PNG_PARALLEL_MAX_BYTES (bit positions in int32) are cut into slices of PNG_SLICE_BYTES; a stream whose chain has more
// than PNG_MAX_WALKED blocks that no slice found goes to png_inflate_kernel.
constexpr int PNG_SLICE_BYTES = 16384, PNG_PARALLEL_MIN_BYTES = 32768, PNG_PARALLEL_MAX_BYTES = 1 << 28;
constexpr int PNG_MAX_WALKED = 8;
constexpr int PNG_STREAM_RECORD = 64, PNG_SLICE_RECORD = 16, PNG_BLOCK_RECORD = 16, PNG_FALLBACK_DESC = PD * 4;
// stream record (int32 fields) and its state: which path the stream took
enum { SR_STATE, SR_BLOCKS, SR_WALKED, SR_CHECK, SR_OUT };
enum { PAR_OK = 1, PAR_WALK = 2, PAR_BOUND = 3, PAR_EXPAND = 4, PAR_RESOLVE = 5 };

__host__ __device__ inline bool png_parallel(int bytes) {
  return bytes >= PNG_PARALLEL_MIN_BYTES && bytes < PNG_PARALLEL_MAX_BYTES;
}
__host__ __device__ inline int png_slices(int bytes) { return (bytes + PNG_SLICE_BYTES - 1) / PNG_SLICE_BYTES; }
__host__ __device__ inline int png_units(int bytes) { return png_slices(bytes) + PNG_MAX_WALKED; }
// a parallel stream's records in the scratch: the stream record, a record per slice, a block record per unit, then the
// uint16 plane of its inflated bytes (0-255 a byte, 256 + j byte j of the 32 KiB window before the block)
__host__ __device__ inline int64_t png_area_bytes(int bytes, int64_t raw) {
  return PNG_STREAM_RECORD + int64_t(png_slices(bytes)) * PNG_SLICE_RECORD + int64_t(png_units(bytes)) * PNG_BLOCK_RECORD +
         (2 * raw + 15) / 16 * 16;
}

__host__ __device__ inline int png_bpp(int depth, int ctype) { return ctype == 2 ? 3 : depth / 8; }
__host__ __device__ inline int64_t png_raw_bytes(const int* d) {
  return int64_t(d[PD_H]) * (1 + int64_t(d[PD_W]) * png_bpp(d[PD_DEPTH], d[PD_CTYPE]));
}
__host__ __device__ inline int png_out_elem(int kind) { return kind == 0 ? 3 : kind == 1 ? 2 : 1; }

__constant__ unsigned short kLenBase[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                            31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ unsigned char kLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5,
                                            5, 5, 5, 0};
__constant__ unsigned short kDistBase[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,   97,
                                             129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193,
                                             12289, 16385, 24577};
__constant__ unsigned char kDistExtra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10,
                                             11, 11, 12, 12, 13, 13};
__constant__ unsigned char kClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// One canonical Huffman code: code-length counts, symbols in code order, and a 9-bit lookup (length << 9 | symbol,
// 0 where the code is longer or absent).
struct Huff {
  short count[16];
  short symbol[288];
  unsigned short look[1 << PNG_LOOK];
};

struct InflateShared {
  Huff lit, dist;
  unsigned char lens[320];
  int ok;
};

// LSB-first bit reader over one stream; bits past its end read as zeros and set `over`.
struct Bits {
  const uint8_t* p;
  int pos, n;
  uint64_t buf;
  int cnt;
  bool over;
  __device__ __forceinline__ void need(int k) {
    while (cnt < k) {
      uint64_t v = 0;
      if (pos < n) v = __ldg(p + pos);
      else over = true;
      ++pos;
      buf |= v << cnt;
      cnt += 8;
    }
  }
  __device__ __forceinline__ uint32_t peek(int k) { need(k); return uint32_t(buf & ((1ull << k) - 1)); }
  __device__ __forceinline__ void drop(int k) { buf >>= k; cnt -= k; }
  __device__ __forceinline__ uint32_t get(int k) {
    if (k == 0) return 0;
    const uint32_t v = peek(k);
    drop(k);
    return v;
  }
  // bits are loaded ahead of use: the stream is overrun only when a bit past its end has been consumed
  __device__ __forceinline__ bool past_end() const { return int64_t(pos) * 8 - cnt > int64_t(n) * 8; }
  __device__ __forceinline__ int64_t bit() const { return int64_t(pos) * 8 - cnt; }
};

// A reader positioned at bit `at` of the stream (whole bytes are loaded, so byte alignment stays drop(cnt & 7)).
__device__ __forceinline__ Bits bits_at(const uint8_t* p, int n, int64_t at) {
  Bits br{p, int(at >> 3), n, 0ull, 0, false};
  br.get(int(at & 7));
  return br;
}

// zlib's canonical walk over `bits` (LSB first): the symbol and code length, or length 0 for no code.
__device__ int huff_walk(const Huff& h, uint32_t bits, int& len) {
  int code = 0, first = 0, index = 0;
  for (int l = 1; l <= 15; ++l) {
    code |= int(bits >> (l - 1)) & 1;
    const int count = h.count[l];
    if (code - count < first) {
      len = l;
      return h.symbol[index + (code - first)];
    }
    index += count;
    first += count;
    first <<= 1;
    code <<= 1;
  }
  len = 0;
  return -1;
}

// Build `h` from lens[0..n): lane 0 counts the lengths and lists the symbols, every lane fills part of the lookup.
// kind 0: code-length code (must be complete), 1: literal / length or distance code (incomplete only when it is a single
// 1-bit code).  false: zlib refuses the set.
__device__ bool huff_build(Huff& h, const unsigned char* lens, int n, int kind, int lane, int& ok) {
  __syncwarp();
  if (lane == 0) {
    for (int l = 0; l < 16; ++l) h.count[l] = 0;
    for (int s = 0; s < n; ++s) ++h.count[lens[s]];
    h.count[0] = 0;
    int max = 15, left = 1;
    while (max >= 1 && h.count[max] == 0) --max;
    ok = 1;
    for (int l = 1; l <= 15 && ok; ++l) {
      left = (left << 1) - h.count[l];
      if (left < 0) ok = 0;                                            // over-subscribed
    }
    if (ok && max > 0 && left > 0 && (kind == 0 || max != 1)) ok = 0;  // incomplete
    int k = 0;
    for (int l = 1; l <= max && ok; ++l)
      for (int s = 0; s < n; ++s)
        if (lens[s] == l) h.symbol[k++] = short(s);
  }
  __syncwarp();
  if (!ok) return false;
  for (int e = lane; e < (1 << PNG_LOOK); e += 32) {
    int len;
    const int s = huff_walk(h, uint32_t(e), len);
    h.look[e] = len >= 1 && len <= PNG_LOOK ? (unsigned short)((len << 9) | s) : 0;
  }
  __syncwarp();
  return true;
}

__device__ __forceinline__ int huff_decode(const Huff& h, Bits& br) {
  const uint32_t bits = br.peek(15);
  const int e = h.look[bits & ((1 << PNG_LOOK) - 1)];
  if (e) {
    br.drop(e >> 9);
    return e & 511;
  }
  int len;
  const int s = huff_walk(h, bits, len);
  if (len == 0) return -1;
  br.drop(len);
  return s;
}

struct Adler {
  uint64_t s1 = 0, s2 = 0;   // sums of b and of (total - position) * b over the bytes this lane stored
  __device__ __forceinline__ void add(int64_t total, int64_t p, int b) {
    s1 += uint64_t(b);
    s2 += uint64_t(uint32_t(total - p) % 65521u) * uint64_t(b);
  }
};

__global__ void __maxnreg__(PNG_INFLATE_REGS)
    png_inflate_kernel(const uint8_t* __restrict__ buf, const int* __restrict__ pd, uint8_t* raw_base, int* status) {
  pdl_prologue();
  __shared__ InflateShared sh;
  const int lane = threadIdx.x;
  const int* d = pd + int64_t(blockIdx.x) * PD;
  uint8_t* out = raw_base + int64_t(d[PD_RAW]) * 16;
  const int64_t total = png_raw_bytes(d);
  Bits br{buf + int64_t(d[PD_DATA]) * 16, 0, d[PD_BYTES], 0ull, 0, false};
  Adler ad;
  int64_t pos = 0;
  int st = PNG_OK;
  {
    const uint32_t cmf = br.get(8), flg = br.get(8);
    if ((cmf * 256 + flg) % 31 != 0 || (cmf & 15) != 8 || (cmf >> 4) > 7 || (flg & 32)) st = PNG_HEADER;
  }
  bool last = false;
  while (st == PNG_OK && !last) {
    last = br.get(1);
    const int type = int(br.get(2));
    if (type == 0) {
      br.drop(br.cnt & 7);
      const uint32_t len = br.get(16), nlen = br.get(16);
      if (len != (~nlen & 0xFFFF)) { st = PNG_BROKEN; break; }
      if (pos + len > total) { st = PNG_SIZE; break; }
      for (uint32_t k = 0; k < len; ++k) {
        const int b = int(br.get(8));
        if (lane == 0) { out[pos] = uint8_t(b); ad.add(total, pos, b); }
        ++pos;
      }
      if (br.past_end()) { st = PNG_SHORT; break; }
      continue;
    }
    if (type == 3) { st = PNG_BROKEN; break; }
    if (type == 1) {
      for (int s = lane; s < 320; s += 32)
        sh.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
      __syncwarp();
      huff_build(sh.lit, sh.lens, 288, 1, lane, sh.ok);
      huff_build(sh.dist, sh.lens + 288, 32, 1, lane, sh.ok);   // symbols 30 and 31 decode, and are refused below
    } else {
      const int nlen = int(br.get(5)) + 257, ndist = int(br.get(5)) + 1, ncode = int(br.get(4)) + 4;
      if (nlen > 286 || ndist > 30) { st = PNG_BROKEN; break; }
      __syncwarp();
      for (int s = lane; s < 19; s += 32) sh.lens[s] = 0;
      __syncwarp();
      for (int k = 0; k < ncode; ++k) {
        const int v = int(br.get(3));
        if (lane == 0) sh.lens[kClOrder[k]] = uint8_t(v);
      }
      __syncwarp();
      if (!huff_build(sh.lit, sh.lens, 19, 0, lane, sh.ok)) { st = PNG_BROKEN; break; }
      int have = 0;   // every lane follows the same walk; lane 0 writes
      while (have < nlen + ndist) {
        const int sym = huff_decode(sh.lit, br);
        if (sym < 0) { st = PNG_BROKEN; break; }
        if (sym < 16) {
          if (lane == 0) sh.lens[have] = uint8_t(sym);
          ++have;
          __syncwarp();
          continue;
        }
        int rep, val = 0;
        if (sym == 16) {
          if (have == 0) { st = PNG_BROKEN; break; }
          val = sh.lens[have - 1];
          rep = 3 + int(br.get(2));
        } else if (sym == 17) {
          rep = 3 + int(br.get(3));
        } else {
          rep = 11 + int(br.get(7));
        }
        if (have + rep > nlen + ndist) { st = PNG_BROKEN; break; }
        __syncwarp();
        for (int k = lane; k < rep; k += 32) sh.lens[have + k] = uint8_t(val);
        have += rep;
        __syncwarp();
      }
      if (st != PNG_OK) break;
      if (sh.lens[256] == 0) { st = PNG_BROKEN; break; }   // no end-of-block code
      if (!huff_build(sh.lit, sh.lens, nlen, 1, lane, sh.ok)) { st = PNG_BROKEN; break; }
      if (!huff_build(sh.dist, sh.lens + nlen, ndist, 1, lane, sh.ok)) { st = PNG_BROKEN; break; }
    }
    // the block's symbols
    for (;;) {
      const int sym = huff_decode(sh.lit, br);
      if (sym < 0 || sym > 285) { st = PNG_BROKEN; break; }
      if (sym < 256) {
        if (pos >= total) { st = PNG_SIZE; break; }
        if (lane == 0) { out[pos] = uint8_t(sym); ad.add(total, pos, sym); }
        ++pos;
        continue;
      }
      if (sym == 256) break;
      const int len = kLenBase[sym - 257] + int(br.get(kLenExtra[sym - 257]));
      const int ds = huff_decode(sh.dist, br);
      if (ds < 0 || ds > 29) { st = PNG_BROKEN; break; }
      const int dist = kDistBase[ds] + int(br.get(kDistExtra[ds]));
      if (dist > pos) { st = PNG_DISTANCE; break; }
      if (pos + len > total) { st = PNG_SIZE; break; }
      const int step = dist < 32 ? dist : 32;   // a run of `step` bytes reads only bytes already stored
      for (int k = 0; k < len; k += step) {
        __syncwarp();
        if (lane < step && k + lane < len) {
          const int64_t p = pos + k + lane;
          const int b = out[p - dist];
          out[p] = uint8_t(b);
          ad.add(total, p, b);
        }
      }
      __syncwarp();
      pos += len;
    }
    if (st == PNG_OK && br.past_end()) st = PNG_SHORT;
  }
  if (st == PNG_OK && br.past_end()) st = PNG_SHORT;
  if (st == PNG_OK && pos != total) st = PNG_SIZE;
  if (st == PNG_OK) {
    br.drop(br.cnt & 7);
    uint32_t want = 0;
    for (int k = 0; k < 4; ++k) want = (want << 8) | br.get(8);   // Adler-32, big-endian
    uint64_t s1 = ad.s1 % 65521, s2 = ad.s2 % 65521;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    const uint32_t a = uint32_t((1 + s1) % 65521), b = uint32_t((uint64_t(total % 65521) + s2) % 65521);
    if (br.past_end()) st = PNG_SHORT;
    else if (((b << 16) | a) != want) st = PNG_CHECK;
  }
  if (lane == 0) status[blockIdx.x] = st;
}

// ---------------------------------------------------------------------------------------------------------------------
// Parallel inflate.
// ---------------------------------------------------------------------------------------------------------------------
struct Area {
  int* sr;          // stream record
  int4* slices;     // {first candidate's start bit or -1, end bit or -1, output bytes, ok | final << 1}
  int4* blocks;     // {start bit, end bit, output offset, output bytes} of the chain's blocks in order
  uint16_t* plane;
};

__device__ __forceinline__ Area png_area(uint8_t* scratch, const int* d) {
  uint8_t* a = scratch + int64_t(d[PD_PAR]) * 16;
  const int ns = png_slices(d[PD_BYTES]), nu = png_units(d[PD_BYTES]);
  int4* slices = reinterpret_cast<int4*>(a + PNG_STREAM_RECORD);
  return {reinterpret_cast<int*>(a), slices, slices + ns, reinterpret_cast<uint16_t*>(slices + ns + nu)};
}

// The stream that owns unit u: the last descriptor whose first unit is at most u.
__device__ int png_unit_owner(const int* pd, int n, int u) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (pd[int64_t(mid) * PD + PD_UNIT] <= u) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// One deflate block from br's position, its 3 header bits first, with every check png_inflate_kernel makes on a block
// except those that need the output before it (a distance reaching before the stream's first byte, the running
// length).  false: the block is refused.  len: its output bytes, at most `limit`; final: its BFINAL bit.  kWrite: the
// block's output goes to plane[0, len) as plane values; a copy source before plane[0] is written as 256 + j, j its
// place in the 32 KiB window before the block.  Every lane runs the same decode; lane 0 writes literals.
template <bool kWrite>
__device__ bool inflate_block(InflateShared& sh, Bits& br, int lane, int64_t limit, uint16_t* plane, int64_t& len,
                              bool& final) {
  final = br.get(1);
  const int type = int(br.get(2));
  len = 0;
  if (type == 0) {
    br.drop(br.cnt & 7);
    const uint32_t n = br.get(16), nn = br.get(16);
    if (n != (~nn & 0xFFFF) || n > limit) return false;
    const int64_t at = br.pos - br.cnt / 8;   // the stored bytes: whole bytes from here
    if (at + n > br.n) return false;
    if (kWrite)
      for (uint32_t k = lane; k < n; k += 32) plane[k] = __ldg(br.p + at + k);
    br.pos = int(at + n);
    br.cnt = 0;
    br.buf = 0;
    len = n;
    return true;
  }
  if (type == 3) return false;
  if (type == 1) {
    __syncwarp();
    for (int s = lane; s < 320; s += 32) sh.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
    __syncwarp();
    huff_build(sh.lit, sh.lens, 288, 1, lane, sh.ok);
    huff_build(sh.dist, sh.lens + 288, 32, 1, lane, sh.ok);
  } else {
    const int nlen = int(br.get(5)) + 257, ndist = int(br.get(5)) + 1, ncode = int(br.get(4)) + 4;
    if (nlen > 286 || ndist > 30) return false;
    __syncwarp();
    for (int s = lane; s < 19; s += 32) sh.lens[s] = 0;
    __syncwarp();
    for (int k = 0; k < ncode; ++k) {
      const int v = int(br.get(3));
      if (lane == 0) sh.lens[kClOrder[k]] = uint8_t(v);
    }
    __syncwarp();
    if (!huff_build(sh.lit, sh.lens, 19, 0, lane, sh.ok)) return false;
    int have = 0;
    while (have < nlen + ndist) {
      const int sym = huff_decode(sh.lit, br);
      if (sym < 0) return false;
      if (sym < 16) {
        if (lane == 0) sh.lens[have] = uint8_t(sym);
        ++have;
        __syncwarp();
        continue;
      }
      int rep, val = 0;
      if (sym == 16) {
        if (have == 0) return false;
        val = sh.lens[have - 1];
        rep = 3 + int(br.get(2));
      } else if (sym == 17) {
        rep = 3 + int(br.get(3));
      } else {
        rep = 11 + int(br.get(7));
      }
      if (have + rep > nlen + ndist) return false;
      __syncwarp();
      for (int k = lane; k < rep; k += 32) sh.lens[have + k] = uint8_t(val);
      have += rep;
      __syncwarp();
    }
    if (sh.lens[256] == 0) return false;
    if (!huff_build(sh.lit, sh.lens, nlen, 1, lane, sh.ok)) return false;
    if (!huff_build(sh.dist, sh.lens + nlen, ndist, 1, lane, sh.ok)) return false;
  }
  for (;;) {
    // past the stream's end the block is refused whatever follows; stop here rather than decode zero bits (a false
    // candidate of the search could otherwise run on until `limit`)
    if (br.past_end()) return false;
    const int sym = huff_decode(sh.lit, br);
    if (sym < 0 || sym > 285) return false;
    if (sym < 256) {
      if (len >= limit) return false;
      if (kWrite && lane == 0) plane[len] = uint16_t(sym);
      ++len;
      continue;
    }
    if (sym == 256) break;
    const int n = kLenBase[sym - 257] + int(br.get(kLenExtra[sym - 257]));
    const int ds = huff_decode(sh.dist, br);
    if (ds < 0 || ds > 29) return false;
    const int dist = kDistBase[ds] + int(br.get(kDistExtra[ds]));
    if (len + n > limit) return false;
    if (kWrite) {
      const int step = dist < 32 ? dist : 32;
      for (int k = 0; k < n; k += step) {
        __syncwarp();
        if (lane < step && k + lane < n) {
          const int64_t q = len + k + lane, src = q - dist;
          plane[q] = src >= 0 ? plane[src] : uint16_t(256 + 32768 + src);
        }
      }
      __syncwarp();
    }
    len += n;
  }
  return !br.past_end();
}

// Whether a dynamic block header at bit `at` passes every check zlib's inflate makes on one (BTYPE 2, HLIT and HDIST
// at most 29, a complete code-length code, exactly HLIT + 257 + HDIST + 1 lengths with no repeat first, literal /
// length and distance codes huff_build accepts, a length for the end-of-block code).  One lane, one position; cnt: the
// lane's 32 counters.
__device__ bool dynamic_header_at(const uint8_t* p, int n, int64_t at, unsigned short* cnt) {
  Bits br = bits_at(p, n, at);
  br.get(1);
  if (br.get(2) != 2) return false;
  const int nlen = int(br.get(5)) + 257, ndist = int(br.get(5)) + 1, ncode = int(br.get(4)) + 4;
  if (nlen > 286 || ndist > 30) return false;
  uint64_t cl = 0, cc = 0;   // 3-bit lengths of the 19 code-length symbols; 5-bit counts per length
  for (int k = 0; k < ncode; ++k) cl |= uint64_t(br.get(3)) << (3 * kClOrder[k]);
  for (int s = 0; s < 19; ++s) cc += 1ull << (5 * ((cl >> (3 * s)) & 7));
  int left = 1;
  for (int l = 1; l <= 7; ++l) {
    left = 2 * left - int((cc >> (5 * l)) & 31);
    if (left < 0) return false;
  }
  if (left != 0) return false;
  for (int l = 0; l < 32; ++l) cnt[l] = 0;
  const int total = nlen + ndist;
  int have = 0, prev = 0, eob = 0;
  while (have < total) {
    int sym = -1;
    for (int l = 1, code = 0, first = 0; l <= 7; ++l) {   // zlib's canonical walk, symbols of a length in order
      code |= int(br.get(1));
      const int c = int((cc >> (5 * l)) & 31);
      if (code - c < first) {
        int want = code - first;
        for (int s = 0; s < 19; ++s)
          if (int((cl >> (3 * s)) & 7) == l && want-- == 0) { sym = s; break; }
        break;
      }
      first = (first + c) << 1;
      code <<= 1;
    }
    if (sym < 0) return false;
    int rep = 1, v = sym;
    if (sym == 16) {
      if (have == 0) return false;
      v = prev;
      rep = 3 + int(br.get(2));
    } else if (sym == 17) {
      v = 0;
      rep = 3 + int(br.get(3));
    } else if (sym == 18) {
      v = 0;
      rep = 11 + int(br.get(7));
    }
    if (have + rep > total) return false;
    const int nl = min(max(nlen - have, 0), rep);
    cnt[v] += nl;
    cnt[16 + v] += rep - nl;
    if (have <= 256 && 256 < have + rep) eob = v;
    prev = v;
    have += rep;
  }
  if (eob == 0 || br.past_end()) return false;
  for (int c = 0; c < 32; c += 16) {   // as huff_build: not over-subscribed, complete unless a single 1-bit code
    int lft = 1, max = 0;
    for (int l = 1; l <= 15; ++l) {
      lft = 2 * lft - cnt[c + l];
      if (lft < 0) return false;
      if (cnt[c + l]) max = l;
    }
    if (max > 0 && lft > 0 && max != 1) return false;
  }
  return true;
}

// 1. Search: one warp per slice.  Slice 0 decodes its block from bit 16; any other takes the first bit of the slice
// where dynamic_header_at holds (32 positions at a time) and decodes that block, storing nothing.
__global__ void __maxnreg__(PNG_INFLATE_REGS)
    png_search_kernel(const uint8_t* __restrict__ buf, const int* __restrict__ pd, int n, uint8_t* scratch) {
  pdl_prologue();
  __shared__ InflateShared sh;
  __shared__ unsigned short cnt[32][32];
  const int lane = threadIdx.x;
  const int* d = pd + int64_t(png_unit_owner(pd, n, blockIdx.x)) * PD;
  const int s = int(blockIdx.x) - d[PD_UNIT], bytes = d[PD_BYTES];
  if (d[PD_PAR] == 0 || s >= png_slices(bytes)) return;
  const Area ar = png_area(scratch, d);
  const uint8_t* p = buf + int64_t(d[PD_DATA]) * 16;
  int64_t start = -1;
  if (s == 0) {
    start = 16;
  } else {
    const int64_t lo = int64_t(s) * PNG_SLICE_BYTES * 8, hi = min(lo + PNG_SLICE_BYTES * 8, int64_t(bytes) * 8);
    for (int64_t b0 = lo; b0 < hi; b0 += 32) {
      const bool hit = b0 + lane < hi && dynamic_header_at(p, bytes, b0 + lane, cnt[lane]);
      const unsigned m = __ballot_sync(0xffffffffu, hit);
      if (m) {
        start = b0 + __ffs(m) - 1;
        break;
      }
    }
  }
  int4 rec = make_int4(int(start), -1, 0, 0);
  if (start >= 0) {
    Bits br = bits_at(p, bytes, start);
    int64_t len;
    bool final;
    if (inflate_block<false>(sh, br, lane, png_raw_bytes(d), nullptr, len, final))
      rec = make_int4(int(start), int(br.bit()), int(len), 1 | (final ? 2 : 0));
  }
  if (lane == 0) ar.slices[s] = rec;
}

// 2. Confirm: one warp per stream walks the chain from bit 16.  A block whose start a slice record holds takes that
// record; any other block is decoded here (at most PNG_MAX_WALKED).  Then the stream's end: the running length equals
// the image's rows, and the Adler-32 follows at the next byte.
__global__ void __maxnreg__(PNG_INFLATE_REGS)
    png_walk_kernel(const uint8_t* __restrict__ buf, const int* __restrict__ pd, uint8_t* scratch) {
  pdl_prologue();
  __shared__ InflateShared sh;
  const int lane = threadIdx.x;
  const int* d = pd + int64_t(blockIdx.x) * PD;
  if (d[PD_PAR] == 0) return;
  const Area ar = png_area(scratch, d);
  const int bytes = d[PD_BYTES];
  const uint8_t* p = buf + int64_t(d[PD_DATA]) * 16;
  const int64_t total = png_raw_bytes(d);
  int state = PAR_OK, nb = 0, walked = 0;
  uint32_t want = 0;
  {
    const uint32_t cmf = p[0], flg = p[1];
    if ((cmf * 256 + flg) % 31 != 0 || (cmf & 15) != 8 || (cmf >> 4) > 7 || (flg & 32)) state = PAR_WALK;
  }
  int64_t at = 16, out = 0;
  bool last = false;
  while (state == PAR_OK && !last) {
    if (at >= int64_t(bytes) * 8) { state = PAR_WALK; break; }
    const int4 r = ar.slices[at / (PNG_SLICE_BYTES * 8)];
    int64_t end, len;
    if (r.x == at && (r.w & 1)) {
      end = r.y;
      len = r.z;
      last = r.w & 2;
    } else {
      if (++walked > PNG_MAX_WALKED) { state = PAR_BOUND; break; }
      Bits br = bits_at(p, bytes, at);
      if (!inflate_block<false>(sh, br, lane, total - out, nullptr, len, last)) { state = PAR_WALK; break; }
      end = br.bit();
    }
    if (out + len > total) { state = PAR_WALK; break; }
    if (lane == 0) ar.blocks[nb] = make_int4(int(at), int(end), int(out), int(len));
    ++nb;
    out += len;
    at = end;
  }
  if (state == PAR_OK && out != total) state = PAR_WALK;
  if (state == PAR_OK) {
    const int64_t b = (at + 7) >> 3;
    if (b + 4 > bytes) state = PAR_WALK;
    else want = (uint32_t(p[b]) << 24) | (uint32_t(p[b + 1]) << 16) | (uint32_t(p[b + 2]) << 8) | p[b + 3];
  }
  if (lane == 0) {
    ar.sr[SR_STATE] = state;
    ar.sr[SR_BLOCKS] = state == PAR_OK ? nb : 0;
    ar.sr[SR_WALKED] = walked;
    ar.sr[SR_CHECK] = int(want);
    ar.sr[SR_OUT] = int(out);
  }
}

// 3. Expand: one warp per block of a confirmed chain decodes it again from its start into the plane at its offset.
__global__ void __maxnreg__(PNG_INFLATE_REGS)
    png_expand_kernel(const uint8_t* __restrict__ buf, const int* __restrict__ pd, int n, uint8_t* scratch) {
  pdl_prologue();
  __shared__ InflateShared sh;
  const int lane = threadIdx.x;
  const int* d = pd + int64_t(png_unit_owner(pd, n, blockIdx.x)) * PD;
  if (d[PD_PAR] == 0) return;
  const Area ar = png_area(scratch, d);
  const int k = int(blockIdx.x) - d[PD_UNIT];
  if (ar.sr[SR_STATE] != PAR_OK || k >= ar.sr[SR_BLOCKS]) return;
  const int4 blk = ar.blocks[k];
  Bits br = bits_at(buf + int64_t(d[PD_DATA]) * 16, d[PD_BYTES], blk.x);
  int64_t len;
  bool final;
  const bool ok = inflate_block<true>(sh, br, lane, blk.w, ar.plane + blk.z, len, final);
  if (lane == 0 && (!ok || len != blk.w || br.bit() != blk.y)) ar.sr[SR_STATE] = PAR_EXPAND;
}

// 4. Resolve: one warp per stream takes its blocks in order and turns the plane into bytes (a window byte reads the
// bytes of the blocks before, final by then), then checks the Adler-32.  Every stream's descriptor is copied for the
// fallback launch, with no stream bytes where the parallel decode succeeded.
__global__ void __maxnreg__(PNG_INFLATE_REGS)
    png_resolve_kernel(const int* __restrict__ pd, uint8_t* raw_base, uint8_t* scratch, int* fallback) {
  pdl_prologue();
  const int lane = threadIdx.x;
  const int* d = pd + int64_t(blockIdx.x) * PD;
  int* fb = fallback + int64_t(blockIdx.x) * PD;
  if (lane < PD) fb[lane] = d[lane];
  if (d[PD_PAR] == 0) return;
  const Area ar = png_area(scratch, d);
  if (ar.sr[SR_STATE] != PAR_OK) return;
  uint8_t* out = raw_base + int64_t(d[PD_RAW]) * 16;
  const int64_t total = png_raw_bytes(d);
  const int nb = ar.sr[SR_BLOCKS];
  Adler ad;
  bool bad = false;
  for (int k = 0; k < nb; ++k) {
    const int4 blk = ar.blocks[k];
    const int64_t o0 = blk.z, o1 = int64_t(blk.z) + blk.w;
    for (int64_t q0 = o0 + lane; q0 < o1; q0 += 4 * 32) {
      int v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = q0 + 32 * j < o1 ? ar.plane[q0 + 32 * j] : 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (v[j] >= 256) {
          const int64_t src = o0 - 32768 + (v[j] - 256);
          bad |= src < 0;
          v[j] = src < 0 ? 0 : out[src];
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (q0 + 32 * j < o1) {
          out[q0 + 32 * j] = uint8_t(v[j]);
          ad.add(total, q0 + 32 * j, v[j]);
        }
      }
    }
    __syncwarp();
  }
  uint64_t s1 = ad.s1 % 65521, s2 = ad.s2 % 65521;
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  bad = __any_sync(0xffffffffu, bad);
  const uint32_t a = uint32_t((1 + s1) % 65521), b = uint32_t((uint64_t(total % 65521) + s2) % 65521);
  if (lane == 0) {
    if (bad || ((b << 16) | a) != uint32_t(ar.sr[SR_CHECK])) ar.sr[SR_STATE] = PAR_RESOLVE;
    else fb[PD_BYTES] = 0;   // png_inflate_kernel stops at the missing zlib header without touching the rows
  }
}

// 6. After png_inflate_kernel has decoded the other streams: status 0 for every stream the parallel decode took.
__global__ void png_merge_kernel(const int* __restrict__ pd, int n, uint8_t* scratch, int* status) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int* d = pd + int64_t(i) * PD;
  if (d[PD_PAR] != 0 && png_area(scratch, d).sr[SR_STATE] == PAR_OK) status[i] = PNG_OK;
}

__device__ __forceinline__ int paeth(int a, int b, int c) {
  const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
  return pa <= pb && pa <= pc ? a : pb <= pc ? b : c;
}

__global__ void __launch_bounds__(PNG_UNFILTER_THREADS)
    png_unfilter_kernel(const uint8_t* __restrict__ buf, const int* __restrict__ pd, uint8_t* raw_base, int* status,
                        uint8_t* out_base) {
  pdl_prologue();   // raw and status are the previous kernel's output: plain loads
  __shared__ uint8_t cur_t[PNG_TILE], pri_t[PNG_TILE];
  __shared__ int bad;
  const int* d = pd + int64_t(blockIdx.x) * PD;
  if (status[blockIdx.x] != PNG_OK) return;
  const int W = d[PD_W], H = d[PD_H], ct = d[PD_CTYPE], kind = d[PD_KIND];
  const int bpp = png_bpp(d[PD_DEPTH], ct);
  const int64_t rb = int64_t(W) * bpp, pitch = rb + 1;
  uint8_t* raw = raw_base + int64_t(d[PD_RAW]) * 16;
  if (threadIdx.x == 0) bad = 0;
  __syncthreads();
  for (int r = threadIdx.x; r < H; r += PNG_UNFILTER_THREADS)
    if (raw[int64_t(r) * pitch] > 4) bad = 1;
  __syncthreads();
  if (bad) {
    if (threadIdx.x == 0) status[blockIdx.x] = PNG_FILTER;
    return;
  }
  const int rows = d[PD_Y0] + d[PD_RH];
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    for (int r = 0; r < rows; ++r) {
      const int f = raw[int64_t(r) * pitch];
      uint8_t* cur = raw + int64_t(r) * pitch + 1;
      const uint8_t* pri = r ? cur - pitch : nullptr;
      if (f == 2 && pri) {
        for (int64_t x = lane; x < rb; x += 32) cur[x] = uint8_t(cur[x] + pri[x]);
      } else if (f == 1 || f == 3 || f == 4) {
        int a = 0, c = 0;   // this lane's byte of the pixel to the left: unfiltered, and the one above it
        for (int64_t t0 = 0; t0 < rb; t0 += PNG_TILE) {
          const int n = int(rb - t0 < PNG_TILE ? rb - t0 : PNG_TILE);
          for (int x = lane; x < n; x += 32) {
            cur_t[x] = cur[t0 + x];
            pri_t[x] = pri ? pri[t0 + x] : 0;
          }
          __syncwarp();
          if (lane < bpp) {
            for (int x = lane; x < n; x += bpp) {
              const int b = pri_t[x];
              const int pred = f == 1 ? a : f == 3 ? (a + b) >> 1 : paeth(a, b, c);
              a = uint8_t(cur_t[x] + pred);
              c = b;
              cur_t[x] = uint8_t(a);
            }
          }
          __syncwarp();
          for (int x = lane; x < n; x += 32) cur[t0 + x] = cur_t[x];
          __syncwarp();
        }
      }
      __syncwarp();
    }
  }
  __syncthreads();
  const int y0 = d[PD_Y0], x0 = d[PD_X0], rw = d[PD_RW];
  const int64_t n = int64_t(d[PD_RH]) * rw;
  const uint8_t* pal = buf + int64_t(d[PD_PALETTE]) * 16;
  uint8_t* o = out_base + int64_t(d[PD_OUT]) * 16;
  for (int64_t t = threadIdx.x; t < n; t += PNG_UNFILTER_THREADS) {
    const int y = y0 + int(t / rw), x = x0 + int(t % rw);
    const uint8_t* row = raw + int64_t(y) * pitch + 1;
    if (kind == 1) {
      reinterpret_cast<uint16_t*>(o)[t] = uint16_t((row[2 * x] << 8) | row[2 * x + 1]);
    } else if (kind == 2) {
      o[t] = row[x];
    } else if (ct == 2) {
      o[3 * t] = row[3 * x];
      o[3 * t + 1] = row[3 * x + 1];
      o[3 * t + 2] = row[3 * x + 2];
    } else if (ct == 3) {
      const int i = row[x];
      o[3 * t] = pal[3 * i];
      o[3 * t + 1] = pal[3 * i + 1];
      o[3 * t + 2] = pal[3 * i + 2];
    } else {
      o[3 * t] = o[3 * t + 1] = o[3 * t + 2] = row[x];
    }
  }
}

}  // namespace
}  // namespace mmae

using namespace mmae;

extern "C" int mmae_png_decode_batch(const void* packed_host, void* packed, int64_t host_bytes, int64_t packed_bytes,
                                     int num_images, int64_t desc_offset, void* scratch, int64_t scratch_bytes,
                                     int* status, void* stream) {
  MMAE_CHECK(packed_host && packed && scratch && status, MMAE_ERR_ARG, "mmae_png_decode_batch: null pointer");
  MMAE_CHECK(num_images >= 1 && num_images <= 65535, MMAE_ERR_ARG, "mmae_png_decode_batch: bad image count %d",
             num_images);
  MMAE_CHECK(((reinterpret_cast<uintptr_t>(packed) | reinterpret_cast<uintptr_t>(scratch)) & 15) == 0, MMAE_ERR_ARG,
             "mmae_png_decode_batch: buffers must be 16-byte aligned");
  MMAE_CHECK(host_bytes >= 0 && host_bytes <= packed_bytes, MMAE_ERR_ARG,
             "mmae_png_decode_batch: host part of %lld bytes, buffer of %lld", (long long)host_bytes,
             (long long)packed_bytes);
  MMAE_CHECK(desc_offset >= 0 && desc_offset * 16 + int64_t(num_images) * PD * 4 <= host_bytes, MMAE_ERR_ARG,
             "mmae_png_decode_batch: descriptors outside the host part");
  const uint8_t* host = static_cast<const uint8_t*>(packed_host);
  const int* pd_host = reinterpret_cast<const int*>(host + desc_offset * 16);
  auto inside = [&](int64_t off16, int64_t bytes) { return off16 >= 0 && off16 * 16 + bytes <= host_bytes; };
  int64_t raw_end = 0, out_end = host_bytes;
  for (int i = 0; i < num_images; ++i) {
    const int* d = pd_host + int64_t(i) * PD;
    const int W = d[PD_W], H = d[PD_H], depth = d[PD_DEPTH], ct = d[PD_CTYPE], kind = d[PD_KIND];
    MMAE_CHECK(W >= 1 && H >= 1, MMAE_ERR_ARG, "mmae_png_decode_batch: image %d: size %d x %d", i, W, H);
    const bool form = (kind == 0 && depth == 8 && (ct == 0 || ct == 2 || ct == 3)) ||
                      (kind == 1 && depth == 16 && ct == 0) || (kind == 2 && depth == 8 && (ct == 0 || ct == 3));
    MMAE_CHECK(form, MMAE_ERR_ARG, "mmae_png_decode_batch: image %d: output kind %d from bit depth %d, colour type %d",
               i, kind, depth, ct);
    MMAE_CHECK(d[PD_Y0] >= 0 && d[PD_X0] >= 0 && d[PD_RH] >= 1 && d[PD_RW] >= 1 && d[PD_Y0] <= H - d[PD_RH] &&
                   d[PD_X0] <= W - d[PD_RW],
               MMAE_ERR_ARG, "mmae_png_decode_batch: image %d: rectangle (%d, %d) + %d x %d outside %d x %d", i,
               d[PD_Y0], d[PD_X0], d[PD_RH], d[PD_RW], H, W);
    const int64_t raw = png_raw_bytes(d);
    MMAE_CHECK(raw <= PNG_MAX_RAW, MMAE_ERR_ARG, "mmae_png_decode_batch: image %d: %lld decoded bytes", i,
               (long long)raw);
    MMAE_CHECK(d[PD_BYTES] >= 0 && inside(d[PD_DATA], d[PD_BYTES]), MMAE_ERR_ARG,
               "mmae_png_decode_batch: image %d: stream outside the host part", i);
    MMAE_CHECK(!(kind == 0 && ct == 3) || inside(d[PD_PALETTE], 768), MMAE_ERR_ARG,
               "mmae_png_decode_batch: image %d: palette outside the host part", i);
    MMAE_CHECK(int64_t(d[PD_RAW]) * 16 == raw_end, MMAE_ERR_ARG,
               "mmae_png_decode_batch: image %d: scratch offset %d, expected %lld", i, d[PD_RAW],
               (long long)(raw_end / 16));
    raw_end += int64_t(align_up(size_t(raw), 16));
    MMAE_CHECK(raw_end / 16 < INT_MAX, MMAE_ERR_ARG, "mmae_png_decode_batch: scratch offsets overflow");
    const int64_t out_bytes = int64_t(d[PD_RH]) * d[PD_RW] * png_out_elem(kind);
    MMAE_CHECK(d[PD_OUT] >= 0 && int64_t(d[PD_OUT]) * 16 >= out_end &&
                   int64_t(d[PD_OUT]) * 16 + out_bytes <= packed_bytes,
               MMAE_ERR_ARG, "mmae_png_decode_batch: image %d: output overlaps the host part or the previous output, "
               "or leaves the buffer", i);
    out_end = int64_t(d[PD_OUT]) * 16 + out_bytes;
  }
  // the parallel streams' records after every image's rows, then the fallback launch's descriptors
  int64_t end = raw_end, units = 0;
  for (int i = 0; i < num_images; ++i) {
    const int* d = pd_host + int64_t(i) * PD;
    const bool par = png_parallel(d[PD_BYTES]);
    MMAE_CHECK(int64_t(d[PD_PAR]) * 16 == (par ? end : 0), MMAE_ERR_ARG,
               "mmae_png_decode_batch: image %d: record offset %d, expected %lld", i, d[PD_PAR],
               (long long)(par ? end / 16 : 0));
    MMAE_CHECK(int64_t(d[PD_UNIT]) == units, MMAE_ERR_ARG, "mmae_png_decode_batch: image %d: first unit %d, expected %lld",
               i, d[PD_UNIT], (long long)units);
    if (par) {
      end += png_area_bytes(d[PD_BYTES], png_raw_bytes(d));
      units += png_units(d[PD_BYTES]);
    }
    MMAE_CHECK(end / 16 < INT_MAX && units < INT_MAX, MMAE_ERR_ARG, "mmae_png_decode_batch: scratch offsets overflow");
  }
  const int64_t fallback_off = end;
  if (units) end += int64_t(num_images) * PNG_FALLBACK_DESC;
  MMAE_CHECK(end <= scratch_bytes, MMAE_ERR_ARG, "mmae_png_decode_batch: scratch of %lld bytes, %lld needed",
             (long long)scratch_bytes, (long long)end);

  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* buf = static_cast<uint8_t*>(packed);
  const int* pd = reinterpret_cast<const int*>(buf + desc_offset * 16);
  uint8_t* raw = static_cast<uint8_t*>(scratch);
  const unsigned n = unsigned(num_images);
  if (units == 0) {
    launch_k(png_inflate_kernel, dim3(n), PNG_INFLATE_THREADS, 0, st, static_cast<const uint8_t*>(buf), pd, raw,
             status);
    count_launch();
    MMAE_LAUNCH_OK();
  } else {
    int* fallback = reinterpret_cast<int*>(raw + fallback_off);
    const uint8_t* cbuf = buf;
    launch_k(png_search_kernel, dim3(unsigned(units)), 32, 0, st, cbuf, pd, num_images, raw);
    count_launch();
    MMAE_LAUNCH_OK();
    launch_k(png_walk_kernel, dim3(n), 32, 0, st, cbuf, pd, raw);
    count_launch();
    MMAE_LAUNCH_OK();
    launch_k(png_expand_kernel, dim3(unsigned(units)), 32, 0, st, cbuf, pd, num_images, raw);
    count_launch();
    MMAE_LAUNCH_OK();
    launch_k(png_resolve_kernel, dim3(n), 32, 0, st, pd, raw, raw, fallback);
    count_launch();
    MMAE_LAUNCH_OK();
    launch_k(png_inflate_kernel, dim3(n), PNG_INFLATE_THREADS, 0, st, cbuf, static_cast<const int*>(fallback), raw,
             status);
    count_launch();
    MMAE_LAUNCH_OK();
    launch_k(png_merge_kernel, dim3((n + 127) / 128), 128, 0, st, pd, num_images, raw, status);
    count_launch();
    MMAE_LAUNCH_OK();
  }
  launch_k(png_unfilter_kernel, dim3(n), PNG_UNFILTER_THREADS, 0, st, static_cast<const uint8_t*>(buf), pd, raw,
           status, buf);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}
