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
#include <climits>

#include "common.cuh"
#include "internal.h"

namespace mmae {
namespace {

constexpr int PD = 16;   // int32 fields of one image's descriptor
enum { PD_W, PD_H, PD_DEPTH, PD_CTYPE, PD_KIND, PD_DATA, PD_BYTES, PD_PALETTE, PD_Y0, PD_X0, PD_RH, PD_RW, PD_OUT,
       PD_RAW };
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
};

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
  MMAE_CHECK(raw_end <= scratch_bytes, MMAE_ERR_ARG, "mmae_png_decode_batch: scratch of %lld bytes, %lld needed",
             (long long)scratch_bytes, (long long)raw_end);

  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* buf = static_cast<uint8_t*>(packed);
  const int* pd = reinterpret_cast<const int*>(buf + desc_offset * 16);
  uint8_t* raw = static_cast<uint8_t*>(scratch);
  const unsigned n = unsigned(num_images);
  launch_k(png_inflate_kernel, dim3(n), PNG_INFLATE_THREADS, 0, st, static_cast<const uint8_t*>(buf), pd, raw, status);
  count_launch();
  MMAE_LAUNCH_OK();
  launch_k(png_unfilter_kernel, dim3(n), PNG_UNFILTER_THREADS, 0, st, static_cast<const uint8_t*>(buf), pd, raw,
           status, buf);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}
