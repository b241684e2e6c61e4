// Classification JPEG decode on the GPU (MMAE_GPU_AUGMENT): the pixel rectangle each sample's transform needs, decoded
// bitwise as libjpeg-turbo decodes it for Pillow's Image.open(f).convert('RGB') on x86-64.
//
// The workers parse the markers (multimae_b200/jpeg.py) and pack, per sample, the entropy-coded segment as it is in the
// file, the byte range of each restart interval, the quantisation tables (natural order) and Huffman lookup tables; the
// decoded rectangle is written to a device-only tail of the same buffer, where mmae_cls_augment_batch's descriptor
// points.  Four kernels for the whole batch:
//   1a. jpeg_parallel_kernel: one CTA of 256 threads per restart interval of at least 16 KiB of entropy-coded data
//      (most files have none, so that is the whole scan) cuts the interval into 512-byte subsequences and decodes them
//      in parallel, synchronising their start states through the Huffman code's self-synchronisation (see the kernel).
//      The interval is left to 1b whenever its decode meets one of libjpeg-turbo's corrupt-data paths or does not end
//      on the interval's last MCU in its last byte.  64 registers (__launch_bounds__(256, 4)), 128 bytes of shared
//      memory, no spills: four CTAs fit an SM, but not beside a 384-thread, 168-register GEMM CTA, so while a training
//      step's GEMMs hold the SMs its CTAs wait for SMs between GEMM CTAs.
//   1b. jpeg_entropy_kernel: one thread per (image, restart interval) runs jdhuff.c's sequential decode up to the last
//      MCU row the rectangle needs, for the intervals 1a does not decode.  Its corrupt-data paths are kept: a code
//      longer than 16 bits is symbol 0 after 17 bits; bits past the interval's data read as zeros, and after the MCU
//      that read them the interval's remaining MCUs stay all-zero (the coefficient scratch is cleared first); DC
//      prediction restarts at every interval.  32 registers, 8 bytes of stack, no shared memory.
//   2. jpeg_idct_kernel: dequantisation and jpeg_idct_islow of the blocks the rectangle and its upsampling context
//      need, with the arithmetic of libjpeg-turbo's x86-64 SIMD version (jidctint-avx2.asm): 16-bit dequantised
//      values, the sums x0 +- x4, x7 + x3, x5 + x1 in 16 bits, outputs saturated to 16 and then 8 bits.  For every
//      coefficient a valid JPEG holds that is jidctint.c's integer result; they differ only on corrupt data.  So the
//      decode equals Pillow's on corrupt data only where Pillow runs that code (x86-64 hosts); on aarch64 hosts
//      (libjpeg-turbo's NEON IDCT) it equals Pillow's on valid files.
//   3. jpeg_color_kernel: h2v1 / h2v2 fancy upsampling (jdsample.c, box replication when the chroma is at most 2
//      samples wide, image-edge rows and columns replicated) and jdcolor.c's fixed-point YCbCr -> RGB; uint8 RGB out.
#include <climits>

#include "common.cuh"
#include "internal.h"

namespace mmae {
namespace {

constexpr int JD = 32;   // int32 fields of one image's descriptor
enum {
  JD_W, JD_H, JD_NCOMP, JD_HMAX, JD_VMAX, JD_RESTART, JD_DATA, JD_DATA_BYTES, JD_NINT, JD_INT, JD_QUANT,
  JD_HUFF,                                       // 6 fields: DC, AC table / 16 of components 0, 1, 2
  JD_Y0 = JD_HUFF + 6, JD_X0, JD_RH, JD_RW, JD_OUT, JD_COEF, JD_PLANE, JD_SUB
};
constexpr int JPEG_LOOKAHEAD = 9;
constexpr int JPEG_TABLE_BYTES = 4 * ((1 << JPEG_LOOKAHEAD) + 18 + 18) + 256;
// The entropy kernel is latency-bound (one sequential thread per interval) and its blocks can hold an SM for tens of
// milliseconds beside a training step on another stream: one warp per block and at most 32 registers a thread (1,024 a
// block, what an SM running a 384-thread, 168-register GEMM CTA has left), no shared and no local memory.
constexpr int JPEG_ENTROPY_THREADS = 32, JPEG_ENTROPY_REGS = 32;
constexpr int JPEG_IDCT_THREADS = 128, JPEG_COLOR_THREADS = 256;
constexpr int JPEG_MAX_SIDE = 65500;   // libjpeg-turbo's JPEG_MAX_DIMENSION
// Parallel entropy decode: subsequences of JPEG_SUB_BYTES bytes of entropy-coded data, one CTA of JPEG_PAR_THREADS per
// restart interval.  Measured on an H100 (700 W) over batches of 128 quality-90 4:2:0 images of 300-600 pixels a side,
// per call: without restart markers 11.1 / 9.2 / 9.1 / 8.9 / 14.1 ms for subsequences of 256 / 512 / 1024 / 2048 /
// 4096 bytes (sequential: 98.6 ms); with a marker every 4 MCU rows (intervals of about 36 KiB) 5.9 / 6.6 / 9.6 / 13.8 /
// 25.0 ms (sequential: 21.9 ms); with one every MCU row (about 9 KiB) 11.2 / 12.0 / 14.7 / 11.8 ms against 8.5 ms
// sequential.  Hence 512 bytes, and intervals under 16 KiB are left to the sequential kernel, as are those of 2^28
// bytes or more (bit positions are int32).  Record slots stay 256 bytes, so the layout does not depend on the choice.
constexpr int JPEG_SLOT_BYTES = 256, JPEG_SUB_BYTES = 512, JPEG_PAR_THREADS = 256;
constexpr int JPEG_PAR_MIN_BYTES = 16384, JPEG_PAR_MAX_BYTES = 1 << 28;
static_assert(JPEG_SUB_BYTES % JPEG_SLOT_BYTES == 0, "subsequences span whole record slots");

// One subsequence's record in the scratch.  An image's records start at its descriptor's JD_SUB; interval k's at
// JD_SUB + (its first byte) / JPEG_SLOT_BYTES + k, which leaves room for ceil(bytes / JPEG_SLOT_BYTES) records.
struct JpegSub {
  int raw, ubyte;      // first byte in the interval's data, and its index once the stuffed zero bytes are removed
  int s_pos, s_bk;     // start state: unstuffed bit position, block in the MCU << 8 | zig-zag index
  int x_pos, x_bk;     // exit state: the first symbol boundary at or past the next subsequence's first bit
  int blocks;          // blocks completed from start to exit; after the scan, the blocks before the start
  unsigned dc[3];      // DC differences summed per component; after the scan, the DC predictions at the start
  int flags;           // JPEG_SUB_DIRTY, JPEG_SUB_BAD
  int fallback;        // the interval's first record: 1 if the sequential kernel decodes the interval
};
constexpr int JPEG_SUB_DIRTY = 1, JPEG_SUB_BAD = 2;

__host__ __device__ inline bool jpeg_parallel_interval(int bytes) {
  return bytes >= JPEG_PAR_MIN_BYTES && bytes < JPEG_PAR_MAX_BYTES;
}

// jpeg_natural_order with the 16 guard entries that keep a corrupt run inside the block.
__constant__ unsigned char kNatural[80] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
    6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
    39, 46, 53, 60, 61, 54, 47, 55, 62, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63};

struct JpegGeom {
  int ncomp, mpr, rows, mcu0, mcu1, bpm;
  int win[3][4];        // per component: first block row, end block row, first block column, end block column
  int64_t plane[3];     // byte offset of each component's plane from the image's first plane
  int64_t plane_bytes;  // all three
  int64_t blocks;       // window blocks, all components
};

__host__ __device__ inline void jpeg_range(int lo, int hi, bool sub, int extent, int& a, int& b) {
  if (sub) {
    lo = (lo >> 1) - 1;
    hi = (hi >> 1) + 1;
    lo = lo < 0 ? 0 : lo;
    hi = hi > extent - 1 ? extent - 1 : hi;
  }
  a = lo;
  b = hi;
}

// multimae_b200/jpeg.py:geometry: the MCU rows and, per component, the blocks the rectangle needs.
__host__ __device__ inline JpegGeom jpeg_geometry(const int* d) {
  JpegGeom g;
  const int W = d[JD_W], H = d[JD_H], hm = d[JD_HMAX], vm = d[JD_VMAX];
  g.ncomp = d[JD_NCOMP];
  g.mpr = (W + 8 * hm - 1) / (8 * hm);
  g.rows = (H + 8 * vm - 1) / (8 * vm);
  g.bpm = g.ncomp == 1 ? 1 : hm * vm + 2;
  g.mcu0 = INT_MAX;
  g.mcu1 = 0;
  g.plane_bytes = 0;
  g.blocks = 0;
#pragma unroll
  for (int c = 0; c < 3; ++c) {   // unrolled: constant indices keep the struct in registers
    if (c >= g.ncomp) break;
    const int hs = c ? 1 : hm, vs = c ? 1 : vm;
    int r0, r1, c0, c1;
    jpeg_range(d[JD_Y0], d[JD_Y0] + d[JD_RH] - 1, vs < vm, (H * vs + vm - 1) / vm, r0, r1);
    jpeg_range(d[JD_X0], d[JD_X0] + d[JD_RW] - 1, hs < hm, (W * hs + hm - 1) / hm, c0, c1);
    int* w = g.win[c];
    w[0] = r0 >> 3;
    w[1] = (r1 >> 3) + 1;
    w[2] = c0 >> 3;
    w[3] = (c1 >> 3) + 1;
    g.mcu0 = w[0] / vs < g.mcu0 ? w[0] / vs : g.mcu0;
    g.mcu1 = (w[1] - 1) / vs + 1 > g.mcu1 ? (w[1] - 1) / vs + 1 : g.mcu1;
    g.plane[c] = g.plane_bytes;
    g.plane_bytes += int64_t(w[1] - w[0]) * (w[3] - w[2]) * 64;
    g.blocks += int64_t(w[1] - w[0]) * (w[3] - w[2]);
  }
  return g;
}

__host__ __device__ inline int64_t jpeg_coef_blocks(const JpegGeom& g) {
  return int64_t(g.mcu1 - g.mcu0) * g.mpr * g.bpm;
}

// ---------------------------------------------------------------------------------------------------------------------
// 1. Entropy decode
// ---------------------------------------------------------------------------------------------------------------------
struct BitReader {
  const uint8_t* p;
  int pos, n;
  uint64_t acc;   // valid bits left-aligned
  int nbits;      // valid bits in acc
  int pad;        // how many of them (the last ones) are zeros read past the data
  bool beyond;    // a bit past the data was consumed
  int bit = 0;         // bits consumed (the parallel decode's position; dead code in the sequential kernel)
  bool long_code = false;   // a code longer than 16 bits was read (likewise)

  __device__ __forceinline__ void fill() {
    while (nbits <= 56) {
      uint32_t v = 0;
      if (pos < n) {
        v = p[pos];
        pos += v == 0xFF ? 2 : 1;   // FF 00 is a stuffed FF data byte
      } else {
        pad += 8;
      }
      acc |= uint64_t(v) << (56 - nbits);
      nbits += 8;
    }
  }
  __device__ __forceinline__ uint32_t peek(int k) const { return uint32_t(acc >> (64 - k)); }
  __device__ __forceinline__ void drop(int k) {
    acc <<= k;
    nbits -= k;
    bit += k;
    if (nbits < pad) beyond = true;
  }
  __device__ __forceinline__ int get(int k) {
    fill();
    const int v = int(peek(k));
    drop(k);
    return v;
  }
  __device__ __forceinline__ int huff(const uint8_t* t) {
    fill();
    const int* lookup = reinterpret_cast<const int*>(t);
    const int* maxcode = lookup + (1 << JPEG_LOOKAHEAD);
    const int* valoffset = maxcode + 18;
    const uint8_t* symbols = reinterpret_cast<const uint8_t*>(valoffset + 18);
    const int e = lookup[peek(JPEG_LOOKAHEAD)];
    const int len = e >> 8;
    if (len >= 1 && len <= JPEG_LOOKAHEAD) {
      drop(len);
      return e & 0xFF;
    }
    for (int l = JPEG_LOOKAHEAD + 1; l <= 16; ++l) {
      const int code = int(peek(l));
      if (code <= maxcode[l]) {
        drop(l);
        return symbols[(code + valoffset[l]) & 0xFF];
      }
    }
    long_code = true;
    drop(17);
    return 0;
  }
};

__device__ __forceinline__ int huff_extend(int v, int s) { return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v; }

__global__ void __maxnreg__(JPEG_ENTROPY_REGS)
    jpeg_entropy_kernel(const uint8_t* __restrict__ buf, const int* __restrict__ jd, const JpegSub* subs,
                        int16_t* coef) {
  pdl_prologue();   // subs: the parallel kernel's output
  const int* d = jd + int64_t(blockIdx.y) * JD;
  const int k = blockIdx.x * JPEG_ENTROPY_THREADS + threadIdx.x;
  if (k >= d[JD_NINT]) return;
  const JpegGeom g = jpeg_geometry(d);
  // MCU counts fit in int: at most ceil(65500 / 8)^2
  const int total = g.mpr * g.rows;
  const int ri = d[JD_RESTART] ? d[JD_RESTART] : total;
  const int first = k * ri, last = min(first + ri, total);   // k < intervals, so k * ri < total + ri
  const int lo = g.mcu0 * g.mpr, hi = min(g.mcu1 * g.mpr, last);
  if (first >= hi || last <= lo) return;
  const int* iv = reinterpret_cast<const int*>(buf + int64_t(d[JD_INT]) * 16) + 2 * k;
  if (jpeg_parallel_interval(iv[1] - iv[0]) && !subs[d[JD_SUB] + iv[0] / JPEG_SLOT_BYTES + k].fallback) return;
  BitReader br{buf + int64_t(d[JD_DATA]) * 16 + iv[0], 0, iv[1] - iv[0], 0ull, 0, 0, false};
  const int bpm = g.bpm, ncomp = g.ncomp;
  int pred0 = 0, pred1 = 0, pred2 = 0;   // DC predictions of the components (scalars: no local memory)
  for (int m = first; m < hi; ++m) {
    int16_t* out = m >= lo ? coef + (int64_t(d[JD_COEF]) + int64_t(m - lo) * bpm) * 64 : nullptr;
    for (int b = 0; b < bpm; ++b) {
      const int c = b < bpm - 2 || ncomp == 1 ? 0 : b - (bpm - 3);
      const uint8_t* dc_tab = buf + int64_t(d[JD_HUFF + 2 * c]) * 16;
      const uint8_t* ac_tab = buf + int64_t(d[JD_HUFF + 2 * c + 1]) * 16;
      int s = br.huff(dc_tab) & 15;
      if (s) s = huff_extend(br.get(s), s);
      const int pred = int(unsigned(c == 0 ? pred0 : c == 1 ? pred1 : pred2) + unsigned(s));
      pred0 = c == 0 ? pred : pred0;
      pred1 = c == 1 ? pred : pred1;
      pred2 = c == 2 ? pred : pred2;
      if (out) out[b * 64] = int16_t(pred);
      for (int kk = 1; kk < 64; ++kk) {
        const int rs = br.huff(ac_tab);
        const int r = rs >> 4;
        s = rs & 15;
        if (s) {
          kk += r;
          const int v = huff_extend(br.get(s), s);
          if (out) out[b * 64 + kNatural[kk]] = int16_t(v);
        } else {
          if (r != 15) break;
          kk += 15;
        }
      }
    }
    if (br.beyond) break;   // libjpeg-turbo leaves the interval's later MCUs zero
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// 1a. Parallel entropy decode (Weissenberger & Schmidt, ICPP 2018): one CTA per restart interval of at least
//     JPEG_PAR_MIN_BYTES, run before jpeg_entropy_kernel, which decodes the intervals this kernel leaves to it.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 add4(uint4 a, uint4 b) { return make_uint4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }

// Exclusive prefix sums (wrapping) of v over the CTA in thread order, starting from `carry`, which becomes carry + the
// CTA's total.  Every thread calls it; `warp_sums` is shared [JPEG_PAR_THREADS / 32].
__device__ uint4 cta_scan(uint4 v, uint4& carry, uint4* warp_sums) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint4 x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint4 y = make_uint4(__shfl_up_sync(~0u, x.x, o), __shfl_up_sync(~0u, x.y, o), __shfl_up_sync(~0u, x.z, o),
                               __shfl_up_sync(~0u, x.w, o));
    if (lane >= o) x = add4(x, y);
  }
  if (lane == 31) warp_sums[w] = x;
  __syncthreads();
  uint4 before = carry, total = carry;
  for (int i = 0; i < JPEG_PAR_THREADS / 32; ++i) {
    if (i < w) before = add4(before, warp_sums[i]);
    total = add4(total, warp_sums[i]);
  }
  __syncthreads();   // warp_sums is reused by the next call
  carry = total;
  return add4(before, make_uint4(x.x - v.x, x.y - v.y, x.z - v.z, x.w - v.w));
}

// Whether the next `n` bits (1 to 7) are all ones: the padding of an interval's last byte.
__device__ __forceinline__ bool padding(BitReader& br, int n) {
  br.fill();
  return br.peek(n) == (1u << n) - 1;
}

// Decode subsequence `s` from its start state up to its exit: the first symbol boundary at or past bit `end` (the
// interval's last subsequence: the first MCU boundary in the last byte followed only by one-bits of padding).  The decode is
// jpeg_entropy_kernel's, symbol for symbol.  Without WRITE it records the exit, the blocks completed and the DC
// differences summed per component, and JPEG_SUB_BAD when it reads a code longer than 16 bits (decoded as the
// sequential kernel does, so that a decode from a guessed start still synchronises) or consumes a bit past the data
// (where it stops): the paths libjpeg-turbo warns on, which only the sequential kernel reproduces.  With WRITE it starts
// from the scanned block count and DC predictions and stores the coefficients of blocks [lo_blk, hi_blk) of the
// interval at coef[(out0 + block) * 64].
template <bool WRITE>
__device__ void jpeg_decode_sub(const uint8_t* buf, const int* d, const uint8_t* data, int bytes, JpegSub* s,
                                int end, bool last, int bpm, int ncomp, int16_t* coef, int64_t out0, int lo_blk,
                                int hi_blk) {
  int pos = s->s_pos, bk = s->s_bk;
  int b = bk >> 8, k = bk & 255;
  int raw = s->raw;
  for (int u = s->ubyte; u < (pos >> 3) && raw < bytes; ++u) raw += data[raw] == 0xFF ? 2 : 1;
  BitReader br{data, raw, bytes, 0ull, 0, 0, false};
  br.fill();
  br.drop(pos & 7);
  const int base = pos & ~7;
  int blk = WRITE ? s->blocks : 0;
  unsigned dc0 = WRITE ? s->dc[0] : 0u, dc1 = WRITE ? s->dc[1] : 0u, dc2 = WRITE ? s->dc[2] : 0u;
  bool bad = false;
  for (;;) {
    pos = base + br.bit;
    if (last ? b == 0 && k == 0 && pos > end - 8 && (pos >= end || padding(br, end - pos)) : pos >= end) break;
    const int c = b < bpm - 2 || ncomp == 1 ? 0 : b - (bpm - 3);
    int16_t* out = WRITE && blk >= lo_blk && blk < hi_blk ? coef + (out0 + blk) * 64 : nullptr;
    if (k == 0) {
      int sz = br.huff(buf + int64_t(d[JD_HUFF + 2 * c]) * 16) & 15;
      const unsigned v = sz ? unsigned(huff_extend(br.get(sz), sz)) : 0u;
      dc0 += c == 0 ? v : 0u;
      dc1 += c == 1 ? v : 0u;
      dc2 += c == 2 ? v : 0u;
      if (WRITE && out) out[0] = int16_t(c == 0 ? dc0 : c == 1 ? dc1 : dc2);
      k = 1;
    } else {
      const int rs = br.huff(buf + int64_t(d[JD_HUFF + 2 * c + 1]) * 16);
      const int r = rs >> 4, sz = rs & 15;
      if (sz) {
        k += r;
        const int v = huff_extend(br.get(sz), sz);
        if (WRITE && out) out[kNatural[k]] = int16_t(v);
        ++k;
      } else {
        k = r != 15 ? 64 : k + 16;
      }
    }
    if (br.beyond) {   // only the last subsequence reaches the end of the data
      bad = true;
      break;
    }
    if (k >= 64) {
      k = 0;
      ++blk;
      b = b + 1 == bpm ? 0 : b + 1;
    }
  }
  if (WRITE) return;
  bad |= br.long_code;
  s->x_pos = pos;
  s->x_bk = b << 8 | k;
  s->blocks = blk;
  s->dc[0] = dc0;
  s->dc[1] = dc1;
  s->dc[2] = dc2;
  s->flags = bad ? JPEG_SUB_BAD : 0;
}

// One CTA per restart interval the parallel decode takes:
//   1. subsequence j starts at byte j * JPEG_SUB_BYTES, one later when that is the zero of a stuffed FF 00 pair;
//      its FF bytes are counted and scanned, which gives each start's index in the unstuffed stream;
//   2. every subsequence decodes from its start state (the first: the interval's start; the others: a guess, block 0
//      of an MCU at their first bit) to its exit; where an exit differs from the next subsequence's start, that start
//      becomes the exit and the next subsequence decodes again; rounds repeat until no start changes.  After round r
//      the starts of subsequences 0..r are the true ones whatever the data, so this ends after at most one round per
//      subsequence; the Huffman code's self-synchronisation usually ends it after two;
//   3. the interval is left to the sequential kernel (`fallback`) if any final decode met a corrupt-data path or the
//      blocks do not add up to the interval's MCUs; otherwise the block counts and per-component DC sums are scanned
//      and every subsequence that touches a block the rectangle needs decodes again from its start, writing them.
__global__ void __launch_bounds__(JPEG_PAR_THREADS, 4)
    jpeg_parallel_kernel(const uint8_t* __restrict__ buf, const int* __restrict__ jd, JpegSub* subs, int16_t* coef) {
  pdl_prologue();
  __shared__ uint4 warp_sums[JPEG_PAR_THREADS / 32];
  const int* d = jd + int64_t(blockIdx.y) * JD;
  const int k = blockIdx.x;
  if (k >= d[JD_NINT]) return;
  const JpegGeom g = jpeg_geometry(d);
  const int total = g.mpr * g.rows;
  const int ri = d[JD_RESTART] ? d[JD_RESTART] : total;
  const int first = k * ri, last = min(first + ri, total);
  const int lo = g.mcu0 * g.mpr, hi = min(g.mcu1 * g.mpr, last);
  if (first >= hi || last <= lo) return;   // as jpeg_entropy_kernel: the rectangle needs nothing of this interval
  const int* iv = reinterpret_cast<const int*>(buf + int64_t(d[JD_INT]) * 16) + 2 * k;
  const int bytes = iv[1] - iv[0];
  if (!jpeg_parallel_interval(bytes)) return;
  const uint8_t* data = buf + int64_t(d[JD_DATA]) * 16 + iv[0];
  JpegSub* S = subs + d[JD_SUB] + iv[0] / JPEG_SLOT_BYTES + k;
  const int n = (bytes + JPEG_SUB_BYTES - 1) / JPEG_SUB_BYTES, bpm = g.bpm, ncomp = g.ncomp;
  const int T = JPEG_PAR_THREADS, tid = threadIdx.x;
  auto start_of = [&](int j) {
    int r = min(j * JPEG_SUB_BYTES, bytes);
    return r > 0 && r < bytes && data[r - 1] == 0xFF ? r + 1 : r;
  };
  // 1. starts, and their indices in the unstuffed stream
  uint4 carry = make_uint4(0, 0, 0, 0);
  for (int j0 = 0; j0 < n; j0 += T) {
    const int j = j0 + tid;
    int r = 0, ff = 0;
    if (j < n) {
      r = start_of(j);
      const int e = start_of(j + 1);
      for (int i = r; i < e; ++i) ff += data[i] == 0xFF;
    }
    const uint4 pre = cta_scan(make_uint4(unsigned(ff), 0, 0, 0), carry, warp_sums);
    if (j < n) {
      S[j].raw = r;
      S[j].ubyte = r - int(pre.x);
      S[j].s_pos = 8 * (r - int(pre.x));
      S[j].s_bk = 0;
      S[j].flags = JPEG_SUB_DIRTY;
    }
  }
  const int end_bits = 8 * (bytes - int(carry.x));
  __syncthreads();
  // 2. synchronisation rounds
  for (;;) {
    for (int j = tid; j < n; j += T)
      if (S[j].flags & JPEG_SUB_DIRTY)
        jpeg_decode_sub<false>(buf, d, data, bytes, S + j, j + 1 < n ? S[j + 1].ubyte * 8 : end_bits, j + 1 == n,
                               bpm, ncomp, coef, 0, 0, 0);
    __syncthreads();
    bool changed = false;
    for (int j = tid; j + 1 < n; j += T)
      if (S[j].x_pos != S[j + 1].s_pos || S[j].x_bk != S[j + 1].s_bk) {
        S[j + 1].s_pos = S[j].x_pos;
        S[j + 1].s_bk = S[j].x_bk;
        S[j + 1].flags |= JPEG_SUB_DIRTY;
        changed = true;
      }
    if (!__syncthreads_or(changed)) break;
  }
  // 3. block counts and DC predictions, or the fallback
  carry = make_uint4(0, 0, 0, 0);
  int bad = 0;
  for (int j0 = 0; j0 < n; j0 += T) {
    const int j = j0 + tid;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (j < n) {
      v = make_uint4(unsigned(S[j].blocks), S[j].dc[0], S[j].dc[1], S[j].dc[2]);
      bad |= S[j].flags & JPEG_SUB_BAD;
    }
    const uint4 pre = cta_scan(v, carry, warp_sums);
    if (j < n) {
      S[j].blocks = int(pre.x);
      S[j].dc[0] = pre.y;
      S[j].dc[1] = pre.z;
      S[j].dc[2] = pre.w;
    }
  }
  const bool fallback = __syncthreads_or(bad) || int(carry.x) != (last - first) * bpm;
  if (tid == 0) S[0].fallback = fallback;
  if (fallback) return;
  const int lo_blk = (lo - first) * bpm, hi_blk = (hi - first) * bpm;
  const int64_t out0 = int64_t(d[JD_COEF]) + int64_t(first - lo) * bpm;
  for (int j = tid; j < n; j += T) {
    const int next = j + 1 < n ? S[j + 1].blocks : int(carry.x);   // the block the exit lies in (or ends)
    if (S[j].blocks < hi_blk && next >= lo_blk)
      jpeg_decode_sub<true>(buf, d, data, bytes, S + j, j + 1 < n ? S[j + 1].ubyte * 8 : end_bits, j + 1 == n, bpm,
                            ncomp, coef, out0, lo_blk, hi_blk);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// 2. Dequantise + islow IDCT (x86-64 SIMD arithmetic)
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int wrap16(int x) { return int(int16_t(x)); }
__device__ __forceinline__ int sat16(int x) { return min(max(x, -32768), 32767); }

// One pass over 8 values: jidctint.c's products regrouped as the SIMD code pairs them; outputs descaled by `shift`
// and saturated to 16 bits.  Every 32-bit sum stays below 2^31 in magnitude for 16-bit inputs.
__device__ __forceinline__ void idct_pass(const int x[8], int shift, int y[8]) {
  const int tmp3 = x[2] * 10703 + x[6] * 4433;
  const int tmp2 = x[2] * 4433 + x[6] * -10704;
  const int tmp0 = wrap16(x[0] + x[4]) * 8192;
  const int tmp1 = wrap16(x[0] - x[4]) * 8192;
  const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  const int z3 = wrap16(x[7] + x[3]), z4 = wrap16(x[5] + x[1]);
  const int z3p = z3 * -6436 + z4 * 9633, z4p = z3 * 9633 + z4 * 6437;
  const int t0 = x[7] * -4927 + x[1] * -7373 + z3p;
  const int t3 = x[7] * -7373 + x[1] * 4926 + z4p;
  const int t1 = x[5] * -4176 + x[3] * -20995 + z4p;
  const int t2 = x[5] * -20995 + x[3] * 4177 + z3p;
  const int r = 1 << (shift - 1);
  y[0] = sat16((tmp10 + t3 + r) >> shift);
  y[7] = sat16((tmp10 - t3 + r) >> shift);
  y[1] = sat16((tmp11 + t2 + r) >> shift);
  y[6] = sat16((tmp11 - t2 + r) >> shift);
  y[2] = sat16((tmp12 + t1 + r) >> shift);
  y[5] = sat16((tmp12 - t1 + r) >> shift);
  y[3] = sat16((tmp13 + t0 + r) >> shift);
  y[4] = sat16((tmp13 - t0 + r) >> shift);
}

__global__ void __launch_bounds__(JPEG_IDCT_THREADS) jpeg_idct_kernel(const uint8_t* __restrict__ buf,
                                                                      const int* __restrict__ jd, const int16_t* coef,
                                                                      uint8_t* planes) {
  pdl_prologue();   // coef is the previous kernel's output: plain loads
  const int* d = jd + int64_t(blockIdx.y) * JD;
  const JpegGeom g = jpeg_geometry(d);
  uint8_t* base = planes + int64_t(d[JD_PLANE]) * 16;
  for (int64_t t = int64_t(blockIdx.x) * JPEG_IDCT_THREADS + threadIdx.x; t < g.blocks;
       t += int64_t(gridDim.x) * JPEG_IDCT_THREADS) {
    int c = 0;
    int64_t i = t;
    while (i >= int64_t(g.win[c][1] - g.win[c][0]) * (g.win[c][3] - g.win[c][2])) {
      i -= int64_t(g.win[c][1] - g.win[c][0]) * (g.win[c][3] - g.win[c][2]);
      ++c;
    }
    const int* w = g.win[c];
    const int bw = w[3] - w[2];
    const int br = w[0] + int(i / bw), bc = w[2] + int(i % bw);
    const int hs = c ? 1 : d[JD_HMAX], vs = c ? 1 : d[JD_VMAX];
    const int within = g.ncomp == 1 ? 0 : c ? d[JD_HMAX] * d[JD_VMAX] + c - 1 : (br % vs) * hs + bc % hs;
    const int64_t blk = int64_t(d[JD_COEF]) + (int64_t(br / vs - g.mcu0) * g.mpr + bc / hs) * g.bpm + within;
    const int16_t* cf = coef + blk * 64;
    const int* q = reinterpret_cast<const int*>(buf + int64_t(d[JD_QUANT]) * 16) + c * 64;
    int x[64];
    bool ac = false;
#pragma unroll
    for (int e = 0; e < 64; ++e) {
      x[e] = wrap16(int(cf[e]) * int(int16_t(q[e])));
      if (e >= 8) ac |= cf[e] != 0;
    }
    int ws[64];
#pragma unroll
    for (int col = 0; col < 8; ++col) {       // pass 1: columns; rows 1..7 all zero take the 16-bit DC shortcut
      int in[8], out[8];
#pragma unroll
      for (int r = 0; r < 8; ++r) in[r] = x[r * 8 + col];
      idct_pass(in, 11, out);
#pragma unroll
      for (int r = 0; r < 8; ++r) ws[r * 8 + col] = ac ? out[r] : wrap16(x[col] * 4);
    }
    uint8_t* dst = base + g.plane[c] + int64_t(br - w[0]) * 8 * (bw * 8) + (bc - w[2]) * 8;
#pragma unroll
    for (int r = 0; r < 8; ++r) {             // pass 2: rows
      int out[8];
      idct_pass(ws + r * 8, 18, out);
      uint32_t lo = 0, hi = 0;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        lo |= uint32_t(min(max(out[e], -128), 127) + 128) << (8 * e);
        hi |= uint32_t(min(max(out[e + 4], -128), 127) + 128) << (8 * e);
      }
      *reinterpret_cast<uint2*>(dst + int64_t(r) * bw * 8) = make_uint2(lo, hi);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// 3. Upsampling + colour conversion
// ---------------------------------------------------------------------------------------------------------------------
struct Plane {
  const uint8_t* p;
  int r0, c0, pitch;   // first sample row / column held, row pitch
  __device__ __forceinline__ int at(int r, int c) const { return p[int64_t(r - r0) * pitch + (c - c0)]; }
};

// Chroma sample of output pixel (y, x): jdsample.c's h2v1 / h2v2 fancy upsampling (plain replication when the
// component is at most 2 samples wide), or the sample itself without subsampling.
__device__ __forceinline__ int chroma(const Plane& p, int y, int x, int hm, int vm, int cw, int ch) {
  if (hm == 1) return p.at(y, x);
  const int cx = x >> 1;
  if (cw <= 2) return p.at(vm == 2 ? y >> 1 : y, cx);
  if (vm == 1) {
    const int v = 3 * p.at(y, cx);
    if (!(x & 1)) return cx == 0 ? p.at(y, 0) : (v + p.at(y, cx - 1) + 1) >> 2;
    return cx == cw - 1 ? p.at(y, cx) : (v + p.at(y, cx + 1) + 2) >> 2;
  }
  const int cy = y >> 1;
  const int ny = (y & 1) ? min(cy + 1, ch - 1) : max(cy - 1, 0);
  const int here = 3 * p.at(cy, cx) + p.at(ny, cx);
  if (!(x & 1)) return cx == 0 ? (here * 4 + 8) >> 4 : (here * 3 + 3 * p.at(cy, cx - 1) + p.at(ny, cx - 1) + 8) >> 4;
  return cx == cw - 1 ? (here * 4 + 7) >> 4 : (here * 3 + 3 * p.at(cy, cx + 1) + p.at(ny, cx + 1) + 7) >> 4;
}

__device__ __forceinline__ uint8_t clamp255(int v) { return uint8_t(min(max(v, 0), 255)); }

__global__ void __launch_bounds__(JPEG_COLOR_THREADS) jpeg_color_kernel(const int* __restrict__ jd,
                                                                        const uint8_t* planes, uint8_t* buf) {
  pdl_prologue();   // planes are the previous kernel's output
  const int* d = jd + int64_t(blockIdx.y) * JD;
  const JpegGeom g = jpeg_geometry(d);
  const int hm = d[JD_HMAX], vm = d[JD_VMAX], W = d[JD_W], H = d[JD_H];
  const int cw = (W + hm - 1) / hm, ch = (H + vm - 1) / vm;
  Plane p[3];
  for (int c = 0; c < g.ncomp; ++c)
    p[c] = Plane{planes + int64_t(d[JD_PLANE]) * 16 + g.plane[c], g.win[c][0] * 8, g.win[c][2] * 8,
                 (g.win[c][3] - g.win[c][2]) * 8};
  uint8_t* out = buf + int64_t(d[JD_OUT]) * 16;
  const int rw = d[JD_RW];
  const int64_t n = int64_t(d[JD_RH]) * rw;
  for (int64_t t = int64_t(blockIdx.x) * JPEG_COLOR_THREADS + threadIdx.x; t < n;
       t += int64_t(gridDim.x) * JPEG_COLOR_THREADS) {
    const int y = d[JD_Y0] + int(t / rw), x = d[JD_X0] + int(t % rw);
    const int Y = p[0].at(y, x);
    uint8_t* o = out + t * 3;
    if (g.ncomp == 1) {
      o[0] = o[1] = o[2] = uint8_t(Y);
      continue;
    }
    const int cb = chroma(p[1], y, x, hm, vm, cw, ch) - 128, cr = chroma(p[2], y, x, hm, vm, cw, ch) - 128;
    o[0] = clamp255(Y + ((91881 * cr + 32768) >> 16));
    o[1] = clamp255(Y + ((-22554 * cb + 32768 + -46802 * cr) >> 16));
    o[2] = clamp255(Y + ((116130 * cb + 32768) >> 16));
  }
}

}  // namespace
}  // namespace mmae

using namespace mmae;

extern "C" int mmae_jpeg_decode_batch(const void* packed_host, void* packed, int64_t host_bytes, int64_t packed_bytes,
                                      int num_images, int64_t desc_offset, void* scratch, int64_t scratch_bytes,
                                      void* stream) {
  MMAE_CHECK(packed_host && packed && scratch, MMAE_ERR_ARG, "mmae_jpeg_decode_batch: null pointer");
  MMAE_CHECK(num_images >= 1 && num_images <= 65535, MMAE_ERR_ARG, "mmae_jpeg_decode_batch: bad image count %d",
             num_images);
  MMAE_CHECK(((reinterpret_cast<uintptr_t>(packed) | reinterpret_cast<uintptr_t>(scratch)) & 15) == 0, MMAE_ERR_ARG,
             "mmae_jpeg_decode_batch: buffers must be 16-byte aligned");
  MMAE_CHECK(host_bytes >= 0 && host_bytes <= packed_bytes, MMAE_ERR_ARG,
             "mmae_jpeg_decode_batch: host part of %lld bytes, buffer of %lld", (long long)host_bytes,
             (long long)packed_bytes);
  MMAE_CHECK(desc_offset >= 0 && desc_offset * 16 + int64_t(num_images) * JD * 4 <= host_bytes, MMAE_ERR_ARG,
             "mmae_jpeg_decode_batch: descriptors outside the host part");
  const uint8_t* host = static_cast<const uint8_t*>(packed_host);
  const int* jd_host = reinterpret_cast<const int*>(host + desc_offset * 16);
  auto inside = [&](int64_t off16, int64_t bytes) { return off16 >= 0 && off16 * 16 + bytes <= host_bytes; };
  int64_t coef_blocks = 0, plane_bytes = 0, sub_slots = 0, out_end = host_bytes;
  int max_nint = 1;
  int64_t max_blocks = 1, max_px = 1;
  for (int i = 0; i < num_images; ++i) {
    const int* d = jd_host + int64_t(i) * JD;
    const int W = d[JD_W], H = d[JD_H], nc = d[JD_NCOMP], hm = d[JD_HMAX], vm = d[JD_VMAX];
    MMAE_CHECK(W >= 1 && H >= 1 && W <= JPEG_MAX_SIDE && H <= JPEG_MAX_SIDE, MMAE_ERR_ARG,
               "mmae_jpeg_decode_batch: image %d: size %d x %d", i, W, H);
    const bool sampling = nc == 1 ? (hm == 1 && vm == 1)
                                  : nc == 3 && ((hm == 1 && vm == 1) || (hm == 2 && vm == 1) || (hm == 2 && vm == 2));
    MMAE_CHECK(sampling, MMAE_ERR_ARG, "mmae_jpeg_decode_batch: image %d: %d components sampled %dx%d", i, nc, hm, vm);
    MMAE_CHECK(d[JD_Y0] >= 0 && d[JD_X0] >= 0 && d[JD_RH] >= 1 && d[JD_RW] >= 1 && d[JD_Y0] <= H - d[JD_RH] &&
                   d[JD_X0] <= W - d[JD_RW],
               MMAE_ERR_ARG, "mmae_jpeg_decode_batch: image %d: rectangle (%d, %d) + %d x %d outside %d x %d", i,
               d[JD_Y0], d[JD_X0], d[JD_RH], d[JD_RW], H, W);
    const JpegGeom g = jpeg_geometry(d);
    const int64_t total = int64_t(g.mpr) * g.rows;
    MMAE_CHECK(d[JD_RESTART] >= 0 && d[JD_RESTART] <= 65535, MMAE_ERR_ARG,
               "mmae_jpeg_decode_batch: image %d: restart interval %d", i, d[JD_RESTART]);
    const int64_t nint = d[JD_RESTART] ? (total + d[JD_RESTART] - 1) / d[JD_RESTART] : 1;
    MMAE_CHECK(d[JD_NINT] == nint, MMAE_ERR_ARG, "mmae_jpeg_decode_batch: image %d: %d intervals, %lld expected", i,
               d[JD_NINT], (long long)nint);
    MMAE_CHECK(d[JD_DATA_BYTES] >= 0 && inside(d[JD_DATA], d[JD_DATA_BYTES]) && inside(d[JD_INT], nint * 8),
               MMAE_ERR_ARG, "mmae_jpeg_decode_batch: image %d: entropy-coded data outside the buffer", i);
    const int* iv = reinterpret_cast<const int*>(host + int64_t(d[JD_INT]) * 16);
    for (int64_t k = 0; k < nint; ++k)
      MMAE_CHECK(iv[2 * k] >= 0 && iv[2 * k] <= iv[2 * k + 1] && iv[2 * k + 1] <= d[JD_DATA_BYTES], MMAE_ERR_ARG,
                 "mmae_jpeg_decode_batch: image %d: interval %lld is [%d, %d) of %d bytes", i, (long long)k, iv[2 * k],
                 iv[2 * k + 1], d[JD_DATA_BYTES]);
    MMAE_CHECK(inside(d[JD_QUANT], int64_t(nc) * 64 * 4), MMAE_ERR_ARG,
               "mmae_jpeg_decode_batch: image %d: quantisation tables outside the buffer", i);
    const int* q = reinterpret_cast<const int*>(host + int64_t(d[JD_QUANT]) * 16);
    for (int e = 0; e < nc * 64; ++e)
      MMAE_CHECK(q[e] >= 0 && q[e] <= 65535, MMAE_ERR_ARG, "mmae_jpeg_decode_batch: image %d: quantiser %d", i, q[e]);
    for (int t = 0; t < 2 * nc; ++t) {
      MMAE_CHECK(inside(d[JD_HUFF + t], JPEG_TABLE_BYTES), MMAE_ERR_ARG,
                 "mmae_jpeg_decode_batch: image %d: Huffman table %d outside the buffer", i, t);
      const uint8_t* sym = host + int64_t(d[JD_HUFF + t]) * 16 + JPEG_TABLE_BYTES - 256;
      for (int s = 0; s < 256 && t % 2 == 0; ++s)
        MMAE_CHECK(sym[s] <= 15, MMAE_ERR_ARG, "mmae_jpeg_decode_batch: image %d: DC symbol %d", i, sym[s]);
    }
    const int64_t out_bytes = int64_t(d[JD_RH]) * d[JD_RW] * 3;
    MMAE_CHECK(d[JD_OUT] >= 0 && int64_t(d[JD_OUT]) * 16 >= out_end && int64_t(d[JD_OUT]) * 16 + out_bytes <= packed_bytes,
               MMAE_ERR_ARG, "mmae_jpeg_decode_batch: image %d: output overlaps the host part or the previous output, "
               "or leaves the buffer", i);
    out_end = int64_t(d[JD_OUT]) * 16 + out_bytes;
    MMAE_CHECK(d[JD_COEF] == coef_blocks && int64_t(d[JD_PLANE]) * 16 == plane_bytes, MMAE_ERR_ARG,
               "mmae_jpeg_decode_batch: image %d: scratch offsets %d / %d, expected %lld / %lld", i, d[JD_COEF],
               d[JD_PLANE], (long long)coef_blocks, (long long)(plane_bytes / 16));
    MMAE_CHECK(d[JD_SUB] == sub_slots, MMAE_ERR_ARG,
               "mmae_jpeg_decode_batch: image %d: subsequence offset %d, expected %lld", i, d[JD_SUB],
               (long long)sub_slots);
    coef_blocks += jpeg_coef_blocks(g);
    plane_bytes += g.plane_bytes;
    sub_slots += d[JD_DATA_BYTES] / JPEG_SLOT_BYTES + nint;
    MMAE_CHECK(coef_blocks < INT_MAX && plane_bytes / 16 < INT_MAX && sub_slots < INT_MAX, MMAE_ERR_ARG,
               "mmae_jpeg_decode_batch: scratch offsets overflow");
    max_nint = std::max<int>(max_nint, int(nint));
    max_blocks = std::max<int64_t>(max_blocks, g.blocks);
    max_px = std::max<int64_t>(max_px, int64_t(d[JD_RH]) * d[JD_RW]);
  }
  const int64_t coef_bytes = coef_blocks * 128;
  const int64_t planes_off = int64_t(align_up(size_t(coef_bytes), 256));
  const int64_t subs_off = planes_off + int64_t(align_up(size_t(plane_bytes), 256));
  const int64_t need = subs_off + sub_slots * int64_t(sizeof(JpegSub));
  MMAE_CHECK(need <= scratch_bytes, MMAE_ERR_ARG, "mmae_jpeg_decode_batch: scratch of %lld bytes, %lld needed",
             (long long)scratch_bytes, (long long)need);

  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* buf = static_cast<uint8_t*>(packed);
  const int* jd = reinterpret_cast<const int*>(buf + desc_offset * 16);
  int16_t* coef = static_cast<int16_t*>(scratch);
  uint8_t* planes = static_cast<uint8_t*>(scratch) + planes_off;
  JpegSub* subs = reinterpret_cast<JpegSub*>(static_cast<uint8_t*>(scratch) + subs_off);
  MMAE_CUDA_OK(cudaMemsetAsync(coef, 0, size_t(coef_bytes), st));
  const unsigned n = unsigned(num_images);
  launch_k(jpeg_parallel_kernel, dim3(unsigned(max_nint), n), JPEG_PAR_THREADS, 0, st,
           static_cast<const uint8_t*>(buf), jd, subs, coef);
  count_launch();
  MMAE_LAUNCH_OK();
  launch_k(jpeg_entropy_kernel, dim3(unsigned((max_nint + JPEG_ENTROPY_THREADS - 1) / JPEG_ENTROPY_THREADS), n),
           JPEG_ENTROPY_THREADS, 0, st, static_cast<const uint8_t*>(buf), jd, static_cast<const JpegSub*>(subs), coef);
  count_launch();
  MMAE_LAUNCH_OK();
  const int64_t cap = 1024;
  launch_k(jpeg_idct_kernel, dim3(unsigned(std::min<int64_t>((max_blocks + JPEG_IDCT_THREADS - 1) / JPEG_IDCT_THREADS,
                                                             cap)), n),
           JPEG_IDCT_THREADS, 0, st, static_cast<const uint8_t*>(buf), jd, static_cast<const int16_t*>(coef), planes);
  count_launch();
  MMAE_LAUNCH_OK();
  launch_k(jpeg_color_kernel, dim3(unsigned(std::min<int64_t>((max_px + JPEG_COLOR_THREADS - 1) / JPEG_COLOR_THREADS,
                                                              cap)), n),
           JPEG_COLOR_THREADS, 0, st, jd, static_cast<const uint8_t*>(planes), buf);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

