// Pre-training augmentation on the GPU (MMAE_GPU_AUGMENT): the resampling half of DataAugmentationForMultiMAE
// (utils/datasets.py:66-111), bitwise equal to Pillow's Image.resize followed by TF.hflip, TF.to_tensor / TF.normalize.
//
// The workers hand over one packed buffer per batch (multimae_b200/data.py: pack_batch): int32 descriptors, resampling
// tables computed on the host (Pillow's precompute_coeffs / normalize_coeffs_8bpc and its nearest map, in double), and the
// uint8 / uint16 crops.  Bicubic resampling is separable as in Pillow: a horizontal pass into a scratch image of the pixel
// type (rounded and clipped as Pillow rounds and clips), then a vertical pass that writes the final fp32 tensors with the
// flip and the normalisation fused.  semseg is one gather through Pillow's two NEAREST maps (crop -> S -> S/4).
//
// The arithmetic must round exactly as the CPU code it restates: every float / double operation below is an explicit
// round-to-nearest intrinsic, so nothing is contracted into an FMA whatever the compiler flags.
#include <unordered_set>

#include "common.cuh"
#include "internal.h"

namespace mmae {
namespace {

constexpr int AUG_THREADS = 256;
constexpr int AUG_DESC = 8;               // kind, src / 16, h, w, flip, column table / 16, row table / 16, scratch / 16
constexpr int AUG_PRECISION_BITS = 22;    // Pillow's fixed-point weights of 8-bit resampling
constexpr int AUG_TABLE_BICUBIC = 1, AUG_TABLE_NEAREST = 2;
constexpr int AUG_MAX_EXTENT = 1 << 15;
constexpr int AUG_MAX_SIZE = 4096;

struct AugOutputs {
  void* p[MMAE_MAX_TASKS];
};
struct AugNorm {
  float mean[3];
  float std[3];
};

// Byte offsets of a bicubic table's sections (header int32[4], bounds int32[2n], fixed-point int32[n*k], double[n*k]).
__host__ __device__ inline int64_t aug_fixed_off(int n) { return 16 + 8 * int64_t(n); }
__host__ __device__ inline int64_t aug_double_off(int n, int k) {
  return (aug_fixed_off(n) + 4 * int64_t(n) * k + 7) / 8 * 8;
}
__host__ __device__ inline int64_t aug_bicubic_bytes(int n, int k) { return aug_double_off(n, k) + 8 * int64_t(n) * k; }

// Pillow's clip8 of a fixed-point sum (half-ulp bias included by the caller).
__device__ __forceinline__ int aug_clip8(int ss) { return min(max(ss >> AUG_PRECISION_BITS, 0), 255); }

// Pillow's 16-bit store of a double sum: round half away from zero, then the low and high bytes clipped separately.
__device__ __forceinline__ int aug_store16(double ss) {
  const int si = int(ss >= 0.0 ? __dadd_rn(ss, 0.5) : __dsub_rn(ss, 0.5));
  const int lo = min(max(si % 256, 0), 255);
  const int hi = min(max(si >> 8, 0), 255);
  return lo | (hi << 8);
}

// Horizontal pass: row y of the crop (h x w) -> row y of the scratch image (h x S), for every rgb / depth item.
__global__ void __launch_bounds__(AUG_THREADS) augment_horizontal_kernel(const uint8_t* __restrict__ buf,
                                                                         const int* __restrict__ desc,
                                                                         uint8_t* __restrict__ scratch, int S) {
  pdl_prologue();
  const int* d = desc + int64_t(blockIdx.y) * AUG_DESC;
  const int kind = d[0];
  if (kind == 2) return;
  const int h = d[2], w = d[3];
  const uint8_t* src = buf + int64_t(d[1]) * 16;
  const uint8_t* tab = buf + int64_t(d[5]) * 16;
  const int ksize = reinterpret_cast<const int*>(tab)[2];
  const int* bounds = reinterpret_cast<const int*>(tab) + 4;
  const int64_t n = int64_t(h) * S;
  for (int64_t idx = int64_t(blockIdx.x) * AUG_THREADS + threadIdx.x; idx < n; idx += int64_t(gridDim.x) * AUG_THREADS) {
    const int y = int(idx / S), xx = int(idx - int64_t(y) * S);
    const int xmin = bounds[2 * xx], xmax = bounds[2 * xx + 1];
    if (kind == 0) {
      const int* k = reinterpret_cast<const int*>(tab + aug_fixed_off(S)) + int64_t(xx) * ksize;
      const uint8_t* row = src + (int64_t(y) * w + xmin) * 3;
      int s0 = 1 << (AUG_PRECISION_BITS - 1), s1 = s0, s2 = s0;
      for (int x = 0; x < xmax; ++x) {
        const int kx = k[x];
        s0 += int(row[3 * x]) * kx;
        s1 += int(row[3 * x + 1]) * kx;
        s2 += int(row[3 * x + 2]) * kx;
      }
      uint8_t* o = scratch + int64_t(d[7]) * 16 + idx * 3;
      o[0] = uint8_t(aug_clip8(s0));
      o[1] = uint8_t(aug_clip8(s1));
      o[2] = uint8_t(aug_clip8(s2));
    } else {
      const double* k = reinterpret_cast<const double*>(tab + aug_double_off(S, ksize)) + int64_t(xx) * ksize;
      const uint16_t* row = reinterpret_cast<const uint16_t*>(src) + int64_t(y) * w + xmin;
      double ss = 0.0;
      for (int x = 0; x < xmax; ++x) ss = __dadd_rn(ss, __dmul_rn(double(row[x]), k[x]));
      reinterpret_cast<uint16_t*>(scratch + int64_t(d[7]) * 16)[idx] = uint16_t(aug_store16(ss));
    }
  }
}

// Vertical pass: column x of the scratch image (h x S) -> the S x S output, flipped and normalised; semseg items gather
// their S/4 x S/4 labels through the nearest maps.
__global__ void __launch_bounds__(AUG_THREADS) augment_vertical_kernel(const uint8_t* __restrict__ buf,
                                                                       const int* __restrict__ desc,
                                                                       const uint8_t* scratch, int S,
                                                                       int num_tasks, const int* __restrict__ map4,
                                                                       AugOutputs out, AugNorm norm) {
  pdl_prologue();   // scratch is the previous kernel's output: read with plain (coherent) loads, no __restrict__
  const int item = blockIdx.y;
  const int* d = desc + int64_t(item) * AUG_DESC;
  const int b = item / num_tasks, t = item - b * num_tasks;
  void* dst_base = nullptr;
#pragma unroll
  for (int i = 0; i < MMAE_MAX_TASKS; ++i)   // a constant index keeps the parameter struct out of local memory
    if (i == t) dst_base = out.p[i];
  const int kind = d[0], flip = d[4];
  const uint8_t* tab = buf + int64_t(d[6]) * 16;
  const int stride = gridDim.x * AUG_THREADS;
  if (kind == 2) {
    const int S4 = S / 4;
    const int* mw = reinterpret_cast<const int*>(buf + int64_t(d[5]) * 16) + 4;
    const int* mh = reinterpret_cast<const int*>(tab) + 4;
    const uint8_t* src = buf + int64_t(d[1]) * 16;
    const int w = d[3];
    int64_t* o = static_cast<int64_t*>(dst_base) + int64_t(b) * S4 * S4;
    for (int idx = blockIdx.x * AUG_THREADS + threadIdx.x; idx < S4 * S4; idx += stride) {
      const int y4 = idx / S4, x4 = idx - y4 * S4;
      const int xs = map4[x4];
      o[idx] = int64_t(src[int64_t(mh[map4[y4]]) * w + mw[flip ? S - 1 - xs : xs]]);
    }
    return;
  }
  const int ksize = reinterpret_cast<const int*>(tab)[2];
  const int* bounds = reinterpret_cast<const int*>(tab) + 4;
  const int64_t plane = int64_t(S) * S;
  for (int idx = blockIdx.x * AUG_THREADS + threadIdx.x; idx < S * S; idx += stride) {
    const int yy = idx / S, x = idx - yy * S;
    const int ymin = bounds[2 * yy], ymax = bounds[2 * yy + 1];
    const int64_t dst = int64_t(yy) * S + (flip ? S - 1 - x : x);
    if (kind == 0) {
      const int* k = reinterpret_cast<const int*>(tab + aug_fixed_off(S)) + int64_t(yy) * ksize;
      const uint8_t* col = scratch + int64_t(d[7]) * 16 + (int64_t(ymin) * S + x) * 3;
      int s0 = 1 << (AUG_PRECISION_BITS - 1), s1 = s0, s2 = s0;
      for (int y = 0; y < ymax; ++y) {
        const int ky = k[y];
        const uint8_t* p = col + int64_t(y) * S * 3;
        s0 += int(p[0]) * ky;
        s1 += int(p[1]) * ky;
        s2 += int(p[2]) * ky;
      }
      float* o = static_cast<float*>(dst_base) + int64_t(b) * 3 * plane + dst;
      const int v[3] = {aug_clip8(s0), aug_clip8(s1), aug_clip8(s2)};
#pragma unroll
      for (int c = 0; c < 3; ++c)   // TF.to_tensor (x / 255), then TF.normalize ((x - mean) / std), each rounded in fp32
        o[c * plane] = __fdiv_rn(__fsub_rn(__fdiv_rn(float(v[c]), 255.0f), norm.mean[c]), norm.std[c]);
    } else {
      const double* k = reinterpret_cast<const double*>(tab + aug_double_off(S, ksize)) + int64_t(yy) * ksize;
      const uint16_t* col = reinterpret_cast<const uint16_t*>(scratch + int64_t(d[7]) * 16) + int64_t(ymin) * S + x;
      double ss = 0.0;
      for (int y = 0; y < ymax; ++y) ss = __dadd_rn(ss, __dmul_rn(double(col[int64_t(y) * S]), k[y]));
      // np.array(img) / 2**16: exact in fp32
      static_cast<float*>(dst_base)[int64_t(b) * plane + dst] = __fmul_rn(float(aug_store16(ss)), 1.0f / 65536.0f);
    }
  }
}

// Host-side check of one table in the host copy of the packed buffer.
int check_table(const uint8_t* host, int64_t bytes, int64_t off16, int kind, int n_in, int n_out, int item,
                std::unordered_set<int64_t>& seen) {
  const int64_t off = off16 * 16;
  MMAE_CHECK(off16 >= 0 && off + 16 <= bytes, MMAE_ERR_ARG, "mmae_augment_batch: item %d: table offset out of range", item);
  const int* hd = reinterpret_cast<const int*>(host + off);
  MMAE_CHECK(hd[3] == kind && hd[0] == n_in && hd[1] == n_out, MMAE_ERR_ARG,
             "mmae_augment_batch: item %d: table at %lld is {in %d, out %d, kind %d}, expected {%d, %d, %d}", item,
             (long long)off, hd[0], hd[1], hd[3], n_in, n_out, kind);
  if (!seen.insert(off).second) return MMAE_OK;
  const int* body = hd + 4;
  if (kind == AUG_TABLE_NEAREST) {
    MMAE_CHECK(off + 16 + 4 * int64_t(n_out) <= bytes, MMAE_ERR_ARG, "mmae_augment_batch: item %d: table is truncated",
               item);
    for (int i = 0; i < n_out; ++i)
      MMAE_CHECK(body[i] >= 0 && body[i] < n_in, MMAE_ERR_ARG,
                 "mmae_augment_batch: item %d: nearest index %d of %d -> %d out of range", item, i, n_in, n_out);
    return MMAE_OK;
  }
  const int ksize = hd[2];
  MMAE_CHECK(ksize >= 1 && ksize <= 4 * AUG_MAX_EXTENT + 1, MMAE_ERR_ARG, "mmae_augment_batch: item %d: bad tap count %d",
             item, ksize);
  MMAE_CHECK(off + aug_bicubic_bytes(n_out, ksize) <= bytes, MMAE_ERR_ARG,
             "mmae_augment_batch: item %d: table is truncated", item);
  for (int i = 0; i < n_out; ++i) {
    const int lo = body[2 * i], cnt = body[2 * i + 1];
    MMAE_CHECK(lo >= 0 && cnt >= 0 && cnt <= ksize && lo + cnt <= n_in, MMAE_ERR_ARG,
               "mmae_augment_batch: item %d: taps [%d, %d + %d) of output %d outside %d inputs", item, lo, lo, cnt, i, n_in);
  }
  return MMAE_OK;
}

}  // namespace
}  // namespace mmae

using namespace mmae;

extern "C" int mmae_augment_batch(const void* packed_host, const void* packed, int64_t packed_bytes, int batch,
                                  int num_tasks, const int* kinds_host, int out_size, int64_t map4_offset, void* scratch,
                                  int64_t scratch_bytes, void* const* out_host, const float* mean_host,
                                  const float* std_host, void* stream) {
  MMAE_CHECK(packed_host && packed && kinds_host && out_host, MMAE_ERR_ARG, "mmae_augment_batch: null pointer");
  MMAE_CHECK(batch >= 1 && num_tasks >= 1 && num_tasks <= MMAE_MAX_TASKS && int64_t(batch) * num_tasks <= 65535,
             MMAE_ERR_ARG, "mmae_augment_batch: bad batch %d / task count %d", batch, num_tasks);
  MMAE_CHECK(out_size >= 4 && out_size <= AUG_MAX_SIZE, MMAE_ERR_ARG, "mmae_augment_batch: output size %d outside [4, %d]",
             out_size, AUG_MAX_SIZE);
  MMAE_CHECK(scratch_bytes >= 0 && (scratch_bytes == 0 || scratch), MMAE_ERR_ARG, "mmae_augment_batch: bad scratch");
  MMAE_CHECK(((reinterpret_cast<uintptr_t>(packed) | reinterpret_cast<uintptr_t>(scratch)) & 15) == 0, MMAE_ERR_ARG,
             "mmae_augment_batch: buffers must be 16-byte aligned");
  const int64_t desc_bytes = int64_t(batch) * num_tasks * AUG_DESC * 4;
  MMAE_CHECK(packed_bytes >= desc_bytes, MMAE_ERR_ARG, "mmae_augment_batch: %lld bytes cannot hold %lld of descriptors",
             (long long)packed_bytes, (long long)desc_bytes);
  bool rgb = false;
  for (int t = 0; t < num_tasks; ++t) {
    MMAE_CHECK(kinds_host[t] >= 0 && kinds_host[t] <= 2, MMAE_ERR_ARG, "mmae_augment_batch: task %d: bad kind %d", t,
               kinds_host[t]);
    MMAE_CHECK(out_host[t] && (reinterpret_cast<uintptr_t>(out_host[t]) & 15) == 0, MMAE_ERR_ARG,
               "mmae_augment_batch: task %d: output pointer null or not 16-byte aligned", t);
    rgb |= kinds_host[t] == 0;
  }
  MMAE_CHECK(!rgb || (mean_host && std_host), MMAE_ERR_ARG, "mmae_augment_batch: rgb needs mean and std");
  AugNorm norm = {};
  for (int c = 0; rgb && c < 3; ++c) {
    MMAE_CHECK(isfinite(mean_host[c]) && isfinite(std_host[c]) && std_host[c] != 0.0f, MMAE_ERR_ARG,
               "mmae_augment_batch: bad mean / std of channel %d", c);
    norm.mean[c] = mean_host[c];
    norm.std[c] = std_host[c];
  }
  const uint8_t* host = static_cast<const uint8_t*>(packed_host);
  std::unordered_set<int64_t> seen;
  int rc = check_table(host, packed_bytes, map4_offset, AUG_TABLE_NEAREST, out_size, out_size / 4, -1, seen);
  if (rc != MMAE_OK) return rc;
  int64_t max_rows = 0;
  const int* desc = reinterpret_cast<const int*>(host);
  for (int i = 0; i < batch * num_tasks; ++i) {
    const int* d = desc + int64_t(i) * AUG_DESC;
    const int kind = d[0], h = d[2], w = d[3];
    MMAE_CHECK(kind == kinds_host[i % num_tasks], MMAE_ERR_ARG, "mmae_augment_batch: item %d: kind %d, task kind %d", i,
               kind, kinds_host[i % num_tasks]);
    MMAE_CHECK(h >= 1 && w >= 1 && h <= AUG_MAX_EXTENT && w <= AUG_MAX_EXTENT && (d[4] == 0 || d[4] == 1), MMAE_ERR_ARG,
               "mmae_augment_batch: item %d: bad crop %d x %d / flip %d", i, h, w, d[4]);
    const int esize = kind == 1 ? 2 : 1, ch = kind == 0 ? 3 : 1;
    MMAE_CHECK(d[1] >= 0 && int64_t(d[1]) * 16 + int64_t(h) * w * ch * esize <= packed_bytes, MMAE_ERR_ARG,
               "mmae_augment_batch: item %d: crop outside the buffer", i);
    const int tk = kind == 2 ? AUG_TABLE_NEAREST : AUG_TABLE_BICUBIC;
    if ((rc = check_table(host, packed_bytes, d[5], tk, w, out_size, i, seen)) != MMAE_OK) return rc;
    if ((rc = check_table(host, packed_bytes, d[6], tk, h, out_size, i, seen)) != MMAE_OK) return rc;
    if (kind != 2) {
      MMAE_CHECK(d[7] >= 0 && int64_t(d[7]) * 16 + int64_t(h) * out_size * ch * esize <= scratch_bytes, MMAE_ERR_ARG,
                 "mmae_augment_batch: item %d: intermediate outside the scratch buffer", i);
      max_rows = std::max<int64_t>(max_rows, h);
    }
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const uint8_t* buf = static_cast<const uint8_t*>(packed);
  const int* desc_dev = reinterpret_cast<const int*>(buf);
  AugOutputs outs = {};
  for (int t = 0; t < num_tasks; ++t) outs.p[t] = out_host[t];
  const unsigned items = unsigned(batch * num_tasks);
  const int64_t cap = 1024;
  if (max_rows > 0) {
    const int64_t bx = std::min<int64_t>((max_rows * out_size + AUG_THREADS - 1) / AUG_THREADS, cap);
    launch_k(augment_horizontal_kernel, dim3(unsigned(bx), items), AUG_THREADS, 0, st, buf, desc_dev,
             static_cast<uint8_t*>(scratch), out_size);
    count_launch();
    MMAE_LAUNCH_OK();
  }
  const int64_t bx = std::min<int64_t>((int64_t(out_size) * out_size + AUG_THREADS - 1) / AUG_THREADS, cap);
  launch_k(augment_vertical_kernel, dim3(unsigned(bx), items), AUG_THREADS, 0, st, buf, desc_dev,
           static_cast<const uint8_t*>(scratch), out_size, num_tasks,
           reinterpret_cast<const int*>(buf + map4_offset * 16) + 4, outs, norm);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}
