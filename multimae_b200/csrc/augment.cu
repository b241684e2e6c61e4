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
constexpr int AUG_TABLE_BICUBIC = 1, AUG_TABLE_NEAREST = 2, AUG_TABLE_BILINEAR = 3;   // 1 and 3: the same layout
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

// A crop sample.  kCoherent: through L2 only (ld.global.cg), for crops the previous kernel of the stream wrote (the JPEG
// / PNG decode's tail): a programmatically launched dependent may otherwise hit a stale L1 line (runtime.cu, MMAE_PDL).
template <bool kCoherent, typename T>
__device__ __forceinline__ int aug_src(const T* p) {
  if constexpr (kCoherent) return int(__ldcg(p));
  return int(*p);
}

// Horizontal pass: row y of the crop (h x w) -> row y of the scratch image (h x S), for every rgb / depth item.
template <bool kCoherent>
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
        s0 += aug_src<kCoherent>(row + 3 * x) * kx;
        s1 += aug_src<kCoherent>(row + 3 * x + 1) * kx;
        s2 += aug_src<kCoherent>(row + 3 * x + 2) * kx;
      }
      uint8_t* o = scratch + int64_t(d[7]) * 16 + idx * 3;
      o[0] = uint8_t(aug_clip8(s0));
      o[1] = uint8_t(aug_clip8(s1));
      o[2] = uint8_t(aug_clip8(s2));
    } else {
      const double* k = reinterpret_cast<const double*>(tab + aug_double_off(S, ksize)) + int64_t(xx) * ksize;
      const uint16_t* row = reinterpret_cast<const uint16_t*>(src) + int64_t(y) * w + xmin;
      double ss = 0.0;
      for (int x = 0; x < xmax; ++x) ss = __dadd_rn(ss, __dmul_rn(double(aug_src<kCoherent>(row + x)), k[x]));
      reinterpret_cast<uint16_t*>(scratch + int64_t(d[7]) * 16)[idx] = uint16_t(aug_store16(ss));
    }
  }
}

// Output pixel (yy, x) of an rgb item's vertical pass, from column x of its scratch image (h x S): Pillow's clip8 values.
__device__ __forceinline__ void aug_vertical_rgb(const uint8_t* tab, const int* d, const uint8_t* scratch, int S, int yy,
                                                 int x, int ksize, int ymin, int ymax, int v[3]) {
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
  v[0] = aug_clip8(s0);
  v[1] = aug_clip8(s1);
  v[2] = aug_clip8(s2);
}

// Vertical pass: column x of the scratch image (h x S) -> the S x S output, flipped and normalised; semseg items gather
// their S/4 x S/4 labels through the nearest maps.
template <bool kCoherent>
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
      const uint8_t* p = &src[int64_t(mh[map4[y4]]) * w + mw[flip ? S - 1 - xs : xs]];
      o[idx] = int64_t(kCoherent ? __ldcg(p) : *p);   // through L2 when kCoherent, as aug_src
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
      float* o = static_cast<float*>(dst_base) + int64_t(b) * 3 * plane + dst;
      int v[3];
      aug_vertical_rgb(tab, d, scratch, S, yy, x, ksize, ymin, ymax, v);
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

// Host-side check of one table in the host part (`host_bytes` long) of the packed buffer; `fn` names the entry point.
int check_table(const char* fn, const uint8_t* host, int64_t host_bytes, int64_t off16, int kind, int n_in, int n_out,
                int item, std::unordered_set<int64_t>& seen) {
  const int64_t off = off16 * 16;
  MMAE_CHECK(off16 >= 0 && off + 16 <= host_bytes, MMAE_ERR_ARG, "%s: item %d: table offset out of range", fn, item);
  const int* hd = reinterpret_cast<const int*>(host + off);
  MMAE_CHECK(hd[3] == kind && hd[0] == n_in && hd[1] == n_out, MMAE_ERR_ARG,
             "%s: item %d: table at %lld is {in %d, out %d, kind %d}, expected {%d, %d, %d}", fn, item, (long long)off,
             hd[0], hd[1], hd[3], n_in, n_out, kind);
  if (!seen.insert(off).second) return MMAE_OK;
  const int* body = hd + 4;
  if (kind == AUG_TABLE_NEAREST) {
    MMAE_CHECK(off + 16 + 4 * int64_t(n_out) <= host_bytes, MMAE_ERR_ARG, "%s: item %d: table is truncated", fn, item);
    for (int i = 0; i < n_out; ++i)
      MMAE_CHECK(body[i] >= 0 && body[i] < n_in, MMAE_ERR_ARG,
                 "%s: item %d: nearest index %d of %d -> %d out of range", fn, item, i, n_in, n_out);
    return MMAE_OK;
  }
  const int ksize = hd[2];
  MMAE_CHECK(ksize >= 1 && ksize <= 4 * AUG_MAX_EXTENT + 1, MMAE_ERR_ARG, "%s: item %d: bad tap count %d", fn, item,
             ksize);
  MMAE_CHECK(off + aug_bicubic_bytes(n_out, ksize) <= host_bytes, MMAE_ERR_ARG, "%s: item %d: table is truncated", fn,
             item);
  for (int i = 0; i < n_out; ++i) {
    const int lo = body[2 * i], cnt = body[2 * i + 1];
    MMAE_CHECK(lo >= 0 && cnt >= 0 && cnt <= ksize && lo + cnt <= n_in, MMAE_ERR_ARG,
               "%s: item %d: taps [%d, %d + %d) of output %d outside %d inputs", fn, item, lo, lo, cnt, i, n_in);
  }
  return MMAE_OK;
}

// Host-side checks of item i shared by both entry points: crop size and flip, the crop inside the buffer (host part or
// device tail), its two tables of type tk (crop extent -> S) inside the host part, and for rgb / depth the intermediate
// offset; inter_end and max_rows grow to the end of its intermediate in the scratch and to its crop height.
int check_item(const char* fn, const uint8_t* host, int64_t host_bytes, int64_t packed_bytes, int i, int tk, int S,
               std::unordered_set<int64_t>& seen, int64_t& inter_end, int64_t& max_rows) {
  const int* d = reinterpret_cast<const int*>(host) + int64_t(i) * AUG_DESC;
  const int kind = d[0], h = d[2], w = d[3];
  MMAE_CHECK(h >= 1 && w >= 1 && h <= AUG_MAX_EXTENT && w <= AUG_MAX_EXTENT && (d[4] == 0 || d[4] == 1), MMAE_ERR_ARG,
             "%s: item %d: bad crop %d x %d / flip %d", fn, i, h, w, d[4]);
  const int64_t px = kind == 0 ? 3 : kind == 1 ? 2 : 1;   // bytes per pixel
  MMAE_CHECK(d[1] >= 0 && int64_t(d[1]) * 16 + int64_t(h) * w * px <= packed_bytes, MMAE_ERR_ARG,
             "%s: item %d: crop outside the buffer", fn, i);
  int rc;
  if ((rc = check_table(fn, host, host_bytes, d[5], tk, w, S, i, seen)) != MMAE_OK) return rc;
  if ((rc = check_table(fn, host, host_bytes, d[6], tk, h, S, i, seen)) != MMAE_OK) return rc;
  if (kind == 2) return MMAE_OK;
  MMAE_CHECK(d[7] >= 0, MMAE_ERR_ARG, "%s: item %d: bad intermediate offset", fn, i);
  inter_end = std::max<int64_t>(inter_end, int64_t(d[7]) * 16 + int64_t(h) * S * px);
  max_rows = std::max<int64_t>(max_rows, h);
  return MMAE_OK;
}

// Host-side check of TF.normalize's mean / std (3 floats each) into `norm`.
int check_norm(const char* fn, const float* mean_host, const float* std_host, AugNorm& norm) {
  for (int c = 0; c < 3; ++c) {
    MMAE_CHECK(isfinite(mean_host[c]) && isfinite(std_host[c]) && std_host[c] != 0.0f, MMAE_ERR_ARG,
               "%s: bad mean / std of channel %d", fn, c);
    norm.mean[c] = mean_host[c];
    norm.std[c] = std_host[c];
  }
  return MMAE_OK;
}


// ---------------------------------------------------------------------------------------------------------------------
// Classification fine-tuning (mmae_cls_augment_batch): resize (the horizontal pass above, then a vertical pass with the
// flip into a uint8 HWC image), RandAugment layers (per layer: a prepare kernel for the per-sample tables, then an apply
// kernel that switches on the op kind; the last one writes the normalised fp32 tensor).  Every image is S x S x 3.
// ---------------------------------------------------------------------------------------------------------------------
enum ClsOpKind {
  CLS_IDENTITY, CLS_INVERT, CLS_POSTERIZE, CLS_SOLARIZE, CLS_SOLARIZE_ADD, CLS_AUTOCONTRAST, CLS_EQUALIZE, CLS_COLOR,
  CLS_CONTRAST, CLS_BRIGHTNESS, CLS_SHARPNESS, CLS_AFFINE, CLS_TRANSPOSE, CLS_OP_KINDS
};
struct ClsOp {
  int kind, filter, iarg, pad;
  double factor;
  double m[6];
};
static_assert(sizeof(ClsOp) == 72, "ClsOp is the host's OP_DTYPE");
constexpr int CLS_FILTER_BILINEAR = 2, CLS_FILTER_BICUBIC = 3;
constexpr int CLS_TAB_INTS = 1024;          // per sample: LUT [3][256], then the Contrast grey level
constexpr int CLS_PREP_THREADS = 1024;
constexpr int CLS_MAX_LAYERS = 16;

struct ClsFill {
  int c[3];
};

__device__ __forceinline__ bool cls_is_lut(int kind) { return kind >= CLS_INVERT && kind <= CLS_EQUALIZE; }

// Pillow's RGB -> L.
__device__ __forceinline__ int cls_luma(const uint8_t* p) {
  return (int(p[0]) * 19595 + int(p[1]) * 38470 + int(p[2]) * 7471 + 0x8000) >> 16;
}

// ImagingBlend(in1, in2, (float) alpha) of one byte: in1 + alpha * (in2 - in1) in float, truncated; clipped when alpha
// is outside [0, 1].
__device__ __forceinline__ int cls_blend(int in1, int in2, float a) {
  const float t = __fadd_rn(float(in1), __fmul_rn(a, float(in2 - in1)));
  if (a >= 0.0f && a <= 1.0f) return int(t);
  return t <= 0.0f ? 0 : (t >= 255.0f ? 255 : int(t));
}

// ImagingFilter3x3's KERNEL1x3: (in[x-1] * k0 + in[x] * k1) + in[x+1] * k2 in float.
__device__ __forceinline__ float cls_k3(const uint8_t* p, float k0, float k1, float k2) {
  return __fadd_rn(__fadd_rn(__fmul_rn(float(p[-3]), k0), __fmul_rn(float(p[0]), k1)), __fmul_rn(float(p[3]), k2));
}

// Geometry.c's BICUBIC of four integer samples (the first, horizontal stage): p2..p4 are integer expressions.
__device__ __forceinline__ double cls_cubic_i(int v1, int v2, int v3, int v4, double d) {
  const double p1 = v2, p2 = -v1 + v3, p3 = 2 * (v1 - v2) + v3 - v4, p4 = -v1 + v2 - v3 + v4;
  return __dadd_rn(p1, __dmul_rn(d, __dadd_rn(p2, __dmul_rn(d, __dadd_rn(p3, __dmul_rn(d, p4))))));
}
__device__ __forceinline__ double cls_cubic_d(double v1, double v2, double v3, double v4, double d) {
  const double p1 = v2;
  const double p2 = __dadd_rn(-v1, v3);
  const double p3 = __dsub_rn(__dadd_rn(__dmul_rn(2.0, __dsub_rn(v1, v2)), v3), v4);
  const double p4 = __dadd_rn(__dsub_rn(__dadd_rn(-v1, v2), v3), v4);
  return __dadd_rn(p1, __dmul_rn(d, __dadd_rn(p2, __dmul_rn(d, __dadd_rn(p3, __dmul_rn(d, p4))))));
}

// Vertical pass of a classification sample into the uint8 image, flipped.
__global__ void __launch_bounds__(AUG_THREADS) cls_vertical_u8_kernel(const uint8_t* __restrict__ buf,
                                                                      const int* __restrict__ desc,
                                                                      const uint8_t* scratch, int S, uint8_t* img) {
  pdl_prologue();
  const int b = blockIdx.y;
  const int* d = desc + int64_t(b) * AUG_DESC;
  const uint8_t* tab = buf + int64_t(d[6]) * 16;
  const int ksize = reinterpret_cast<const int*>(tab)[2];
  const int* bounds = reinterpret_cast<const int*>(tab) + 4;
  const int flip = d[4];
  for (int idx = blockIdx.x * AUG_THREADS + threadIdx.x; idx < S * S; idx += gridDim.x * AUG_THREADS) {
    const int yy = idx / S, x = idx - yy * S;
    int v[3];
    aug_vertical_rgb(tab, d, scratch, S, yy, x, ksize, bounds[2 * yy], bounds[2 * yy + 1], v);
    uint8_t* o = img + ((int64_t(b) * S + yy) * S + (flip ? S - 1 - x : x)) * 3;
    o[0] = uint8_t(v[0]);
    o[1] = uint8_t(v[1]);
    o[2] = uint8_t(v[2]);
  }
}

// One block per sample: the LUT of a LUT op (ImageOps' tables; AutoContrast and Equalize from the channel histograms) or
// the grey level of Contrast (ImageStat's mean of the L image, rounded as ImageEnhance rounds it).
__global__ void __launch_bounds__(CLS_PREP_THREADS) cls_prepare_kernel(const ClsOp* __restrict__ ops, int layer,
                                                                       int num_layers, const uint8_t* img, int S,
                                                                       int* tabs) {
  pdl_prologue();
  __shared__ int hist[4][256];
  __shared__ int lohi[3][2];
  const int b = blockIdx.x, tid = threadIdx.x;
  const ClsOp& op = ops[int64_t(b) * num_layers + layer];
  const int kind = op.kind;
  if (!cls_is_lut(kind) && kind != CLS_CONTRAST) return;
  int* t = tabs + int64_t(b) * CLS_TAB_INTS;
  const bool need_hist = kind == CLS_AUTOCONTRAST || kind == CLS_EQUALIZE || kind == CLS_CONTRAST;
  if (need_hist) {
    for (int i = tid; i < 4 * 256; i += CLS_PREP_THREADS) (&hist[0][0])[i] = 0;
    __syncthreads();
    const uint8_t* p = img + int64_t(b) * S * S * 3;
    for (int i = tid; i < S * S; i += CLS_PREP_THREADS) {
      if (kind == CLS_CONTRAST) {
        atomicAdd(&hist[3][cls_luma(p + 3 * i)], 1);
      } else {
        atomicAdd(&hist[0][p[3 * i]], 1);
        atomicAdd(&hist[1][p[3 * i + 1]], 1);
        atomicAdd(&hist[2][p[3 * i + 2]], 1);
      }
    }
    __syncthreads();
  }
  if (kind == CLS_CONTRAST) {
    if (tid == 0) {
      long long sum = 0, count = 0;
      for (int j = 0; j < 256; ++j) {
        sum += (long long)j * hist[3][j];
        count += hist[3][j];
      }
      t[768] = int(__dadd_rn(__ddiv_rn(double(sum), double(count)), 0.5));
    }
    return;
  }
  if (kind == CLS_EQUALIZE) {
    if (tid < 3) {
      const int* h = hist[tid];
      int nonzero = 0, last = 0;
      long long total = 0;
      for (int i = 0; i < 256; ++i)
        if (h[i]) {
          ++nonzero;
          last = h[i];
          total += h[i];
        }
      const long long step = nonzero <= 1 ? 0 : (total - last) / 255;
      long long n = step / 2;
      for (int i = 0; i < 256; ++i) {
        t[tid * 256 + i] = step ? int(min(n / step, 255LL)) : i;   // Image.point clips the table
        n += h[i];
      }
    }
    return;
  }
  if (kind == CLS_AUTOCONTRAST) {
    if (tid < 3) {
      int lo = 0, hi = 255;
      while (lo < 256 && !hist[tid][lo]) ++lo;
      while (hi >= 0 && !hist[tid][hi]) --hi;
      lohi[tid][0] = lo;
      lohi[tid][1] = hi;
    }
    __syncthreads();
  }
  if (tid < 768) {
    const int c = tid >> 8, i = tid & 255;
    int v = i;
    switch (kind) {
      case CLS_INVERT: v = 255 - i; break;
      case CLS_POSTERIZE: v = i & ~((1 << (8 - op.iarg)) - 1); break;
      case CLS_SOLARIZE: v = i < op.iarg ? i : 255 - i; break;
      case CLS_SOLARIZE_ADD: v = i < 128 ? min(255, i + op.iarg) : i; break;
      default: {   // AutoContrast: scale = 255.0 / (hi - lo), offset = -lo * scale, int(i * scale + offset) clipped
        const int lo = lohi[c][0], hi = lohi[c][1];
        if (hi > lo) {
          const double scale = __ddiv_rn(255.0, double(hi - lo));
          const double offset = __dmul_rn(double(-lo), scale);
          v = min(max(int(__dadd_rn(__dmul_rn(double(i), scale), offset)), 0), 255);
        }
      }
    }
    t[tid] = v;
  }
}

// One RandAugment layer for every sample: reads `src`, writes `dst` (uint8) or, for the last layer, the normalised fp32
// output.
__global__ void __launch_bounds__(AUG_THREADS) cls_apply_kernel(const ClsOp* __restrict__ ops, int layer, int num_layers,
                                                                const uint8_t* src, uint8_t* dst, const int* tabs, int S,
                                                                ClsFill fill, float* out, AugNorm norm) {
  pdl_prologue();
  __shared__ uint8_t lut[768];
  const int b = blockIdx.y;
  const ClsOp& op = ops[int64_t(b) * num_layers + layer];
  const int kind = op.kind;
  const int* t = tabs + int64_t(b) * CLS_TAB_INTS;
  if (cls_is_lut(kind)) {
    for (int i = threadIdx.x; i < 768; i += AUG_THREADS) lut[i] = uint8_t(t[i]);
    __syncthreads();
  }
  const int grey = kind == CLS_CONTRAST ? t[768] : 0;
  const float alpha = __double2float_rn(op.factor);
  const float k1 = __fdiv_rn(1.0f, 13.0f), k5 = __fdiv_rn(5.0f, 13.0f);
  const uint8_t* im = src + int64_t(b) * S * S * 3;
  const int64_t plane = int64_t(S) * S;
  for (int idx = blockIdx.x * AUG_THREADS + threadIdx.x; idx < S * S; idx += gridDim.x * AUG_THREADS) {
    const int y = idx / S, x = idx - y * S;
    const uint8_t* p = im + int64_t(idx) * 3;
    int v[3] = {p[0], p[1], p[2]};
    if (cls_is_lut(kind)) {
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = lut[c * 256 + v[c]];
    } else if (kind == CLS_COLOR) {
      const int g = cls_luma(p);
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = cls_blend(g, v[c], alpha);
    } else if (kind == CLS_CONTRAST) {
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = cls_blend(grey, v[c], alpha);
    } else if (kind == CLS_BRIGHTNESS) {
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = cls_blend(0, v[c], alpha);
    } else if (kind == CLS_SHARPNESS) {
      if (y > 0 && y < S - 1 && x > 0 && x < S - 1) {   // SMOOTH leaves the border unfiltered: the blend keeps it
        const int64_t row = int64_t(S) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          float ss = 0.5f;
          ss = __fadd_rn(ss, cls_k3(p + row + c, k1, k1, k1));
          ss = __fadd_rn(ss, cls_k3(p + c, k1, k5, k1));
          ss = __fadd_rn(ss, cls_k3(p - row + c, k1, k1, k1));
          const int sm = ss <= 0.0f ? 0 : (ss >= 255.0f ? 255 : int(ss));
          v[c] = cls_blend(sm, v[c], alpha);
        }
      }
    } else if (kind == CLS_TRANSPOSE) {
      const int sy = op.iarg == 180 ? S - 1 - y : (op.iarg == 90 ? x : S - 1 - x);
      const int sx = op.iarg == 180 ? S - 1 - x : (op.iarg == 90 ? S - 1 - y : y);
      const uint8_t* q = im + (int64_t(sy) * S + sx) * 3;
      v[0] = q[0];
      v[1] = q[1];
      v[2] = q[2];
    } else if (kind == CLS_AFFINE) {
      const double xs = double(x) + 0.5, ys = double(y) + 0.5;
      double xin = __dadd_rn(__dadd_rn(__dmul_rn(op.m[0], xs), __dmul_rn(op.m[1], ys)), op.m[2]);
      double yin = __dadd_rn(__dadd_rn(__dmul_rn(op.m[3], xs), __dmul_rn(op.m[4], ys)), op.m[5]);
      if (!(xin >= 0.0 && xin < double(S) && yin >= 0.0 && yin < double(S))) {
        v[0] = fill.c[0];
        v[1] = fill.c[1];
        v[2] = fill.c[2];
      } else {
        xin = __dsub_rn(xin, 0.5);
        yin = __dsub_rn(yin, 0.5);
        const int xi = int(floor(xin)), yi = int(floor(yin));
        const double dx = __dsub_rn(xin, double(xi)), dy = __dsub_rn(yin, double(yi));
        auto at = [&](int yy, int xx, int c) -> int {
          yy = min(max(yy, 0), S - 1);
          xx = min(max(xx, 0), S - 1);
          return im[(int64_t(yy) * S + xx) * 3 + c];
        };
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          if (op.filter == CLS_FILTER_BILINEAR) {
            auto row = [&](int yy) {
              const int a = at(yy, xi, c), bb = at(yy, xi + 1, c);
              return __dadd_rn(double(a), __dmul_rn(double(bb - a), dx));
            };
            double v1 = row(yi);
            if (yi + 1 >= 0 && yi + 1 < S) {
              const double v2 = row(yi + 1);
              v1 = __dadd_rn(v1, __dmul_rn(__dsub_rn(v2, v1), dy));
            }
            v[c] = int(v1);
          } else {
            const int x0 = xi - 1, y0 = yi - 1;
            auto row = [&](int yy) {
              return cls_cubic_i(at(yy, x0, c), at(yy, x0 + 1, c), at(yy, x0 + 2, c), at(yy, x0 + 3, c), dx);
            };
            const double r1 = row(y0);
            const double r2 = (y0 + 1 >= 0 && y0 + 1 < S) ? row(y0 + 1) : r1;
            const double r3 = (y0 + 2 >= 0 && y0 + 2 < S) ? row(y0 + 2) : r2;
            const double r4 = (y0 + 3 >= 0 && y0 + 3 < S) ? row(y0 + 3) : r3;
            const double r = cls_cubic_d(r1, r2, r3, r4, dy);
            v[c] = r <= 0.0 ? 0 : (r >= 255.0 ? 255 : int(r));
          }
        }
      }
    }
    if (out) {
      float* o = out + int64_t(b) * 3 * plane + idx;
#pragma unroll
      for (int c = 0; c < 3; ++c)
        o[c * plane] = __fdiv_rn(__fsub_rn(__fdiv_rn(float(v[c]), 255.0f), norm.mean[c]), norm.std[c]);
    } else {
      uint8_t* o = dst + (int64_t(b) * plane + idx) * 3;
      o[0] = uint8_t(v[0]);
      o[1] = uint8_t(v[1]);
      o[2] = uint8_t(v[2]);
    }
  }
}

int check_cls_op(const ClsOp& op, int item, int layer) {
  MMAE_CHECK(op.kind >= 0 && op.kind < CLS_OP_KINDS, MMAE_ERR_ARG, "mmae_cls_augment_batch: item %d layer %d: bad op %d",
             item, layer, op.kind);
  bool ok = true;
  switch (op.kind) {
    case CLS_POSTERIZE: ok = op.iarg >= 0 && op.iarg <= 8; break;
    case CLS_SOLARIZE: ok = op.iarg >= 0 && op.iarg <= 256; break;
    case CLS_SOLARIZE_ADD: ok = op.iarg >= 0 && op.iarg <= 255; break;
    case CLS_TRANSPOSE: ok = op.iarg == 90 || op.iarg == 180 || op.iarg == 270; break;
    case CLS_COLOR: case CLS_CONTRAST: case CLS_BRIGHTNESS: case CLS_SHARPNESS: ok = isfinite(op.factor); break;
    case CLS_AFFINE:
      ok = op.filter == CLS_FILTER_BILINEAR || op.filter == CLS_FILTER_BICUBIC;
      for (int i = 0; i < 6; ++i) ok = ok && isfinite(op.m[i]);
      break;
    default: break;
  }
  MMAE_CHECK(ok, MMAE_ERR_ARG, "mmae_cls_augment_batch: item %d layer %d: bad arguments of op %d", item, layer, op.kind);
  return MMAE_OK;
}

}  // namespace
}  // namespace mmae

using namespace mmae;

extern "C" int mmae_augment_batch(const void* packed_host, const void* packed, int64_t host_bytes, int64_t packed_bytes,
                                  int batch, int num_tasks, const int* kinds_host, int out_size, int64_t map4_offset,
                                  void* scratch, int64_t scratch_bytes, void* const* out_host, const float* mean_host,
                                  const float* std_host, void* stream) {
  MMAE_CHECK(packed_host && packed && kinds_host && out_host, MMAE_ERR_ARG, "mmae_augment_batch: null pointer");
  MMAE_CHECK(batch >= 1 && num_tasks >= 1 && num_tasks <= MMAE_MAX_TASKS && int64_t(batch) * num_tasks <= 65535,
             MMAE_ERR_ARG, "mmae_augment_batch: bad batch %d / task count %d", batch, num_tasks);
  MMAE_CHECK(out_size >= 4 && out_size <= AUG_MAX_SIZE, MMAE_ERR_ARG, "mmae_augment_batch: output size %d outside [4, %d]",
             out_size, AUG_MAX_SIZE);
  MMAE_CHECK(scratch_bytes >= 0 && (scratch_bytes == 0 || scratch), MMAE_ERR_ARG, "mmae_augment_batch: bad scratch");
  MMAE_CHECK(((reinterpret_cast<uintptr_t>(packed) | reinterpret_cast<uintptr_t>(scratch)) & 15) == 0, MMAE_ERR_ARG,
             "mmae_augment_batch: buffers must be 16-byte aligned");
  MMAE_CHECK(host_bytes >= 0 && host_bytes <= packed_bytes, MMAE_ERR_ARG,
             "mmae_augment_batch: host part of %lld bytes, buffer of %lld", (long long)host_bytes,
             (long long)packed_bytes);
  const int64_t desc_bytes = int64_t(batch) * num_tasks * AUG_DESC * 4;
  MMAE_CHECK(host_bytes >= desc_bytes, MMAE_ERR_ARG, "mmae_augment_batch: %lld bytes cannot hold %lld of descriptors",
             (long long)host_bytes, (long long)desc_bytes);
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
  int rc;
  if (rgb && (rc = check_norm("mmae_augment_batch", mean_host, std_host, norm)) != MMAE_OK) return rc;
  const uint8_t* host = static_cast<const uint8_t*>(packed_host);
  std::unordered_set<int64_t> seen;
  rc = check_table("mmae_augment_batch", host, host_bytes, map4_offset, AUG_TABLE_NEAREST, out_size, out_size / 4, -1,
                   seen);
  if (rc != MMAE_OK) return rc;
  int64_t inter_end = 0, max_rows = 0;
  for (int i = 0; i < batch * num_tasks; ++i) {
    const int kind = reinterpret_cast<const int*>(host)[int64_t(i) * AUG_DESC];
    MMAE_CHECK(kind == kinds_host[i % num_tasks], MMAE_ERR_ARG, "mmae_augment_batch: item %d: kind %d, task kind %d", i,
               kind, kinds_host[i % num_tasks]);
    rc = check_item("mmae_augment_batch", host, host_bytes, packed_bytes, i,
                    kind == 2 ? AUG_TABLE_NEAREST : AUG_TABLE_BICUBIC, out_size, seen, inter_end, max_rows);
    if (rc != MMAE_OK) return rc;
  }
  MMAE_CHECK(inter_end <= scratch_bytes, MMAE_ERR_ARG, "mmae_augment_batch: scratch of %lld bytes, %lld needed",
             (long long)scratch_bytes, (long long)inter_end);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const uint8_t* buf = static_cast<const uint8_t*>(packed);
  const int* desc_dev = reinterpret_cast<const int*>(buf);
  AugOutputs outs = {};
  for (int t = 0; t < num_tasks; ++t) outs.p[t] = out_host[t];
  const unsigned items = unsigned(batch * num_tasks);
  const int64_t cap = 1024;
  const bool coherent = host_bytes < packed_bytes;   // crops past the host part: written by the JPEG / PNG decode
  if (max_rows > 0) {
    const int64_t bx = std::min<int64_t>((max_rows * out_size + AUG_THREADS - 1) / AUG_THREADS, cap);
    launch_k(coherent ? augment_horizontal_kernel<true> : augment_horizontal_kernel<false>, dim3(unsigned(bx), items),
             AUG_THREADS, 0, st, buf, desc_dev, static_cast<uint8_t*>(scratch), out_size);
    count_launch();
    MMAE_LAUNCH_OK();
  }
  const int64_t bx = std::min<int64_t>((int64_t(out_size) * out_size + AUG_THREADS - 1) / AUG_THREADS, cap);
  launch_k(coherent ? augment_vertical_kernel<true> : augment_vertical_kernel<false>, dim3(unsigned(bx), items),
           AUG_THREADS, 0, st, buf, desc_dev, static_cast<const uint8_t*>(scratch), out_size, num_tasks,
           reinterpret_cast<const int*>(buf + map4_offset * 16) + 4, outs, norm);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

extern "C" int mmae_cls_augment_batch(const void* packed_host, const void* packed, int64_t host_bytes,
                                      int64_t packed_bytes, int batch, int num_layers, int64_t ops_offset, int out_size,
                                      const int* fill_host, void* scratch, int64_t scratch_bytes, float* out,
                                      const float* mean_host, const float* std_host, void* stream) {
  MMAE_CHECK(packed_host && packed && fill_host && scratch && out && mean_host && std_host, MMAE_ERR_ARG,
             "mmae_cls_augment_batch: null pointer");
  MMAE_CHECK(batch >= 1 && batch <= 65535 && num_layers >= 0 && num_layers <= CLS_MAX_LAYERS, MMAE_ERR_ARG,
             "mmae_cls_augment_batch: bad batch %d / layer count %d", batch, num_layers);
  MMAE_CHECK(out_size >= 4 && out_size <= AUG_MAX_SIZE, MMAE_ERR_ARG,
             "mmae_cls_augment_batch: output size %d outside [4, %d]", out_size, AUG_MAX_SIZE);
  MMAE_CHECK(((reinterpret_cast<uintptr_t>(packed) | reinterpret_cast<uintptr_t>(scratch) |
               reinterpret_cast<uintptr_t>(out)) & 15) == 0,
             MMAE_ERR_ARG, "mmae_cls_augment_batch: buffers must be 16-byte aligned");
  AugNorm norm = {};
  ClsFill fill = {};
  int rc = check_norm("mmae_cls_augment_batch", mean_host, std_host, norm);
  if (rc != MMAE_OK) return rc;
  for (int c = 0; c < 3; ++c) {
    MMAE_CHECK(fill_host[c] >= 0 && fill_host[c] <= 255, MMAE_ERR_ARG, "mmae_cls_augment_batch: bad fill %d",
               fill_host[c]);
    fill.c[c] = fill_host[c];
  }
  const int S = out_size;
  const int64_t desc_bytes = int64_t(batch) * AUG_DESC * 4;
  const int64_t ops_bytes = int64_t(batch) * num_layers * int64_t(sizeof(ClsOp));
  MMAE_CHECK(host_bytes >= 0 && host_bytes <= packed_bytes, MMAE_ERR_ARG,
             "mmae_cls_augment_batch: host part of %lld bytes, buffer of %lld", (long long)host_bytes,
             (long long)packed_bytes);
  MMAE_CHECK(ops_offset * 16 >= desc_bytes && ops_offset * 16 + ops_bytes <= host_bytes, MMAE_ERR_ARG,
             "mmae_cls_augment_batch: op records [%lld, +%lld) overlap the descriptors or leave the %lld-byte host part",
             (long long)(ops_offset * 16), (long long)ops_bytes, (long long)host_bytes);
  const uint8_t* host = static_cast<const uint8_t*>(packed_host);
  std::unordered_set<int64_t> seen;
  int64_t inter_end = 0, max_rows = 0;
  for (int i = 0; i < batch; ++i) {
    const int* d = reinterpret_cast<const int*>(host) + int64_t(i) * AUG_DESC;
    MMAE_CHECK(d[0] == 0, MMAE_ERR_ARG, "mmae_cls_augment_batch: item %d: kind %d, expected 0 (rgb)", i, d[0]);
    MMAE_CHECK(d[5] >= 0 && int64_t(d[5]) * 16 + 16 <= host_bytes, MMAE_ERR_ARG,
               "mmae_cls_augment_batch: item %d: table offset out of range", i);
    const int tk = reinterpret_cast<const int*>(host + int64_t(d[5]) * 16)[3];
    MMAE_CHECK(tk == AUG_TABLE_BICUBIC || tk == AUG_TABLE_BILINEAR, MMAE_ERR_ARG,
               "mmae_cls_augment_batch: item %d: table type %d", i, tk);
    rc = check_item("mmae_cls_augment_batch", host, host_bytes, packed_bytes, i, tk, S, seen, inter_end, max_rows);
    if (rc != MMAE_OK) return rc;
    for (int l = 0; l < num_layers; ++l) {
      ClsOp op;
      memcpy(&op, host + ops_offset * 16 + (int64_t(i) * num_layers + l) * int64_t(sizeof(ClsOp)), sizeof(ClsOp));
      if ((rc = check_cls_op(op, i, l)) != MMAE_OK) return rc;
    }
  }
  const int64_t img_bytes = int64_t(batch) * S * S * 3;
  const int64_t img0 = int64_t(align_up(size_t(inter_end), 256));
  const int64_t img1 = img0 + int64_t(align_up(size_t(img_bytes), 256));
  const int64_t tabs = img1 + int64_t(align_up(size_t(img_bytes), 256));
  const int64_t need = num_layers ? tabs + int64_t(batch) * CLS_TAB_INTS * 4 : inter_end;
  MMAE_CHECK(need <= scratch_bytes, MMAE_ERR_ARG, "mmae_cls_augment_batch: scratch of %lld bytes, %lld needed",
             (long long)scratch_bytes, (long long)need);

  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const uint8_t* buf = static_cast<const uint8_t*>(packed);
  const int* desc_dev = reinterpret_cast<const int*>(buf);
  uint8_t* sc = static_cast<uint8_t*>(scratch);
  const int64_t cap = 1024;
  const int64_t bx_h = std::min<int64_t>((max_rows * S + AUG_THREADS - 1) / AUG_THREADS, cap);
  const bool coherent = host_bytes < packed_bytes;   // crops past the host part: written by the JPEG decode
  launch_k(coherent ? augment_horizontal_kernel<true> : augment_horizontal_kernel<false>,
           dim3(unsigned(bx_h), unsigned(batch)), AUG_THREADS, 0, st, buf, desc_dev, sc, S);
  count_launch();
  MMAE_LAUNCH_OK();
  const unsigned bx = unsigned(std::min<int64_t>((int64_t(S) * S + AUG_THREADS - 1) / AUG_THREADS, cap));
  if (num_layers == 0) {
    AugOutputs outs = {};
    outs.p[0] = out;
    launch_k(coherent ? augment_vertical_kernel<true> : augment_vertical_kernel<false>, dim3(bx, unsigned(batch)),
             AUG_THREADS, 0, st, buf, desc_dev, static_cast<const uint8_t*>(sc), S, 1, static_cast<const int*>(nullptr),
             outs, norm);
    count_launch();
    MMAE_LAUNCH_OK();
    return MMAE_OK;
  }
  uint8_t* img[2] = {sc + img0, sc + img1};
  int* tab = reinterpret_cast<int*>(sc + tabs);
  const ClsOp* ops = reinterpret_cast<const ClsOp*>(buf + ops_offset * 16);
  launch_k(cls_vertical_u8_kernel, dim3(bx, unsigned(batch)), AUG_THREADS, 0, st, buf, desc_dev,
           static_cast<const uint8_t*>(sc), S, img[0]);
  count_launch();
  MMAE_LAUNCH_OK();
  for (int l = 0; l < num_layers; ++l) {
    const bool last = l == num_layers - 1;
    launch_k(cls_prepare_kernel, dim3(unsigned(batch)), CLS_PREP_THREADS, 0, st, ops, l, num_layers,
             static_cast<const uint8_t*>(img[l & 1]), S, tab);
    count_launch();
    MMAE_LAUNCH_OK();
    launch_k(cls_apply_kernel, dim3(bx, unsigned(batch)), AUG_THREADS, 0, st, ops, l, num_layers,
             static_cast<const uint8_t*>(img[l & 1]), last ? static_cast<uint8_t*>(nullptr) : img[(l + 1) & 1],
             static_cast<const int*>(tab), S, fill, last ? out : static_cast<float*>(nullptr), norm);
    count_launch();
    MMAE_LAUNCH_OK();
  }
  return MMAE_OK;
}
