// Trainable positional tables of the input adapters (learnable_pos_emb=True or sincos_pos_emb=False):
//   forward : rows[p, d] = F.interpolate(pos_emb [1, D, h, w], (nh, nw))[0, d, p / nw, p % nw]
//             (bicubic, A = -0.75, for PatchedInputAdapter, multimae/input_adapters.py:113; bilinear for
//             SemSegInputAdapter, :235; align_corners=False in both), or the transpose when (nh, nw) == (h, w)
//   backward: dpos_emb[0, d, y, x] += sum over the rows p that read (y, x) of weight(p; y, x) * drows[p, d]
// and the gradient of those rows from the encoder-input gradient, dx -> drows (mmae_embed_pos_backward).
// Everything is written in gather form: each output element is owned by one thread and summed in a fixed order, so the
// results are bitwise repeatable and no atomics are needed.  The tables are small (32 x 32 x 768 at most in the shipped
// configurations); the kernels read the parameter in place, so a captured CUDA graph sees the optimizer's latest values.
#include "common.cuh"
#include "../../include/multimae_b200.h"

#include "internal.h"

#define RUN(expr)                   \
  do {                              \
    int _rc = (expr);               \
    if (_rc != MMAE_OK) return _rc; \
  } while (0)

namespace mmae {
namespace {

constexpr int POS_THREADS = 256;
constexpr int POS_MAX_TAPS = 4;

// The source taps of output index `dst` along one axis of length `in` resized to `out`, as ATen computes them
// (aten/src/ATen/native/UpSample.h): scale = in / out, src = scale * (dst + 0.5) - 0.5.
//   bilinear: src clamped below at 0, i0 = floor(src), i1 = i0 + (i0 < in - 1), weights (1 - l, l) with l = src - i0;
//   bicubic : i = floor(src) - 1 .. floor(src) + 2 clamped to [0, in - 1], weights of the cubic convolution with A = -0.75
//             at t = src - floor(src) (a clamped tap keeps its weight, so border pixels collect several);
//   in == out: the single tap dst with weight 1 (the same values the formulas give there, and what F.interpolate returns).
struct Taps {
  int i[POS_MAX_TAPS];
  float w[POS_MAX_TAPS];
  int n;
};

__device__ __forceinline__ float cubic1(float x, float A) { return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; }
__device__ __forceinline__ float cubic2(float x, float A) { return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; }

__device__ __forceinline__ Taps axis_taps(int dst, int in, int out, int mode) {
  Taps t;
  if (in == out) {
    t.n = 1;
    t.i[0] = dst;
    t.w[0] = 1.f;
    return t;
  }
  const float scale = (float)in / (float)out;
  const float src = scale * (dst + 0.5f) - 0.5f;
  if (mode == MMAE_POS_BILINEAR) {
    const float s = fmaxf(src, 0.f);
    const int i0 = (int)s;
    const float l1 = s - (float)i0;
    t.n = 2;
    t.i[0] = i0;
    t.i[1] = i0 + (i0 < in - 1 ? 1 : 0);
    t.w[0] = 1.f - l1;
    t.w[1] = l1;
    return t;
  }
  const int f = (int)floorf(src);
  const float x = src - (float)f, A = -0.75f;
  t.n = 4;
  t.w[0] = cubic2(x + 1.f, A);
  t.w[1] = cubic1(x, A);
  t.w[2] = cubic1(1.f - x, A);
  t.w[3] = cubic2(2.f - x, A);
#pragma unroll
  for (int k = 0; k < 4; ++k) t.i[k] = min(max(f - 1 + k, 0), in - 1);
  return t;
}

// weight with which output index `dst` reads source index `src` along one axis (0: it does not read it)
__device__ __forceinline__ float axis_weight(int dst, int src, int in, int out, int mode) {
  const Taps t = axis_taps(dst, in, out, mode);
  float w = 0.f;
  for (int k = 0; k < t.n; ++k)
    if (t.i[k] == src) w += t.w[k];
  return w;
}

// One CTA per output row p = (oy, ox); thread d of the row reads the table at its (at most 4 x 4) taps.
__global__ void __launch_bounds__(POS_THREADS) pos_resample_fwd_kernel(const float* __restrict__ table, int D, int h, int w,
                                                                       int nh, int nw, int mode, float* __restrict__ rows) {
  pdl_prologue();
  const int p = blockIdx.x, oy = p / nw, ox = p % nw;
  const Taps ty = axis_taps(oy, h, nh, mode), tx = axis_taps(ox, w, nw, mode);
  const int64_t plane = int64_t(h) * w;
  for (int d = threadIdx.x; d < D; d += POS_THREADS) {
    const float* td = table + d * plane;
    float acc = 0.f;
    for (int a = 0; a < ty.n; ++a) {
      float r = 0.f;
      for (int b = 0; b < tx.n; ++b) r = fmaf(tx.w[b], __ldg(td + ty.i[a] * w + tx.i[b]), r);
      acc = fmaf(ty.w[a], r, acc);
    }
    rows[int64_t(p) * D + d] = acc;
  }
}

// Adjoint, one CTA per table position (y, x): the per-axis weights of every output index on y / x go to shared memory
// first, then thread d sums wy(oy) * wx(ox) * drows[oy * nw + ox, d] over the outputs that read (y, x), oy then ox in
// increasing order, and adds the sum to dtable[d, y, x].
__global__ void __launch_bounds__(POS_THREADS) pos_resample_bwd_kernel(const float* __restrict__ drows, int D, int h, int w,
                                                                       int nh, int nw, int mode, float* __restrict__ dtable) {
  pdl_prologue();
  extern __shared__ float wsm[];                        // [nh] weights on y, then [nw] weights on x
  const int y = blockIdx.x / w, x = blockIdx.x % w;
  for (int i = threadIdx.x; i < nh + nw; i += POS_THREADS)
    wsm[i] = i < nh ? axis_weight(i, y, h, nh, mode) : axis_weight(i - nh, x, w, nw, mode);
  __syncthreads();
  const float* wy = wsm;
  const float* wx = wsm + nh;
  const int64_t plane = int64_t(h) * w;
  for (int d = threadIdx.x; d < D; d += POS_THREADS) {
    float acc = 0.f;
    for (int oy = 0; oy < nh; ++oy) {
      if (wy[oy] == 0.f) continue;
      float r = 0.f;
      const float* g = drows + int64_t(oy) * nw * D + d;
      for (int ox = 0; ox < nw; ++ox)
        if (wx[ox] != 0.f) r = fmaf(wx[ox], __ldg(g + int64_t(ox) * D), r);
      acc = fmaf(wy[oy], r, acc);
    }
    dtable[d * plane + blockIdx.x] += acc;
  }
}

struct PosRows {
  float* p[MMAE_MAX_TASKS];
};

// One CTA per token g of the full (unmasked) sequence, i.e. per row p of task t's table: drows_t[p, :] = sum over samples
// b with slot = ids_restore[b, g] < T of dx[b, slot, :], b in increasing order.  Tasks without a destination are skipped.
// A kernel of its own rather than a fold into embed_assemble_bwd_kernel (index_ops.cu): that kernel walks dx by sequence
// row, and the B tokens of one patch lie in different CTAs there, so the sum would need atomics and lose repeatability.
// The extra read of dx is B*T*D*4 bytes (12.6 MB for the ADE fine-tuning step at batch 4).
__global__ void __launch_bounds__(POS_THREADS) embed_pos_bwd_kernel(mmae_embed_layout L, const int64_t* __restrict__ ids_restore,
                                                                    int B, int T, int G, int D, const float* __restrict__ dx,
                                                                    PosRows out) {
  pdl_prologue();
  const int g = blockIdx.x, total = L.tok_offset[L.num_tasks];
  int t = 0;
  for (int i = 1; i < L.num_tasks; ++i)
    if (g >= L.tok_offset[i]) t = i;
  float* dst = out.p[t];
  if (dst == nullptr) return;
  const int p = g - L.tok_offset[t];
  for (int c = threadIdx.x; c < D / 4; c += POS_THREADS) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int b = 0; b < B; ++b) {
      const int64_t slot = __ldg(ids_restore + int64_t(b) * total + g);
      if (slot >= T) continue;                          // the patch is masked in sample b: it reaches no token
      const float4 v = __ldg(reinterpret_cast<const float4*>(dx + (int64_t(b) * (T + G) + slot) * D) + c);
      acc.x += v.x;
      acc.y += v.y;
      acc.z += v.z;
      acc.w += v.w;
    }
    reinterpret_cast<float4*>(dst + int64_t(p) * D)[c] = acc;
  }
}

int check_resample(const char* what, const void* a, const void* b, int D, int h, int w, int nh, int nw, int mode) {
  MMAE_CHECK(a && b && D > 0 && h > 0 && w > 0 && nh > 0 && nw > 0, MMAE_ERR_ARG, "%s: bad args", what);
  MMAE_CHECK(mode == MMAE_POS_BICUBIC || mode == MMAE_POS_BILINEAR, MMAE_ERR_ARG, "%s: mode %d is neither "
             "MMAE_POS_BICUBIC nor MMAE_POS_BILINEAR", what, mode);
  MMAE_CHECK(nh + nw <= 8192, MMAE_ERR_UNSUPPORTED, "%s: output grid %d x %d is too large", what, nh, nw);
  return MMAE_OK;
}

}  // namespace
}  // namespace mmae

using namespace mmae;

extern "C" int mmae_pos_resample_forward(const float* table, int D, int h, int w, int nh, int nw, int mode, float* rows,
                                         void* st) {
  RUN(check_resample("mmae_pos_resample_forward", table, rows, D, h, w, nh, nw, mode));
  launch_k(pos_resample_fwd_kernel, nh * nw, POS_THREADS, 0, reinterpret_cast<cudaStream_t>(st), table, D, h, w, nh, nw,
           mode, rows);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

extern "C" int mmae_pos_resample_backward(const float* drows, int D, int h, int w, int nh, int nw, int mode, float* dtable,
                                          void* st) {
  RUN(check_resample("mmae_pos_resample_backward", drows, dtable, D, h, w, nh, nw, mode));
  launch_k(pos_resample_bwd_kernel, h * w, POS_THREADS, size_t(nh + nw) * sizeof(float), reinterpret_cast<cudaStream_t>(st),
           drows, D, h, w, nh, nw, mode, dtable);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

extern "C" int mmae_embed_pos_backward(const mmae_embed_layout* Lp, const int64_t* ids_restore, int B, int T, int G, int D,
                                       const float* dx, float* const* drows_host, void* st) {
  MMAE_CHECK(Lp && ids_restore && dx && drows_host && B > 0 && T > 0 && G >= 0 && D > 0 && D % 4 == 0, MMAE_ERR_ARG,
             "mmae_embed_pos_backward: bad args");
  const mmae_embed_layout& L = *Lp;
  MMAE_CHECK(L.num_tasks >= 1 && L.num_tasks <= MMAE_MAX_TASKS, MMAE_ERR_ARG, "mmae_embed_pos_backward: bad task count");
  PosRows out;
  bool any = false;
  for (int t = 0; t < MMAE_MAX_TASKS; ++t) {
    out.p[t] = t < L.num_tasks ? drows_host[t] : nullptr;
    any = any || out.p[t] != nullptr;
  }
  if (!any) return MMAE_OK;
  launch_k(embed_pos_bwd_kernel, L.tok_offset[L.num_tasks], POS_THREADS, 0, reinterpret_cast<cudaStream_t>(st), L,
           ids_restore, B, T, G, D, dx, out);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}
