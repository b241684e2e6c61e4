// Classification head of fine-tuning: LinearOutputAdapter.forward (multimae/output_adapters.py:345-356),
//   x = encoder_tokens.mean(1)  (use_mean_pooling)  or  encoder_tokens[:, -1]  (the global token),
//   logits = head(norm(x)).
// The pool reads the whole fp32 encoder output once and its backward writes a gradient of the same size, so both are
// HBM-bound; the LayerNorm works on B rows only and the head is a small GEMM through mmae_gemm_bf16.
//
// Forward:  cls_pool_kernel        - grid (splits, B): each CTA sums a run of tokens of one sample for every column
//           cls_pool_ln_kernel     - grid B: adds a sample's partial rows in a fixed order, scales by 1/N, LayerNorm
//           mmae_gemm_bf16         - logits = xn W^T + b (fp32 accumulation and output)
// Backward: mmae_cast_colsum_f32   - bf16(dlogits), head bias gradient
//           mmae_gemm_bf16 x 2     - head weight gradient, dxn = dlogits W
//           cls_head_bwd_kernel    - grid (splits, B): LayerNorm backward of the sample's pooled row, written to its run
//                                    of token rows (dpooled / N, or dpooled on the last row and zeros elsewhere)
//           mmae_cast_colsum_f32 x 2 - LayerNorm weight / bias gradients from per-sample partial rows
// No atomics: every result is a fixed-order sum, so repeated calls are bitwise equal.
//
// The GEMM needs N % 8 == 0.  For other class counts (101, 37, 1) the head runs on a padded width Cp = round_up(C, 8):
// the bf16 weight gets zero rows, and logits, bias, logit gradient and head gradients go through padded workspace
// buffers, so nothing outside the caller's [B, C] / [C, D] / [C] tensors is read or written.
#include <cstring>

#include "internal.h"

namespace mmae {
namespace {

constexpr int POOL_MAX_THREADS = 256;
constexpr int LN_THREADS = 256;

int pool_threads(int D) { return std::min(POOL_MAX_THREADS, (D / 4 + 31) / 32 * 32); }

// token runs per sample: enough CTAs for ~4 per SM, but at most one per token
int pool_splits(int B, int N) {
  const int want = std::max(1, ceil_div(4 * reduce_sm_count(), B));
  const int chunk = ceil_div(N, std::min(want, N));
  return ceil_div(N, chunk);
}

// partial[b, s, :] = sum of x[b, t, :] over the tokens t of run s
__global__ void __launch_bounds__(POOL_MAX_THREADS) cls_pool_kernel(const float* __restrict__ x, int N, int D, int chunk,
                                                                    float* __restrict__ partial) {
  pdl_prologue();
  const int s = blockIdx.x, b = blockIdx.y;
  const int t0 = s * chunk, t1 = min(N, t0 + chunk);
  const int D4 = D / 4;
  const float* xb = x + (int64_t(b) * N + t0) * D;
  for (int c = threadIdx.x; c < D4; c += blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    const float* p = xb + 4 * c;
    int t = t0;
#pragma unroll 1
    for (; t + 8 <= t1; t += 8) {            // eight independent 16-byte loads in flight per thread
      uint4 v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = ld_stream_16(p + int64_t(j) * D);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        acc.x += __uint_as_float(v[j].x);
        acc.y += __uint_as_float(v[j].y);
        acc.z += __uint_as_float(v[j].z);
        acc.w += __uint_as_float(v[j].w);
      }
      p += int64_t(8) * D;
    }
    for (; t < t1; ++t) {
      const uint4 v = ld_stream_16(p);
      acc.x += __uint_as_float(v.x);
      acc.y += __uint_as_float(v.y);
      acc.z += __uint_as_float(v.z);
      acc.w += __uint_as_float(v.w);
      p += D;
    }
    *reinterpret_cast<float4*>(partial + (int64_t(b) * gridDim.x + s) * D + 4 * c) = acc;
  }
}

// sum over the CTA; `red` holds one float per warp.  Every thread returns the total.
__device__ __forceinline__ float block_sum(float v, float* red) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  v = warp_sum(v);
  __syncthreads();                           // `red` may still be read by the previous call
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = lane < nw ? red[lane] : 0.f;
  return warp_sum(t);
}

// pooled[b] = scale * sum_{s < parts} src[b * sample_stride + s * part_stride + :], then LayerNorm of that row.
// Writes pooled (fp32), mean / rstd, and the normalised row as bf16 (xn, the GEMM operand) and / or fp32 (y).
__global__ void __launch_bounds__(LN_THREADS) cls_pool_ln_kernel(const float* __restrict__ src, int64_t sample_stride,
                                                                 int parts, int64_t part_stride, float scale, int D,
                                                                 const float* __restrict__ gamma,
                                                                 const float* __restrict__ beta, float eps,
                                                                 float* __restrict__ pooled, float* __restrict__ mean_out,
                                                                 float* __restrict__ rstd_out, bf16* __restrict__ xn,
                                                                 float* __restrict__ y) {
  pdl_prologue();
  extern __shared__ float row[];             // D floats
  __shared__ float red[LN_THREADS / 32];
  const int b = blockIdx.x, D4 = D / 4;
  const float* sb = src + int64_t(b) * sample_stride;
  float s1 = 0.f;
  for (int c = threadIdx.x; c < D4; c += blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = 0; s < parts; ++s) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(sb + s * part_stride + 4 * c));
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    acc.x *= scale; acc.y *= scale; acc.z *= scale; acc.w *= scale;
    reinterpret_cast<float4*>(row)[c] = acc;
    *reinterpret_cast<float4*>(pooled + int64_t(b) * D + 4 * c) = acc;
    s1 += acc.x + acc.y + acc.z + acc.w;
  }
  const float mean = block_sum(s1, red) / D;
  float s2 = 0.f;
  for (int c = threadIdx.x; c < D4; c += blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(row)[c];
    const float a = v.x - mean, bb = v.y - mean, cc = v.z - mean, d = v.w - mean;
    s2 += a * a + bb * bb + cc * cc + d * d;
  }
  const float rstd = rsqrtf(block_sum(s2, red) / D + eps);
  if (threadIdx.x == 0) {
    mean_out[b] = mean;
    rstd_out[b] = rstd;
  }
  for (int c = threadIdx.x; c < D4; c += blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(row)[c];
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + 4 * c));
    const float4 be = __ldg(reinterpret_cast<const float4*>(beta + 4 * c));
    float4 o;
    o.x = (v.x - mean) * rstd * g.x + be.x;
    o.y = (v.y - mean) * rstd * g.y + be.y;
    o.z = (v.z - mean) * rstd * g.z + be.z;
    o.w = (v.w - mean) * rstd * g.w + be.w;
    if (xn) {
      uint2 p;
      p.x = pack_bf16x2(o.x, o.y);
      p.y = pack_bf16x2(o.z, o.w);
      *reinterpret_cast<uint2*>(xn + int64_t(b) * D + 4 * c) = p;
    }
    if (y) *reinterpret_cast<float4*>(y + int64_t(b) * D + 4 * c) = o;
  }
}

// LayerNorm backward of sample b's pooled row (recomputed by each of the sample's CTAs: D elements), then the gradient
// of the CTA's run of token rows.  CTA s == 0 also writes the sample's partial row of the LayerNorm parameter gradients:
// dgb[b, 0:D] = dy * xhat, dgb[b, D:2D] = dy.
__global__ void __launch_bounds__(LN_THREADS) cls_head_bwd_kernel(const float* __restrict__ dy,
                                                                  const float* __restrict__ pooled,
                                                                  const float* __restrict__ mean_in,
                                                                  const float* __restrict__ rstd_in,
                                                                  const float* __restrict__ gamma, int N, int D,
                                                                  int chunk, int mean_pool, float* __restrict__ dx,
                                                                  float* __restrict__ dgb) {
  pdl_prologue();
  extern __shared__ float drow[];            // D floats: the gradient of the pooled row, already scaled for the tokens
  __shared__ float red[LN_THREADS / 32];
  const int s = blockIdx.x, b = blockIdx.y, D4 = D / 4;
  const float mean = mean_in[b], rstd = rstd_in[b];
  const float* dyb = dy + int64_t(b) * D;
  const float* pb = pooled + int64_t(b) * D;
  float sg = 0.f, sgx = 0.f;
  for (int c = threadIdx.x; c < D4; c += blockDim.x) {
    const float4 d = __ldg(reinterpret_cast<const float4*>(dyb + 4 * c));
    const float4 p = __ldg(reinterpret_cast<const float4*>(pb + 4 * c));
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + 4 * c));
    const float4 xh = make_float4((p.x - mean) * rstd, (p.y - mean) * rstd, (p.z - mean) * rstd, (p.w - mean) * rstd);
    const float4 gd = make_float4(d.x * g.x, d.y * g.y, d.z * g.z, d.w * g.w);
    sg += gd.x + gd.y + gd.z + gd.w;
    sgx += gd.x * xh.x + gd.y * xh.y + gd.z * xh.z + gd.w * xh.w;
    if (s == 0) {
      *reinterpret_cast<float4*>(dgb + int64_t(b) * 2 * D + 4 * c) =
          make_float4(d.x * xh.x, d.y * xh.y, d.z * xh.z, d.w * xh.w);
      *reinterpret_cast<float4*>(dgb + int64_t(b) * 2 * D + D + 4 * c) = d;
    }
  }
  const float mg = block_sum(sg, red) / D;
  const float mgx = block_sum(sgx, red) / D;
  const float f = mean_pool ? rstd / N : rstd;
  for (int c = threadIdx.x; c < D4; c += blockDim.x) {
    const float4 d = __ldg(reinterpret_cast<const float4*>(dyb + 4 * c));
    const float4 p = __ldg(reinterpret_cast<const float4*>(pb + 4 * c));
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + 4 * c));
    float4 o;
    o.x = f * (d.x * g.x - mg - (p.x - mean) * rstd * mgx);
    o.y = f * (d.y * g.y - mg - (p.y - mean) * rstd * mgx);
    o.z = f * (d.z * g.z - mg - (p.z - mean) * rstd * mgx);
    o.w = f * (d.w * g.w - mg - (p.w - mean) * rstd * mgx);
    reinterpret_cast<float4*>(drow)[c] = o;
  }
  __syncthreads();
  const int t0 = s * chunk, t1 = min(N, t0 + chunk);
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int t = t0; t < t1; ++t) {
    const bool hot = mean_pool || t == N - 1;
    float4* out = reinterpret_cast<float4*>(dx + (int64_t(b) * N + t) * D);
    for (int c = threadIdx.x; c < D4; c += blockDim.x) __stcs(out + c, hot ? reinterpret_cast<const float4*>(drow)[c] : zero);
  }
}

}  // namespace

// dst[i] += src[i]
__global__ void add_f32_kernel(float* __restrict__ dst, const float* __restrict__ src, int64_t n) {
  pdl_prologue();
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x)
    dst[i] += src[i];
}

int add_f32(float* dst, const float* src, int64_t n, cudaStream_t st) {
  const int threads = 256;
  const int64_t blocks = std::min<int64_t>((n + threads - 1) / threads, int64_t(sm_count()) * 4);
  launch_k(add_f32_kernel, dim3((unsigned)blocks), dim3(threads), 0, st, dst, src, n);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

namespace {

int round8(int c) { return (c + 7) / 8 * 8; }

struct Carve {
  uint8_t* base;
  size_t off = 0;
  template <typename T>
  T* take(size_t n) {
    off = align_up(off, 256);
    T* p = reinterpret_cast<T*>(base + off);
    off += n * sizeof(T);
    return p;
  }
};

struct ClsSaved {
  float *pooled, *mean, *rstd;
  bf16 *xn, *w_b;           // w_b: [Cp, D] bf16 head weight when no registered mirror can serve it
  size_t bytes;
};
ClsSaved cls_saved(void* base, int B, int D, int C) {
  Carve c{reinterpret_cast<uint8_t*>(base)};
  ClsSaved s;
  s.pooled = c.take<float>(size_t(B) * D);
  s.mean = c.take<float>(B);
  s.rstd = c.take<float>(B);
  s.xn = c.take<bf16>(size_t(B) * D);
  s.w_b = C > 0 ? c.take<bf16>(size_t(round8(C)) * D) : nullptr;
  s.bytes = align_up(c.off, 256);
  return s;
}

struct ClsWs {
  float* partial;            // [B, splits, D] token-run sums
  float *logits_p, *bias_p;  // padded width only
  float *dlogits_p, *db_p, *dw_p;
  bf16* dlogits_b;           // [B, Cp]
  float *dxn, *dgb;          // [B, D] gradient of the normalised row, [B, 2D] LayerNorm parameter-gradient partials
  size_t bytes;
};
ClsWs cls_ws(void* base, int B, int N, int D, int C) {
  Carve c{reinterpret_cast<uint8_t*>(base)};
  ClsWs w;
  const int Cp = round8(C);
  const bool pad = C > 0 && Cp != C;
  w.partial = c.take<float>(size_t(B) * pool_splits(B, N) * D);
  w.logits_p = pad ? c.take<float>(size_t(B) * Cp) : nullptr;
  w.bias_p = pad ? c.take<float>(Cp) : nullptr;
  w.dlogits_p = pad ? c.take<float>(size_t(B) * Cp) : nullptr;
  w.db_p = pad ? c.take<float>(Cp) : nullptr;
  w.dw_p = pad ? c.take<float>(size_t(Cp) * D) : nullptr;
  w.dlogits_b = C > 0 ? c.take<bf16>(size_t(B) * Cp) : nullptr;
  w.dxn = C > 0 ? c.take<float>(size_t(B) * D) : nullptr;
  w.dgb = c.take<float>(size_t(B) * 2 * D);
  w.bytes = align_up(c.off, 256);
  return w;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

#define RUN(expr)                   \
  do {                              \
    int _rc = (expr);               \
    if (_rc != MMAE_OK) return _rc; \
  } while (0)

int check_dims(const char* what, int B, int N, int D, int C) {
  MMAE_CHECK(B > 0 && N > 0 && C >= 0, MMAE_ERR_ARG, "%s: bad shape B=%d N=%d C=%d", what, B, N, C);
  MMAE_CHECK(D > 0 && D % 8 == 0 && D <= 8192, MMAE_ERR_UNSUPPORTED, "%s: D=%d must be a multiple of 8, at most 8192",
             what, D);
  return MMAE_OK;
}

}  // namespace
}  // namespace mmae

using namespace mmae;

extern "C" int64_t mmae_clshead_saved_bytes(int B, int N, int D, int C) {
  (void)N;
  return (int64_t)cls_saved(nullptr, B, D, C).bytes;
}
extern "C" int64_t mmae_clshead_workspace_bytes(int B, int N, int D, int C) {
  return (int64_t)cls_ws(nullptr, B, N, D, C).bytes;
}

extern "C" int mmae_clshead_forward(const float* x, int B, int N, int D, int C, int mean_pool, float eps,
                                    const float* norm_w, const float* norm_b, const float* head_w, const float* head_b,
                                    float* out, void* saved, void* ws, void* stream) {
  RUN(check_dims("mmae_clshead_forward", B, N, D, C));
  MMAE_CHECK(x && norm_w && norm_b && out && saved && ws && (C == 0 || (head_w && head_b)), MMAE_ERR_ARG,
             "mmae_clshead_forward: bad args");
  MMAE_CHECK(aligned16(x) && aligned16(norm_w) && aligned16(norm_b) && aligned16(out), MMAE_ERR_ARG,
             "mmae_clshead_forward: tensors must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ClsSaved s = cls_saved(saved, B, D, C);
  ClsWs w = cls_ws(ws, B, N, D, C);
  const int Cp = round8(C);
  const bool pad = C > 0 && Cp != C;
  // pool (multimae/output_adapters.py:349-353) + norm (:355)
  const float* src;
  int64_t sample_stride, part_stride = D;
  int parts;
  float scale;
  if (mean_pool) {
    parts = pool_splits(B, N);
    const int chunk = ceil_div(N, parts);
    launch_k(cls_pool_kernel, dim3(parts, B), dim3(pool_threads(D)), 0, st, x, N, D, chunk, w.partial);
    count_launch();
    MMAE_LAUNCH_OK();
    src = w.partial;
    sample_stride = int64_t(parts) * D;
    scale = 1.0f / N;
  } else {                                   // the global token, appended last (multimae/multimae.py:346-347)
    src = x + int64_t(N - 1) * D;
    sample_stride = int64_t(N) * D;
    parts = 1;
    scale = 1.0f;
  }
  launch_k(cls_pool_ln_kernel, dim3(B), dim3(LN_THREADS), D * sizeof(float), st, src, sample_stride, parts, part_stride,
           scale, D, norm_w, norm_b, eps, s.pooled, s.mean, s.rstd, C > 0 ? s.xn : nullptr, C > 0 ? nullptr : out);
  count_launch();
  MMAE_LAUNCH_OK();
  if (C == 0) return MMAE_OK;                // head = nn.Identity(): the output is the fp32 normalised row
  // head (:355): bf16 operands like the autocast Linear, fp32 accumulation and logits
  const bf16* W = mirror_lookup(head_w);
  if (!pad && W == nullptr) {
    RUN(mmae_cast_f32_to_bf16(head_w, s.w_b, int64_t(C) * D, st));
    W = s.w_b;
  } else if (pad) {                          // zero rows C..Cp-1; a mirror is copied, not read past its tensor
    if (W != nullptr)
      MMAE_CUDA_OK(cudaMemcpyAsync(s.w_b, W, size_t(C) * D * sizeof(bf16), cudaMemcpyDeviceToDevice, st));
    else
      RUN(mmae_cast_f32_to_bf16(head_w, s.w_b, int64_t(C) * D, st));
    MMAE_CUDA_OK(cudaMemsetAsync(s.w_b + size_t(C) * D, 0, size_t(Cp - C) * D * sizeof(bf16), st));
    W = s.w_b;
    MMAE_CUDA_OK(cudaMemsetAsync(w.bias_p, 0, Cp * sizeof(float), st));
    MMAE_CUDA_OK(cudaMemcpyAsync(w.bias_p, head_b, C * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  mmae_gemm_epilogue ep;
  memset(&ep, 0, sizeof(ep));
  ep.alpha = 1.0f;
  ep.bias = pad ? w.bias_p : head_b;
  ep.out_f32 = pad ? w.logits_p : out;
  ep.ld_out_f32 = Cp;
  RUN(mmae_gemm_bf16(s.xn, D, 0, W, D, 0, B, Cp, D, 1, &ep, st));
  if (pad)
    MMAE_CUDA_OK(cudaMemcpy2DAsync(out, C * sizeof(float), w.logits_p, Cp * sizeof(float), C * sizeof(float), B,
                                   cudaMemcpyDeviceToDevice, st));
  return MMAE_OK;
}

extern "C" int mmae_clshead_backward(const float* dout, int B, int N, int D, int C, int mean_pool, const float* norm_w,
                                     const float* head_w, float* d_norm_w, float* d_norm_b, float* d_head_w,
                                     float* d_head_b, float* dx, const void* saved, void* ws, void* stream) {
  RUN(check_dims("mmae_clshead_backward", B, N, D, C));
  MMAE_CHECK(dout && norm_w && d_norm_w && d_norm_b && dx && saved && ws && (C == 0 || (head_w && d_head_w && d_head_b)),
             MMAE_ERR_ARG, "mmae_clshead_backward: bad args");
  MMAE_CHECK(aligned16(dout) && aligned16(dx) && aligned16(norm_w), MMAE_ERR_ARG,
             "mmae_clshead_backward: tensors must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ClsSaved s = cls_saved(const_cast<void*>(saved), B, D, C);
  ClsWs w = cls_ws(ws, B, N, D, C);
  const int Cp = round8(C);
  const bool pad = C > 0 && Cp != C;
  const float* dy = dout;                    // gradient of the normalised row
  if (C > 0) {
    const float* dl = dout;
    if (pad) {
      MMAE_CUDA_OK(cudaMemsetAsync(w.dlogits_p, 0, size_t(B) * Cp * sizeof(float), st));
      MMAE_CUDA_OK(cudaMemcpy2DAsync(w.dlogits_p, Cp * sizeof(float), dout, C * sizeof(float), C * sizeof(float), B,
                                     cudaMemcpyDeviceToDevice, st));
      MMAE_CUDA_OK(cudaMemsetAsync(w.db_p, 0, Cp * sizeof(float), st));
      MMAE_CUDA_OK(cudaMemsetAsync(w.dw_p, 0, size_t(Cp) * D * sizeof(float), st));
      dl = w.dlogits_p;
    }
    RUN(mmae_cast_colsum_f32(dl, Cp, w.dlogits_b, Cp, pad ? w.db_p : d_head_b, B, Cp, st));
    const bf16* W = pad ? nullptr : mirror_lookup(head_w);
    if (W == nullptr) W = s.w_b;             // cast (and padded) by the forward
    mmae_gemm_epilogue ep;
    memset(&ep, 0, sizeof(ep));
    ep.alpha = 1.0f;
    ep.accumulate = 1;                       // dW[Cp, D] += dlogits^T xn
    ep.out_f32 = pad ? w.dw_p : d_head_w;
    ep.ld_out_f32 = D;
    RUN(mmae_gemm_bf16(w.dlogits_b, Cp, 1, s.xn, D, 1, Cp, D, B, 0, &ep, st));
    memset(&ep, 0, sizeof(ep));
    ep.alpha = 1.0f;
    ep.out_f32 = w.dxn;                      // dxn[B, D] = dlogits W
    ep.ld_out_f32 = D;
    RUN(mmae_gemm_bf16(w.dlogits_b, Cp, 0, W, D, 1, B, D, Cp, 1, &ep, st));
    if (pad) {
      RUN(add_f32(d_head_b, w.db_p, C, st));
      RUN(add_f32(d_head_w, w.dw_p, int64_t(C) * D, st));
    }
    dy = w.dxn;
  }
  const int parts = pool_splits(B, N), chunk = ceil_div(N, parts);
  launch_k(cls_head_bwd_kernel, dim3(parts, B), dim3(LN_THREADS), D * sizeof(float), st, dy, s.pooled, s.mean, s.rstd,
           norm_w, N, D, chunk, mean_pool, dx, w.dgb);
  count_launch();
  MMAE_LAUNCH_OK();
  RUN(mmae_cast_colsum_f32(w.dgb, 2 * D, nullptr, 0, d_norm_w, B, D, st));
  RUN(mmae_cast_colsum_f32(w.dgb + D, 2 * D, nullptr, 0, d_norm_b, B, D, st));
  return MMAE_OK;
}
