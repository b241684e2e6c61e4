// LayerNorm forward / backward (fp32 statistics, eps as given), one warp per row, rows kept in registers.
// Replaces nn.LayerNorm(eps=1e-6) at multimae/multimae_utils.py:222,225,230-231 and
// multimae/output_adapters.py:120-122,265-266 (autocast keeps LayerNorm in fp32: SURVEY.md §A.2).
// HBM-bound: fwd reads 4 B/elem, writes 2 B/elem (bf16 operand for the next GEMM) + 8 B/row of statistics.
#include "common.cuh"
#include "../../include/multimae_b200.h"
#include "internal.h"

namespace mmae {
void count_launch();
namespace {

constexpr int LN_WARPS = 8;

// D = NVEC * 128 (each lane owns NVEC float4, strided by 32 lanes)
template <int NVEC, bool DROP>
__global__ void __launch_bounds__(LN_WARPS * 32) ln_fwd_kernel(const float* __restrict__ x, int64_t ldx,
                                                               const bf16* __restrict__ addend, int64_t ldadd,
                                                               float* __restrict__ x_sum, int64_t ldsum,
                                                               const float* __restrict__ gamma,
                                                               const float* __restrict__ beta, bf16* __restrict__ y_bf16,
                                                               int64_t ldy, float* __restrict__ y_f32, int64_t ldyf,
                                                               float* __restrict__ mean_out,
                                                               float* __restrict__ rstd_out,
                                                               const float* __restrict__ add_scale, int rows_per_sample,
                                                               int M, float eps, DropSite drop) {
  pdl_prologue();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * LN_WARPS + warp;
  if (row >= M) return;
  constexpr int D = NVEC * 128;
  const float* xr = x + int64_t(row) * ldx;
  // per-sample factor of the addend (stochastic depth: 0 or 1/keep); 1 when none is given, which leaves x + a exact
  const float sc = add_scale != nullptr ? __ldg(add_scale + row / rows_per_sample) : 1.0f;
  const uint64_t dseed = DROP ? *drop.seed : 0;
  float4 v[NVEC];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NVEC; ++i) {
    const int c = (i * 32 + lane) * 4;
    v[i] = __ldg(reinterpret_cast<const float4*>(xr + c));
    if (addend != nullptr) {   // residual add fused in front of the normalisation: x <- x + bf16 branch output
      const uint2 u = __ldg(reinterpret_cast<const uint2*>(addend + int64_t(row) * ldadd + c));
      const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y);
      if constexpr (DROP) {   // dropout of the branch: per-element factor 0 or 1/(1-p)
        const float4 f = dropout_factor4(drop, dseed, uint64_t(row), c);
        v[i].x += sc * f.x * a.x; v[i].y += sc * f.y * a.y; v[i].z += sc * f.z * b.x; v[i].w += sc * f.w * b.y;
      } else {
        v[i].x += sc * a.x; v[i].y += sc * a.y; v[i].z += sc * b.x; v[i].w += sc * b.y;
      }
      if (x_sum != nullptr) *reinterpret_cast<float4*>(x_sum + int64_t(row) * ldsum + c) = v[i];
    }
    s += v[i].x + v[i].y + v[i].z + v[i].w;
  }
  const float mean = warp_sum(s) * (1.0f / D);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NVEC; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += a * a + b * b + c * c + d * d;
  }
  const float rstd = rsqrtf(warp_sum(q) * (1.0f / D) + eps);
  if (lane == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
#pragma unroll
  for (int i = 0; i < NVEC; ++i) {
    const int c = (i * 32 + lane) * 4;
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + c));
    const float4 b = __ldg(reinterpret_cast<const float4*>(beta + c));
    float4 o;
    o.x = (v[i].x - mean) * rstd * g.x + b.x;
    o.y = (v[i].y - mean) * rstd * g.y + b.y;
    o.z = (v[i].z - mean) * rstd * g.z + b.z;
    o.w = (v[i].w - mean) * rstd * g.w + b.w;
    if (y_bf16) {
      uint2 p;
      p.x = pack_bf16x2(o.x, o.y);
      p.y = pack_bf16x2(o.z, o.w);
      *reinterpret_cast<uint2*>(y_bf16 + int64_t(row) * ldy + c) = p;
    }
    if (y_f32) *reinterpret_cast<float4*>(y_f32 + int64_t(row) * ldyf + c) = o;
  }
}

// Backward.  dx_out = dx_resid (optional) + rstd * (g - mean(g) - xhat * mean(g*xhat)),  g = dy * gamma.
// dgamma/dbeta: per-lane register partials over the block's rows -> smem reduce over warps -> one partial row per block.
//
// Persistent: the grid is one wave (blocks = SMs x resident blocks), warps stride over the rows, so there is no partial
// last wave (12672 rows in 64-row blocks are 198 blocks: on 132 SMs half of the time would run at half occupancy) and the
// column-sum atomics drop to one set per resident block.  The next row's x / dy loads are issued before the current
// row's reductions (the per-lane column accumulators cap residency at 8 warps per SM for D = 768, so a warp has to
// carry its own memory-level parallelism).
template <int NVEC, bool DY_BF16>
struct LnRow {
  float4 x[NVEC];
  float4 d[DY_BF16 ? (NVEC + 1) / 2 : NVEC];   // bf16 dy stays packed: 8 bytes per float4 slot
};

template <int NVEC, bool DY_BF16>
__device__ __forceinline__ void ln_row_load(LnRow<NVEC, DY_BF16>& r, const void* dy_, int64_t lddy, const float* x,
                                            int64_t ldx, int row, int lane) {
#pragma unroll
  for (int i = 0; i < NVEC; ++i) {
    const int c = (i * 32 + lane) * 4;
    r.x[i] = __ldg(reinterpret_cast<const float4*>(x + int64_t(row) * ldx + c));
    if constexpr (DY_BF16) {
      const uint2 u = __ldg(reinterpret_cast<const uint2*>(reinterpret_cast<const bf16*>(dy_) + int64_t(row) * lddy + c));
      float* slot = reinterpret_cast<float*>(&r.d[i >> 1]) + (i & 1) * 2;
      slot[0] = __uint_as_float(u.x);
      slot[1] = __uint_as_float(u.y);
    } else {
      r.d[i] = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(dy_) + int64_t(row) * lddy + c));
    }
  }
}

template <int NVEC, bool DY_BF16>
__device__ __forceinline__ float4 ln_row_dy(const LnRow<NVEC, DY_BF16>& r, int i) {
  if constexpr (DY_BF16) {
    const float* slot = reinterpret_cast<const float*>(&r.d[i >> 1]) + (i & 1) * 2;
    const float2 a = unpack_bf16x2(__float_as_uint(slot[0])), b = unpack_bf16x2(__float_as_uint(slot[1]));
    return make_float4(a.x, a.y, b.x, b.y);
  } else {
    return r.d[i];
  }
}

template <int NVEC, bool DY_BF16, bool DROP>
__global__ void __launch_bounds__(LN_WARPS * 32) ln_bwd_kernel(const void* __restrict__ dy_, int64_t lddy,
                                                               const float* __restrict__ x, int64_t ldx,
                                                               const float* __restrict__ mean_in,
                                                               const float* __restrict__ rstd_in,
                                                               const float* __restrict__ gamma,
                                                               const float* __restrict__ dx_resid, int64_t ldr,
                                                               float* __restrict__ dx, int64_t lddx,
                                                               float* __restrict__ partial, bool want_colsum,
                                                               bf16* __restrict__ dx_bf16, int64_t lddxb,
                                                               const float* __restrict__ out_scale, int rows_per_sample,
                                                               int M, DropSite drop) {
  pdl_prologue();
  constexpr int D = NVEC * 128;
  __shared__ float4 red[LN_WARPS][32];
  __shared__ float4 sgamma[NVEC * 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < NVEC * 32; i += LN_WARPS * 32) sgamma[i] = __ldg(reinterpret_cast<const float4*>(gamma) + i);
  __syncthreads();
  float4 dg[NVEC], db[NVEC], cs[NVEC];
#pragma unroll
  for (int i = 0; i < NVEC; ++i) {
    dg[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    db[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    cs[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const int row_stride = gridDim.x * LN_WARPS;
  int row = blockIdx.x * LN_WARPS + warp;
  const uint64_t dseed = DROP ? *drop.seed : 0;
  LnRow<NVEC, DY_BF16> cur, nxt;
  float mean = 0.f, rstd = 0.f, mean_n = 0.f, rstd_n = 0.f;
  if (row < M) {
    ln_row_load(cur, dy_, lddy, x, ldx, row, lane);
    mean = __ldg(mean_in + row);
    rstd = __ldg(rstd_in + row);
  }
  for (; row < M; row += row_stride) {
    const int row_n = row + row_stride;
    if (row_n < M) {   // next row's loads fly while this row is reduced and written
      ln_row_load(nxt, dy_, lddy, x, ldx, row_n, lane);
      mean_n = __ldg(mean_in + row_n);
      rstd_n = __ldg(rstd_in + row_n);
    }
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NVEC; ++i) {
      const float4 d = ln_row_dy(cur, i);
      const float4 gm = sgamma[i * 32 + lane];
      const float4 xh = make_float4((cur.x[i].x - mean) * rstd, (cur.x[i].y - mean) * rstd, (cur.x[i].z - mean) * rstd,
                                    (cur.x[i].w - mean) * rstd);
      const float4 g = make_float4(d.x * gm.x, d.y * gm.y, d.z * gm.z, d.w * gm.w);
      s1 += g.x + g.y + g.z + g.w;
      s2 += g.x * xh.x + g.y * xh.y + g.z * xh.z + g.w * xh.w;
      dg[i].x += d.x * xh.x; dg[i].y += d.y * xh.y; dg[i].z += d.z * xh.z; dg[i].w += d.w * xh.w;
      db[i].x += d.x; db[i].y += d.y; db[i].z += d.z; db[i].w += d.w;
    }
    const float c1 = warp_sum(s1) * (1.0f / D), c2 = warp_sum(s2) * (1.0f / D);
    // per-sample factor of the bf16 copy and its column sums (the gradient entering a drop-path branch); dx stays unscaled
    const float sc = out_scale != nullptr ? __ldg(out_scale + row / rows_per_sample) : 1.0f;
#pragma unroll
    for (int i = 0; i < NVEC; ++i) {
      const int c = (i * 32 + lane) * 4;
      const float4 d = ln_row_dy(cur, i);
      const float4 gm = sgamma[i * 32 + lane];
      const float4 xh = make_float4((cur.x[i].x - mean) * rstd, (cur.x[i].y - mean) * rstd, (cur.x[i].z - mean) * rstd,
                                    (cur.x[i].w - mean) * rstd);
      float4 o;
      o.x = rstd * (d.x * gm.x - c1 - xh.x * c2);
      o.y = rstd * (d.y * gm.y - c1 - xh.y * c2);
      o.z = rstd * (d.z * gm.z - c1 - xh.z * c2);
      o.w = rstd * (d.w * gm.w - c1 - xh.w * c2);
      if (dx_resid) {
        const float4 r = __ldg(reinterpret_cast<const float4*>(dx_resid + int64_t(row) * ldr + c));
        o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
      }
      *reinterpret_cast<float4*>(dx + int64_t(row) * lddx + c) = o;
      if (dx_bf16 != nullptr) {   // bf16 copy of dx (next GEMM operand) and its column sums (next bias gradient)
        uint2 pk;
        float4 os = make_float4(sc * o.x, sc * o.y, sc * o.z, sc * o.w);
        if constexpr (DROP) {   // the gradient entering a dropout branch: the forward's mask and 1/(1-p)
          const float4 f = dropout_factor4(drop, dseed, uint64_t(row), c);
          os = make_float4(os.x * f.x, os.y * f.y, os.z * f.z, os.w * f.w);
        }
        pk.x = pack_bf16x2(os.x, os.y);
        pk.y = pack_bf16x2(os.z, os.w);
        *reinterpret_cast<uint2*>(dx_bf16 + int64_t(row) * lddxb + c) = pk;
        cs[i].x += os.x; cs[i].y += os.y; cs[i].z += os.z; cs[i].w += os.w;
      }
    }
    cur = nxt;
    mean = mean_n;
    rstd = rstd_n;
  }
  // column reductions across the block's warps -> this block's row of partial sums [dgamma | dbeta | colsum(dx)], added up
  // by colred_finalize (no atomics: blocks x 3D scalar atomics on a few cache lines cost more than the streaming pass)
#pragma unroll
  for (int pass = 0; pass < 3; ++pass) {
    if (pass == 2 && !want_colsum) continue;
    float* dst = partial + (int64_t(blockIdx.x) * 3 + pass) * D;
#pragma unroll
    for (int i = 0; i < NVEC; ++i) {
      __syncthreads();
      red[warp][lane] = pass == 0 ? dg[i] : (pass == 1 ? db[i] : cs[i]);
      __syncthreads();
      if (warp == 0) {
        float4 a = red[0][lane];
#pragma unroll
        for (int w = 1; w < LN_WARPS; ++w) {
          const float4 o = red[w][lane];
          a.x += o.x; a.y += o.y; a.z += o.z; a.w += o.w;
        }
        const int c = (i * 32 + lane) * 4;
        *reinterpret_cast<float4*>(dst + c) = a;
      }
    }
  }
}

}  // namespace
}  // namespace mmae

using namespace mmae;

static int ln_forward_impl(const float* x, int64_t ldx, const bf16* addend, int64_t ldadd, float* x_sum, int64_t ldsum,
                           const float* gamma, const float* beta, void* y_bf16, int64_t ldy, float* y_f32, int64_t ldyf,
                           float* mean, float* rstd, const float* add_scale, int rows_per_sample, int M, int D, float eps,
                           void* stream, DropSite drop = DropSite()) {
  MMAE_CHECK(x && gamma && beta && (y_bf16 || y_f32) && M > 0, MMAE_ERR_ARG, "mmae_layernorm_forward: bad args");
  MMAE_CHECK(!add_scale || (addend && rows_per_sample > 0 && M % rows_per_sample == 0), MMAE_ERR_ARG,
             "mmae_add_layernorm_forward: a row scale needs an addend and rows-per-sample dividing M=%d", M);
  MMAE_CHECK(D % 128 == 0 && D <= 1024 && ldx % 4 == 0 && ldy % 4 == 0 && ldyf % 4 == 0, MMAE_ERR_UNSUPPORTED,
             "mmae_layernorm_forward: D=%d must be a multiple of 128 and <= 1024", D);
  dim3 grid(ceil_div(M, LN_WARPS)), block(LN_WARPS * 32);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  bf16* yb = reinterpret_cast<bf16*>(y_bf16);
#define LN_CASE(NV)                                                                                                         \
  case NV:                                                                                                                  \
    launch_k(drop.seed ? ln_fwd_kernel<NV, true> : ln_fwd_kernel<NV, false>, grid, block, 0, st, x, ldx, addend, ldadd, x_sum, \
             ldsum, gamma, beta, yb, ldy, y_f32, ldyf, mean, rstd, add_scale, rows_per_sample, M, eps, drop);                  \
    break;
  switch (D / 128) {
    LN_CASE(1) LN_CASE(2) LN_CASE(3) LN_CASE(4) LN_CASE(5) LN_CASE(6) LN_CASE(7) LN_CASE(8)
    default: MMAE_CHECK(false, MMAE_ERR_UNSUPPORTED, "mmae_layernorm_forward: unsupported D=%d", D);
  }
#undef LN_CASE
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

extern "C" int mmae_layernorm_forward(const float* x, int64_t ldx, const float* gamma, const float* beta, void* y_bf16,
                                      int64_t ldy, float* y_f32, int64_t ldyf, float* mean, float* rstd, int M, int D,
                                      float eps, void* stream) {
  return ln_forward_impl(x, ldx, nullptr, 0, nullptr, 0, gamma, beta, y_bf16, ldy, y_f32, ldyf, mean, rstd, nullptr, 1, M, D,
                         eps, stream);
}

// x_sum = x + addend (fp32, written when non-NULL), then LayerNorm of x_sum: the residual add of
// `x = x + attn(...)` (multimae/multimae_utils.py:230) fused in front of the next norm (:231)
// x_sum = x + row_scale[row / rows_per_sample] * addend: the same with a per-sample factor on the branch (stochastic depth)
int mmae::add_layernorm_forward_scaled(const float* x, int64_t ldx, const bf16* addend, int64_t ldadd, const float* row_scale,
                                       int rows_per_sample, float* x_sum, int64_t ldsum, const float* gamma, const float* beta,
                                       bf16* y_bf16, int64_t ldy, float* mean, float* rstd, int M, int D, float eps,
                                       void* stream, DropSite drop) {
  MMAE_CHECK(addend && ldadd % 4 == 0 && (!x_sum || ldsum % 4 == 0), MMAE_ERR_ARG, "mmae_add_layernorm_forward: bad args");
  return ln_forward_impl(x, ldx, addend, ldadd, x_sum, ldsum, gamma, beta, y_bf16, ldy, nullptr, 0, mean, rstd, row_scale,
                         rows_per_sample, M, D, eps, stream, drop);
}

extern "C" int mmae_add_layernorm_forward(const float* x, int64_t ldx, const void* addend_bf16, int64_t ldadd, float* x_sum,
                                          int64_t ldsum, const float* gamma, const float* beta, void* y_bf16, int64_t ldy,
                                          float* mean, float* rstd, int M, int D, float eps, void* stream) {
  return add_layernorm_forward_scaled(x, ldx, reinterpret_cast<const bf16*>(addend_bf16), ldadd, nullptr, 1, x_sum, ldsum,
                                      gamma, beta, reinterpret_cast<bf16*>(y_bf16), ldy, mean, rstd, M, D, eps, stream);
}

static int ln_backward_impl(const void* dy, int dy_is_bf16, int64_t lddy, const float* x, int64_t ldx, const float* mean,
                            const float* rstd, const float* gamma, const float* dx_resid, int64_t ldr, float* dx,
                            int64_t lddx, float* dgamma, float* dbeta, bf16* dx_bf16, int64_t lddxb, float* dx_colsum,
                            const float* out_scale, int rows_per_sample, int M, int D, void* stream,
                            DropSite drop = DropSite()) {
  MMAE_CHECK(dy && x && mean && rstd && gamma && dx && M > 0, MMAE_ERR_ARG, "mmae_layernorm_backward: bad args");
  MMAE_CHECK(!out_scale || (dx_bf16 && rows_per_sample > 0 && M % rows_per_sample == 0), MMAE_ERR_ARG,
             "mmae_layernorm_backward_ex: a row scale needs the bf16 output and rows-per-sample dividing M=%d", M);
  MMAE_CHECK(!drop.seed || dx_bf16, MMAE_ERR_ARG, "mmae_layernorm_backward_ex: a dropout mask needs the bf16 output");
  MMAE_CHECK(D % 128 == 0 && D <= 1024 && ldx % 4 == 0 && lddy % 4 == 0 && lddx % 4 == 0 && ldr % 4 == 0,
             MMAE_ERR_UNSUPPORTED, "mmae_layernorm_backward: D=%d must be a multiple of 128 and <= 1024", D);
  // one wave: resident blocks per SM follow from the register footprint of the per-lane column accumulators
  static const int tune = []() {
    const char* e = getenv("MMAE_TUNE_LNB");
    return e ? atoi(e) : 0;
  }();
  int per_sm = D <= 256 ? 3 : (D <= 384 ? 2 : 1);
  if (tune > 0) per_sm = std::min(per_sm, tune);
  dim3 grid(std::min(ceil_div(M, LN_WARPS), sm_count() * per_sm)), block(LN_WARPS * 32);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  MMAE_CHECK(dgamma && dbeta, MMAE_ERR_ARG, "mmae_layernorm_backward: dgamma / dbeta are required");
  float* partial = colred_scratch(size_t(grid.x) * 3 * D, st);
  if (!partial) return MMAE_ERR_CUDA;
#define LNB_CASE(NV)                                                                                              \
  case NV:                                                                                                        \
    launch_k(dy_is_bf16 ? (drop.seed ? ln_bwd_kernel<NV, true, true> : ln_bwd_kernel<NV, true, false>)             \
                        : (drop.seed ? ln_bwd_kernel<NV, false, true> : ln_bwd_kernel<NV, false, false>),          \
             grid, block, 0, st, dy, lddy, x, ldx, mean, rstd, gamma, dx_resid, ldr, dx, lddx, partial,           \
             dx_colsum != nullptr, dx_bf16, lddxb, out_scale, rows_per_sample, M, drop);                          \
    break;
  switch (D / 128) {
    LNB_CASE(1) LNB_CASE(2) LNB_CASE(3) LNB_CASE(4) LNB_CASE(5) LNB_CASE(6) LNB_CASE(7) LNB_CASE(8)
    default: MMAE_CHECK(false, MMAE_ERR_UNSUPPORTED, "mmae_layernorm_backward: unsupported D=%d", D);
  }
#undef LNB_CASE
  count_launch();
  MMAE_LAUNCH_OK();
  // partial row = [dgamma | dbeta | colsum]; without a colsum destination only the first two segments are summed
  return colred_finalize(partial, grid.x, 3 * D, D, dgamma, dbeta, dx_colsum, st);
}

extern "C" int mmae_layernorm_backward(const void* dy, int dy_is_bf16, int64_t lddy, const float* x, int64_t ldx,
                                       const float* mean, const float* rstd, const float* gamma, const float* dx_resid,
                                       int64_t ldr, float* dx, int64_t lddx, float* dgamma, float* dbeta, int M, int D,
                                       void* stream) {
  return ln_backward_impl(dy, dy_is_bf16, lddy, x, ldx, mean, rstd, gamma, dx_resid, ldr, dx, lddx, dgamma, dbeta, nullptr, 0,
                          nullptr, nullptr, 1, M, D, stream);
}

// the _ex form with bf16(dx) and its column sums multiplied by row_scale[row / rows_per_sample] (the fp32 dx is not): the
// gradient entering a branch that stochastic depth scaled per sample, while dx itself continues down the residual path
int mmae::layernorm_backward_ex_scaled(const void* dy, int dy_is_bf16, int64_t lddy, const float* x, int64_t ldx,
                                       const float* mean, const float* rstd, const float* gamma, const float* dx_resid,
                                       int64_t ldr, float* dx, int64_t lddx, float* dgamma, float* dbeta, bf16* dx_bf16,
                                       int64_t lddxb, float* dx_colsum, const float* row_scale, int rows_per_sample, int M,
                                       int D, void* stream, DropSite drop) {
  MMAE_CHECK(!dx_bf16 || lddxb % 4 == 0, MMAE_ERR_ARG, "mmae_layernorm_backward_ex: bad bf16 leading dimension");
  return ln_backward_impl(dy, dy_is_bf16, lddy, x, ldx, mean, rstd, gamma, dx_resid, ldr, dx, lddx, dgamma, dbeta, dx_bf16,
                          lddxb, dx_colsum, row_scale, rows_per_sample, M, D, stream, drop);
}

// same, additionally emitting bf16(dx) and colsum += sum_rows(dx): the operand and bias gradient of the next Linear backward
extern "C" int mmae_layernorm_backward_ex(const void* dy, int dy_is_bf16, int64_t lddy, const float* x, int64_t ldx,
                                          const float* mean, const float* rstd, const float* gamma, const float* dx_resid,
                                          int64_t ldr, float* dx, int64_t lddx, float* dgamma, float* dbeta, void* dx_bf16,
                                          int64_t lddxb, float* dx_colsum, int M, int D, void* stream) {
  return layernorm_backward_ex_scaled(dy, dy_is_bf16, lddy, x, ldx, mean, rstd, gamma, dx_resid, ldr, dx, lddx, dgamma, dbeta,
                                      reinterpret_cast<bf16*>(dx_bf16), lddxb, dx_colsum, nullptr, 1, M, D, stream);
}
