// fp32-tier primitives for `fp32_output_adapters` (multimae/multimae.py:367-377: the listed output adapters run outside
// autocast, i.e. every Linear / softmax / GELU of theirs in fp32 - the shipped pre-training config lists ['semseg'],
// cfgs/pretrain/multimae-b_98_rgb+-depth-semseg_1600e.yaml:28).
//
//   * fp32-accurate Linear on the bf16 tensor cores: x = x_hi + x_lo, W = W_hi + W_lo (two bf16 pieces each, 16 mantissa
//     bits) and  x W^T ~= x_hi W_hi^T + x_hi W_lo^T + x_lo W_hi^T  is ONE wgmma GEMM over a K-concatenated operand pair
//     A' = [x_hi | x_hi | x_lo], B' = [W_hi | W_lo | W_hi] (fp32 accumulation; the dropped x_lo W_lo^T term and the
//     split residuals are ~2^-16 relative).  dgrad / wgrad use the same trick with row-stacked (MN-major) operands.
//   * attention, GELU in plain fp32 CUDA-core kernels (decoder sizes: 196 x <= 196 keys, head_dim 32 - 5 GFLOP per call).
#include <cstdlib>

#include "common.cuh"
#include "../../include/multimae_b200.h"
#include "internal.h"

namespace mmae {
void count_launch();
namespace {

// debugging aid: MMAE_F32_NOPDL bit mask launches the fp32-tier kernels fully serialised (1 split, 2 attention, 4 gelu)
int g_f32_nopdl = []() {
  const char* e = getenv("MMAE_F32_NOPDL");
  return e ? atoi(e) : 0;
}();
template <typename... KArgs, typename... Args>
cudaError_t launch_f32(int klass, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  if (g_f32_nopdl & klass) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
  }
  return launch_k(kernel, grid, block, smem, st, static_cast<Args&&>(args)...);
}

// dst pieces of src [R, C] (fp32): slot s in {0,1,2} holds the low piece if bit s of `pat` is set, else the high piece.
// stack = 0: slots are column blocks of a [R, 3C] matrix; stack = 1: row blocks of a [3R, C] matrix.
__global__ void __launch_bounds__(256) split3_kernel(const float* __restrict__ src, int64_t ld, int R, int C,
                                                     bf16* __restrict__ dst, int64_t ld_dst, int pat, int stack) {
  pdl_prologue();
  const int c4 = C >> 2;
  const int64_t total = int64_t(R) * c4;
  for (int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += int64_t(gridDim.x) * blockDim.x) {
    const int r = int(idx / c4), c = int(idx - int64_t(r) * c4) * 4;
    const float4 v = __ldg(reinterpret_cast<const float4*>(src + int64_t(r) * ld + c));
    const bf16 h0 = __float2bfloat16_rn(v.x), h1 = __float2bfloat16_rn(v.y), h2 = __float2bfloat16_rn(v.z), h3 = __float2bfloat16_rn(v.w);
    uint2 hi, lo;
    hi.x = pack_bf16x2(__bfloat162float(h0), __bfloat162float(h1));
    hi.y = pack_bf16x2(__bfloat162float(h2), __bfloat162float(h3));
    lo.x = pack_bf16x2(v.x - __bfloat162float(h0), v.y - __bfloat162float(h1));
    lo.y = pack_bf16x2(v.z - __bfloat162float(h2), v.w - __bfloat162float(h3));
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      const uint2 val = (pat >> s) & 1 ? lo : hi;
      bf16* d = stack ? dst + (int64_t(s) * R + r) * ld_dst + c : dst + int64_t(r) * ld_dst + int64_t(s) * C + c;
      *reinterpret_cast<uint2*>(d) = val;
    }
  }
}

int launch_split3(const float* src, int64_t ld, int R, int C, bf16* dst, int64_t ld_dst, int pat, int stack, cudaStream_t st) {
  const int64_t total = int64_t(R) * (C / 4);
  const unsigned blocks = (unsigned)std::min<int64_t>((total + 255) / 256, int64_t(sm_count()) * 16);
  launch_f32(1, split3_kernel, std::max(1u, blocks), 256, 0, st, src, ld, R, C, dst, ld_dst, pat, stack);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

constexpr int PAT_A = 4;   // (hi, hi, lo)
constexpr int PAT_B = 2;   // (hi, lo, hi)

__global__ void __launch_bounds__(256) gelu_f32_kernel(const float* __restrict__ z, float* __restrict__ io, int64_t n, int backward) {
  pdl_prologue();
  const int64_t stride = int64_t(gridDim.x) * blockDim.x * 4;
  for (int64_t i = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) * 4; i < n; i += stride) {
    const float4 a = *reinterpret_cast<const float4*>(z + i);
    float4 o;
    const float* av = reinterpret_cast<const float*>(&a);
    float* ov = reinterpret_cast<float*>(&o);
    if (backward) o = *reinterpret_cast<const float4*>(io + i);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float x = av[k];
      const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752440f));
      if (backward)
        ov[k] *= cdf + x * 0.39894228040143267794f * expf(-0.5f * x * x);
      else
        ov[k] = x * cdf;
    }
    *reinterpret_cast<float4*>(io + i) = o;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// fp32 attention (CUDA cores).  One thread per query (forward, dQ) or per key (dK / dV); the other side is streamed through
// shared memory in chunks of 64 rows.  q/k/v/o views: row-major [B*N, ld], head h = columns [h*DH, (h+1)*DH).
// Inputs are read with plain (coherent) loads and without __restrict__: these kernels start with loads of what the
// PREVIOUS kernel wrote, and under programmatic dependent launch a non-coherent load (ld.global.nc / __ldg: "read-only for
// the lifetime of the kernel") is not ordered behind griddepcontrol.wait - measured: wrong gradients with PDL on, exact
// with the attention kernels launched serialised.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int FA_ROWS = 128, FA_CHUNK = 64;

template <int DH>
__device__ __forceinline__ void fa_load_chunk(float (*dst)[DH], const float* src, int64_t ld, int row0, int nrows_total) {
  for (int i = threadIdx.x; i < FA_CHUNK * (DH / 4); i += FA_ROWS) {
    const int r = i / (DH / 4), c = (i % (DH / 4)) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row0 + r < nrows_total) v = (*reinterpret_cast<const float4*>(src + int64_t(row0 + r) * ld + c));
    *reinterpret_cast<float4*>(&dst[r][c]) = v;
  }
}

template <int DH>
__global__ void __launch_bounds__(FA_ROWS) attn_f32_fwd_kernel(const float* Q, int64_t ldq, const float* K,
                                                               int64_t ldk, const float* V, int64_t ldv,
                                                               float* O, int64_t ldo, float* lse,
                                                               int Nq, int Nk, int H, float scale) {
  pdl_prologue();
  __shared__ __align__(16) float Ks[FA_CHUNK][DH], Vs[FA_CHUNK][DH];
  const int h = blockIdx.y, b = blockIdx.z;
  const int qi = blockIdx.x * FA_ROWS + threadIdx.x;
  const bool ok = qi < Nq;
  const float* Kb = K + int64_t(b) * Nk * ldk + h * DH;
  const float* Vb = V + int64_t(b) * Nk * ldv + h * DH;
  float q[DH], acc[DH];
#pragma unroll
  for (int d = 0; d < DH; ++d) {
    q[d] = ok ? *(Q + (int64_t(b) * Nq + qi) * ldq + h * DH + d) * scale : 0.f;
    acc[d] = 0.f;
  }
  float m = -INFINITY, l = 0.f;
  for (int k0 = 0; k0 < Nk; k0 += FA_CHUNK) {
    __syncthreads();
    fa_load_chunk<DH>(Ks, Kb, ldk, k0, Nk);
    fa_load_chunk<DH>(Vs, Vb, ldv, k0, Nk);
    __syncthreads();
    const int nj = min(FA_CHUNK, Nk - k0);
    for (int j = 0; j < nj; ++j) {
      float s = 0.f;
#pragma unroll
      for (int d = 0; d < DH; ++d) s = fmaf(q[d], Ks[j][d], s);
      if (s > m) {                       // rare after the first few keys: rescale the running sums
        const float corr = expf(m - s);
        l *= corr;
#pragma unroll
        for (int d = 0; d < DH; ++d) acc[d] *= corr;
        m = s;
      }
      const float pj = expf(s - m);
      l += pj;
#pragma unroll
      for (int d = 0; d < DH; ++d) acc[d] = fmaf(pj, Vs[j][d], acc[d]);
    }
  }
  if (ok) {
    const float inv = 1.0f / l;
    float* o = O + (int64_t(b) * Nq + qi) * ldo + h * DH;
#pragma unroll
    for (int d = 0; d < DH; ++d) o[d] = acc[d] * inv;
    lse[(int64_t(b) * H + h) * Nq + qi] = m + logf(l);
  }
}

// dQ: thread = query.  Also writes delta[b,h,q] = sum_d dO O for the dK / dV kernel.
template <int DH>
__global__ void __launch_bounds__(FA_ROWS) attn_f32_bwd_dq_kernel(const float* Q, int64_t ldq, const float* K,
                                                                  int64_t ldk, const float* V, int64_t ldv,
                                                                  const float* O, int64_t ldo,
                                                                  const float* dO, int64_t lddo,
                                                                  const float* lse, float* delta,
                                                                  float* dQ, int64_t lddq, int Nq, int Nk, int H,
                                                                  float scale) {
  pdl_prologue();
  __shared__ __align__(16) float Ks[FA_CHUNK][DH], Vs[FA_CHUNK][DH];
  const int h = blockIdx.y, b = blockIdx.z;
  const int qi = blockIdx.x * FA_ROWS + threadIdx.x;
  const bool ok = qi < Nq;
  const float* Kb = K + int64_t(b) * Nk * ldk + h * DH;
  const float* Vb = V + int64_t(b) * Nk * ldv + h * DH;
  float q[DH], g[DH], dq[DH];
  float del = 0.f;
#pragma unroll
  for (int d = 0; d < DH; ++d) {
    q[d] = ok ? *(Q + (int64_t(b) * Nq + qi) * ldq + h * DH + d) * scale : 0.f;
    g[d] = ok ? *(dO + (int64_t(b) * Nq + qi) * lddo + h * DH + d) : 0.f;
    const float o = ok ? *(O + (int64_t(b) * Nq + qi) * ldo + h * DH + d) : 0.f;
    del = fmaf(g[d], o, del);
    dq[d] = 0.f;
  }
  const float L = ok ? lse[(int64_t(b) * H + h) * Nq + qi] : 0.f;
  if (ok) delta[(int64_t(b) * H + h) * Nq + qi] = del;
  for (int k0 = 0; k0 < Nk; k0 += FA_CHUNK) {
    __syncthreads();
    fa_load_chunk<DH>(Ks, Kb, ldk, k0, Nk);
    fa_load_chunk<DH>(Vs, Vb, ldv, k0, Nk);
    __syncthreads();
    const int nj = min(FA_CHUNK, Nk - k0);
    for (int j = 0; j < nj; ++j) {
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int d = 0; d < DH; ++d) {
        s = fmaf(q[d], Ks[j][d], s);
        dp = fmaf(g[d], Vs[j][d], dp);
      }
      const float ds = expf(s - L) * (dp - del);
#pragma unroll
      for (int d = 0; d < DH; ++d) dq[d] = fmaf(ds, Ks[j][d], dq[d]);
    }
  }
  if (ok) {
    float* o = dQ + (int64_t(b) * Nq + qi) * lddq + h * DH;
#pragma unroll
    for (int d = 0; d < DH; ++d) o[d] = dq[d] * scale;
  }
}

// dK, dV: thread = key; queries (with dO, lse, delta) streamed in chunks
template <int DH>
__global__ void __launch_bounds__(FA_ROWS) attn_f32_bwd_dkv_kernel(const float* Q, int64_t ldq, const float* K,
                                                                   int64_t ldk, const float* V, int64_t ldv,
                                                                   const float* dO, int64_t lddo,
                                                                   const float* lse, const float* delta,
                                                                   float* dK, int64_t lddk, float* dV,
                                                                   int64_t lddv, int Nq, int Nk, int H, float scale) {
  pdl_prologue();
  __shared__ __align__(16) float Qs[FA_CHUNK][DH], Gs[FA_CHUNK][DH];
  __shared__ float Ls[FA_CHUNK], Ds[FA_CHUNK];
  const int h = blockIdx.y, b = blockIdx.z;
  const int kj = blockIdx.x * FA_ROWS + threadIdx.x;
  const bool ok = kj < Nk;
  const float* Qb = Q + int64_t(b) * Nq * ldq + h * DH;
  const float* Gb = dO + int64_t(b) * Nq * lddo + h * DH;
  float k[DH], v[DH], dk[DH], dv[DH];
#pragma unroll
  for (int d = 0; d < DH; ++d) {
    k[d] = ok ? *(K + (int64_t(b) * Nk + kj) * ldk + h * DH + d) * scale : 0.f;
    v[d] = ok ? *(V + (int64_t(b) * Nk + kj) * ldv + h * DH + d) : 0.f;
    dk[d] = dv[d] = 0.f;
  }
  for (int q0 = 0; q0 < Nq; q0 += FA_CHUNK) {
    __syncthreads();
    fa_load_chunk<DH>(Qs, Qb, ldq, q0, Nq);
    fa_load_chunk<DH>(Gs, Gb, lddo, q0, Nq);
    if (threadIdx.x < FA_CHUNK) {
      const int qi = q0 + threadIdx.x;
      Ls[threadIdx.x] = qi < Nq ? lse[(int64_t(b) * H + h) * Nq + qi] : INFINITY;
      Ds[threadIdx.x] = qi < Nq ? delta[(int64_t(b) * H + h) * Nq + qi] : 0.f;
    }
    __syncthreads();
    const int ni = min(FA_CHUNK, Nq - q0);
    for (int i = 0; i < ni; ++i) {
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int d = 0; d < DH; ++d) {
        s = fmaf(Qs[i][d], k[d], s);
        dp = fmaf(Gs[i][d], v[d], dp);
      }
      const float pij = expf(s - Ls[i]);
      const float ds = pij * (dp - Ds[i]);
#pragma unroll
      for (int d = 0; d < DH; ++d) {
        dv[d] = fmaf(pij, Gs[i][d], dv[d]);
        dk[d] = fmaf(ds, Qs[i][d], dk[d]);
      }
    }
  }
  if (ok) {
    float* ok_ = dK + (int64_t(b) * Nk + kj) * lddk + h * DH;
    float* ov = dV + (int64_t(b) * Nk + kj) * lddv + h * DH;
#pragma unroll
    for (int d = 0; d < DH; ++d) {
      ok_[d] = dk[d] * scale;
      ov[d] = dv[d];
    }
  }
}

}  // namespace

// y[M,N] = x[M,K] W[N,K]^T (+ bias) (+ residual[M,N]) with fp32-level accuracy; wsA >= 3*M*K bf16, wsB >= 3*N*K bf16
int linear_f32x3_forward(const float* x, const float* W, const float* bias, const float* resid, float* y, int M, int N, int K,
                         bf16* wsA, bf16* wsB, void* st) {
  cudaStream_t cst = reinterpret_cast<cudaStream_t>(st);
  int rc;
  if ((rc = launch_split3(x, K, M, K, wsA, 3 * int64_t(K), PAT_A, 0, cst))) return rc;
  if ((rc = launch_split3(W, K, N, K, wsB, 3 * int64_t(K), PAT_B, 0, cst))) return rc;
  mmae_gemm_epilogue ep;
  memset(&ep, 0, sizeof(ep));
  ep.alpha = 1.0f;
  ep.bias = bias;
  ep.residual = resid;
  ep.ld_residual = N;
  ep.out_f32 = y;
  ep.ld_out_f32 = N;
  return mmae_gemm_bf16(wsA, 3 * int64_t(K), 0, wsB, 3 * int64_t(K), 0, M, N, 3 * K, 1, &ep, st);
}

// dx[M,K] (+)= dy[M,N] W[N,K]; wsA >= 3*M*N, wsB >= 3*N*K
int linear_f32x3_dgrad(const float* dy, const float* W, float* dx, int M, int N, int K, int accumulate, bf16* wsA, bf16* wsB,
                       void* st) {
  cudaStream_t cst = reinterpret_cast<cudaStream_t>(st);
  int rc;
  if ((rc = launch_split3(dy, N, M, N, wsA, 3 * int64_t(N), PAT_A, 0, cst))) return rc;
  if ((rc = launch_split3(W, K, N, K, wsB, K, PAT_B, 1, cst))) return rc;      // [3N, K]: K-dim rows, MN-major B
  mmae_gemm_epilogue ep;
  memset(&ep, 0, sizeof(ep));
  ep.alpha = 1.0f;
  ep.accumulate = accumulate;
  ep.out_f32 = dx;
  ep.ld_out_f32 = K;
  return mmae_gemm_bf16(wsA, 3 * int64_t(N), 0, wsB, K, 1, M, K, 3 * N, 1, &ep, st);
}

// dW[N,K] += dy[M,N]^T x[M,K]; db[N] += colsum(dy) when db != NULL; wsA >= 3*M*N, wsB >= 3*M*K
int linear_f32x3_wgrad(const float* dy, const float* x, float* dW, float* db, int M, int N, int K, bf16* wsA, bf16* wsB, void* st) {
  cudaStream_t cst = reinterpret_cast<cudaStream_t>(st);
  int rc;
  if (db != nullptr && (rc = mmae_cast_colsum_f32(dy, N, nullptr, 0, db, M, N, st))) return rc;
  if ((rc = launch_split3(dy, N, M, N, wsA, N, PAT_A, 1, cst))) return rc;      // [3M, N]
  if ((rc = launch_split3(x, K, M, K, wsB, K, PAT_B, 1, cst))) return rc;       // [3M, K]
  mmae_gemm_epilogue ep;
  memset(&ep, 0, sizeof(ep));
  ep.alpha = 1.0f;
  ep.accumulate = 1;
  ep.out_f32 = dW;
  ep.ld_out_f32 = K;
  return mmae_gemm_bf16(wsA, N, 1, wsB, K, 1, N, K, 3 * M, 0, &ep, st);
}

int gelu_f32(const float* z, float* io, int64_t n, int backward, void* st) {
  if (n == 0) return MMAE_OK;
  int64_t blocks = (n / 4 + 255) / 256;
  blocks = std::min<int64_t>(blocks, int64_t(sm_count()) * 16);
  launch_f32(4, gelu_f32_kernel, (unsigned)std::max<int64_t>(blocks, 1), 256, 0, reinterpret_cast<cudaStream_t>(st), z, io, n, backward);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

}  // namespace mmae

using namespace mmae;

extern "C" int mmae_linear_f32_forward(const float* x, const float* W, const float* bias, const float* residual, float* y, int M,
                                       int N, int K, void* ws, void* stream) {
  MMAE_CHECK(x && W && y && ws && M > 0 && N > 0 && K > 0 && N % 8 == 0 && K % 8 == 0, MMAE_ERR_ARG,
             "mmae_linear_f32_forward: bad args (N, K multiples of 8)");
  bf16* wsA = reinterpret_cast<bf16*>(ws);
  bf16* wsB = wsA + align_up(size_t(3) * M * K, 128);
  return linear_f32x3_forward(x, W, bias, residual, y, M, N, K, wsA, wsB, stream);
}
extern "C" int64_t mmae_linear_f32_workspace_bytes(int M, int N, int K) {
  const size_t big = std::max(std::max(size_t(M) * K, size_t(M) * N), size_t(N) * K);
  return (int64_t)(2 * (align_up(3 * big, 128) * sizeof(bf16)));
}
extern "C" int mmae_linear_f32_backward(const float* x, const float* W, const float* dy, float* dx, float* dW, float* db, int M,
                                        int N, int K, void* ws, void* stream) {
  MMAE_CHECK(x && W && dy && ws && M > 0 && N % 8 == 0 && K % 8 == 0 && M % 8 == 0, MMAE_ERR_ARG,
             "mmae_linear_f32_backward: bad args (M, N, K multiples of 8)");
  const size_t big = std::max(std::max(size_t(M) * K, size_t(M) * N), size_t(N) * K);
  bf16* wsA = reinterpret_cast<bf16*>(ws);
  bf16* wsB = wsA + align_up(3 * big, 128);
  int rc;
  if (dx != nullptr && (rc = linear_f32x3_dgrad(dy, W, dx, M, N, K, 0, wsA, wsB, stream))) return rc;
  if (dW != nullptr && (rc = linear_f32x3_wgrad(dy, x, dW, db, M, N, K, wsA, wsB, stream))) return rc;
  return MMAE_OK;
}

extern "C" int mmae_gelu_f32(const float* z, float* io, int64_t n, int backward, void* stream) {
  MMAE_CHECK(z && io && n >= 0 && n % 4 == 0, MMAE_ERR_ARG, "mmae_gelu_f32: bad args (n %% 4)");
  return gelu_f32(z, io, n, backward, stream);
}

extern "C" int mmae_attention_f32_forward(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv,
                                          float* o, int64_t ldo, float* lse, int B, int H, int Nq, int Nk, int head_dim,
                                          float scale, void* stream) {
  MMAE_CHECK(q && k && v && o && lse && B > 0 && H > 0 && Nq > 0 && Nk > 0, MMAE_ERR_ARG, "mmae_attention_f32_forward: bad args");
  MMAE_CHECK(head_dim == 32, MMAE_ERR_UNSUPPORTED, "mmae_attention_f32_forward: head_dim %d (the fp32 tier covers the decoders' 32)", head_dim);
  MMAE_CHECK(ldk % 4 == 0 && ldv % 4 == 0, MMAE_ERR_ARG, "mmae_attention_f32_forward: ldk / ldv %% 4");
  launch_f32(2, attn_f32_fwd_kernel<32>, dim3(ceil_div(Nq, FA_ROWS), H, B), FA_ROWS, 0, reinterpret_cast<cudaStream_t>(stream), q, ldq, k,
           ldk, v, ldv, o, ldo, lse, Nq, Nk, H, scale);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

extern "C" int mmae_attention_f32_backward(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv,
                                           const float* o, int64_t ldo, const float* d_o, int64_t lddo, const float* lse,
                                           float* delta_ws, float* dq, int64_t lddq, float* dk, int64_t lddk, float* dv,
                                           int64_t lddv, int B, int H, int Nq, int Nk, int head_dim, float scale, void* stream) {
  MMAE_CHECK(q && k && v && o && d_o && lse && delta_ws && dq && dk && dv, MMAE_ERR_ARG, "mmae_attention_f32_backward: bad args");
  MMAE_CHECK(head_dim == 32, MMAE_ERR_UNSUPPORTED, "mmae_attention_f32_backward: head_dim %d (32 only)", head_dim);
  MMAE_CHECK(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0 && lddo % 4 == 0, MMAE_ERR_ARG, "mmae_attention_f32_backward: ld %% 4");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  launch_f32(2, attn_f32_bwd_dq_kernel<32>, dim3(ceil_div(Nq, FA_ROWS), H, B), FA_ROWS, 0, st, q, ldq, k, ldk, v, ldv, o, ldo, d_o, lddo,
           lse, delta_ws, dq, lddq, Nq, Nk, H, scale);
  count_launch();
  MMAE_LAUNCH_OK();
  launch_f32(2, attn_f32_bwd_dkv_kernel<32>, dim3(ceil_div(Nk, FA_ROWS), H, B), FA_ROWS, 0, st, q, ldq, k, ldk, v, ldv, d_o, lddo, lse,
           delta_ws, dk, lddk, dv, lddv, Nq, Nk, H, scale);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}
