// Attention on the Hopper warpgroup tensor cores.  Forward for up to 256 keys (the encoder's 99 x 99 and the decoders'
// 196 x 99 / 196 x 196 problems): one warpgroup per 64 queries of one (batch, head).
//   S = Q K^T : wgmma 64 x KP x 16 (KP = keys padded to 128 or 256), Q and K K-major in shared memory
//   softmax   : in registers, exact (every key of the row is in S: no running rescale)
//   O = P V   : wgmma 64 x head_dim x 16 with P as the register A operand (the S accumulator layout IS the A fragment
//               layout), V transposed into a K-major shared-memory tile while it is staged
// Shared memory holds 8 x 8 core matrices without swizzle, filled by plain 16-byte loads (rows beyond Nq / Nk are zero).
#include "common.cuh"
#include "../../include/multimae_b200.h"

namespace mmae {
void count_launch();

namespace {

constexpr int WA_ROWS = 64;
constexpr int WA_THREADS = 128;
constexpr float WA_LOG2E = 1.4426950408889634f;

// byte offset of element (r, k) in a K-major tile of `kdim` columns made of 8 x 8 core matrices
__device__ __forceinline__ int core_off(int r, int k, int kdim) {
  return (((r >> 3) * (kdim >> 3) + (k >> 3)) << 7) + ((r & 7) << 4) + ((k & 7) << 1);
}

template <int DH, int KP>
__global__ void __launch_bounds__(WA_THREADS) attn_wg_fwd_kernel(const bf16* __restrict__ Q, int64_t ldq,
                                                                 const bf16* __restrict__ K, int64_t ldk,
                                                                 const bf16* __restrict__ V, int64_t ldv, bf16* __restrict__ O,
                                                                 int64_t ldo, float* __restrict__ lse, int Nq, int Nk, int H,
                                                                 float scale) {
  pdl_prologue();
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* sQ = smem;                          // [64][DH]
  uint8_t* sK = sQ + WA_ROWS * DH * 2;         // [KP][DH]
  uint8_t* sVt = sK + KP * DH * 2;             // [DH][KP]
  const int q0 = blockIdx.x * WA_ROWS, h = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x;
  const bf16* Qb = Q + int64_t(b) * Nq * ldq + h * DH;
  const bf16* Kb = K + int64_t(b) * Nk * ldk + h * DH;
  const bf16* Vb = V + int64_t(b) * Nk * ldv + h * DH;

  for (int i = tid; i < WA_ROWS * DH / 8; i += WA_THREADS) {
    const int r = i / (DH / 8), c = (i % (DH / 8)) * 8;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (q0 + r < Nq) v = __ldg(reinterpret_cast<const uint4*>(Qb + int64_t(q0 + r) * ldq + c));
    *reinterpret_cast<uint4*>(sQ + core_off(r, c, DH)) = v;
  }
  for (int i = tid; i < KP * DH / 8; i += WA_THREADS) {
    const int r = i / (DH / 8), c = (i % (DH / 8)) * 8;
    uint4 kv = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);
    if (r < Nk) {
      kv = __ldg(reinterpret_cast<const uint4*>(Kb + int64_t(r) * ldk + c));
      vv = __ldg(reinterpret_cast<const uint4*>(Vb + int64_t(r) * ldv + c));
    }
    *reinterpret_cast<uint4*>(sK + core_off(r, c, DH)) = kv;
    const bf16* ve = reinterpret_cast<const bf16*>(&vv);
#pragma unroll
    for (int e = 0; e < 8; ++e) *reinterpret_cast<bf16*>(sVt + core_off(c + e, r, KP)) = ve[e];
  }
  fence_proxy_async_smem();   // generic-proxy stores -> wgmma operand reads
  __syncthreads();

  float s[KP / 2];   // written by the first wgmma (scale-d = 0)
  const uint32_t q_addr = smem_u32(sQ), k_addr = smem_u32(sK), vt_addr = smem_u32(sVt);
  wgmma_fence();
#pragma unroll
  for (int j = 0; j < DH / 16; ++j) {
    const uint64_t da = gmma_desc_noswz(q_addr + j * 256, 128, (DH / 8) * 128);
    const uint64_t db = gmma_desc_noswz(k_addr + j * 256, 128, (DH / 8) * 128);
    if constexpr (KP == 256) wgmma_m64n256k16<0, 0>(s, da, db, j != 0);
    else wgmma_m64n128k16<0, 0>(s, da, db, j != 0);
  }
  wgmma_commit();
  wgmma_wait<0>();
#pragma unroll
  for (int i = 0; i < KP / 2; ++i) reg_fence(s[i]);

  // rows rl and rl + 8 of this warp's 16; columns 8 j + 2 (lane % 4) (+ 1)
  const int lane = tid & 31, rl = (tid >> 5) * 16 + (lane >> 2), cq = 2 * (lane & 3);
  float m_a = -INFINITY, m_b = -INFINITY;
#pragma unroll
  for (int j = 0; j < KP / 8; ++j) {
    const int c = j * 8 + cq;
    if (c >= Nk) s[4 * j] = s[4 * j + 2] = -INFINITY;
    if (c + 1 >= Nk) s[4 * j + 1] = s[4 * j + 3] = -INFINITY;
    m_a = fmaxf(m_a, fmaxf(s[4 * j], s[4 * j + 1]));
    m_b = fmaxf(m_b, fmaxf(s[4 * j + 2], s[4 * j + 3]));
  }
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    m_a = fmaxf(m_a, __shfl_xor_sync(0xffffffffu, m_a, o));
    m_b = fmaxf(m_b, __shfl_xor_sync(0xffffffffu, m_b, o));
  }
  const float sl = scale * WA_LOG2E;
  float l_a = 0.f, l_b = 0.f;
#pragma unroll
  for (int j = 0; j < KP / 8; ++j) {
    s[4 * j] = fast_exp2((s[4 * j] - m_a) * sl);
    s[4 * j + 1] = fast_exp2((s[4 * j + 1] - m_a) * sl);
    s[4 * j + 2] = fast_exp2((s[4 * j + 2] - m_b) * sl);
    s[4 * j + 3] = fast_exp2((s[4 * j + 3] - m_b) * sl);
    l_a += s[4 * j] + s[4 * j + 1];
    l_b += s[4 * j + 2] + s[4 * j + 3];
  }
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    l_a += __shfl_xor_sync(0xffffffffu, l_a, o);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, o);
  }

  float acc[DH / 2];   // written by the first wgmma (scale-d = 0)
  uint32_t pa[KP / 16][4];
#pragma unroll
  for (int kk = 0; kk < KP / 16; ++kk) {
    pa[kk][0] = pack_bf16x2(s[8 * kk], s[8 * kk + 1]);
    pa[kk][1] = pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]);
    pa[kk][2] = pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]);
    pa[kk][3] = pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7]);
  }
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < KP / 16; ++kk) {
    const uint64_t db = gmma_desc_noswz(vt_addr + kk * 256, 128, (KP / 8) * 128);
    if constexpr (DH == 64) wgmma_m64n64k16_rs<0>(acc, pa[kk], db, kk != 0);
    else wgmma_m64n32k16_rs<0>(acc, pa[kk], db, kk != 0);
  }
  wgmma_commit();
  wgmma_wait<0>();
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) reg_fence(acc[i]);

  const float inv_a = 1.f / l_a, inv_b = 1.f / l_b;
  const int row_a = q0 + rl, row_b = row_a + 8;
  bf16* Ob = O + int64_t(b) * Nq * ldo + h * DH;
#pragma unroll
  for (int j = 0; j < DH / 8; ++j) {
    const int c = j * 8 + cq;
    if (row_a < Nq)
      *reinterpret_cast<uint32_t*>(Ob + int64_t(row_a) * ldo + c) = pack_bf16x2(acc[4 * j] * inv_a, acc[4 * j + 1] * inv_a);
    if (row_b < Nq)
      *reinterpret_cast<uint32_t*>(Ob + int64_t(row_b) * ldo + c) = pack_bf16x2(acc[4 * j + 2] * inv_b, acc[4 * j + 3] * inv_b);
  }
  if ((lane & 3) == 0) {
    float* L = lse + (int64_t(b) * H + h) * Nq;
    if (row_a < Nq) L[row_a] = m_a * scale + logf(l_a);
    if (row_b < Nq) L[row_b] = m_b * scale + logf(l_b);
  }
}

template <int DH, int KP>
int launch_wg(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o, int64_t ldo,
              float* lse, int B, int H, int Nq, int Nk, float scale, cudaStream_t st) {
  constexpr int SMEM = (WA_ROWS + 2 * KP) * DH * 2;
  auto kern = attn_wg_fwd_kernel<DH, KP>;
  static bool configured = false;
  if (!configured) {
    MMAE_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    configured = true;
  }
  launch_k(kern, dim3(ceil_div(Nq, WA_ROWS), H, B), WA_THREADS, SMEM, st, (const bf16*)q, ldq, (const bf16*)k, ldk,
           (const bf16*)v, ldv, (bf16*)o, ldo, lse, Nq, Nk, H, scale);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Backward (any Nq, Nk; head_dim 32 / 64), after the delta kernel of attention.cu (delta = rowsum(dO o O)):
//   dK / dV : one warpgroup per 64 keys, looping over 64-query tiles:  S^T = K Q^T, dP^T = V dO^T (wgmma from shared
//             memory), P^T = exp(S^T scale - lse), dS^T = P^T (dP^T - delta), then dV += P^T dO and dK += dS^T Q with P^T /
//             dS^T as register A operands and dO^T / Q^T staged K-major
//   dQ      : one warpgroup per 64 queries, looping over 64-key tiles:  S = Q K^T, dP = dO V^T, dS = P (dP - delta),
//             dQ += dS K with K^T staged K-major
// ---------------------------------------------------------------------------------------------------------------------
// stage rows [r0, r0 + 64) of a [rows, ld] bf16 head slice: `nt` K-major [64][DH] (may be null) and `t` its transpose
// [DH][64] (may be null); rows >= valid are zero
template <int DH>
__device__ __forceinline__ void stage64(uint8_t* nt, uint8_t* t, const bf16* base, int64_t ld, int r0, int valid, int tid) {
  for (int i = tid; i < 64 * DH / 8; i += WA_THREADS) {
    const int r = i / (DH / 8), c = (i % (DH / 8)) * 8;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r0 + r < valid) v = __ldg(reinterpret_cast<const uint4*>(base + int64_t(r0 + r) * ld + c));
    if (nt) *reinterpret_cast<uint4*>(nt + core_off(r, c, DH)) = v;
    if (t) {
      const bf16* e = reinterpret_cast<const bf16*>(&v);
#pragma unroll
      for (int x = 0; x < 8; ++x) *reinterpret_cast<bf16*>(t + core_off(c + x, r, 64)) = e[x];
    }
  }
}

// 64 x 64 scores of two [64][DH] K-major tiles: d = A B^T
template <int DH>
__device__ __forceinline__ void mm64(float (&d)[32], uint32_t a_addr, uint32_t b_addr) {
  wgmma_fence();
#pragma unroll
  for (int j = 0; j < DH / 16; ++j)
    wgmma_m64n64k16<0, 0>(d, gmma_desc_noswz(a_addr + j * 256, 128, (DH / 8) * 128),
                          gmma_desc_noswz(b_addr + j * 256, 128, (DH / 8) * 128), j != 0);
  wgmma_commit();
  wgmma_wait<0>();
#pragma unroll
  for (int i = 0; i < 32; ++i) reg_fence(d[i]);
}

// acc (+)= P B with P a 64 x 64 register operand (accumulator layout) and B^T staged K-major as [DH][64]
template <int DH>
__device__ __forceinline__ void mm_rs(float (&acc)[DH / 2], const float (&p)[32], uint32_t bt_addr, bool accumulate) {
  uint32_t pa[4][4];
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    pa[kk][0] = pack_bf16x2(p[8 * kk], p[8 * kk + 1]);
    pa[kk][1] = pack_bf16x2(p[8 * kk + 2], p[8 * kk + 3]);
    pa[kk][2] = pack_bf16x2(p[8 * kk + 4], p[8 * kk + 5]);
    pa[kk][3] = pack_bf16x2(p[8 * kk + 6], p[8 * kk + 7]);
  }
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint64_t db = gmma_desc_noswz(bt_addr + kk * 256, 128, 8 * 128);
    if constexpr (DH == 64) wgmma_m64n64k16_rs<0>(acc, pa[kk], db, (accumulate || kk != 0) ? 1u : 0u);
    else wgmma_m64n32k16_rs<0>(acc, pa[kk], db, (accumulate || kk != 0) ? 1u : 0u);
  }
  wgmma_commit();
  wgmma_wait<0>();
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) reg_fence(acc[i]);
}

template <int DH>
__device__ __forceinline__ void store_rows(bf16* base, int64_t ld, int r0, int valid, const float (&acc)[DH / 2], float mul,
                                           int rl, int cq) {
#pragma unroll
  for (int j = 0; j < DH / 8; ++j) {
    const int c = j * 8 + cq;
    if (r0 + rl < valid)
      *reinterpret_cast<uint32_t*>(base + int64_t(r0 + rl) * ld + c) = pack_bf16x2(acc[4 * j] * mul, acc[4 * j + 1] * mul);
    if (r0 + rl + 8 < valid)
      *reinterpret_cast<uint32_t*>(base + int64_t(r0 + rl + 8) * ld + c) = pack_bf16x2(acc[4 * j + 2] * mul, acc[4 * j + 3] * mul);
  }
}

template <int DH>
__global__ void __launch_bounds__(WA_THREADS) attn_wg_bwd_dkv_kernel(const bf16* __restrict__ Q, int64_t ldq,
                                                                     const bf16* __restrict__ K, int64_t ldk,
                                                                     const bf16* __restrict__ V, int64_t ldv,
                                                                     const bf16* __restrict__ dO, int64_t lddo,
                                                                     const float* __restrict__ lse, const float* __restrict__ delta,
                                                                     bf16* __restrict__ dK, int64_t lddk, bf16* __restrict__ dV,
                                                                     int64_t lddv, int Nq, int Nk, int H, float scale) {
  pdl_prologue();
  extern __shared__ __align__(128) uint8_t smem[];
  constexpr int T = 64 * DH * 2;
  uint8_t *sK = smem, *sV = sK + T, *sQ = sV + T, *sdO = sQ + T, *sQt = sdO + T, *sdOt = sQt + T;
  const int k0 = blockIdx.x * 64, h = blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
  const bf16* Qb = Q + int64_t(b) * Nq * ldq + h * DH;
  const bf16* dOb = dO + int64_t(b) * Nq * lddo + h * DH;
  const float* Lb = lse + (int64_t(b) * H + h) * Nq;
  const float* Db = delta + (int64_t(b) * H + h) * Nq;
  stage64<DH>(sK, nullptr, K + int64_t(b) * Nk * ldk + h * DH, ldk, k0, Nk, tid);
  stage64<DH>(sV, nullptr, V + int64_t(b) * Nk * ldv + h * DH, ldv, k0, Nk, tid);
  const int lane = tid & 31, rl = (tid >> 5) * 16 + (lane >> 2), cq = 2 * (lane & 3);
  const float sl = scale * WA_LOG2E;
  float dk[DH / 2], dv[DH / 2];   // written by the first query tile's wgmma (scale-d = 0)
  for (int q0 = 0; q0 < Nq; q0 += 64) {
    if (q0 > 0) __syncthreads();   // every warp's MMAs on the previous tile have completed
    stage64<DH>(sQ, sQt, Qb, ldq, q0, Nq, tid);
    stage64<DH>(sdO, sdOt, dOb, lddo, q0, Nq, tid);
    fence_proxy_async_smem();
    __syncthreads();
    float st[32], dpt[32];
    mm64<DH>(st, smem_u32(sK), smem_u32(sQ));     // S^T  [keys][queries]
    mm64<DH>(dpt, smem_u32(sV), smem_u32(sdO));   // dP^T
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int q = q0 + j * 8 + cq + e;
        const bool ok = q < Nq;
        const float L = ok ? __ldg(Lb + q) * WA_LOG2E : 0.f, D = ok ? __ldg(Db + q) : 0.f;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int i = 4 * j + 2 * hr + e;
          const float pv = ok ? fast_exp2(st[i] * sl - L) : 0.f;
          st[i] = pv;
          dpt[i] = pv * (dpt[i] - D);
        }
      }
    }
    mm_rs<DH>(dv, st, smem_u32(sdOt), q0 > 0);    // dV += P^T dO
    mm_rs<DH>(dk, dpt, smem_u32(sQt), q0 > 0);    // dK += dS^T Q
  }
  store_rows<DH>(dK + int64_t(b) * Nk * lddk + h * DH, lddk, k0, Nk, dk, scale, rl, cq);
  store_rows<DH>(dV + int64_t(b) * Nk * lddv + h * DH, lddv, k0, Nk, dv, 1.f, rl, cq);
}

template <int DH>
__global__ void __launch_bounds__(WA_THREADS) attn_wg_bwd_dq_kernel(const bf16* __restrict__ Q, int64_t ldq,
                                                                    const bf16* __restrict__ K, int64_t ldk,
                                                                    const bf16* __restrict__ V, int64_t ldv,
                                                                    const bf16* __restrict__ dO, int64_t lddo,
                                                                    const float* __restrict__ lse, const float* __restrict__ delta,
                                                                    bf16* __restrict__ dQ, int64_t lddq, int Nq, int Nk, int H,
                                                                    float scale) {
  pdl_prologue();
  extern __shared__ __align__(128) uint8_t smem[];
  constexpr int T = 64 * DH * 2;
  uint8_t *sQ = smem, *sdO = sQ + T, *sK = sdO + T, *sV = sK + T, *sKt = sV + T;
  const int q0 = blockIdx.x * 64, h = blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
  const bf16* Kb = K + int64_t(b) * Nk * ldk + h * DH;
  const bf16* Vb = V + int64_t(b) * Nk * ldv + h * DH;
  stage64<DH>(sQ, nullptr, Q + int64_t(b) * Nq * ldq + h * DH, ldq, q0, Nq, tid);
  stage64<DH>(sdO, nullptr, dO + int64_t(b) * Nq * lddo + h * DH, lddo, q0, Nq, tid);
  const int lane = tid & 31, rl = (tid >> 5) * 16 + (lane >> 2), cq = 2 * (lane & 3);
  const float sl = scale * WA_LOG2E;
  const float* Lb = lse + (int64_t(b) * H + h) * Nq;
  const float* Db = delta + (int64_t(b) * H + h) * Nq;
  float L[2], D[2];
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int q = q0 + rl + 8 * hr;
    L[hr] = q < Nq ? __ldg(Lb + q) * WA_LOG2E : 0.f;
    D[hr] = q < Nq ? __ldg(Db + q) : 0.f;
  }
  float dq[DH / 2];   // written by the first key tile's wgmma (scale-d = 0)
  for (int k0 = 0; k0 < Nk; k0 += 64) {
    if (k0 > 0) __syncthreads();
    stage64<DH>(sK, sKt, Kb, ldk, k0, Nk, tid);
    stage64<DH>(sV, nullptr, Vb, ldv, k0, Nk, tid);
    fence_proxy_async_smem();
    __syncthreads();
    float sc[32], dp[32];
    mm64<DH>(sc, smem_u32(sQ), smem_u32(sK));     // S  [queries][keys]
    mm64<DH>(dp, smem_u32(sdO), smem_u32(sV));    // dP
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const bool ok = k0 + j * 8 + cq + e < Nk;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int i = 4 * j + 2 * hr + e;
          const float pv = ok ? fast_exp2(sc[i] * sl - L[hr]) : 0.f;
          dp[i] = pv * (dp[i] - D[hr]);
        }
      }
    }
    mm_rs<DH>(dq, dp, smem_u32(sKt), k0 > 0);     // dQ += dS K
  }
  store_rows<DH>(dQ + int64_t(b) * Nq * lddq + h * DH, lddq, q0, Nq, dq, scale, rl, cq);
}

template <int DH>
int launch_wg_bwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, const void* d_o,
                  int64_t lddo, const float* lse, const float* delta, void* dq, int64_t lddq, void* dk, int64_t lddk, void* dv,
                  int64_t lddv, int B, int H, int Nq, int Nk, float scale, cudaStream_t st) {
  constexpr int T = 64 * DH * 2;
  auto kkv = attn_wg_bwd_dkv_kernel<DH>;
  auto kq = attn_wg_bwd_dq_kernel<DH>;
  static bool configured = false;
  if (!configured) {
    MMAE_CUDA_OK(cudaFuncSetAttribute(kkv, cudaFuncAttributeMaxDynamicSharedMemorySize, 6 * T));
    MMAE_CUDA_OK(cudaFuncSetAttribute(kq, cudaFuncAttributeMaxDynamicSharedMemorySize, 5 * T));
    configured = true;
  }
  launch_k(kkv, dim3(ceil_div(Nk, 64), H, B), WA_THREADS, 6 * T, st, (const bf16*)q, ldq, (const bf16*)k, ldk, (const bf16*)v,
           ldv, (const bf16*)d_o, lddo, lse, delta, (bf16*)dk, lddk, (bf16*)dv, lddv, Nq, Nk, H, scale);
  count_launch();
  launch_k(kq, dim3(ceil_div(Nq, 64), H, B), WA_THREADS, 5 * T, st, (const bf16*)q, ldq, (const bf16*)k, ldk, (const bf16*)v,
           ldv, (const bf16*)d_o, lddo, lse, delta, (bf16*)dq, lddq, Nq, Nk, H, scale);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

}  // namespace

bool attn_wg_fwd_supported(int Nk, int head_dim) { return (head_dim == 32 || head_dim == 64) && Nk >= 1 && Nk <= 256; }

int attn_wg_forward(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o, int64_t ldo,
                    float* lse, int B, int H, int Nq, int Nk, int head_dim, float scale, cudaStream_t st) {
  if (head_dim == 64)
    return Nk <= 128 ? launch_wg<64, 128>(q, ldq, k, ldk, v, ldv, o, ldo, lse, B, H, Nq, Nk, scale, st)
                     : launch_wg<64, 256>(q, ldq, k, ldk, v, ldv, o, ldo, lse, B, H, Nq, Nk, scale, st);
  return Nk <= 128 ? launch_wg<32, 128>(q, ldq, k, ldk, v, ldv, o, ldo, lse, B, H, Nq, Nk, scale, st)
                   : launch_wg<32, 256>(q, ldq, k, ldk, v, ldv, o, ldo, lse, B, H, Nq, Nk, scale, st);
}

}  // namespace mmae

namespace mmae {
int attn_wg_backward(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, const void* d_o,
                     int64_t lddo, const float* lse, const float* delta, void* dq, int64_t lddq, void* dk, int64_t lddk,
                     void* dv, int64_t lddv, int B, int H, int Nq, int Nk, int head_dim, float scale, cudaStream_t st) {
  if (head_dim == 64)
    return launch_wg_bwd<64>(q, ldq, k, ldk, v, ldv, d_o, lddo, lse, delta, dq, lddq, dk, lddk, dv, lddv, B, H, Nq, Nk, scale, st);
  return launch_wg_bwd<32>(q, ldq, k, ldk, v, ldv, d_o, lddo, lse, delta, dq, lddq, dk, lddk, dv, lddv, B, H, Nq, Nk, scale, st);
}
}  // namespace mmae
