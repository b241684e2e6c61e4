// Fused multi-head attention, forward and backward (flash-style: scores never touch HBM).
//
// v1 kernel family: warp-level mma.sync.m16n8k16 (bf16 in, fp32 accumulate), 4 warps x 16 stationary rows per CTA,
// the other sequence dimension streamed through shared memory in chunks of 64.  Softmax in fp32 with exp2.
// Works for any (Nq, Nk) and head_dim in {32, 64}: encoder MHSA (99x99, dh 64), decoder cross-attention
// (196x99, dh 32) and decoder self-attention (196x196, dh 32), and the 448^2 / MultiMAE-L variants.
//
// Replaces multimae/multimae_utils.py:172-179 (Attention) and :203-211 (CrossAttention): q@k^T*scale -> softmax ->
// @v, the two permute copies around it, and their autograd backward.
//
// Layout contract: Q/K/V/O live inside row-major [B*N, ld] projection buffers; head h occupies columns
// [h*DH, (h+1)*DH) relative to the given base pointer; batch b occupies rows [b*N, (b+1)*N).
#include "common.cuh"
#include "../../include/multimae_b200.h"

#include <cstdlib>

namespace mmae {
void count_launch();
bool attn_wg_fwd_supported(int Nk, int head_dim);
int attn_wg_forward(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o, int64_t ldo,
                    float* lse, int B, int H, int Nq, int Nk, int head_dim, float scale, cudaStream_t st);
int attn_wg_backward(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, const void* d_o,
                     int64_t lddo, const float* lse, const float* delta, void* dq, int64_t lddq, void* dk, int64_t lddk,
                     void* dv, int64_t lddv, int B, int H, int Nq, int Nk, int head_dim, float scale, cudaStream_t st);
namespace {

constexpr int ATT_ROWS = 64;    // stationary rows per CTA (4 warps x 16)
constexpr int ATT_CHUNK = 64;   // streamed rows per shared-memory stage
constexpr int ATT_THREADS = 128;
constexpr float LOG2E = 1.4426950408889634f;

__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// Fragment loads with ldmatrix (one instruction per fragment instead of 2-4 scalar LDS; the 80-byte row pitch keeps the
// eight 16-byte row segments of a matrix on distinct banks).
// A fragment (16 rows x 16 k) from row-major smem s[row][k]
__device__ __forceinline__ void load_a_frag(uint32_t (&a)[4], const bf16* s, int ld, int row0, int k0, int g, int t) {
  const int lane = g * 4 + t;
  const bf16* p = s + (row0 + (lane & 7) + ((lane >> 3) & 1) * 8) * ld + k0 + (lane >> 4) * 8;
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(a[0]), "=r"(a[1]), "=r"(a[2]), "=r"(a[3])
               : "r"(smem_u32(p)));
}
// B fragment (16 k x 8 n) from smem stored as s[n][k] (k contiguous)
__device__ __forceinline__ void load_b_frag(uint32_t (&b)[2], const bf16* s, int ld, int n0, int k0, int g, int t) {
  const int lane = (g * 4 + t) & 15;
  const bf16* p = s + (n0 + (lane & 7)) * ld + k0 + (lane >> 3) * 8;
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];" : "=r"(b[0]), "=r"(b[1]) : "r"(smem_u32(p)));
}
// B fragment (16 k x 8 n) from smem stored as s[k][n] (n contiguous: a row-major [rows = k][cols = n] tile as it was
// loaded) - the transposing ldmatrix replaces a transposed copy of the tile in shared memory
__device__ __forceinline__ void load_b_frag_t(uint32_t (&b)[2], const bf16* s, int ld, int k0, int n0, int g, int t) {
  const int lane = (g * 4 + t) & 15;
  const bf16* p = s + (k0 + (lane & 7) + (lane >> 3) * 8) * ld + n0;
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];" : "=r"(b[0]), "=r"(b[1]) : "r"(smem_u32(p)));
}

// Copy `ATT_CHUNK` rows x DH columns of a global [rows, ld] matrix into row-major smem (pitch DH+8), zero-filling
// rows >= rows_valid.  Optionally also writes the transpose st[d][row] (pitch ATT_CHUNK+8).
template <int DH, bool ROWMAJOR, bool TRANSPOSED>
__device__ __forceinline__ void load_chunk(bf16* s, bf16* st, const bf16* gbase, int64_t ld, int row0, int rows_valid) {
  constexpr int LDS = DH + 8, LDT = ATT_CHUNK + 8, VPR = DH / 8;
  for (int idx = threadIdx.x; idx < ATT_CHUNK * VPR; idx += ATT_THREADS) {
    const int r = idx / VPR, cv = idx % VPR;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (row0 + r < rows_valid) v = __ldg(reinterpret_cast<const uint4*>(gbase + int64_t(row0 + r) * ld + cv * 8));
    if constexpr (ROWMAJOR) *reinterpret_cast<uint4*>(s + r * LDS + cv * 8) = v;
    if constexpr (TRANSPOSED) {
      const bf16* e = reinterpret_cast<const bf16*>(&v);
#pragma unroll
      for (int i = 0; i < 8; ++i) st[(cv * 8 + i) * LDT + r] = e[i];
    }
  }
}

// Asynchronous variant for the streamed operand: 16-byte cp.async per (row, 8 columns), rows >= rows_valid zero-filled
// (src-size 0), so the next chunk is in flight while the current one is consumed.
__device__ __forceinline__ void cp_async_16(void* smem_dst, const void* gsrc, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(valid ? 16 : 0)
               : "memory");
}
__device__ __forceinline__ void cp_async_4(void* smem_dst, const void* gsrc, bool valid) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(valid ? 4 : 0)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
template <int DH>
__device__ __forceinline__ void load_chunk_async(bf16* s, const bf16* gbase, int64_t ld, int row0, int rows_valid) {
  constexpr int LDS = DH + 8, VPR = DH / 8;
  for (int idx = threadIdx.x; idx < ATT_CHUNK * VPR; idx += ATT_THREADS) {
    const int r = idx / VPR, cv = idx % VPR;
    const bool ok = row0 + r < rows_valid;
    cp_async_16(s + r * LDS + cv * 8, gbase + int64_t(ok ? row0 + r : 0) * ld + cv * 8, ok);
  }
}

// =====================================================================================================================
// forward
// =====================================================================================================================
// Attention dropout (Attention.attn_drop, multimae/multimae_utils.py:177) acts on the softmax probabilities P before P V.
// Its site matrix is [B*H*Nq, Nk]: row (b*H + h)*Nq + i, column j.  With DROP the forward keeps lse undropped and multiplies
// P by the mask before P V (the 1/(1-p) joins the final 1/l); the backward uses dV = (P*M/(1-p))^T dO and
// dP = (dO V^T)*M/(1-p), and dS = P*(dP - delta) with delta = rowsum(dO * O) of the dropped O, unchanged.
// factors of columns col, col + 1 (col even) of `row`
__device__ __forceinline__ float2 dropout_factor2(const DropSite& d, uint64_t seed, uint64_t row, int col) {
  const uint4 w = dropout_words(seed, d.site, row, col);
  const bool hi = col & 2;
  return make_float2((hi ? w.z : w.x) < d.thresh ? d.scale : 0.f, (hi ? w.w : w.y) < d.thresh ? d.scale : 0.f);
}

template <int DH, bool DROP>
__global__ void __launch_bounds__(ATT_THREADS) attn_fwd_kernel(const bf16* __restrict__ Q, int64_t ldq,
                                                               const bf16* __restrict__ K, int64_t ldk,
                                                               const bf16* __restrict__ V, int64_t ldv,
                                                               bf16* __restrict__ O, int64_t ldo,
                                                               float* __restrict__ lse, int Nq, int Nk, int H,
                                                               float scale, DropSite drop) {
  pdl_prologue();
  constexpr int LDS = DH + 8, LDT = ATT_CHUNK + 8;
  __shared__ __align__(16) bf16 sQ[ATT_ROWS * LDS];
  __shared__ __align__(16) bf16 sKb[2][ATT_CHUNK * LDS];
  __shared__ __align__(16) bf16 sVb[2][ATT_CHUNK * LDS];

  const int q0 = blockIdx.x * ATT_ROWS, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const bf16* Qb = Q + int64_t(b) * Nq * ldq + h * DH;
  const bf16* Kb = K + int64_t(b) * Nk * ldk + h * DH;
  const bf16* Vb = V + int64_t(b) * Nk * ldv + h * DH;

  load_chunk_async<DH>(sKb[0], Kb, ldk, 0, Nk);      // first key chunk flies while Q is staged
  load_chunk_async<DH>(sVb[0], Vb, ldv, 0, Nk);
  cp_async_commit();
  load_chunk<DH, true, false>(sQ, nullptr, Qb, ldq, q0, Nq);
  __syncthreads();
  uint32_t qa[DH / 16][4];
#pragma unroll
  for (int kk = 0; kk < DH / 16; ++kk) load_a_frag(qa[kk], sQ, LDS, warp * 16, kk * 16, g, t);

  float acc[DH / 8][4];
#pragma unroll
  for (int j = 0; j < DH / 8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const float sl2 = scale * LOG2E;
  const bool live = q0 + warp * 16 < Nq;
  uint64_t dseed = 0, drow_a = 0;
  if constexpr (DROP) {
    dseed = *drop.seed;
    drow_a = (uint64_t(b) * H + h) * Nq + q0 + warp * 16 + g;
  }

  for (int k0 = 0, it = 0; k0 < Nk; k0 += ATT_CHUNK, ++it) {
    const bf16* sK = sKb[it & 1];
    const bf16* sV = sVb[it & 1];
    if (k0 + ATT_CHUNK < Nk) {      // prefetch the next chunk into the other buffer (its readers finished last iteration)
      load_chunk_async<DH>(sKb[(it + 1) & 1], Kb, ldk, k0 + ATT_CHUNK, Nk);
      load_chunk_async<DH>(sVb[(it + 1) & 1], Vb, ldv, k0 + ATT_CHUNK, Nk);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();

    // a warp whose 16 query rows all lie past Nq only stages chunks (decoder 196 queries: 3 of the last CTA's 4 warps)
    if (live) {
      float s[ATT_CHUNK / 8][4];
#pragma unroll
      for (int j = 0; j < ATT_CHUNK / 8; ++j) {
        s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
        for (int kk = 0; kk < DH / 16; ++kk) {
          uint32_t bfr[2];
          load_b_frag(bfr, sK, LDS, j * 8, kk * 16, g, t);
          mma_bf16_16816(s[j], qa[kk], bfr);
        }
      }
      // mask padded keys, running max
      float mx[2] = {m_run[0], m_run[1]};
#pragma unroll
      for (int j = 0; j < ATT_CHUNK / 8; ++j) {
        const int key = k0 + j * 8 + 2 * t;
        if (key >= Nk) s[j][0] = s[j][2] = -INFINITY;
        if (key + 1 >= Nk) s[j][1] = s[j][3] = -INFINITY;
        mx[0] = fmaxf(mx[0], fmaxf(s[j][0], s[j][1]));
        mx[1] = fmaxf(mx[1], fmaxf(s[j][2], s[j][3]));
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      }
      const float alpha0 = fast_exp2((m_run[0] - mx[0]) * sl2), alpha1 = fast_exp2((m_run[1] - mx[1]) * sl2);
      m_run[0] = mx[0];
      m_run[1] = mx[1];
      const float mo0 = mx[0] * sl2, mo1 = mx[1] * sl2;
      float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
      for (int j = 0; j < ATT_CHUNK / 8; ++j) {
        s[j][0] = fast_exp2(s[j][0] * sl2 - mo0);
        s[j][1] = fast_exp2(s[j][1] * sl2 - mo0);
        s[j][2] = fast_exp2(s[j][2] * sl2 - mo1);
        s[j][3] = fast_exp2(s[j][3] * sl2 - mo1);
        rs0 += s[j][0] + s[j][1];
        rs1 += s[j][2] + s[j][3];
      }
      l_run[0] = l_run[0] * alpha0 + rs0;
      l_run[1] = l_run[1] * alpha1 + rs1;
#pragma unroll
      for (int j = 0; j < DH / 8; ++j) {
        acc[j][0] *= alpha0; acc[j][1] *= alpha0;
        acc[j][2] *= alpha1; acc[j][3] *= alpha1;
      }
      if constexpr (DROP) {   // the row sums above stay undropped; 0 / 1 here, 1/(1-p) at the end
#pragma unroll
        for (int j = 0; j < ATT_CHUNK / 8; ++j) {
          const int key = k0 + j * 8 + 2 * t;
          const float2 fa = dropout_factor2(drop, dseed, drow_a, key), fb = dropout_factor2(drop, dseed, drow_a + 8, key);
          if (fa.x == 0.f) s[j][0] = 0.f;
          if (fa.y == 0.f) s[j][1] = 0.f;
          if (fb.x == 0.f) s[j][2] = 0.f;
          if (fb.y == 0.f) s[j][3] = 0.f;
        }
      }
      // O += P V
#pragma unroll
      for (int ks = 0; ks < ATT_CHUNK / 16; ++ks) {
        uint32_t pa[4];
        pa[0] = pack_bf16x2(s[2 * ks][0], s[2 * ks][1]);
        pa[1] = pack_bf16x2(s[2 * ks][2], s[2 * ks][3]);
        pa[2] = pack_bf16x2(s[2 * ks + 1][0], s[2 * ks + 1][1]);
        pa[3] = pack_bf16x2(s[2 * ks + 1][2], s[2 * ks + 1][3]);
#pragma unroll
        for (int jd = 0; jd < DH / 8; ++jd) {
          uint32_t bfr[2];
          load_b_frag_t(bfr, sV, LDS, ks * 16, jd * 8, g, t);
          mma_bf16_16816(acc[jd], pa, bfr);
        }
      }
    }
    __syncthreads();   // every warp is done with this buffer before the next iteration's prefetch overwrites it
  }

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  const int row_a = q0 + warp * 16 + g, row_b = row_a + 8;
  float inv0 = 1.0f / l_run[0], inv1 = 1.0f / l_run[1];
  if constexpr (DROP) {
    inv0 *= drop.scale;
    inv1 *= drop.scale;
  }
  bf16* Ob = O + int64_t(b) * Nq * ldo + h * DH;
#pragma unroll
  for (int jd = 0; jd < DH / 8; ++jd) {
    const int c = jd * 8 + 2 * t;
    if (row_a < Nq) *reinterpret_cast<uint32_t*>(Ob + int64_t(row_a) * ldo + c) = pack_bf16x2(acc[jd][0] * inv0, acc[jd][1] * inv0);
    if (row_b < Nq) *reinterpret_cast<uint32_t*>(Ob + int64_t(row_b) * ldo + c) = pack_bf16x2(acc[jd][2] * inv1, acc[jd][3] * inv1);
  }
  if (lse != nullptr && t == 0) {
    float* L = lse + (int64_t(b) * H + h) * Nq;
    if (row_a < Nq) L[row_a] = m_run[0] * scale + logf(l_run[0]);
    if (row_b < Nq) L[row_b] = m_run[1] * scale + logf(l_run[1]);
  }
}

// =====================================================================================================================
// backward, part 0: delta[b,h,q] = sum_d dO[q,d] * O[q,d]
// =====================================================================================================================
template <int DH>
__global__ void __launch_bounds__(256) attn_delta_kernel(const bf16* __restrict__ O, int64_t ldo,
                                                         const bf16* __restrict__ dO, int64_t lddo,
                                                         float* __restrict__ delta, int Nq, int H, int64_t rows) {
  pdl_prologue();
  // one 16-byte segment (8 columns) per thread; a head is TPH consecutive segments = TPH consecutive lanes
  constexpr int TPH = DH / 8;
  const int S = H * TPH;                                    // segments per row
  const int64_t total = rows * S;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t g0 = int64_t(blockIdx.x) * blockDim.x; g0 < total; g0 += stride) {
    const int64_t g = g0 + threadIdx.x;
    const bool ok = g < total;
    const int64_t row = ok ? g / S : 0;
    const int idx = ok ? int(g - row * S) : 0;
    float p = 0.f;
    if (ok) {
      const uint4 o = __ldg(reinterpret_cast<const uint4*>(O + row * ldo + idx * 8));
      const uint4 d = __ldg(reinterpret_cast<const uint4*>(dO + row * lddo + idx * 8));
      const uint32_t* ou = reinterpret_cast<const uint32_t*>(&o);
      const uint32_t* du = reinterpret_cast<const uint32_t*>(&d);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 a = unpack_bf16x2(ou[i]), c = unpack_bf16x2(du[i]);
        p += a.x * c.x + a.y * c.y;
      }
    }
#pragma unroll
    for (int o = TPH / 2; o > 0; o >>= 1) p += __shfl_xor_sync(0xffffffffu, p, o);
    if (ok && (idx % TPH) == 0) {
      const int64_t b = row / Nq;
      const int q = int(row - b * Nq);
      delta[(b * H + idx / TPH) * Nq + q] = p;
    }
  }
}

// =====================================================================================================================
// backward, part 1: dQ (query-stationary)
// =====================================================================================================================
template <int DH, bool DROP>
__global__ void __launch_bounds__(ATT_THREADS) attn_bwd_dq_kernel(const bf16* __restrict__ Q, int64_t ldq,
                                                                  const bf16* __restrict__ K, int64_t ldk,
                                                                  const bf16* __restrict__ V, int64_t ldv,
                                                                  const bf16* __restrict__ dO, int64_t lddo,
                                                                  const float* __restrict__ lse,
                                                                  const float* __restrict__ delta,
                                                                  bf16* __restrict__ dQ, int64_t lddq, int Nq, int Nk,
                                                                  int H, float scale, DropSite drop) {
  pdl_prologue();
  constexpr int LDS = DH + 8, LDT = ATT_CHUNK + 8;
  __shared__ __align__(16) bf16 sA[ATT_ROWS * LDS];   // Q tile, then dO tile (staging for the A fragments)
  __shared__ __align__(16) bf16 sKb[2][ATT_CHUNK * LDS];
  __shared__ __align__(16) bf16 sVb[2][ATT_CHUNK * LDS];

  const int q0 = blockIdx.x * ATT_ROWS, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const bf16* Qb = Q + int64_t(b) * Nq * ldq + h * DH;
  const bf16* Kb = K + int64_t(b) * Nk * ldk + h * DH;
  const bf16* Vb = V + int64_t(b) * Nk * ldv + h * DH;
  const bf16* dOb = dO + int64_t(b) * Nq * lddo + h * DH;

  uint32_t qa[DH / 16][4], doa[DH / 16][4];
  load_chunk_async<DH>(sKb[0], Kb, ldk, 0, Nk);      // first key chunk flies while Q / dO are staged
  load_chunk_async<DH>(sVb[0], Vb, ldv, 0, Nk);
  cp_async_commit();
  load_chunk<DH, true, false>(sA, nullptr, Qb, ldq, q0, Nq);
  __syncthreads();
#pragma unroll
  for (int kk = 0; kk < DH / 16; ++kk) load_a_frag(qa[kk], sA, LDS, warp * 16, kk * 16, g, t);
  __syncthreads();
  load_chunk<DH, true, false>(sA, nullptr, dOb, lddo, q0, Nq);
  __syncthreads();
#pragma unroll
  for (int kk = 0; kk < DH / 16; ++kk) load_a_frag(doa[kk], sA, LDS, warp * 16, kk * 16, g, t);

  const int row_a = q0 + warp * 16 + g, row_b = row_a + 8;
  const float* Lp = lse + (int64_t(b) * H + h) * Nq;
  const float* Dp = delta + (int64_t(b) * H + h) * Nq;
  const float lse_a = row_a < Nq ? Lp[row_a] * LOG2E : INFINITY, lse_b = row_b < Nq ? Lp[row_b] * LOG2E : INFINITY;
  const float del_a = row_a < Nq ? Dp[row_a] : 0.f, del_b = row_b < Nq ? Dp[row_b] : 0.f;
  const float sl2 = scale * LOG2E;
  uint64_t dseed = 0;
  const uint64_t drow_a = (uint64_t(b) * H + h) * Nq + row_a;
  if constexpr (DROP) dseed = *drop.seed;

  float acc[DH / 8][4];
#pragma unroll
  for (int j = 0; j < DH / 8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;

  for (int k0 = 0, it = 0; k0 < Nk; k0 += ATT_CHUNK, ++it) {
    const bf16* sK = sKb[it & 1];
    const bf16* sV = sVb[it & 1];
    if (k0 + ATT_CHUNK < Nk) {
      load_chunk_async<DH>(sKb[(it + 1) & 1], Kb, ldk, k0 + ATT_CHUNK, Nk);
      load_chunk_async<DH>(sVb[(it + 1) & 1], Vb, ldv, k0 + ATT_CHUNK, Nk);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
#pragma unroll
    for (int ks = 0; ks < ATT_CHUNK / 16; ++ks) {
      uint32_t dsa[4];
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int n0 = ks * 16 + half * 8;
        float s[4] = {0.f, 0.f, 0.f, 0.f}, dp[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int kk = 0; kk < DH / 16; ++kk) {
          uint32_t bk[2], bv[2];
          load_b_frag(bk, sK, LDS, n0, kk * 16, g, t);
          load_b_frag(bv, sV, LDS, n0, kk * 16, g, t);
          mma_bf16_16816(s, qa[kk], bk);
          mma_bf16_16816(dp, doa[kk], bv);
        }
        const int key = k0 + n0 + 2 * t;
        if constexpr (DROP) {   // dP = (dO V^T) * M / (1-p)
          const float2 fa = dropout_factor2(drop, dseed, drow_a, key), fb = dropout_factor2(drop, dseed, drow_a + 8, key);
          dp[0] *= fa.x; dp[1] *= fa.y; dp[2] *= fb.x; dp[3] *= fb.y;
        }
        const bool v0 = key < Nk, v1 = key + 1 < Nk;
        const float p0 = v0 ? fast_exp2(s[0] * sl2 - lse_a) : 0.f, p1 = v1 ? fast_exp2(s[1] * sl2 - lse_a) : 0.f;
        const float p2 = v0 ? fast_exp2(s[2] * sl2 - lse_b) : 0.f, p3 = v1 ? fast_exp2(s[3] * sl2 - lse_b) : 0.f;
        dsa[half * 2 + 0] = pack_bf16x2(p0 * (dp[0] - del_a), p1 * (dp[1] - del_a));
        dsa[half * 2 + 1] = pack_bf16x2(p2 * (dp[2] - del_b), p3 * (dp[3] - del_b));
      }
#pragma unroll
      for (int jd = 0; jd < DH / 8; ++jd) {
        uint32_t bfr[2];
        load_b_frag_t(bfr, sK, LDS, ks * 16, jd * 8, g, t);
        mma_bf16_16816(acc[jd], dsa, bfr);
      }
    }
    __syncthreads();   // buffer free for the prefetch of the next iteration
  }
  bf16* dQb = dQ + int64_t(b) * Nq * lddq + h * DH;
#pragma unroll
  for (int jd = 0; jd < DH / 8; ++jd) {
    const int c = jd * 8 + 2 * t;
    if (row_a < Nq) *reinterpret_cast<uint32_t*>(dQb + int64_t(row_a) * lddq + c) = pack_bf16x2(acc[jd][0] * scale, acc[jd][1] * scale);
    if (row_b < Nq) *reinterpret_cast<uint32_t*>(dQb + int64_t(row_b) * lddq + c) = pack_bf16x2(acc[jd][2] * scale, acc[jd][3] * scale);
  }
}

// =====================================================================================================================
// backward, part 2: dK, dV (key-stationary; works on transposed score tiles S^T = K Q^T)
// =====================================================================================================================
// factors of the transposed tile elements a thread holds: keys key_a, key_a + 8 (rows of S^T) x queries q, q + 1 (columns)
// -> {(key_a, q), (key_a, q+1), (key_a + 8, q), (key_a + 8, q+1)}, the order of an mma accumulator fragment
__device__ __forceinline__ float4 dropout_factor_t(const DropSite& d, uint64_t seed, uint64_t qrow, int key_a) {
  return make_float4(dropout_factor(d, seed, qrow, key_a), dropout_factor(d, seed, qrow + 1, key_a),
                     dropout_factor(d, seed, qrow, key_a + 8), dropout_factor(d, seed, qrow + 1, key_a + 8));
}

template <int DH, bool DROP>
__global__ void __launch_bounds__(ATT_THREADS) attn_bwd_dkv_kernel(const bf16* __restrict__ Q, int64_t ldq,
                                                                   const bf16* __restrict__ K, int64_t ldk,
                                                                   const bf16* __restrict__ V, int64_t ldv,
                                                                   const bf16* __restrict__ dO, int64_t lddo,
                                                                   const float* __restrict__ lse,
                                                                   const float* __restrict__ delta,
                                                                   bf16* __restrict__ dK, int64_t lddk,
                                                                   bf16* __restrict__ dV, int64_t lddv, int Nq, int Nk,
                                                                   int H, float scale, DropSite drop) {
  pdl_prologue();
  constexpr int LDS = DH + 8, LDT = ATT_CHUNK + 8;
  __shared__ __align__(16) bf16 sQb[2][ATT_CHUNK * LDS];
  __shared__ __align__(16) bf16 sdOb[2][ATT_CHUNK * LDS];
  __shared__ float sLseb[2][ATT_CHUNK], sDelb[2][ATT_CHUNK];
  bf16* sQ = sQb[0];      // the stationary K / V tiles are staged through buffer 0 first
  bf16* sdO = sdOb[0];

  const int k0 = blockIdx.x * ATT_ROWS, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const bf16* Qb = Q + int64_t(b) * Nq * ldq + h * DH;
  const bf16* Kb = K + int64_t(b) * Nk * ldk + h * DH;
  const bf16* Vb = V + int64_t(b) * Nk * ldv + h * DH;
  const bf16* dOb = dO + int64_t(b) * Nq * lddo + h * DH;
  const float* Lp = lse + (int64_t(b) * H + h) * Nq;
  const float* Dp = delta + (int64_t(b) * H + h) * Nq;

  // stationary K / V fragments (staged through sQ / sdO)
  uint32_t ka[DH / 16][4], va[DH / 16][4];
  load_chunk<DH, true, false>(sQ, nullptr, Kb, ldk, k0, Nk);
  load_chunk<DH, true, false>(sdO, nullptr, Vb, ldv, k0, Nk);
  __syncthreads();
#pragma unroll
  for (int kk = 0; kk < DH / 16; ++kk) {
    load_a_frag(ka[kk], sQ, LDS, warp * 16, kk * 16, g, t);
    load_a_frag(va[kk], sdO, LDS, warp * 16, kk * 16, g, t);
  }

  float dk[DH / 8][4], dv[DH / 8][4];
#pragma unroll
  for (int j = 0; j < DH / 8; ++j) {
    dk[j][0] = dk[j][1] = dk[j][2] = dk[j][3] = 0.f;
    dv[j][0] = dv[j][1] = dv[j][2] = dv[j][3] = 0.f;
  }
  const float sl2 = scale * LOG2E;
  uint64_t dseed = 0;
  const uint64_t dbase = (uint64_t(b) * H + h) * Nq;
  if constexpr (DROP) dseed = *drop.seed;

  // query chunks stream through two buffers: Q, dO rows and their lse / delta arrive by cp.async while the previous chunk
  // is consumed.  Rows past Nq are zero-filled: Q = dO = 0 and delta = 0 make their P and dS contributions vanish.
  auto issue_chunk = [&](int buf, int q0) {
    load_chunk_async<DH>(sQb[buf], Qb, ldq, q0, Nq);
    load_chunk_async<DH>(sdOb[buf], dOb, lddo, q0, Nq);
    if (threadIdx.x < ATT_CHUNK) {
      const int q = q0 + threadIdx.x;
      const bool ok = q < Nq;
      cp_async_4(&sLseb[buf][threadIdx.x], Lp + (ok ? q : 0), ok);
      cp_async_4(&sDelb[buf][threadIdx.x], Dp + (ok ? q : 0), ok);
    }
    cp_async_commit();
  };
  __syncthreads();          // all K / V fragments are in registers: buffer 0 may be overwritten
  issue_chunk(0, 0);
  for (int q0 = 0, it = 0; q0 < Nq; q0 += ATT_CHUNK, ++it) {
    sQ = sQb[it & 1];
    sdO = sdOb[it & 1];
    const float* sLse = sLseb[it & 1];
    const float* sDel = sDelb[it & 1];
    if (q0 + ATT_CHUNK < Nq) {
      issue_chunk((it + 1) & 1, q0 + ATT_CHUNK);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
#pragma unroll
    for (int qs = 0; qs < ATT_CHUNK / 16; ++qs) {
      uint32_t pa[4], dsa[4];
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int n0 = qs * 16 + half * 8;   // query columns n0 .. n0+7 of this chunk
        float s[4] = {0.f, 0.f, 0.f, 0.f}, dp[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int kk = 0; kk < DH / 16; ++kk) {
          uint32_t bq[2], bd[2];
          load_b_frag(bq, sQ, LDS, n0, kk * 16, g, t);
          load_b_frag(bd, sdO, LDS, n0, kk * 16, g, t);
          mma_bf16_16816(s, ka[kk], bq);    // S^T[key, q]
          mma_bf16_16816(dp, va[kk], bd);   // dP^T[key, q]
        }
        const int qc = n0 + 2 * t;
        const float l0 = sLse[qc] * LOG2E, l1 = sLse[qc + 1] * LOG2E, d0 = sDel[qc], d1 = sDel[qc + 1];
        const float p0 = fast_exp2(s[0] * sl2 - l0), p1 = fast_exp2(s[1] * sl2 - l1);
        const float p2 = fast_exp2(s[2] * sl2 - l0), p3 = fast_exp2(s[3] * sl2 - l1);
        if constexpr (DROP) {
          const float4 f = dropout_factor_t(drop, dseed, dbase + q0 + qc, k0 + warp * 16 + g);
          pa[half * 2 + 0] = pack_bf16x2(p0 * f.x, p1 * f.y);
          pa[half * 2 + 1] = pack_bf16x2(p2 * f.z, p3 * f.w);
          dp[0] *= f.x; dp[1] *= f.y; dp[2] *= f.z; dp[3] *= f.w;
        } else {
          pa[half * 2 + 0] = pack_bf16x2(p0, p1);
          pa[half * 2 + 1] = pack_bf16x2(p2, p3);
        }
        dsa[half * 2 + 0] = pack_bf16x2(p0 * (dp[0] - d0), p1 * (dp[1] - d1));
        dsa[half * 2 + 1] = pack_bf16x2(p2 * (dp[2] - d0), p3 * (dp[3] - d1));
      }
#pragma unroll
      for (int jd = 0; jd < DH / 8; ++jd) {
        uint32_t b1[2], b2[2];
        load_b_frag_t(b1, sdO, LDS, qs * 16, jd * 8, g, t);
        load_b_frag_t(b2, sQ, LDS, qs * 16, jd * 8, g, t);
        mma_bf16_16816(dv[jd], pa, b1);    // dV += P^T dO
        mma_bf16_16816(dk[jd], dsa, b2);   // dK += dS^T Q
      }
    }
    __syncthreads();   // buffer free for the prefetch of the next iteration
  }
  const int row_a = k0 + warp * 16 + g, row_b = row_a + 8;
  bf16* dKb = dK + int64_t(b) * Nk * lddk + h * DH;
  bf16* dVb = dV + int64_t(b) * Nk * lddv + h * DH;
#pragma unroll
  for (int jd = 0; jd < DH / 8; ++jd) {
    const int c = jd * 8 + 2 * t;
    if (row_a < Nk) {
      *reinterpret_cast<uint32_t*>(dKb + int64_t(row_a) * lddk + c) = pack_bf16x2(dk[jd][0] * scale, dk[jd][1] * scale);
      *reinterpret_cast<uint32_t*>(dVb + int64_t(row_a) * lddv + c) = pack_bf16x2(dv[jd][0], dv[jd][1]);
    }
    if (row_b < Nk) {
      *reinterpret_cast<uint32_t*>(dKb + int64_t(row_b) * lddk + c) = pack_bf16x2(dk[jd][2] * scale, dk[jd][3] * scale);
      *reinterpret_cast<uint32_t*>(dVb + int64_t(row_b) * lddv + c) = pack_bf16x2(dv[jd][2], dv[jd][3]);
    }
  }
}

// =====================================================================================================================
// fused backward for Nk <= 256: one CTA per (b, h) owns every key, so each score tile is computed once (5 matmuls instead
// of the 7 of the dQ + dK/dV pair above, and half the exp2) and dQ is written without atomics.
//
// Warp w owns keys [16w, 16w + 16) (keys padded to a multiple of 16, not 64); all of the head's K stays in shared memory
// and the warp's V rows are held as A fragments.  Query
// chunks of ATT_CHUNK rows (Q, dO, O, lse) stream through a cp.async double buffer.  Per chunk:
//   A  delta = rowsum(dO * O) from the staged chunk (replaces attn_delta_kernel)
//   B  every warp: S^T, dP^T for its keys, P and dS in registers, dV += P^T dO, dK += dS^T Q; dS^T (bf16) -> smem
//   C  dQ(chunk) = dS K from smem, spread over the warps in 16 x 16 output tiles, stored straight to global
// 16-query sub-tiles wholly past Nq are skipped.  Rows past Nq are zero-filled (Q = dO = O = 0, lse = 0): their P
// multiplies dO = 0 and their dS is 0.  Keys past Nk have K = V = 0 and P forced to 0.
// ptxas (sm_90a): 128 registers at dh 64, 124 at dh 32, no spills; the K A fragments are re-read from sK (which dQ needs
// anyway) instead of being held, which is what keeps dh 64 within 128.  At the bench shapes the dynamic shared memory is
// 88 KB (encoder, 7 warps: 2 CTAs per SM), 57 KB (decoder cross, 7 warps: 2) and 78 KB (decoder self, 13 warps: 1 CTA
// per SM, register-bound; capping dh 32 at 72 registers for 2 spills, see the table below).
// =====================================================================================================================
constexpr int FB_MAX_KEYS = 256;
constexpr int FB_LDD = ATT_CHUNK + 8;   // pitch of the dS^T tile [key][query] (144-byte rows: conflict-free ldmatrix)

template <int DH>
__host__ __device__ constexpr int fb_stream_elems() { return ATT_CHUNK * (DH + 8); }
// dynamic shared memory: sK [Nkp][DH+8] | sdS [Nkp][FB_LDD] (V is staged here first) | 2 x (Q, dO, O) | 2 x lse | delta
template <int DH>
__host__ __device__ constexpr size_t fb_smem_bytes(int Nkp) {
  return size_t(Nkp) * (DH + 8 + FB_LDD) * sizeof(bf16) + 6 * fb_stream_elems<DH>() * sizeof(bf16) +
         3 * ATT_CHUNK * sizeof(float);
}

template <int DH>
__device__ __forceinline__ void load_rows_async(bf16* s, const bf16* gbase, int64_t ld, int row0, int nrows, int rows_valid) {
  constexpr int LDS = DH + 8, VPR = DH / 8;
  for (int idx = threadIdx.x; idx < nrows * VPR; idx += blockDim.x) {
    const int r = idx / VPR, cv = idx % VPR;
    const bool ok = row0 + r < rows_valid;
    cp_async_16(s + r * LDS + cv * 8, gbase + int64_t(ok ? row0 + r : 0) * ld + cv * 8, ok);
  }
}

// A fragment (16 rows x 16 k) from smem stored transposed, s[k][row] (row contiguous)
__device__ __forceinline__ void load_a_frag_t(uint32_t (&a)[4], const bf16* s, int ld, int row0, int k0, int lane) {
  const int m = lane >> 3;
  const bf16* p = s + (k0 + (lane & 7) + (m >> 1) * 8) * ld + row0 + (m & 1) * 8;
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(a[0]), "=r"(a[1]), "=r"(a[2]), "=r"(a[3])
               : "r"(smem_u32(p)));
}

template <int DH, bool DROP>
__global__ void __launch_bounds__(FB_MAX_KEYS / 16 * 32) attn_bwd_fused_kernel(
    const bf16* __restrict__ Q, int64_t ldq, const bf16* __restrict__ K, int64_t ldk, const bf16* __restrict__ V,
    int64_t ldv, const bf16* __restrict__ O, int64_t ldo, const bf16* __restrict__ dO, int64_t lddo,
    const float* __restrict__ lse, bf16* __restrict__ dQ, int64_t lddq, bf16* __restrict__ dK, int64_t lddk,
    bf16* __restrict__ dV, int64_t lddv, int Nq, int Nk, int H, float scale, DropSite drop) {
  pdl_prologue();
  constexpr int LDS = DH + 8, SE = fb_stream_elems<DH>();
  static_assert(LDS <= FB_LDD, "V is staged in the dS^T tile");
  extern __shared__ __align__(16) unsigned char fb_smem[];
  const int nwarps = blockDim.x >> 5, Nkp = nwarps * 16;
  bf16* sK = reinterpret_cast<bf16*>(fb_smem);
  bf16* sdS = sK + Nkp * LDS;
  bf16* sStream = sdS + Nkp * FB_LDD;               // [buf][Q | dO | O]
  float* sLse = reinterpret_cast<float*>(sStream + 6 * SE);   // [buf][ATT_CHUNK]
  float* sDel = sLse + 2 * ATT_CHUNK;

  const int h = blockIdx.x % H, b = blockIdx.x / H;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const bf16* Qb = Q + int64_t(b) * Nq * ldq + h * DH;
  const bf16* Kb = K + int64_t(b) * Nk * ldk + h * DH;
  const bf16* Vb = V + int64_t(b) * Nk * ldv + h * DH;
  const bf16* Ob = O + int64_t(b) * Nq * ldo + h * DH;
  const bf16* dOb = dO + int64_t(b) * Nq * lddo + h * DH;
  const float* Lp = lse + (int64_t(b) * H + h) * Nq;

  auto issue_chunk = [&](int buf, int q0) {
    bf16* s = sStream + buf * 3 * SE;
    load_rows_async<DH>(s, Qb, ldq, q0, ATT_CHUNK, Nq);
    load_rows_async<DH>(s + SE, dOb, lddo, q0, ATT_CHUNK, Nq);
    load_rows_async<DH>(s + 2 * SE, Ob, ldo, q0, ATT_CHUNK, Nq);
    for (int i = threadIdx.x; i < ATT_CHUNK; i += blockDim.x) {
      const bool ok = q0 + i < Nq;
      cp_async_4(&sLse[buf * ATT_CHUNK + i], Lp + (ok ? q0 + i : 0), ok);
    }
    cp_async_commit();
  };
  load_rows_async<DH>(sK, Kb, ldk, 0, Nkp, Nk);
  load_rows_async<DH>(sdS, Vb, ldv, 0, Nkp, Nk);    // rows of pitch LDS inside the dS^T area, read once below
  issue_chunk(0, 0);
  cp_async_wait<0>();
  __syncthreads();
  uint32_t va[DH / 16][4];
#pragma unroll
  for (int kk = 0; kk < DH / 16; ++kk) load_a_frag(va[kk], sdS, LDS, warp * 16, kk * 16, g, t);
  float dk[DH / 8][4], dv[DH / 8][4];
#pragma unroll
  for (int j = 0; j < DH / 8; ++j) {
    dk[j][0] = dk[j][1] = dk[j][2] = dk[j][3] = 0.f;
    dv[j][0] = dv[j][1] = dv[j][2] = dv[j][3] = 0.f;
  }
  const float sl2 = scale * LOG2E;
  const bool key_a = warp * 16 + g < Nk, key_b = warp * 16 + g + 8 < Nk;
  uint64_t dseed = 0;
  const uint64_t dbase = (uint64_t(b) * H + h) * Nq;
  if constexpr (DROP) dseed = *drop.seed;

  for (int q0 = 0, it = 0; q0 < Nq; q0 += ATT_CHUNK, ++it) {
    const int buf = it & 1;
    // the other buffer was last read before the previous chunk's dS^T barrier, and V before the first one
    if (q0 + ATT_CHUNK < Nq) {
      issue_chunk(buf ^ 1, q0 + ATT_CHUNK);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();   // chunk landed; every warp is done with the previous chunk's dS^T and delta
    const bf16* sQ = sStream + buf * 3 * SE;
    const bf16* sdO = sQ + SE;
    const float* sL = sLse + buf * ATT_CHUNK;
    // A: delta
    for (int r = threadIdx.x; r < ATT_CHUNK; r += blockDim.x) {
      const bf16* o = sQ + 2 * SE + r * LDS;
      const bf16* d = sdO + r * LDS;
      float p = 0.f;
#pragma unroll
      for (int c = 0; c < DH; c += 8) {
        const uint4 ov = *reinterpret_cast<const uint4*>(o + c), dv4 = *reinterpret_cast<const uint4*>(d + c);
        const uint32_t* ou = reinterpret_cast<const uint32_t*>(&ov);
        const uint32_t* du = reinterpret_cast<const uint32_t*>(&dv4);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 x = unpack_bf16x2(ou[i]), y = unpack_bf16x2(du[i]);
          p += x.x * y.x + x.y * y.y;
        }
      }
      sDel[r] = p;
    }
    __syncthreads();
    // B: S^T, dP^T, dV, dK for this warp's keys
#pragma unroll
    for (int qs = 0; qs < ATT_CHUNK / 16; ++qs) {
      if (q0 + qs * 16 >= Nq) break;
      uint32_t pa[4], dsa[4];
      float s[2][4] = {}, dp[2][4] = {};
#pragma unroll
      for (int kk = 0; kk < DH / 16; ++kk) {
        uint32_t ka[4];   // K fragments come from sK (kept for dQ) rather than registers: no spills at dh 64
        load_a_frag(ka, sK, LDS, warp * 16, kk * 16, g, t);
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          uint32_t bq[2], bd[2];
          load_b_frag(bq, sQ, LDS, qs * 16 + half * 8, kk * 16, g, t);
          load_b_frag(bd, sdO, LDS, qs * 16 + half * 8, kk * 16, g, t);
          mma_bf16_16816(s[half], ka, bq);       // S^T[key, q]
          mma_bf16_16816(dp[half], va[kk], bd);  // dP^T[key, q]
        }
      }
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int qc = qs * 16 + half * 8 + 2 * t;
        const float l0 = sL[qc] * LOG2E, l1 = sL[qc + 1] * LOG2E, d0 = sDel[qc], d1 = sDel[qc + 1];
        const float p0 = key_a ? fast_exp2(s[half][0] * sl2 - l0) : 0.f, p1 = key_a ? fast_exp2(s[half][1] * sl2 - l1) : 0.f;
        const float p2 = key_b ? fast_exp2(s[half][2] * sl2 - l0) : 0.f, p3 = key_b ? fast_exp2(s[half][3] * sl2 - l1) : 0.f;
        if constexpr (DROP) {
          const float4 f = dropout_factor_t(drop, dseed, dbase + q0 + qc, warp * 16 + g);
          pa[half * 2 + 0] = pack_bf16x2(p0 * f.x, p1 * f.y);
          pa[half * 2 + 1] = pack_bf16x2(p2 * f.z, p3 * f.w);
          dp[half][0] *= f.x; dp[half][1] *= f.y; dp[half][2] *= f.z; dp[half][3] *= f.w;
        } else {
          pa[half * 2 + 0] = pack_bf16x2(p0, p1);
          pa[half * 2 + 1] = pack_bf16x2(p2, p3);
        }
        dsa[half * 2 + 0] = pack_bf16x2(p0 * (dp[half][0] - d0), p1 * (dp[half][1] - d1));
        dsa[half * 2 + 1] = pack_bf16x2(p2 * (dp[half][2] - d0), p3 * (dp[half][3] - d1));
      }
#pragma unroll
      for (int jd = 0; jd < DH / 8; ++jd) {
        uint32_t b1[2], b2[2];
        load_b_frag_t(b1, sdO, LDS, qs * 16, jd * 8, g, t);
        load_b_frag_t(b2, sQ, LDS, qs * 16, jd * 8, g, t);
        mma_bf16_16816(dv[jd], pa, b1);    // dV += P^T dO
        mma_bf16_16816(dk[jd], dsa, b2);   // dK += dS^T Q
      }
      bf16* r0 = sdS + (warp * 16 + g) * FB_LDD + qs * 16 + 2 * t;
      *reinterpret_cast<uint32_t*>(r0) = dsa[0];
      *reinterpret_cast<uint32_t*>(r0 + 8 * FB_LDD) = dsa[1];
      *reinterpret_cast<uint32_t*>(r0 + 8) = dsa[2];
      *reinterpret_cast<uint32_t*>(r0 + 8 * FB_LDD + 8) = dsa[3];
    }
    __syncthreads();
    // C: dQ(chunk) = dS K, one 16-query x 16-column tile per warp at a time
    for (int u = warp; u < (ATT_CHUNK / 16) * (DH / 16); u += nwarps) {
      const int qt = u / (DH / 16), c0 = (u % (DH / 16)) * 16;
      if (q0 + qt * 16 >= Nq) continue;
      float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
      for (int ks = 0; ks < Nkp; ks += 16) {
        uint32_t a[4], b0[2], b1[2];
        load_a_frag_t(a, sdS, FB_LDD, qt * 16, ks, lane);
        load_b_frag_t(b0, sK, LDS, ks, c0, g, t);
        load_b_frag_t(b1, sK, LDS, ks, c0 + 8, g, t);
        mma_bf16_16816(acc[0], a, b0);
        mma_bf16_16816(acc[1], a, b1);
      }
      const int row_a = q0 + qt * 16 + g, row_b = row_a + 8;
      bf16* dQb = dQ + int64_t(b) * Nq * lddq + h * DH;
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int c = c0 + j * 8 + 2 * t;
        if (row_a < Nq) *reinterpret_cast<uint32_t*>(dQb + int64_t(row_a) * lddq + c) = pack_bf16x2(acc[j][0] * scale, acc[j][1] * scale);
        if (row_b < Nq) *reinterpret_cast<uint32_t*>(dQb + int64_t(row_b) * lddq + c) = pack_bf16x2(acc[j][2] * scale, acc[j][3] * scale);
      }
    }
  }
  const int row_a = warp * 16 + g, row_b = row_a + 8;
  bf16* dKb = dK + int64_t(b) * Nk * lddk + h * DH;
  bf16* dVb = dV + int64_t(b) * Nk * lddv + h * DH;
#pragma unroll
  for (int jd = 0; jd < DH / 8; ++jd) {
    const int c = jd * 8 + 2 * t;
    if (row_a < Nk) {
      *reinterpret_cast<uint32_t*>(dKb + int64_t(row_a) * lddk + c) = pack_bf16x2(dk[jd][0] * scale, dk[jd][1] * scale);
      *reinterpret_cast<uint32_t*>(dVb + int64_t(row_a) * lddv + c) = pack_bf16x2(dv[jd][0], dv[jd][1]);
    }
    if (row_b < Nk) {
      *reinterpret_cast<uint32_t*>(dKb + int64_t(row_b) * lddk + c) = pack_bf16x2(dk[jd][2] * scale, dk[jd][3] * scale);
      *reinterpret_cast<uint32_t*>(dVb + int64_t(row_b) * lddv + c) = pack_bf16x2(dv[jd][2], dv[jd][3]);
    }
  }
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <int DH, bool DROP>
int launch_bwd_fused(const bf16* q, int64_t ldq, const bf16* k, int64_t ldk, const bf16* v, int64_t ldv, const bf16* o,
                     int64_t ldo, const bf16* d_o, int64_t lddo, const float* lse, bf16* dq, int64_t lddq, bf16* dk,
                     int64_t lddk, bf16* dv, int64_t lddv, int B, int H, int Nq, int Nk, float scale, DropSite drop,
                     cudaStream_t st) {
  auto kern = attn_bwd_fused_kernel<DH, DROP>;
  static bool configured = false;
  if (!configured) {
    MMAE_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(fb_smem_bytes<DH>(FB_MAX_KEYS))));
    configured = true;
  }
  const int nwarps = ceil_div(Nk, 16);
  launch_k(kern, dim3(B * H), dim3(nwarps * 32), fb_smem_bytes<DH>(nwarps * 16), st, q, ldq, k, ldk, v, ldv, o, ldo, d_o,
           lddo, lse, dq, lddq, dk, lddk, dv, lddv, Nq, Nk, H, scale, drop);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

unsigned delta_grid(int B, int Nq, int H, int dh) {
  const int64_t total = int64_t(B) * Nq * H * (dh / 8);
  return (unsigned)std::min<int64_t>((total + 255) / 256, int64_t(sm_count()) * 16);
}

// backward above FB_MAX_KEYS keys: delta, then dQ (query-stationary) and dK / dV (key-stationary)
template <int DH, bool DROP>
int launch_bwd_split(const bf16* q, int64_t ldq, const bf16* k, int64_t ldk, const bf16* v, int64_t ldv, const bf16* o,
                     int64_t ldo, const bf16* d_o, int64_t lddo, const float* lse, float* delta_ws, bf16* dq, int64_t lddq,
                     bf16* dk, int64_t lddk, bf16* dv, int64_t lddv, int B, int H, int Nq, int Nk, float scale,
                     DropSite drop, cudaStream_t st) {
  dim3 gq(ceil_div(Nq, ATT_ROWS), H, B), gk(ceil_div(Nk, ATT_ROWS), H, B);
  launch_k(attn_delta_kernel<DH>, delta_grid(B, Nq, H, DH), 256, 0, st, o, ldo, d_o, lddo, delta_ws, Nq, H, int64_t(B) * Nq);
  launch_k(attn_bwd_dq_kernel<DH, DROP>, gq, ATT_THREADS, 0, st, q, ldq, k, ldk, v, ldv, d_o, lddo, lse, delta_ws, dq, lddq,
           Nq, Nk, H, scale, drop);
  launch_k(attn_bwd_dkv_kernel<DH, DROP>, gk, ATT_THREADS, 0, st, q, ldq, k, ldk, v, ldv, d_o, lddo, lse, delta_ws, dk, lddk,
           dv, lddv, Nq, Nk, H, scale, drop);
  count_launch();
  count_launch();
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

template <int DH, bool DROP>
int launch_bwd(const bf16* q, int64_t ldq, const bf16* k, int64_t ldk, const bf16* v, int64_t ldv, const bf16* o,
               int64_t ldo, const bf16* d_o, int64_t lddo, const float* lse, float* delta_ws, bf16* dq, int64_t lddq,
               bf16* dk, int64_t lddk, bf16* dv, int64_t lddv, int B, int H, int Nq, int Nk, float scale, DropSite drop,
               cudaStream_t st) {
  if (Nk <= FB_MAX_KEYS)   // one fused kernel per (b, h); delta_ws is not used
    return launch_bwd_fused<DH, DROP>(q, ldq, k, ldk, v, ldv, o, ldo, d_o, lddo, lse, dq, lddq, dk, lddk, dv, lddv, B, H, Nq,
                                      Nk, scale, drop, st);
  return launch_bwd_split<DH, DROP>(q, ldq, k, ldk, v, ldv, o, ldo, d_o, lddo, lse, delta_ws, dq, lddq, dk, lddk, dv, lddv,
                                    B, H, Nq, Nk, scale, drop, st);
}

// keep bits of rows x cols elements of one site, 0 / 1 bytes (mmae_dropout_keep_mask)
__global__ void __launch_bounds__(256) dropout_keep_mask_kernel(DropSite drop, int64_t rows, int cols, uint8_t* __restrict__ out) {
  pdl_prologue();
  const uint64_t seed = *drop.seed;
  const int64_t n = rows * cols;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t r = i / cols;
    const int c = int(i - r * cols);
    out[i] = uint8_t(word_at(dropout_words(seed, drop.site, uint64_t(r), c), c & 3) < drop.thresh);
  }
}

}  // namespace
}  // namespace mmae

using namespace mmae;

// Kernel families, as a bit mask (the values keep the meaning they had on earlier architectures where Hopper has a
// counterpart): 1 = wgmma forward (attention_wgmma.cu) for <= 128 keys; 2 | 8 | 32 | 128 = wgmma forward for 129..256 keys;
// 4 | 64 = wgmma backward (any length); the forward above 256 keys and the backward without those bits use the warp-level
// mma.sync kernels of this file (bit 16 selected a persistent variant that has no Hopper kernel and is ignored).
// 0 = mma.sync kernels everywhere; their backward is the fused kernel up to 256 keys, delta + dQ + dK/dV above.
// Attention dropout (dropout_p > 0) runs the mma.sync kernels whatever the mask selects: the wgmma kernels have no dropout.
// Default 0 (env MMAE_ATTN_TC), from scripts/gpu_time_attention.py on one H100 80GB HBM3 at a 700 W power limit,
// MultiMAE-B bs 128, us per call (forward mma.sync / wgmma, backward mma.sync fused / wgmma; in brackets, from the same
// run, the forward before idle warps skipped their work and the delta + dQ + dK/dV backward the fused kernel replaced):
//   encoder 99 x 99, dh 64      46.8 (51.8) / 77.4    109.1 (155.4) / 340.1
//   decoder 196 x 99, dh 32     43.9 (53.0) / 48.5     74.1 (115.5) / 198.8
//   decoder 196 x 196, dh 32    65.6 (69.0) / 125.4   127.0 (180.1) / 333.1
// The wgmma kernels stage every tile with plain loads and no pipelining.  Also measured and not kept (400 W limit): the
// forward skipping the 16-key groups of its last key chunk that lie wholly past Nk (6 to 9 % slower at all three
// shapes), and the fused backward capped at 72 registers at dh 32 for 2 CTAs per SM (it spills: decoder self 4 %
// faster, decoder cross 8 % slower).
// A negative value restores the start-up default.
static int g_attn_tc = []() {
  const char* e = getenv("MMAE_ATTN_TC");
  return e ? atoi(e) : 0;
}();
static const int g_attn_tc_default = g_attn_tc;
extern "C" int mmae_attention_set_tc(int enable) {
  g_attn_tc = enable < 0 ? g_attn_tc_default : enable;
  return MMAE_OK;
}

// Dropout (dropout_p > 0) always runs the mma.sync kernels of this file, whatever MMAE_ATTN_TC selects: the wgmma kernels
// have no dropout.  At dropout_p = 0 the seed is not read and the kernels are those without dropout.
extern "C" int mmae_attention_forward(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                      void* o, int64_t ldo, float* lse, int B, int H, int Nq, int Nk, int head_dim,
                                      float scale, float dropout_p, const uint64_t* seed, void* stream) {
  MMAE_CHECK(q && k && v && o && B > 0 && H > 0 && Nq > 0 && Nk > 0, MMAE_ERR_ARG, "mmae_attention_forward: bad args");
  MMAE_CHECK(head_dim == 32 || head_dim == 64, MMAE_ERR_UNSUPPORTED, "mmae_attention_forward: head_dim %d (32|64)", head_dim);
  MMAE_CHECK(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && aligned16(q) && aligned16(k) &&
                 aligned16(v) && aligned16(o),
             MMAE_ERR_ARG, "mmae_attention_forward: 16-byte alignment / ld %% 8 required");
  MMAE_CHECK(dropout_p >= 0.f && dropout_p <= 1.f && (dropout_p == 0.f || seed), MMAE_ERR_ARG,
             "mmae_attention_forward: dropout p in [0, 1] and, when p > 0, a seed are required");
  const DropSite drop = make_drop_site(seed, MMAE_DROP_SITE_ATTN, dropout_p);
  dim3 grid(ceil_div(Nq, ATT_ROWS), H, B);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (!drop.seed && attn_wg_fwd_supported(Nk, head_dim) &&
      ((Nk <= 128 && (g_attn_tc & 1)) || (Nk > 128 && (g_attn_tc & (2 | 8 | 32 | 128)))))
    return attn_wg_forward(q, ldq, k, ldk, v, ldv, o, ldo, lse, B, H, Nq, Nk, head_dim, scale, st);
  const bf16 *qp = (const bf16*)q, *kp = (const bf16*)k, *vp = (const bf16*)v;
  auto kern = head_dim == 64 ? (drop.seed ? attn_fwd_kernel<64, true> : attn_fwd_kernel<64, false>)
                             : (drop.seed ? attn_fwd_kernel<32, true> : attn_fwd_kernel<32, false>);
  launch_k(kern, grid, ATT_THREADS, 0, st, qp, ldq, kp, ldk, vp, ldv, (bf16*)o, ldo, lse, Nq, Nk, H, scale, drop);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

extern "C" int mmae_attention_backward(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                                       int64_t ldv, const void* o, int64_t ldo, const void* d_o, int64_t lddo,
                                       const float* lse, float* delta_ws, void* dq, int64_t lddq, void* dk,
                                       int64_t lddk, void* dv, int64_t lddv, int B, int H, int Nq, int Nk,
                                       int head_dim, float scale, float dropout_p, const uint64_t* seed, void* stream) {
  MMAE_CHECK(q && k && v && o && d_o && lse && delta_ws && dq && dk && dv && B > 0 && H > 0 && Nq > 0 && Nk > 0,
             MMAE_ERR_ARG, "mmae_attention_backward: bad args");
  MMAE_CHECK(head_dim == 32 || head_dim == 64, MMAE_ERR_UNSUPPORTED, "mmae_attention_backward: head_dim %d (32|64)", head_dim);
  MMAE_CHECK(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && lddo % 8 == 0 && lddq % 8 == 0 &&
                 lddk % 8 == 0 && lddv % 8 == 0 && aligned16(q) && aligned16(k) && aligned16(v) && aligned16(o) &&
                 aligned16(d_o) && aligned16(dq) && aligned16(dk) && aligned16(dv),
             MMAE_ERR_ARG, "mmae_attention_backward: 16-byte alignment / ld %% 8 required");
  MMAE_CHECK(dropout_p >= 0.f && dropout_p <= 1.f && (dropout_p == 0.f || seed), MMAE_ERR_ARG,
             "mmae_attention_backward: dropout p in [0, 1] and, when p > 0, a seed are required");
  const DropSite drop = make_drop_site(seed, MMAE_DROP_SITE_ATTN, dropout_p);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const bf16 *qp = (const bf16*)q, *kp = (const bf16*)k, *vp = (const bf16*)v, *op = (const bf16*)o,
             *dop = (const bf16*)d_o;
  if (!drop.seed && (g_attn_tc & (4 | 64))) {   // wgmma backward (attention_wgmma.cu) behind the delta kernel
    if (head_dim == 64)
      launch_k(attn_delta_kernel<64>, delta_grid(B, Nq, H, 64), 256, 0, st, op, ldo, dop, lddo, delta_ws, Nq, H, int64_t(B) * Nq);
    else
      launch_k(attn_delta_kernel<32>, delta_grid(B, Nq, H, 32), 256, 0, st, op, ldo, dop, lddo, delta_ws, Nq, H, int64_t(B) * Nq);
    count_launch();
    MMAE_LAUNCH_OK();
    return attn_wg_backward(q, ldq, k, ldk, v, ldv, d_o, lddo, lse, delta_ws, dq, lddq, dk, lddk, dv, lddv, B, H, Nq, Nk,
                            head_dim, scale, st);
  }
  auto run = head_dim == 64 ? (drop.seed ? launch_bwd<64, true> : launch_bwd<64, false>)
                            : (drop.seed ? launch_bwd<32, true> : launch_bwd<32, false>);
  return run(qp, ldq, kp, ldk, vp, ldv, op, ldo, dop, lddo, lse, delta_ws, (bf16*)dq, lddq, (bf16*)dk, lddk, (bf16*)dv, lddv,
             B, H, Nq, Nk, scale, drop, st);
}

extern "C" int mmae_dropout_keep_mask(const uint64_t* seed, int site, int64_t rows, int cols, float p, void* out,
                                      void* stream) {
  MMAE_CHECK(seed && out && rows > 0 && cols > 0 && p >= 0.f && p <= 1.f, MMAE_ERR_ARG, "mmae_dropout_keep_mask: bad args");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (p == 0.f) {   // a site at p = 0 drops nothing
    MMAE_CUDA_OK(cudaMemsetAsync(out, 1, size_t(rows) * cols, st));
    return MMAE_OK;
  }
  const int64_t n = rows * cols;
  launch_k(dropout_keep_mask_kernel, (unsigned)std::min<int64_t>((n + 255) / 256, int64_t(sm_count()) * 16), 256, 0, st,
           make_drop_site(seed, site, p), rows, cols, static_cast<uint8_t*>(out));
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}
