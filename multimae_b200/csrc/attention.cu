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
template <int DH>
__global__ void __launch_bounds__(ATT_THREADS) attn_fwd_kernel(const bf16* __restrict__ Q, int64_t ldq,
                                                               const bf16* __restrict__ K, int64_t ldk,
                                                               const bf16* __restrict__ V, int64_t ldv,
                                                               bf16* __restrict__ O, int64_t ldo,
                                                               float* __restrict__ lse, int Nq, int Nk, int H,
                                                               float scale) {
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
    __syncthreads();   // every warp is done with this buffer before the next iteration's prefetch overwrites it
  }

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  const int row_a = q0 + warp * 16 + g, row_b = row_a + 8;
  const float inv0 = 1.0f / l_run[0], inv1 = 1.0f / l_run[1];
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
template <int DH>
__global__ void __launch_bounds__(ATT_THREADS) attn_bwd_dq_kernel(const bf16* __restrict__ Q, int64_t ldq,
                                                                  const bf16* __restrict__ K, int64_t ldk,
                                                                  const bf16* __restrict__ V, int64_t ldv,
                                                                  const bf16* __restrict__ dO, int64_t lddo,
                                                                  const float* __restrict__ lse,
                                                                  const float* __restrict__ delta,
                                                                  bf16* __restrict__ dQ, int64_t lddq, int Nq, int Nk,
                                                                  int H, float scale) {
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
template <int DH>
__global__ void __launch_bounds__(ATT_THREADS) attn_bwd_dkv_kernel(const bf16* __restrict__ Q, int64_t ldq,
                                                                   const bf16* __restrict__ K, int64_t ldk,
                                                                   const bf16* __restrict__ V, int64_t ldv,
                                                                   const bf16* __restrict__ dO, int64_t lddo,
                                                                   const float* __restrict__ lse,
                                                                   const float* __restrict__ delta,
                                                                   bf16* __restrict__ dK, int64_t lddk,
                                                                   bf16* __restrict__ dV, int64_t lddv, int Nq, int Nk,
                                                                   int H, float scale) {
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
        pa[half * 2 + 0] = pack_bf16x2(p0, p1);
        pa[half * 2 + 1] = pack_bf16x2(p2, p3);
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

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace
}  // namespace mmae

using namespace mmae;

// Kernel families, as a bit mask (the values keep the meaning they had on earlier architectures where Hopper has a
// counterpart): 1 = wgmma forward (attention_wgmma.cu) for <= 128 keys; 2 | 8 | 32 | 128 = wgmma forward for 129..256 keys;
// 4 | 64 = wgmma backward (any length); the forward above 256 keys and the backward without those bits use the warp-level
// mma.sync kernels of this file (bit 16 selected a persistent variant that has no Hopper kernel and is ignored).
// 0 = mma.sync kernels everywhere.
// Default 0 (env MMAE_ATTN_TC), from scripts/gpu_time_attention.py and bench.py on one H100 80GB HBM3 capped at 400 W,
// MultiMAE-B bs 128, us per call (forward mma.sync / wgmma, backward mma.sync / wgmma):
//   encoder 99 x 99, dh 64      55.3 / 77.4    165.3 / 337.9
//   decoder 196 x 99, dh 32     46.1 / 48.1    118.9 / 198.5
//   decoder 196 x 196, dh 32    72.7 / 122.3   193.2 / 331.5
// and the step: 44.5 ms (0), 47.8 ms (64: wgmma backward), 48.5 ms (195: wgmma forward + backward).  The wgmma kernels
// stage every tile with plain loads and no pipelining.  A negative value restores the start-up default.
static int g_attn_tc = []() {
  const char* e = getenv("MMAE_ATTN_TC");
  return e ? atoi(e) : 0;
}();
static const int g_attn_tc_default = g_attn_tc;
extern "C" int mmae_attention_set_tc(int enable) {
  g_attn_tc = enable < 0 ? g_attn_tc_default : enable;
  return MMAE_OK;
}

extern "C" int mmae_attention_forward(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                      void* o, int64_t ldo, float* lse, int B, int H, int Nq, int Nk, int head_dim,
                                      float scale, void* stream) {
  MMAE_CHECK(q && k && v && o && B > 0 && H > 0 && Nq > 0 && Nk > 0, MMAE_ERR_ARG, "mmae_attention_forward: bad args");
  MMAE_CHECK(head_dim == 32 || head_dim == 64, MMAE_ERR_UNSUPPORTED, "mmae_attention_forward: head_dim %d (32|64)", head_dim);
  MMAE_CHECK(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && aligned16(q) && aligned16(k) &&
                 aligned16(v) && aligned16(o),
             MMAE_ERR_ARG, "mmae_attention_forward: 16-byte alignment / ld %% 8 required");
  dim3 grid(ceil_div(Nq, ATT_ROWS), H, B);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (attn_wg_fwd_supported(Nk, head_dim) && ((Nk <= 128 && (g_attn_tc & 1)) || (Nk > 128 && (g_attn_tc & (2 | 8 | 32 | 128)))))
    return attn_wg_forward(q, ldq, k, ldk, v, ldv, o, ldo, lse, B, H, Nq, Nk, head_dim, scale, st);
  const bf16 *qp = (const bf16*)q, *kp = (const bf16*)k, *vp = (const bf16*)v;
  if (head_dim == 64)
    launch_k(attn_fwd_kernel<64>, grid, ATT_THREADS, 0, st, qp, ldq, kp, ldk, vp, ldv, (bf16*)o, ldo, lse, Nq, Nk, H, scale);
  else
    launch_k(attn_fwd_kernel<32>, grid, ATT_THREADS, 0, st, qp, ldq, kp, ldk, vp, ldv, (bf16*)o, ldo, lse, Nq, Nk, H, scale);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

static unsigned delta_grid(int B, int Nq, int H, int dh) {
  const int64_t total = int64_t(B) * Nq * H * (dh / 8);
  return (unsigned)std::min<int64_t>((total + 255) / 256, int64_t(sm_count()) * 16);
}

extern "C" int mmae_attention_backward(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                                       int64_t ldv, const void* o, int64_t ldo, const void* d_o, int64_t lddo,
                                       const float* lse, float* delta_ws, void* dq, int64_t lddq, void* dk,
                                       int64_t lddk, void* dv, int64_t lddv, int B, int H, int Nq, int Nk,
                                       int head_dim, float scale, void* stream) {
  MMAE_CHECK(q && k && v && o && d_o && lse && delta_ws && dq && dk && dv && B > 0 && H > 0 && Nq > 0 && Nk > 0,
             MMAE_ERR_ARG, "mmae_attention_backward: bad args");
  MMAE_CHECK(head_dim == 32 || head_dim == 64, MMAE_ERR_UNSUPPORTED, "mmae_attention_backward: head_dim %d (32|64)", head_dim);
  MMAE_CHECK(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && lddo % 8 == 0 && lddq % 8 == 0 &&
                 lddk % 8 == 0 && lddv % 8 == 0 && aligned16(q) && aligned16(k) && aligned16(v) && aligned16(o) &&
                 aligned16(d_o) && aligned16(dq) && aligned16(dk) && aligned16(dv),
             MMAE_ERR_ARG, "mmae_attention_backward: 16-byte alignment / ld %% 8 required");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const bf16 *qp = (const bf16*)q, *kp = (const bf16*)k, *vp = (const bf16*)v, *op = (const bf16*)o,
             *dop = (const bf16*)d_o;
  dim3 gq(ceil_div(Nq, ATT_ROWS), H, B), gk(ceil_div(Nk, ATT_ROWS), H, B);
  if (g_attn_tc & (4 | 64)) {   // wgmma backward (attention_wgmma.cu) behind the delta kernel
    if (head_dim == 64)
      launch_k(attn_delta_kernel<64>, delta_grid(B, Nq, H, 64), 256, 0, st, op, ldo, dop, lddo, delta_ws, Nq, H, int64_t(B) * Nq);
    else
      launch_k(attn_delta_kernel<32>, delta_grid(B, Nq, H, 32), 256, 0, st, op, ldo, dop, lddo, delta_ws, Nq, H, int64_t(B) * Nq);
    count_launch();
    MMAE_LAUNCH_OK();
    return attn_wg_backward(q, ldq, k, ldk, v, ldv, d_o, lddo, lse, delta_ws, dq, lddq, dk, lddk, dv, lddv, B, H, Nq, Nk,
                            head_dim, scale, st);
  }
  if (head_dim == 64) {
    launch_k(attn_delta_kernel<64>, delta_grid(B, Nq, H, 64), 256, 0, st, op, ldo, dop, lddo, delta_ws, Nq, H, int64_t(B) * Nq);
    launch_k(attn_bwd_dq_kernel<64>, gq, ATT_THREADS, 0, st, qp, ldq, kp, ldk, vp, ldv, dop, lddo, lse, delta_ws, (bf16*)dq,
                                                       lddq, Nq, Nk, H, scale);
    launch_k(attn_bwd_dkv_kernel<64>, gk, ATT_THREADS, 0, st, qp, ldq, kp, ldk, vp, ldv, dop, lddo, lse, delta_ws, (bf16*)dk,
                                                        lddk, (bf16*)dv, lddv, Nq, Nk, H, scale);
  } else {
    launch_k(attn_delta_kernel<32>, delta_grid(B, Nq, H, 32), 256, 0, st, op, ldo, dop, lddo, delta_ws, Nq, H, int64_t(B) * Nq);
    launch_k(attn_bwd_dq_kernel<32>, gq, ATT_THREADS, 0, st, qp, ldq, kp, ldk, vp, ldv, dop, lddo, lse, delta_ws, (bf16*)dq,
                                                       lddq, Nq, Nk, H, scale);
    launch_k(attn_bwd_dkv_kernel<32>, gk, ATT_THREADS, 0, st, qp, ldq, kp, ldk, vp, ldv, dop, lddo, lse, delta_ws, (bf16*)dk,
                                                        lddk, (bf16*)dv, lddv, Nq, Nk, H, scale);
  }
  count_launch();
  count_launch();
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}
