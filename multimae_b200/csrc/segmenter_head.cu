// Segmenter head of semantic-segmentation fine-tuning: SegmenterMaskTransformerAdapter.forward
// (multimae/output_adapters.py:450-478):
//   x = cat(proj_dec(cat_t encoder_tokens[:, task t]), cls_emb)       [B, n + K, E]: n patch tokens, then one token per class
//   x = blocks(x)                                                     ordinary transformer Blocks (mmae_block_*)
//   x = decoder_norm(x)
//   P = patch_proj(x[:, :n]),  C = classes_proj(x[:, n:])             Linear E -> E, no bias
//   masks = normalize(P) @ normalize(C)^T                             cosine of every (patch, class) pair, [B, n, K]
//   masks = mask_norm(masks)                                          LayerNorm over the CLASS axis (width K)
//   out = interpolate("b (nh nw) k -> b k nh nw", (H, W), bilinear)
//
// Entry points:
//   proj : mmae_convnext_proj_forward (token gather + proj_dec GEMM with bias) into a [B*n, E] scratch, then
//          seg_assemble_kernel writes the [B, n + K, E] sequence (patch rows, then cls_emb).  Backward: seg_unassemble_kernel
//          (patch rows back to [B*n, E]), seg_colsum_add_kernel (dcls_emb[k] += sum_b dseq[b, n + k], fixed order) and
//          mmae_convnext_proj_backward.
//   mask : seg_mask_kernel<BN, false> - the fused cosine mask + class LayerNorm.  One CTA owns 64 patch rows of one sample
//          and all K classes: P and C tiles stream through a 3-stage cp.async ring in chunks of 32 columns of E, the product
//          accumulates on mma.sync.m16n8k16 bf16 (each warp 16 rows x all classes, so a row's statistics stay in one quad),
//          and the epilogue scales by 1 / max(|p_i|, 1e-12) and 1 / max(|c_j|, 1e-12), normalises over the classes and
//          writes the fp32 class map [B*n, Kp] once (Kp = round_up(K, 8), pad columns zero).
//          Backward: seg_mask_kernel<BN, true> recomputes the product tile, applies the LayerNorm backward and leaves
//            Gs[i, j] = dM[i, j] rp_i rc_j (bf16), t_i = sum_j dM[i, j] M[i, j], and one partial row per CTA of
//            u_j = sum_i dM[i, j] M[i, j], dgamma_j and dbeta_j (summed in a fixed order afterwards: no atomics);
//          seg_dproj_kernel<false>: dP_b = Gs_b C_b - rp_i^2 t_i P_b      ([n, K] x [K, E], normalise backward in the epilogue)
//          seg_dproj_kernel<true> : dC_b = Gs_b^T P_b - rc_j^2 u_j C_b    ([K, n] x [n, E])
//          with y = x r, dx = (dy - y (y . dy)) r  and  y_i . dy_i = t_i  (u_j for the classes).
//   tail : mmae_layernorm_forward over all B (n + K) rows, seg_rows_kernel<false> (patch rows and class rows into two
//          contiguous bf16 matrices), the two projection GEMMs (fp32 out), seg_rownorm_kernel (bf16 copy + 1 / max(norm,
//          1e-12) per row), the mask kernel, the ConvNeXt head's bilinear upsample (s = 1).  Backward in reverse; the two
//          weight-gradient GEMMs accumulate with the library's split-K atomics, everything else is free of atomics, so the
//          input gradient, dcls_emb and the mask_norm gradients are bitwise repeatable.
//
// ptxas (sm_90a, CUDA 12.9), registers / static + dynamic shared memory, no spills in any of them (BN = the accumulator
// width that holds Kp: 64, 160 or 256):
//   seg_mask_kernel<64, false>  96 / 1024 + 30720 B    <160, false> 143 / 2560 + 53760 B    <256, false> 255 / 4096 + 76800 B
//   seg_mask_kernel<64, true>   80 /  512 + 30720 B    <160, true>  167 / 1280 + 53760 B    <256, true>  238 / 2048 + 76800 B
//   seg_dproj_kernel<false>    126 / 41472 B           seg_dproj_kernel<true> 127 / 39936 B
// The products run on HMMA.16816.F32.BF16.
#include <cstring>

#include "internal.h"

namespace mmae {
namespace {

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

#define RUN(expr)                   \
  do {                              \
    int _rc = (expr);               \
    if (_rc != MMAE_OK) return _rc; \
  } while (0)

int round8(int c) { return (c + 7) / 8 * 8; }
bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <typename K, typename... A>
int launch(K kernel, dim3 grid, dim3 block, size_t smem, void* st, A... args) {
  launch_k(kernel, grid, block, smem, reinterpret_cast<cudaStream_t>(st), args...);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

// ------------------------------------------------------------------------------------------------ row movers
// seq[b, r, :] = r < n ? tmp[b*n + r, :] : cls_emb[r - n, :]
__global__ void __launch_bounds__(256) seg_assemble_kernel(const float* __restrict__ tmp, const float* __restrict__ cls_emb,
                                                           int n, int K, int E, float* __restrict__ seq) {
  pdl_prologue();
  const int row = blockIdx.x, b = row / (n + K), r = row % (n + K);
  const float4* src = reinterpret_cast<const float4*>(r < n ? tmp + (int64_t(b) * n + r) * E : cls_emb + int64_t(r - n) * E);
  float4* dst = reinterpret_cast<float4*>(seq + int64_t(row) * E);
  for (int c = threadIdx.x; c < E / 4; c += blockDim.x) dst[c] = __ldg(src + c);
}

// tmp[b*n + t, :] = dseq[b, t, :]  (the patch rows)
__global__ void __launch_bounds__(256) seg_unassemble_kernel(const float* __restrict__ dseq, int n, int K, int E,
                                                             float* __restrict__ tmp) {
  pdl_prologue();
  const int row = blockIdx.x, b = row / n, t = row % n;
  const float4* src = reinterpret_cast<const float4*>(dseq + (int64_t(b) * (n + K) + t) * E);
  float4* dst = reinterpret_cast<float4*>(tmp + int64_t(row) * E);
  for (int c = threadIdx.x; c < E / 4; c += blockDim.x) dst[c] = __ldg(src + c);
}

// dst[c] += sum_r src[r * ld + c], r ascending (bitwise repeatable)
__global__ void __launch_bounds__(256) seg_colsum_add_kernel(const float* __restrict__ src, int rows, int64_t ld, int cols,
                                                             float* __restrict__ dst) {
  pdl_prologue();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  float s = 0.f;
  for (int r = 0; r < rows; ++r) s += __ldg(src + int64_t(r) * ld + c);
  dst[c] += s;
}

// Row r = b*(n+K) + q of the [B, n + K, E] bf16 sequence <-> row (q < n ? b*n + q : B*n + b*K + q - n) of the compact matrix
// that holds all patch rows, then all class rows.  MERGE = false: sequence -> compact; true: compact -> sequence.
template <bool MERGE>
__global__ void __launch_bounds__(128) seg_rows_kernel(bf16* __restrict__ seq, bf16* __restrict__ compact, int B, int n, int K,
                                                       int E) {
  pdl_prologue();
  const int row = blockIdx.x, b = row / (n + K), q = row % (n + K);
  const int64_t crow = q < n ? int64_t(b) * n + q : int64_t(B) * n + int64_t(b) * K + q - n;
  uint4* s = reinterpret_cast<uint4*>(seq + int64_t(row) * E);
  uint4* c = reinterpret_cast<uint4*>(compact + crow * E);
  for (int i = threadIdx.x; i < E / 8; i += blockDim.x) {
    if (MERGE) s[i] = c[i];
    else c[i] = s[i];
  }
}

// one warp per row: dst = bf16(src), r = 1 / max(||src||_2, 1e-12)   (F.normalize's denominator)
__global__ void __launch_bounds__(256) seg_rownorm_kernel(const float* __restrict__ src, int rows, int E, bf16* __restrict__ dst,
                                                          float* __restrict__ r) {
  pdl_prologue();
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float4* s = reinterpret_cast<const float4*>(src + int64_t(row) * E);
  uint2* d = reinterpret_cast<uint2*>(dst + int64_t(row) * E);
  float ss = 0.f;
  for (int i = lane_id(); i < E / 4; i += 32) {
    const float4 v = __ldg(s + i);
    ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    d[i] = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  }
  ss = warp_sum(ss);
  if (lane_id() == 0) r[row] = 1.f / fmaxf(sqrtf(ss), 1e-12f);
}

// ------------------------------------------------------------------------------------------------ mma.sync mainloop
constexpr int SG_BM = 64, SG_BK = 32, SG_STAGES = 3, SG_THREADS = 128;

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  const int bytes = valid ? 16 : 0;                  // 0: nothing is read, the 16 bytes are zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <bool TRANS>
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  if (TRANS)
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
  else
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// [R][CC] tile of a row-major bf16 matrix (rows x cols valid, cols a multiple of 8) at (r0, c0) -> shared memory with rows
// CC + 8 elements apart (conflict-free ldmatrix); everything outside the matrix is zero-filled
template <int R, int CC>
__device__ __forceinline__ void load_tile(bf16* sm, const bf16* __restrict__ g, int ld, int r0, int c0, int rows, int cols) {
  constexpr int V = CC / 8;
  for (int i = threadIdx.x; i < R * V; i += SG_THREADS) {
    const int r = i / V, v = i % V, gr = r0 + r, gc = c0 + v * 8;
    const bool ok = gr < rows && gc < cols;
    cp_async16(smem_u32(sm + r * (CC + 8) + v * 8), ok ? g + gr * ld + gc : g, ok);
  }
}

template <int BN, bool AT, bool BT>
struct SgTile {
  static constexpr int A_ELEMS = AT ? SG_BK * (SG_BM + 8) : SG_BM * (SG_BK + 8);
  static constexpr int B_ELEMS = BT ? SG_BK * (BN + 8) : BN * (SG_BK + 8);
  static constexpr int STAGE = A_ELEMS + B_ELEMS;
  static constexpr size_t BYTES = size_t(SG_STAGES) * STAGE * sizeof(bf16);
};

// acc[j][.] (m16n8 tile j of warp w: rows m0 + 16 w .. + 15, columns n0 + 8 j .. + 7) = A[M, K] B over the whole K.
//   AT = false: A is stored [M][K] (K contiguous);  true: [K][M]
//   BT = false: B is stored [N][K] (K contiguous);  true: [K][N]
// Fragment layout of mma.m16n8k16: thread (g = lane / 4, tg = lane % 4) holds rows g, g + 8 and columns 2 tg, 2 tg + 1.
template <int BN, bool AT, bool BT>
__device__ __forceinline__ void sg_mainloop(float (&acc)[BN / 8][4], bf16* smem, const bf16* __restrict__ A, int lda,
                                            const bf16* __restrict__ Bm, int ldb, int M, int N, int K, int m0, int n0) {
  using T = SgTile<BN, AT, BT>;
  constexpr int SA = AT ? SG_BM + 8 : SG_BK + 8, SB = BT ? BN + 8 : SG_BK + 8;
  const int nk = (K + SG_BK - 1) / SG_BK;
  const int lane = lane_id(), wm0 = (threadIdx.x >> 5) * 16, mat = lane >> 3, l8 = lane & 7;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[j][e] = 0.f;

  auto issue = [&](int kb) {
    if (kb < nk) {
      bf16* sa = smem + (kb % SG_STAGES) * T::STAGE;
      bf16* sb = sa + T::A_ELEMS;
      const int k0 = kb * SG_BK;
      if (AT) load_tile<SG_BK, SG_BM>(sa, A, lda, k0, m0, K, M);
      else load_tile<SG_BM, SG_BK>(sa, A, lda, m0, k0, M, K);
      if (BT) load_tile<SG_BK, BN>(sb, Bm, ldb, k0, n0, K, N);
      else load_tile<BN, SG_BK>(sb, Bm, ldb, n0, k0, N, K);
    }
    cp_async_commit();
  };
#pragma unroll
  for (int s = 0; s < SG_STAGES - 1; ++s) issue(s);
  for (int kb = 0; kb < nk; ++kb) {
    cp_async_wait<SG_STAGES - 2>();
    __syncthreads();                       // stage kb has landed; stage kb - 1 is no longer read by anyone
    issue(kb + SG_STAGES - 1);
    const bf16* sa = smem + (kb % SG_STAGES) * T::STAGE;
    const bf16* sb = sa + T::A_ELEMS;
#pragma unroll
    for (int kk = 0; kk < SG_BK; kk += 16) {
      uint32_t a[4];
      if (AT) ldmatrix_x4<true>(a, smem_u32(sa + (kk + (mat >> 1) * 8 + l8) * SA + wm0 + (mat & 1) * 8));
      else ldmatrix_x4<false>(a, smem_u32(sa + (wm0 + (mat & 1) * 8 + l8) * SA + kk + (mat >> 1) * 8));
#pragma unroll
      for (int j = 0; j < BN / 8; j += 2) {
        uint32_t b[4];                     // (tile j, k lo), (tile j, k hi), (tile j + 1, k lo), (tile j + 1, k hi)
        if (BT) ldmatrix_x4<true>(b, smem_u32(sb + (kk + (mat & 1) * 8 + l8) * SB + j * 8 + (mat >> 1) * 8));
        else ldmatrix_x4<false>(b, smem_u32(sb + (j * 8 + (mat >> 1) * 8 + l8) * SB + kk + (mat & 1) * 8));
        mma_bf16(acc[j], a, b[0], b[1]);
        mma_bf16(acc[j + 1], a, b[2], b[3]);
      }
    }
  }
  cp_async_wait<0>();
}

__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}
// sum over the 8 row groups of a warp (lanes with equal lane % 4)
__device__ __forceinline__ float rowgroup_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  v += __shfl_xor_sync(0xffffffffu, v, 8);
  v += __shfl_xor_sync(0xffffffffu, v, 16);
  return v;
}

// ------------------------------------------------------------------------------------------------ cosine mask + class LN
struct MaskArgs {
  const bf16 *P, *C;             // [B*n, E], [B*K, E]
  const float *rp, *rc;          // [B*n], [B*K]
  const float *gamma, *beta;     // mask_norm [K]
  float eps;
  int n, K, Kp, E, tiles;        // tiles = ceil(n / 64)
  float *cmap, *mean, *rstd;     // forward: written; backward: mean / rstd read
  const float* dcmap;            // backward: [B*n, Kp]
  bf16* Gs;                      // backward: [B*n, Kp]
  float *t, *part;               // backward: [B*n], [B*tiles][3][Kp] (u, dgamma, dbeta)
};

// grid (tiles, B).  BN >= Kp: the accumulator tile of a warp is 16 x BN.
template <int BN, bool BWD>
__global__ void __launch_bounds__(SG_THREADS) seg_mask_kernel(MaskArgs a) {
  pdl_prologue();
  extern __shared__ __align__(16) uint8_t sg_smem[];
  __shared__ float s_rc[BN], s_gamma[BN], s_beta[BN], s_valid[BN];      // zero in the pad columns K..BN-1
  const int b = blockIdx.y, m0 = blockIdx.x * SG_BM, n = a.n, K = a.K, Kp = a.Kp;
  for (int c = threadIdx.x; c < BN; c += SG_THREADS) {
    s_rc[c] = c < K ? __ldg(a.rc + int64_t(b) * K + c) : 0.f;
    s_gamma[c] = c < K ? __ldg(a.gamma + c) : 0.f;
    s_beta[c] = c < K && !BWD ? __ldg(a.beta + c) : 0.f;
    s_valid[c] = c < K ? 1.f : 0.f;
  }
  float acc[BN / 8][4];
  sg_mainloop<BN, false, false>(acc, reinterpret_cast<bf16*>(sg_smem), a.P + int64_t(b) * n * a.E, a.E,
                                a.C + int64_t(b) * K * a.E, a.E, n, K, a.E, m0, 0);
  const int lane = lane_id(), warp = threadIdx.x >> 5, g = lane >> 2, tg = lane & 3;
  const float invK = 1.f / float(K);
  int row[2];
  bool ok[2];
  float rp[2], mean[2], rstd[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    row[h] = m0 + warp * 16 + g + 8 * h;
    ok[h] = row[h] < n;
    rp[h] = ok[h] ? __ldg(a.rp + int64_t(b) * n + row[h]) : 0.f;
  }
  __syncthreads();               // the tiles are free (the backward reuses them), and no epilogue load is hoisted into the loop
  // masks = S rp_i rc_j (zero in the pad columns: s_rc is zero there)
#pragma unroll
  for (int j = 0; j < BN / 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[j][e] *= rp[e >> 1] * s_rc[j * 8 + tg * 2 + (e & 1)];

  if (!BWD) {
    // one row at a time: mean, variance around it, then the row of the class map (gamma and beta are zero in the pad
    // columns, so those are written as zeros)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float s = 0.f, q = 0.f;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) s += acc[j][2 * h] + acc[j][2 * h + 1];
      const float mu = quad_sum(s) * invK;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float d = (acc[j][2 * h + e] - mu) * s_valid[j * 8 + tg * 2 + e];
          q += d * d;
        }
      const float rs = rsqrtf(quad_sum(q) * invK + a.eps);
      const int r = m0 + warp * 16 + g + 8 * h;
      if (r < n) {
        if (tg == 0) {
          a.mean[b * n + r] = mu;
          a.rstd[b * n + r] = rs;
        }
        float* orow = a.cmap + int64_t(b * n + r) * Kp + tg * 2;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          if (j * 8 < Kp) {
            const int c = j * 8 + tg * 2;
            float2 y;
            y.x = (acc[j][2 * h] - mu) * rs * s_gamma[c] + s_beta[c];
            y.y = (acc[j][2 * h + 1] - mu) * rs * s_gamma[c + 1] + s_beta[c + 1];
            *reinterpret_cast<float2*>(orow + j * 8) = y;
          }
        }
      }
    }
  } else {
    // LayerNorm backward over the class axis: xhat = (M - mean) rstd, dxh = dy gamma,
    // dM = rstd (dxh - mean_j(dxh) - xhat mean_j(dxh xhat))
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mean[h] = ok[h] ? __ldg(a.mean + int64_t(b) * n + row[h]) : 0.f;
      rstd[h] = ok[h] ? __ldg(a.rstd + int64_t(b) * n + row[h]) : 0.f;
    }
    float s1[2] = {0.f, 0.f}, s2[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int c = j * 8 + tg * 2;
      if (c < Kp) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float2 dy = ok[h] ? __ldg(reinterpret_cast<const float2*>(a.dcmap + (int64_t(b) * n + row[h]) * Kp + c))
                                  : make_float2(0.f, 0.f);
          const float d0 = dy.x * s_gamma[c], d1 = dy.y * s_gamma[c + 1];      // gamma is zero in the pad columns
          s1[h] += d0 + d1;
          s2[h] += d0 * (acc[j][2 * h] - mean[h]) * rstd[h] + d1 * (acc[j][2 * h + 1] - mean[h]) * rstd[h];
        }
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      s1[h] = quad_sum(s1[h]) * invK;
      s2[h] = quad_sum(s2[h]) * invK;
    }
    float* red = reinterpret_cast<float*>(sg_smem);        // [4 warps][3][BN]; the mainloop's tiles are no longer read
    float tsum[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int c = j * 8 + tg * 2;
      if (c < Kp) {                                        // uniform over the warp
        float u[2] = {0.f, 0.f}, dg[2] = {0.f, 0.f}, db[2] = {0.f, 0.f};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float2 dy = ok[h] ? __ldg(reinterpret_cast<const float2*>(a.dcmap + (int64_t(b) * n + row[h]) * Kp + c))
                                  : make_float2(0.f, 0.f);
          float gs[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float m = acc[j][2 * h + e], xh = (m - mean[h]) * rstd[h], dyv = e ? dy.y : dy.x;
            const bool valid = c + e < K;
            const float dm = valid ? rstd[h] * (dyv * s_gamma[c + e] - s1[h] - xh * s2[h]) : 0.f;
            tsum[h] += dm * m;
            u[e] += dm * m;
            dg[e] += valid ? dyv * xh : 0.f;
            db[e] += valid ? dyv : 0.f;
            gs[e] = dm * rp[h] * s_rc[c + e];
          }
          if (ok[h]) *reinterpret_cast<uint32_t*>(a.Gs + (int64_t(b) * n + row[h]) * Kp + c) = pack_bf16x2(gs[0], gs[1]);
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          u[e] = rowgroup_sum(u[e]);
          dg[e] = rowgroup_sum(dg[e]);
          db[e] = rowgroup_sum(db[e]);
          if (g == 0) {
            red[(warp * 3 + 0) * BN + c + e] = u[e];
            red[(warp * 3 + 1) * BN + c + e] = dg[e];
            red[(warp * 3 + 2) * BN + c + e] = db[e];
          }
        }
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      tsum[h] = quad_sum(tsum[h]);
      if (ok[h] && tg == 0) a.t[int64_t(b) * n + row[h]] = tsum[h];
    }
    __syncthreads();
    float* out = a.part + (int64_t(b) * a.tiles + blockIdx.x) * 3 * Kp;
    for (int i = threadIdx.x; i < 3 * Kp; i += SG_THREADS) {
      const int which = i / Kp, c = i % Kp;
      out[i] = (red[(0 * 3 + which) * BN + c] + red[(1 * 3 + which) * BN + c]) +
               (red[(2 * 3 + which) * BN + c] + red[(3 * 3 + which) * BN + c]);
    }
  }
}

// Normalise backward around the two per-sample products.  grid (E / 128, row tiles, B).
//   CLASSES = false: rows = patches i of sample b:  out[i, :] = sum_j Gs[i, j] C[j, :] - rp_i^2 t_i P[i, :]
//   CLASSES = true : rows = classes j of sample b:  out[j, :] = sum_i Gs[i, j] P[i, :] - rc_j^2 u_j C[j, :]
constexpr int DP_BN = 128;
struct DprojArgs {
  const bf16 *P, *C, *Gs;
  const float *rp, *rc, *t, *part;
  int n, K, Kp, E, tiles;
  bf16 *dP, *dC;                 // [B*n, E], [B*K, E]
};
template <bool CLASSES>
__global__ void __launch_bounds__(SG_THREADS) seg_dproj_kernel(DprojArgs a) {
  pdl_prologue();
  extern __shared__ __align__(16) uint8_t sg_smem[];
  const int b = blockIdx.z, m0 = blockIdx.y * SG_BM, n0 = blockIdx.x * DP_BN, n = a.n, K = a.K, Kp = a.Kp, E = a.E;
  const bf16* Pb = a.P + int64_t(b) * n * E;
  const bf16* Cb = a.C + int64_t(b) * K * E;
  const bf16* Gb = a.Gs + int64_t(b) * n * Kp;
  float acc[DP_BN / 8][4];
  if (CLASSES) sg_mainloop<DP_BN, true, true>(acc, reinterpret_cast<bf16*>(sg_smem), Gb, Kp, Pb, E, Kp, E, n, m0, n0);
  else sg_mainloop<DP_BN, false, true>(acc, reinterpret_cast<bf16*>(sg_smem), Gb, Kp, Cb, E, n, E, K, m0, n0);
  const int lane = lane_id(), warp = threadIdx.x >> 5, g = lane >> 2, tg = lane & 3;
  const int rows = CLASSES ? K : n;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = m0 + warp * 16 + g + 8 * h;
    if (r >= rows) continue;
    float coef;
    if (CLASSES) {
      float u = 0.f;
      for (int tl = 0; tl < a.tiles; ++tl) u += __ldg(a.part + (int64_t(b) * a.tiles + tl) * 3 * Kp + r);
      const float rc = __ldg(a.rc + int64_t(b) * K + r);
      coef = rc * rc * u;
    } else {
      const float rp = __ldg(a.rp + int64_t(b) * n + r);
      coef = rp * rp * __ldg(a.t + int64_t(b) * n + r);
    }
    const bf16* self = (CLASSES ? Cb : Pb) + int64_t(r) * E;
    bf16* out = (CLASSES ? a.dC + int64_t(b) * K * E : a.dP + int64_t(b) * n * E) + int64_t(r) * E;
#pragma unroll
    for (int j = 0; j < DP_BN / 8; ++j) {
      const int c = n0 + j * 8 + tg * 2;
      if (c < E) {
        const float2 x = unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(self + c)));
        *reinterpret_cast<uint32_t*>(out + c) = pack_bf16x2(acc[j][2 * h] - coef * x.x, acc[j][2 * h + 1] - coef * x.y);
      }
    }
  }
}

template <typename Kern>
int opt_in_smem(Kern kernel, size_t bytes) {
  if (bytes > 48 * 1024) MMAE_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return MMAE_OK;
}

template <int BN, bool BWD>
int launch_mask(const MaskArgs& a, int B, void* stream) {
  const size_t bytes = SgTile<BN, false, false>::BYTES;            // >= the backward's 4 x 3 x BN floats
  RUN(opt_in_smem(seg_mask_kernel<BN, BWD>, bytes));
  return launch(seg_mask_kernel<BN, BWD>, dim3(a.tiles, B), dim3(SG_THREADS), bytes, stream, a);
}
template <bool BWD>
int launch_mask_any(const MaskArgs& a, int B, void* stream) {
  if (a.Kp <= 64) return launch_mask<64, BWD>(a, B, stream);
  if (a.Kp <= 160) return launch_mask<160, BWD>(a, B, stream);
  return launch_mask<256, BWD>(a, B, stream);
}

int check_mask(const char* what, int B, int n, int K, int E) {
  MMAE_CHECK(B > 0 && n > 0, MMAE_ERR_ARG, "%s: bad shape B=%d n=%d", what, B, n);
  MMAE_CHECK(K >= 8 && K <= 256, MMAE_ERR_UNSUPPORTED,
             "%s: K=%d classes; the mask kernel holds 8 to 256 classes in one accumulator tile", what, K);
  MMAE_CHECK(E > 0 && E % 128 == 0 && E <= 1024, MMAE_ERR_UNSUPPORTED,
             "%s: E=%d must be a multiple of 128, at most 1024", what, E);
  MMAE_CHECK(int64_t(B) * (n + K) * E < (int64_t(1) << 31), MMAE_ERR_UNSUPPORTED, "%s: too many tokens", what);
  return MMAE_OK;
}

struct MaskWs {
  bf16* Gs;
  float *t, *part;
  size_t bytes;
};
MaskWs mask_ws(void* base, int B, int n, int K) {
  Carve c{reinterpret_cast<uint8_t*>(base)};
  const int Kp = round8(K);
  MaskWs w;
  w.Gs = c.take<bf16>(size_t(B) * n * Kp);
  w.t = c.take<float>(size_t(B) * n);
  w.part = c.take<float>(size_t(B) * ceil_div(n, SG_BM) * 3 * Kp);
  w.bytes = align_up(c.off, 256);
  return w;
}

int colsum_add(const float* src, int rows, int64_t ld, int cols, float* dst, void* stream) {
  return launch(seg_colsum_add_kernel, dim3(ceil_div(cols, 256)), dim3(256), 0, stream, src, rows, ld, cols, dst);
}

}  // namespace
}  // namespace mmae

using namespace mmae;

// ====================================================================================================== mask
extern "C" int64_t mmae_segmenter_mask_workspace_bytes(int B, int n, int K) { return (int64_t)mask_ws(nullptr, B, n, K).bytes; }

extern "C" int mmae_segmenter_mask_forward(const void* P, const void* C, const float* rp, const float* rc, const float* gamma,
                                           const float* beta, float eps, int B, int n, int K, int E, float* cmap, float* mean,
                                           float* rstd, void* stream) {
  RUN(check_mask("mmae_segmenter_mask_forward", B, n, K, E));
  MMAE_CHECK(P && C && rp && rc && gamma && beta && cmap && mean && rstd && aligned16(P) && aligned16(C) && aligned16(cmap),
             MMAE_ERR_ARG, "mmae_segmenter_mask_forward: bad args (tensors must be 16-byte aligned)");
  MaskArgs a{};
  a.P = reinterpret_cast<const bf16*>(P);
  a.C = reinterpret_cast<const bf16*>(C);
  a.rp = rp, a.rc = rc, a.gamma = gamma, a.beta = beta, a.eps = eps;
  a.n = n, a.K = K, a.Kp = round8(K), a.E = E, a.tiles = ceil_div(n, SG_BM);
  a.cmap = cmap, a.mean = mean, a.rstd = rstd;
  return launch_mask_any<false>(a, B, stream);
}

extern "C" int mmae_segmenter_mask_backward(const void* P, const void* C, const float* rp, const float* rc, const float* gamma,
                                            const float* mean, const float* rstd, const float* dcmap, int B, int n, int K,
                                            int E, void* dP, void* dC, float* d_gamma, float* d_beta, void* ws, void* stream) {
  RUN(check_mask("mmae_segmenter_mask_backward", B, n, K, E));
  MMAE_CHECK(P && C && rp && rc && gamma && mean && rstd && dcmap && dP && dC && d_gamma && d_beta && ws && aligned16(P) &&
                 aligned16(C) && aligned16(dcmap) && aligned16(dP) && aligned16(dC),
             MMAE_ERR_ARG, "mmae_segmenter_mask_backward: bad args (tensors must be 16-byte aligned)");
  MaskWs w = mask_ws(ws, B, n, K);
  MaskArgs a{};
  a.P = reinterpret_cast<const bf16*>(P);
  a.C = reinterpret_cast<const bf16*>(C);
  a.rp = rp, a.rc = rc, a.gamma = gamma, a.beta = nullptr, a.eps = 0.f;
  a.n = n, a.K = K, a.Kp = round8(K), a.E = E, a.tiles = ceil_div(n, SG_BM);
  a.mean = const_cast<float*>(mean), a.rstd = const_cast<float*>(rstd);
  a.dcmap = dcmap, a.Gs = w.Gs, a.t = w.t, a.part = w.part;
  RUN(launch_mask_any<true>(a, B, stream));
  RUN(colsum_add(w.part + a.Kp, B * a.tiles, int64_t(3) * a.Kp, K, d_gamma, stream));
  RUN(colsum_add(w.part + 2 * a.Kp, B * a.tiles, int64_t(3) * a.Kp, K, d_beta, stream));
  DprojArgs d{};
  d.P = a.P, d.C = a.C, d.Gs = w.Gs, d.rp = rp, d.rc = rc, d.t = w.t, d.part = w.part;
  d.n = n, d.K = K, d.Kp = a.Kp, d.E = E, d.tiles = a.tiles;
  d.dP = reinterpret_cast<bf16*>(dP), d.dC = reinterpret_cast<bf16*>(dC);
  RUN(launch(seg_dproj_kernel<false>, dim3(ceil_div(E, DP_BN), ceil_div(n, SG_BM), B), dim3(SG_THREADS),
             SgTile<DP_BN, false, true>::BYTES, stream, d));
  return launch(seg_dproj_kernel<true>, dim3(ceil_div(E, DP_BN), ceil_div(a.Kp, SG_BM), B), dim3(SG_THREADS),
                SgTile<DP_BN, true, true>::BYTES, stream, d);
}

// ====================================================================================================== proj
namespace {
size_t proj_tmp_off(int B, int n, int D_in, int E) { return align_up((size_t)mmae_convnext_proj_workspace_bytes(B, n, D_in, E), 256); }
}  // namespace

extern "C" int64_t mmae_segmenter_proj_saved_bytes(int B, int n, int D_in, int E) {
  return mmae_convnext_proj_saved_bytes(B, n, D_in, E);
}
extern "C" int64_t mmae_segmenter_proj_workspace_bytes(int B, int n, int D_in, int E) {
  return (int64_t)(proj_tmp_off(B, n, D_in, E) + align_up(size_t(B) * n * E * sizeof(float), 256));
}

extern "C" int mmae_segmenter_proj_forward(const float* enc, int B, int N, int D, int n, int num_tasks, const int* start_host,
                                           int E, int K, const float* w, const float* bias, const float* cls_emb, float* seq,
                                           void* saved, void* ws, void* stream) {
  MMAE_CHECK(cls_emb && seq && ws && K > 0 && E > 0 && E % 8 == 0 && aligned16(cls_emb) && aligned16(seq), MMAE_ERR_ARG,
             "mmae_segmenter_proj_forward: bad args (tensors must be 16-byte aligned)");
  float* tmp = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(ws) + proj_tmp_off(B, n, num_tasks * D, E));
  RUN(mmae_convnext_proj_forward(enc, B, N, D, n, num_tasks, start_host, E, w, bias, tmp, saved, ws, stream));
  return launch(seg_assemble_kernel, dim3(B * (n + K)), dim3(std::min(256, std::max(32, E / 4))), 0, stream, (const float*)tmp,
                cls_emb, n, K, E, seq);
}

extern "C" int mmae_segmenter_proj_backward(const float* dseq, int B, int N, int D, int n, int num_tasks,
                                            const int* start_host, int E, int K, const float* w, float* d_w, float* d_b,
                                            float* d_cls, float* denc, const void* saved, void* ws, void* stream) {
  MMAE_CHECK(dseq && d_cls && ws && B > 0 && n > 0 && K > 0 && E > 0 && E % 8 == 0 && aligned16(dseq), MMAE_ERR_ARG,
             "mmae_segmenter_proj_backward: bad args (tensors must be 16-byte aligned)");
  float* tmp = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(ws) + proj_tmp_off(B, n, num_tasks * D, E));
  RUN(launch(seg_unassemble_kernel, dim3(B * n), dim3(std::min(256, std::max(32, E / 4))), 0, stream, dseq, n, K, E, tmp));
  RUN(colsum_add(dseq + int64_t(n) * E, B, int64_t(n + K) * E, K * E, d_cls, stream));
  return mmae_convnext_proj_backward(tmp, B, N, D, n, num_tasks, start_host, E, w, d_w, d_b, denc, saved, ws, stream);
}

// ====================================================================================================== tail
namespace {
struct TailSaved {
  bf16 *wp, *wc, *Xpc, *PCb;     // Xpc: decoder_norm output, patch rows then class rows; PCb: the projections, same order
  float *dmean, *drstd, *r, *lmean, *lrstd;
  size_t bytes;
};
TailSaved tl_saved(void* base, int B, int n, int E, int K) {
  Carve c{reinterpret_cast<uint8_t*>(base)};
  const size_t rows = size_t(B) * (n + K);
  TailSaved s;
  s.wp = c.take<bf16>(size_t(E) * E);
  s.wc = c.take<bf16>(size_t(E) * E);
  s.Xpc = c.take<bf16>(rows * E);
  s.PCb = c.take<bf16>(rows * E);
  s.dmean = c.take<float>(rows);
  s.drstd = c.take<float>(rows);
  s.r = c.take<float>(rows);
  s.lmean = c.take<float>(size_t(B) * n);
  s.lrstd = c.take<float>(size_t(B) * n);
  s.bytes = align_up(c.off, 256);
  return s;
}
struct TailWs {
  bf16 *seq_b, *dPC, *dXpc;      // seq_b: decoder_norm output / its gradient in sequence order
  float *PC32, *cmap;            // cmap: the [B*n, Kp] class map (forward) or its gradient (backward)
  void* mask;
  size_t bytes;
};
TailWs tl_ws(void* base, int B, int n, int E, int K) {
  Carve c{reinterpret_cast<uint8_t*>(base)};
  const size_t rows = size_t(B) * (n + K);
  TailWs w;
  w.seq_b = c.take<bf16>(rows * E);
  w.dPC = c.take<bf16>(rows * E);
  w.dXpc = c.take<bf16>(rows * E);
  w.PC32 = c.take<float>(rows * E);
  w.cmap = c.take<float>(size_t(B) * n * round8(K));
  w.mask = c.take<uint8_t>(mask_ws(nullptr, B, n, K).bytes);
  w.bytes = align_up(c.off, 256);
  return w;
}
// order of the parameter / gradient pointer arrays of the tail entry points
enum { DEC_W, DEC_B, PATCH_W, CLASSES_W, MASK_W, MASK_B, NUM_TAIL_PARAMS };
}  // namespace

extern "C" int64_t mmae_segmenter_tail_saved_bytes(int B, int nh, int nw, int E, int K) {
  return (int64_t)tl_saved(nullptr, B, nh * nw, E, K).bytes;
}
extern "C" int64_t mmae_segmenter_tail_workspace_bytes(int B, int nh, int nw, int E, int K) {
  return (int64_t)tl_ws(nullptr, B, nh * nw, E, K).bytes;
}

extern "C" int mmae_segmenter_tail_forward(const float* x, int B, int nh, int nw, int E, int K, int H, int W, float eps_dec,
                                           float eps_mask, const float* const* p, float* out, void* saved, void* ws,
                                           void* stream) {
  MMAE_CHECK(nh > 0 && nw > 0, MMAE_ERR_ARG, "mmae_segmenter_tail_forward: bad grid %d x %d", nh, nw);
  const int n = nh * nw, rows = B * (n + K);
  RUN(check_mask("mmae_segmenter_tail_forward", B, n, K, E));
  RUN(upsample_check("mmae_segmenter_tail_forward", nh, nw, 1, K, H, W));
  MMAE_CHECK(x && p && out && saved && ws && aligned16(x), MMAE_ERR_ARG, "mmae_segmenter_tail_forward: bad args");
  TailSaved sv = tl_saved(saved, B, n, E, K);
  TailWs wk = tl_ws(ws, B, n, E, K);
  RUN(weight_operand(p[PATCH_W], &sv.wp, int64_t(E) * E, true, stream));
  RUN(weight_operand(p[CLASSES_W], &sv.wc, int64_t(E) * E, true, stream));
  // decoder_norm (output_adapters.py:463), then the patch rows and the class rows as two contiguous matrices
  RUN(mmae_layernorm_forward(x, E, p[DEC_W], p[DEC_B], wk.seq_b, E, nullptr, 0, sv.dmean, sv.drstd, rows, E, eps_dec, stream));
  RUN(launch(seg_rows_kernel<false>, dim3(rows), dim3(128), 0, stream, wk.seq_b, sv.Xpc, B, n, K, E));
  // patch_proj, classes_proj (:465-466)
  const size_t coff = size_t(B) * n * E;
  RUN(linear_f32(sv.Xpc, sv.wp, nullptr, nullptr, wk.PC32, B * n, E, E, stream));
  RUN(linear_f32(sv.Xpc + coff, sv.wc, nullptr, nullptr, wk.PC32 + coff, B * K, E, E, stream));
  RUN(launch(seg_rownorm_kernel, dim3(ceil_div(rows, 8)), dim3(256), 0, stream, (const float*)wk.PC32, rows, E, sv.PCb, sv.r));
  // normalize, product, mask_norm (:468-472)
  RUN(mmae_segmenter_mask_forward(sv.PCb, sv.PCb + coff, sv.r, sv.r + size_t(B) * n, p[MASK_W], p[MASK_B], eps_mask, B, n, K, E,
                                  wk.cmap, sv.lmean, sv.lrstd, stream));
  // F.interpolate(size=(H, W), mode="bilinear") (:476)
  return launch_upsample_fwd(wk.cmap, round8(K), K, B, nh, nw, 1, H, W, out, stream);
}

extern "C" int mmae_segmenter_tail_backward(const float* x, const float* dout, float* dx, int B, int nh, int nw, int E, int K,
                                            int H, int W, const float* const* p, float* const* gr, const void* saved, void* ws,
                                            void* stream) {
  MMAE_CHECK(nh > 0 && nw > 0, MMAE_ERR_ARG, "mmae_segmenter_tail_backward: bad grid %d x %d", nh, nw);
  const int n = nh * nw, rows = B * (n + K);
  RUN(check_mask("mmae_segmenter_tail_backward", B, n, K, E));
  RUN(upsample_check("mmae_segmenter_tail_backward", nh, nw, 1, K, H, W));
  MMAE_CHECK(x && dout && dx && p && gr && saved && ws && aligned16(x) && aligned16(dx), MMAE_ERR_ARG,
             "mmae_segmenter_tail_backward: bad args");
  TailSaved sv = tl_saved(const_cast<void*>(saved), B, n, E, K);
  TailWs wk = tl_ws(ws, B, n, E, K);
  RUN(weight_operand(p[PATCH_W], &sv.wp, 0, false, stream));
  RUN(weight_operand(p[CLASSES_W], &sv.wc, 0, false, stream));
  const size_t coff = size_t(B) * n * E;
  RUN(launch_upsample_bwd(dout, round8(K), K, B, nh, nw, 1, H, W, wk.cmap, stream));
  RUN(mmae_segmenter_mask_backward(sv.PCb, sv.PCb + coff, sv.r, sv.r + size_t(B) * n, p[MASK_W], sv.lmean, sv.lrstd, wk.cmap, B,
                                   n, K, E, wk.dPC, wk.dPC + coff, gr[MASK_W], gr[MASK_B], wk.mask, stream));
  RUN(wgrad(wk.dPC, E, sv.Xpc, E, gr[PATCH_W], B * n, E, E, stream));
  RUN(wgrad(wk.dPC + coff, E, sv.Xpc + coff, E, gr[CLASSES_W], B * K, E, E, stream));
  RUN(dgrad_bf16(wk.dPC, E, sv.wp, nullptr, wk.dXpc, B * n, E, E, stream));
  RUN(dgrad_bf16(wk.dPC + coff, E, sv.wc, nullptr, wk.dXpc + coff, B * K, E, E, stream));
  RUN(launch(seg_rows_kernel<true>, dim3(rows), dim3(128), 0, stream, wk.seq_b, wk.dXpc, B, n, K, E));
  return mmae_layernorm_backward(wk.seq_b, 1, E, x, E, sv.dmean, sv.drstd, p[DEC_W], nullptr, 0, dx, E, gr[DEC_W], gr[DEC_B],
                                 rows, E, stream);
}
