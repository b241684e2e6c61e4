// HBM-bound cast / column-sum / transpose kernels (vectorised, coalesced; no data reuse -> no tensor cores).
#include <cstdlib>

#include "common.cuh"
#include "../../include/multimae_b200.h"
#include "internal.h"

namespace mmae {
void count_launch();
namespace {

// ---------------------------------------------------------------------------------------------------------------------
// Column reductions without a finalize launch.  Row-blocked kernels (grid.y row blocks per column block) write one partial
// row per block; the block that takes the LAST ticket of its column block (atomic counter per blockIdx.x, self-resetting)
// adds the partial rows up and accumulates into the destination: no same-address atomics on the data (they serialise in
// one or two L2 slices), a deterministic summation order, and 84 fewer launches per MultiMAE-B step than with a separate
// colred_finalize kernel.  Block shape (32, 8); W = columns per thread (4 or 8); `red` holds 8 x 32 x (W + 1) floats.
// ---------------------------------------------------------------------------------------------------------------------
template <int W>
__device__ __forceinline__ void colred_last_block_add(const float* partial, unsigned int* counters, int N, int col,
                                                      float* __restrict__ colsum, float* red) {
  __shared__ int s_last;
  __threadfence();                       // this block's partial row is visible device-wide before its ticket
  __syncthreads();
  if (threadIdx.x == 0 && threadIdx.y == 0) {
    const unsigned int t = atomicAdd(&counters[blockIdx.x], 1u);
    s_last = t == gridDim.y - 1;
    if (s_last) counters[blockIdx.x] = 0u;   // every other block of this column block has already taken its ticket
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  float acc[W];
#pragma unroll
  for (int k = 0; k < W; ++k) acc[k] = 0.f;
  if (col < N) {
    for (int y = threadIdx.y; y < int(gridDim.y); y += 8) {
      const float4* src = reinterpret_cast<const float4*>(partial + int64_t(y) * N + col);
#pragma unroll
      for (int k = 0; k < W / 4; ++k) {
        const float4 v = __ldcg(src + k);   // written by other SMs: read through L2
        acc[4 * k] += v.x; acc[4 * k + 1] += v.y; acc[4 * k + 2] += v.z; acc[4 * k + 3] += v.w;
      }
    }
  }
  float* mine = red + (threadIdx.y * 32 + threadIdx.x) * (W + 1);
#pragma unroll
  for (int k = 0; k < W; ++k) mine[k] = acc[k];
  __syncthreads();
  if (threadIdx.y == 0 && col < N) {
#pragma unroll
    for (int k = 0; k < W; ++k) {
      float t = 0.f;
#pragma unroll
      for (int y = 0; y < 8; ++y) t += red[(y * 32 + threadIdx.x) * (W + 1) + k];
      colsum[col + k] += t;
    }
  }
}

__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, bf16* __restrict__ dst, int64_t n) {
  pdl_prologue();
  const int64_t stride = int64_t(gridDim.x) * blockDim.x * 8;
  for (int64_t i = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) * 8; i < n; i += stride) {
    if (i + 8 <= n) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(src + i));
      const float4 b = __ldg(reinterpret_cast<const float4*>(src + i + 4));
      uint4 o;
      o.x = pack_bf16x2(a.x, a.y); o.y = pack_bf16x2(a.z, a.w);
      o.z = pack_bf16x2(b.x, b.y); o.w = pack_bf16x2(b.z, b.w);
      *reinterpret_cast<uint4*>(dst + i) = o;
    } else {
      for (int64_t j = i; j < n; ++j) dst[j] = __float2bfloat16_rn(src[j]);
    }
  }
}

// Tile: ROWS_PER_BLOCK rows x 128 columns; block (32, 8).  Each thread owns 4 consecutive columns.

template <bool SRC_BF16, bool DROP>
__global__ void __launch_bounds__(256) cast_colsum_kernel(const void* __restrict__ src_, int64_t ld_src,
                                                          bf16* __restrict__ dst, int64_t ld_dst,
                                                          float* __restrict__ colsum, float* __restrict__ partial,
                                                          unsigned int* __restrict__ counters, int M, int N,
                                                          int rows_per_block, const float* __restrict__ row_scale,
                                                          int rows_per_sample, DropSite drop) {
  pdl_prologue();
  const uint64_t dseed = DROP ? *drop.seed : 0;
  __shared__ float4 red[8][32];
  __shared__ float red2[8 * 32 * 5];
  const int col = blockIdx.x * 128 + threadIdx.x * 4;
  const int r0 = blockIdx.y * rows_per_block;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (col < N) {
#pragma unroll 4
    for (int r = r0 + threadIdx.y; r < min(r0 + rows_per_block, M); r += 8) {
      float4 v;
      if constexpr (SRC_BF16) {
        const uint2 u = __ldg(reinterpret_cast<const uint2*>(reinterpret_cast<const bf16*>(src_) + int64_t(r) * ld_src + col));
        const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y);
        v = make_float4(a.x, a.y, b.x, b.y);
      } else {
        v = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(src_) + int64_t(r) * ld_src + col));
        if (row_scale != nullptr) {   // per-sample factor (stochastic depth) on the cast copy and on the column sums
          const float sc = __ldg(row_scale + r / rows_per_sample);
          v = make_float4(sc * v.x, sc * v.y, sc * v.z, sc * v.w);
        }
        if constexpr (DROP) {   // dropout of the branch this gradient enters: its mask and 1/(1-p)
          const float4 f = dropout_factor4(drop, dseed, uint64_t(r), col);
          v = make_float4(f.x * v.x, f.y * v.y, f.z * v.z, f.w * v.w);
        }
        if (dst) {
          uint2 o;
          o.x = pack_bf16x2(v.x, v.y);
          o.y = pack_bf16x2(v.z, v.w);
          *reinterpret_cast<uint2*>(dst + int64_t(r) * ld_dst + col) = o;
        }
      }
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  }
  if (colsum == nullptr) return;
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && col < N) {
#pragma unroll
    for (int y = 1; y < 8; ++y) {
      const float4 o = red[y][threadIdx.x];
      acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w;
    }
    // one partial row per row-block (added up by the block with the last ticket), or the only block adds directly
    if (gridDim.y == 1) {
      float4 c = *reinterpret_cast<float4*>(colsum + col);
      c.x += acc.x; c.y += acc.y; c.z += acc.z; c.w += acc.w;
      *reinterpret_cast<float4*>(colsum + col) = c;
    } else {
      *reinterpret_cast<float4*>(partial + int64_t(blockIdx.y) * N + col) = acc;
    }
  }
  if (gridDim.y > 1 && counters != nullptr) colred_last_block_add<4>(partial, counters, N, col, colsum, red2);
}

// dst[c] += sum_y partial[y, c]: block (32, 32) per 32 columns, y strided over the 32 thread rows (a latency-bound
// kernel: ~Y/32 dependent-free loads per thread, all issued before the first add)
__global__ void __launch_bounds__(1024) colred_finalize_kernel(const float* __restrict__ partial, int Y, int ld, int C, int seg,
                                                               const ColredDst dsts) {
  pdl_prologue();
  __shared__ float red[32][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  float acc = 0.f;
  if (c < C) {
    int y = threadIdx.y;
    for (; y + 96 < Y; y += 128) {
      const float a0 = partial[int64_t(y) * ld + c], a1 = partial[int64_t(y + 32) * ld + c];
      const float a2 = partial[int64_t(y + 64) * ld + c], a3 = partial[int64_t(y + 96) * ld + c];
      acc += (a0 + a1) + (a2 + a3);
    }
    for (; y < Y; y += 32) acc += partial[int64_t(y) * ld + c];
  }
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  // transpose-reduce: warp w sums column w's 32 partials
  float v = red[threadIdx.x][threadIdx.y];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int cc = blockIdx.x * 32 + threadIdx.y;
  if (threadIdx.x == 0 && cc < C) {
    const int k = cc / seg;
    float* d = dsts.p[k];
    if (d != nullptr) d[cc - k * seg] += v;
  }
}

// colsum[n] += sum_m src[m, n] for a bf16 matrix: 8 columns (16 bytes) per thread, 4 rows in flight, block (32, 8)
__global__ void __launch_bounds__(256) colsum_bf16_kernel(const bf16* __restrict__ src, int64_t ld, float* __restrict__ colsum,
                                                          float* __restrict__ partial, unsigned int* __restrict__ counters, int M,
                                                          int N, int rows_per_block) {
  pdl_prologue();
  __shared__ float red[8][32][9];
  const int col = blockIdx.x * 256 + threadIdx.x * 8;
  const int r0 = blockIdx.y * rows_per_block;
  const int r_end = min(r0 + rows_per_block, M);
  float acc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) acc[k] = 0.f;
  if (col < N) {
    constexpr int U = 4;
    for (int rb = r0 + threadIdx.y; rb < r_end; rb += 8 * U) {
      uint4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (rb + 8 * u < r_end) v[u] = ld_stream_16(src + int64_t(rb + 8 * u) * ld + col);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (rb + 8 * u >= r_end) break;
        const uint32_t* w = reinterpret_cast<const uint32_t*>(&v[u]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 a = unpack_bf16x2(w[k]);
          acc[2 * k] += a.x;
          acc[2 * k + 1] += a.y;
        }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) red[threadIdx.y][threadIdx.x][k] = acc[k];
  __syncthreads();
  if (threadIdx.y == 0 && col < N) {
    float t[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      t[k] = 0.f;
#pragma unroll
      for (int y = 0; y < 8; ++y) t[k] += red[y][threadIdx.x][k];
    }
    float* dst = gridDim.y == 1 ? colsum + col : partial + int64_t(blockIdx.y) * N + col;
    if (gridDim.y == 1) {
#pragma unroll
      for (int k = 0; k < 8; ++k) t[k] += dst[k];
    }
    *reinterpret_cast<float4*>(dst) = make_float4(t[0], t[1], t[2], t[3]);
    *reinterpret_cast<float4*>(dst + 4) = make_float4(t[4], t[5], t[6], t[7]);
  }
  if (gridDim.y > 1 && counters != nullptr) {
    __syncthreads();                     // `red` is reused by the last block's reduction
    colred_last_block_add<8>(partial, counters, N, col, colsum, &red[0][0][0]);
  }
}

// a = gelu(z)  /  dz *= gelu'(z): bf16 streams, 8 elements per thread.  Used when the GELU is NOT fused into the GEMM
// epilogue (mmae_set_fuse_gelu(0), the default: faster on H100, see modules.cu).
template <bool BACKWARD>
__global__ void __launch_bounds__(256) gelu_stream_kernel(const bf16* __restrict__ z, bf16* __restrict__ io, int64_t n) {
  pdl_prologue();
  constexpr int U = 2;   // independent 16-byte loads in flight per thread and stream
  const int64_t stride = int64_t(gridDim.x) * blockDim.x * 8;
  for (int64_t i0 = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) * 8; i0 < n; i0 += stride * U) {
    uint4 zv[U], dv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + u * stride;
      if (i < n) {
        zv[u] = ld_stream_16(z + i);
        if constexpr (BACKWARD) dv[u] = ld_stream_16_rw(io + i);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + u * stride;
      if (i >= n) break;
      const uint32_t* zu = reinterpret_cast<const uint32_t*>(&zv[u]);
      uint4 ov;
      uint32_t* ou = reinterpret_cast<uint32_t*>(&ov);
      if constexpr (BACKWARD) {
        const uint32_t* du = reinterpret_cast<const uint32_t*>(&dv[u]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 a = unpack_bf16x2(zu[k]), d = unpack_bf16x2(du[k]);
          ou[k] = pack_bf16x2(d.x * dgelu_erf(a.x), d.y * dgelu_erf(a.y));
        }
      } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 a = unpack_bf16x2(zu[k]);
          ou[k] = pack_bf16x2(gelu_erf(a.x), gelu_erf(a.y));
        }
      }
      *reinterpret_cast<uint4*>(io + i) = ov;
    }
  }
}

// dz[m,n] *= gelu'(z[m,n]) in place AND colsum[n] += sum_m dz[m,n] (the fc1 bias gradient): one pass instead of a GELU'
// pass plus a column-sum pass.  Block (32, 8): 8 rows x 256 columns per iteration, 64 rows per block.
__global__ void __launch_bounds__(256) dgelu_colsum_kernel(const bf16* __restrict__ z, bf16* __restrict__ dz, int64_t ld,
                                                           float* __restrict__ colsum, float* __restrict__ partial,
                                                           unsigned int* __restrict__ counters, int M, int N,
                                                           int rows_per_block) {
  pdl_prologue();
  __shared__ float red[8][32][9];
  const int col = blockIdx.x * 256 + threadIdx.x * 8;
  const int r0 = blockIdx.y * rows_per_block;
  float acc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) acc[k] = 0.f;
  if (col < N) {
    const int r_end = min(r0 + rows_per_block, M);
    constexpr int U = 4;   // rows in flight per thread (loads issued before any of the in-place stores)
    for (int rb = r0 + threadIdx.y; rb < r_end; rb += 8 * U) {
      uint4 zv[U], dv[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int r = rb + 8 * u;
        if (r < r_end) {
          zv[u] = ld_stream_16(z + int64_t(r) * ld + col);
          dv[u] = ld_stream_16_rw(dz + int64_t(r) * ld + col);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int r = rb + 8 * u;
        if (r >= r_end) break;
        const uint32_t* zu = reinterpret_cast<const uint32_t*>(&zv[u]);
        const uint32_t* du = reinterpret_cast<const uint32_t*>(&dv[u]);
        uint4 ov;
        uint32_t* ou = reinterpret_cast<uint32_t*>(&ov);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 a = unpack_bf16x2(zu[k]), d = unpack_bf16x2(du[k]);
          const float o0 = d.x * dgelu_erf(a.x), o1 = d.y * dgelu_erf(a.y);
          ou[k] = pack_bf16x2(o0, o1);
          const float2 rbk = unpack_bf16x2(ou[k]);      // sum what is stored (bf16-rounded), as a separate pass would
          acc[2 * k] += rbk.x;
          acc[2 * k + 1] += rbk.y;
        }
        *reinterpret_cast<uint4*>(dz + int64_t(r) * ld + col) = ov;
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) red[threadIdx.y][threadIdx.x][k] = acc[k];
  __syncthreads();
  if (threadIdx.y == 0 && col < N) {
    float t[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      t[k] = 0.f;
#pragma unroll
      for (int y = 0; y < 8; ++y) t[k] += red[y][threadIdx.x][k];
    }
    float* dst = gridDim.y == 1 ? colsum + col : partial + int64_t(blockIdx.y) * N + col;
    if (gridDim.y == 1) {
#pragma unroll
      for (int k = 0; k < 8; ++k) t[k] += dst[k];
    }
    *reinterpret_cast<float4*>(dst) = make_float4(t[0], t[1], t[2], t[3]);
    *reinterpret_cast<float4*>(dst + 4) = make_float4(t[4], t[5], t[6], t[7]);
  }
  if (gridDim.y > 1 && counters != nullptr) {
    __syncthreads();                     // `red` is reused by the last block's reduction
    colred_last_block_add<8>(partial, counters, N, col, colsum, &red[0][0][0]);
  }
}

// out[i] = x[i] + s * y[i]   (residual add of a branch output onto the fp32 stream; y bf16 or fp32)
// s = row_scale[i / per_sample] (stochastic depth: 0 or 1/keep per sample), 1 without row_scale - then x + 1 * y == x + y
// exactly, with or without FMA contraction.  x == null: out = s * y (the fp32 tier's scaled copy of a branch gradient).
template <bool Y_BF16, bool DROP>
__global__ void __launch_bounds__(256) add_bf16_f32_kernel(const float* __restrict__ x, const void* __restrict__ y_,
                                                           float* __restrict__ out, int64_t n,
                                                           const float* __restrict__ row_scale, int64_t per_sample,
                                                           DropSite drop, int drop_cols) {
  pdl_prologue();
  const uint64_t dseed = DROP ? *drop.seed : 0;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x * 8;
  for (int64_t i = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) * 8; i < n; i += stride) {
    const float4 a = x != nullptr ? __ldg(reinterpret_cast<const float4*>(x + i)) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 b = x != nullptr ? __ldg(reinterpret_cast<const float4*>(x + i + 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 y0, y1;
    if constexpr (Y_BF16) {
      const uint4 yv = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const bf16*>(y_) + i));
      const float2 p0 = unpack_bf16x2(yv.x), p1 = unpack_bf16x2(yv.y), p2 = unpack_bf16x2(yv.z), p3 = unpack_bf16x2(yv.w);
      y0 = make_float4(p0.x, p0.y, p1.x, p1.y);
      y1 = make_float4(p2.x, p2.y, p3.x, p3.y);
    } else {
      y0 = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(y_) + i));
      y1 = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(y_) + i + 4));
    }
    const float s = row_scale != nullptr ? __ldg(row_scale + i / per_sample) : 1.0f;   // per_sample % 8 == 0
    if constexpr (DROP) {   // dropout of the branch, element (i / drop_cols, i % drop_cols); drop_cols % 8 == 0
      const int64_t r = i / drop_cols;
      const int c = int(i - r * drop_cols);
      const float4 f0 = dropout_factor4(drop, dseed, uint64_t(r), c), f1 = dropout_factor4(drop, dseed, uint64_t(r), c + 4);
      y0 = make_float4(f0.x * y0.x, f0.y * y0.y, f0.z * y0.z, f0.w * y0.w);
      y1 = make_float4(f1.x * y1.x, f1.y * y1.y, f1.z * y1.z, f1.w * y1.w);
    }
    *reinterpret_cast<float4*>(out + i) = make_float4(a.x + s * y0.x, a.y + s * y0.y, a.z + s * y0.z, a.w + s * y0.w);
    *reinterpret_cast<float4*>(out + i + 4) = make_float4(b.x + s * y1.x, b.y + s * y1.y, b.z + s * y1.z, b.w + s * y1.w);
  }
}

// 64x64 bf16 tile transpose through padded shared memory; block 256 threads
__global__ void __launch_bounds__(256) transpose_bf16_kernel(const bf16* __restrict__ src, int64_t ld_src,
                                                             bf16* __restrict__ dst, int64_t ld_dst, int M, int N) {
  pdl_prologue();
  __shared__ bf16 tile[64][66];
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  // load: each thread reads 2 consecutive columns; 32 threads cover 64 columns, 8 row groups
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = ty + i * 8;
    const int gm = m0 + r, gn = n0 + tx * 2;
    __nv_bfloat162 v = __floats2bfloat162_rn(0.f, 0.f);
    if (gm < M && gn < N) v = *reinterpret_cast<const __nv_bfloat162*>(src + int64_t(gm) * ld_src + gn);
    tile[r][tx * 2] = v.x;
    tile[r][tx * 2 + 1] = v.y;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = ty + i * 8;  // row of the transposed tile = column n
    const int gn = n0 + r, gm = m0 + tx * 2;
    if (gn < N && gm < M) {
      __nv_bfloat162 v;
      v.x = tile[tx * 2][r];
      v.y = tile[tx * 2 + 1][r];
      *reinterpret_cast<__nv_bfloat162*>(dst + int64_t(gn) * ld_dst + gm) = v;
    }
  }
}

}  // namespace
}  // namespace mmae

using namespace mmae;

// Row blocking of the column-sum kernels: about `blocks_per_sm` resident blocks per SM in ONE wave.  Each block ends with
// one fp32 atomic per column, so fewer, longer blocks also mean fewer same-address atomics (64-row blocks meant 392
// atomics per column on a 25088-row matrix, which cost more than reading it).  MMAE_TUNE_CS overrides blocks_per_sm.
static int colsum_rows_per_block(int M, int col_blocks, int blocks_per_sm) {
  static const int tune = []() {
    const char* e = getenv("MMAE_TUNE_CS");
    return e ? atoi(e) : 0;
  }();
  if (tune > 0) blocks_per_sm = tune;
  const int target = std::max(1, reduce_sm_count() * blocks_per_sm / std::max(col_blocks, 1));
  int rpb = ceil_div(M, target);
  rpb = std::max(32, (rpb + 7) / 8 * 8);
  return rpb;
}

// MMAE_COLRED_FOLD=0: separate colred_finalize launches instead of the last-block reduction (A/B measurements)
static int g_colred_fold = []() {
  const char* e = getenv("MMAE_COLRED_FOLD");
  return e ? atoi(e) : 1;
}();

namespace mmae {
// Every scratch buffer starts with a zero-initialised header of ticket counters (one per column block of the kernel using
// the buffer; the block that takes the last ticket resets it), followed by the partial rows.
float* colred_scratch(size_t floats, cudaStream_t st) {
  // One buffer per stream: kernels of different streams (the task decoders) run concurrently.  All buffers are created
  // by the first call (which must not be inside a stream capture), so a stream first seen during a capture still gets one.
  constexpr int MAX_SLOTS = 12;
  constexpr size_t DEFAULT_FLOATS = size_t(2) << 20;   // 8 MB each covers every shape of the MultiMAE-B step
  struct Slot {
    cudaStream_t st;
    bool bound;
    float* buf;
    size_t cap;
    uint64_t last_use;
  };
  static Slot slots[MAX_SLOTS];
  static bool created = false;
  static uint64_t tick = 0;
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(st, &cs);
  const bool capturing = cs != cudaStreamCaptureStatusNone;
  if (!created) {
    if (capturing) {
      set_last_error("column-reduction scratch must be created outside stream capture: run the step once eagerly first");
      return nullptr;
    }
    for (int i = 0; i < MAX_SLOTS; ++i) {
      slots[i] = {nullptr, false, nullptr, 0, 0};
      if (cudaMalloc(&slots[i].buf, (DEFAULT_FLOATS + COLRED_HEADER_FLOATS) * sizeof(float)) != cudaSuccess ||
          cudaMemset(slots[i].buf, 0, COLRED_HEADER_FLOATS * sizeof(float)) != cudaSuccess) {
        set_last_error("cudaMalloc of the column-reduction scratch failed");
        return nullptr;
      }
      slots[i].cap = DEFAULT_FLOATS;
    }
    created = true;
  }
  Slot* s = nullptr;
  for (int i = 0; i < MAX_SLOTS && s == nullptr; ++i)
    if (slots[i].bound && slots[i].st == st) s = &slots[i];
  for (int i = 0; i < MAX_SLOTS && s == nullptr; ++i)
    if (!slots[i].bound) {
      s = &slots[i];
      s->bound = true;
      s->st = st;
    }
  if (s == nullptr) {   // every slot is bound: hand the least recently used one to this stream
    s = &slots[0];
    for (int i = 1; i < MAX_SLOTS; ++i)
      if (slots[i].last_use < s->last_use) s = &slots[i];
    s->st = st;
  }
  s->last_use = ++tick;
  if (floats <= s->cap) return s->buf + COLRED_HEADER_FLOATS;
  if (capturing) {
    set_last_error("column-reduction scratch must grow to %zu floats during stream capture: run the step once eagerly first",
                   floats);
    return nullptr;
  }
  // The old buffer stays allocated: a CUDA graph captured before the growth still uses it.  Growth after a capture
  // happens when a later eager step needs more, e.g. one in deterministic mode (the ordered split-K workspace).  The
  // capacity at least doubles, so a slot leaves behind buffers that add up to less than its current one.
  floats = std::max(floats, 2 * s->cap);
  s->buf = nullptr;
  s->cap = 0;
  if (cudaMalloc(&s->buf, (floats + COLRED_HEADER_FLOATS) * sizeof(float)) != cudaSuccess ||
      cudaMemset(s->buf, 0, COLRED_HEADER_FLOATS * sizeof(float)) != cudaSuccess) {
    set_last_error("cudaMalloc of the column-reduction scratch (%zu bytes) failed", floats * sizeof(float));
    return nullptr;
  }
  s->cap = floats;
  return s->buf + COLRED_HEADER_FLOATS;
}

int colred_finalize_n(const float* partial, int Y, int ld, int seg, const ColredDst& dst, int nseg, cudaStream_t st) {
  dim3 grid(ceil_div(seg * nseg, 32)), block(32, 32);
  launch_k(colred_finalize_kernel, grid, block, 0, st, partial, Y, ld, seg * nseg, seg, dst);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}
int colred_finalize(const float* partial, int Y, int ld, int seg, float* dst0, float* dst1, float* dst2, cudaStream_t st) {
  ColredDst dst;
  for (int i = 0; i < 9; ++i) dst.p[i] = nullptr;
  dst.p[0] = dst0;
  dst.p[1] = dst1;
  dst.p[2] = dst2;
  return colred_finalize_n(partial, Y, ld, seg, dst, dst2 ? 3 : (dst1 ? 2 : 1), st);
}
}  // namespace mmae

extern "C" int mmae_cast_f32_to_bf16(const float* src, void* dst_bf16, int64_t n, void* stream) {
  MMAE_CHECK(src && dst_bf16 && n >= 0, MMAE_ERR_ARG, "mmae_cast_f32_to_bf16: bad args");
  if (n == 0) return MMAE_OK;
  MMAE_CHECK((reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst_bf16) & 15) == 0,
             MMAE_ERR_ARG, "mmae_cast_f32_to_bf16: pointers must be 16-byte aligned");
  const int threads = 256;
  int64_t blocks = (n / 8 + threads - 1) / threads;
  const int64_t cap = int64_t(sm_count()) * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  launch_k(cast_f32_bf16_kernel, (unsigned)blocks, threads, 0, reinterpret_cast<cudaStream_t>(stream), src, reinterpret_cast<bf16*>(dst_bf16), n);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

int mmae::cast_colsum_f32_scaled(const float* src, int64_t ld_src, bf16* dst_bf16, int64_t ld_dst, float* colsum,
                                 const float* row_scale, int rows_per_sample, int M, int N, void* stream, DropSite drop) {
  MMAE_CHECK(src && M > 0 && N > 0 && N % 4 == 0 && ld_src % 4 == 0 && (!dst_bf16 || ld_dst % 4 == 0), MMAE_ERR_ARG,
             "mmae_cast_colsum_f32: bad args (N, ld must be multiples of 4)");
  MMAE_CHECK(!row_scale || (rows_per_sample > 0 && M % rows_per_sample == 0), MMAE_ERR_ARG,
             "mmae_cast_colsum_f32: rows-per-sample must divide M=%d", M);
  cudaStream_t cst = reinterpret_cast<cudaStream_t>(stream);
  const int rpb = colsum_rows_per_block(M, ceil_div(N, 128), 4);
  dim3 grid(ceil_div(N, 128), ceil_div(M, rpb)), block(32, 8);
  float* partial = nullptr;
  if (colsum && grid.y > 1) {
    partial = colred_scratch(size_t(grid.y) * N, cst);
    if (!partial) return MMAE_ERR_CUDA;
  }
  launch_k(drop.seed ? cast_colsum_kernel<false, true> : cast_colsum_kernel<false, false>, grid, block, 0, cst, src, ld_src, dst_bf16, ld_dst, colsum, partial,
                                                     g_colred_fold ? colred_counters(partial) : nullptr, M, N, rpb, row_scale,
                                                     rows_per_sample, drop);
  count_launch();
  MMAE_LAUNCH_OK();
  if (partial && !g_colred_fold) return colred_finalize(partial, grid.y, N, N, colsum, nullptr, nullptr, cst);
  return MMAE_OK;
}

extern "C" int mmae_cast_colsum_f32(const float* src, int64_t ld_src, void* dst_bf16, int64_t ld_dst, float* colsum,
                                    int M, int N, void* stream) {
  return cast_colsum_f32_scaled(src, ld_src, reinterpret_cast<bf16*>(dst_bf16), ld_dst, colsum, nullptr, 1, M, N, stream);
}

extern "C" int mmae_colsum_bf16(const void* src_bf16, int64_t ld_src, float* colsum, int M, int N, void* stream) {
  MMAE_CHECK(src_bf16 && colsum && M > 0 && N > 0 && N % 4 == 0 && ld_src % 4 == 0, MMAE_ERR_ARG,
             "mmae_colsum_bf16: bad args");
  cudaStream_t cst = reinterpret_cast<cudaStream_t>(stream);
  const bool wide = N % 8 == 0 && ld_src % 8 == 0 && (reinterpret_cast<uintptr_t>(src_bf16) & 15) == 0;
  const int cols = wide ? 256 : 128;
  const int rpb = colsum_rows_per_block(M, ceil_div(N, cols), 4);
  dim3 grid(ceil_div(N, cols), ceil_div(M, rpb)), block(32, 8);
  float* partial = nullptr;
  if (grid.y > 1) {
    partial = colred_scratch(size_t(grid.y) * N, cst);
    if (!partial) return MMAE_ERR_CUDA;
  }
  if (wide)
    launch_k(colsum_bf16_kernel, grid, block, 0, cst, reinterpret_cast<const bf16*>(src_bf16), ld_src, colsum, partial,
                                                g_colred_fold ? colred_counters(partial) : nullptr, M, N, rpb);
  else
    launch_k(cast_colsum_kernel<true, false>, grid, block, 0, cst, src_bf16, ld_src, nullptr, 0, colsum, partial,
                                                      g_colred_fold ? colred_counters(partial) : nullptr, M, N, rpb,
                                                      nullptr, 1, DropSite());
  count_launch();
  MMAE_LAUNCH_OK();
  if (partial && !g_colred_fold) return colred_finalize(partial, grid.y, N, N, colsum, nullptr, nullptr, cst);
  return MMAE_OK;
}

extern "C" int mmae_transpose_bf16(const void* src, int64_t ld_src, void* dst, int64_t ld_dst, int M, int N,
                                   void* stream) {
  MMAE_CHECK(src && dst && M > 0 && N > 0 && M % 2 == 0 && N % 2 == 0 && ld_src % 2 == 0 && ld_dst % 2 == 0,
             MMAE_ERR_ARG, "mmae_transpose_bf16: bad args");
  dim3 grid(ceil_div(N, 64), ceil_div(M, 64));
  launch_k(transpose_bf16_kernel, grid, 256, 0, reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const bf16*>(src), ld_src, reinterpret_cast<bf16*>(dst), ld_dst, M, N);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

// a[i] = gelu(z[i]) (backward = 0)   or   dz[i] *= gelu'(z[i]) in place (backward = 1); n must be a multiple of 8
extern "C" int mmae_gelu_bf16(const void* z, void* io, int64_t n, int backward, void* stream) {
  MMAE_CHECK(z && io && n >= 0 && n % 8 == 0, MMAE_ERR_ARG, "mmae_gelu_bf16: bad args (n %% 8)");
  if (n == 0) return MMAE_OK;
  int64_t blocks = (n / 8 + 255) / 256;
  const int64_t cap = int64_t(sm_count()) * 16;
  if (blocks > cap) blocks = cap;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (backward)
    launch_k(gelu_stream_kernel<true>, (unsigned)blocks, 256, 0, st, reinterpret_cast<const bf16*>(z), reinterpret_cast<bf16*>(io), n);
  else
    launch_k(gelu_stream_kernel<false>, (unsigned)blocks, 256, 0, st, reinterpret_cast<const bf16*>(z), reinterpret_cast<bf16*>(io), n);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

int mmae::add_scaled_f32(const float* x, const void* y, int y_is_bf16, const float* row_scale, int64_t per_sample, float* out,
                         int64_t n, void* stream, DropSite drop, int drop_cols) {
  MMAE_CHECK(y && out && n >= 0 && n % 8 == 0, MMAE_ERR_ARG, "mmae_add_bf16_f32: bad args (n %% 8)");
  MMAE_CHECK(x || row_scale, MMAE_ERR_ARG, "mmae_add_bf16_f32: null x");
  MMAE_CHECK(!row_scale || (per_sample > 0 && per_sample % 8 == 0 && n % per_sample == 0), MMAE_ERR_ARG,
             "mmae_add_bf16_f32: a row scale needs a multiple of 8 elements per sample dividing n");
  MMAE_CHECK(!drop.seed || (drop_cols > 0 && drop_cols % 8 == 0 && n % drop_cols == 0), MMAE_ERR_ARG,
             "mmae_add_bf16_f32: a dropout mask needs a multiple of 8 columns dividing n");
  if (n == 0) return MMAE_OK;
  int64_t blocks = (n / 8 + 255) / 256;
  const int64_t cap = int64_t(sm_count()) * 16;
  if (blocks > cap) blocks = cap;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  auto kern = y_is_bf16 ? (drop.seed ? add_bf16_f32_kernel<true, true> : add_bf16_f32_kernel<true, false>)
                        : (drop.seed ? add_bf16_f32_kernel<false, true> : add_bf16_f32_kernel<false, false>);
  launch_k(kern, (unsigned)blocks, 256, 0, st, x, y, out, n, row_scale, per_sample, drop, drop_cols);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

extern "C" int mmae_add_bf16_f32(const float* x, const void* y_bf16, float* out, int64_t n, void* stream) {
  MMAE_CHECK(x, MMAE_ERR_ARG, "mmae_add_bf16_f32: bad args (n %% 8)");
  return add_scaled_f32(x, y_bf16, 1, nullptr, 1, out, n, stream);
}

extern "C" int mmae_dgelu_colsum_bf16(const void* z, void* dz, int64_t ld, float* colsum, int M, int N, void* stream) {
  MMAE_CHECK(z && dz && colsum && M > 0 && N > 0 && N % 8 == 0 && ld % 8 == 0, MMAE_ERR_ARG, "mmae_dgelu_colsum_bf16: bad args");
  cudaStream_t cst = reinterpret_cast<cudaStream_t>(stream);
  const int rpb = colsum_rows_per_block(M, ceil_div(N, 256), 3);
  dim3 grid(ceil_div(N, 256), ceil_div(M, rpb)), block(32, 8);
  float* partial = nullptr;
  if (grid.y > 1) {
    partial = colred_scratch(size_t(grid.y) * N, cst);
    if (!partial) return MMAE_ERR_CUDA;
  }
  launch_k(dgelu_colsum_kernel, grid, block, 0, cst, reinterpret_cast<const bf16*>(z), reinterpret_cast<bf16*>(dz), ld, colsum,
                                               partial, g_colred_fold ? colred_counters(partial) : nullptr, M, N, rpb);
  count_launch();
  MMAE_LAUNCH_OK();
  if (partial && !g_colred_fold) return colred_finalize(partial, grid.y, N, N, colsum, nullptr, nullptr, cst);
  return MMAE_OK;
}
