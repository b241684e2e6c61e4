// wgmma / TMA GEMM for sm_90a:  C[M,N] = epilogue(alpha * A * B^T), bf16 operands, fp32 accumulate in registers.
//
// Persistent: the grid holds at most one CTA (or two-CTA cluster) per SM, and each walks a fixed sequence of work items.
// A work item is one 128 x BN output tile (BN = 64 / 128 / 192 / 256) over one K range (split-K).  CTA c of a grid of
// g takes items c, c + g, c + 2g, ...; items are ordered n-tile fastest, then m-tile, then split, so the CTAs running
// at the same time share their A rows (the large, token-sized operand) and the whole of B stays in L2.  Three
// warpgroups:
//   warpgroup 0    : TMA producer (one thread: cp.async.bulk.tensor -> 128B-swizzled shared-memory ring, mbarrier
//                    complete_tx); gives its registers to the consumers (setmaxnreg).  Ring slot and phase follow a
//                    k-block count that runs across work items, so the next item's stages load during an epilogue.
//   warpgroups 1-2 : consumers, 64 rows of the tile each: wgmma 64 x BN x 16 straight from the ring (K-major or MN-major
//                    operands through the descriptor's transpose bit), then the fused epilogue from the accumulator
//                    registers (bias / GELU / dGELU / residual, bf16 and fp32 outputs, red.global adds for split-K), or
//                    for plain bf16 / fp32 outputs through a staging area of its own and TMA tile stores / reduce-adds
// CL = 2: a cluster of two CTAs along M shares the B tile - each CTA loads half of it and multicasts it to both, so a
// 256 x BN output tile reads B from L2 once.  Both CTAs walk the same item sequence (one M-half each), so their rings
// stay in lockstep; a stage is refilled only after the consumers of BOTH CTAs released it.
//
#include <algorithm>
#include <cstdlib>

#include "common.cuh"
#include "../../include/multimae_b200.h"

namespace mmae {

void count_launch();
bool gemm_profile_begin(cudaStream_t st, double flops, int M, int N, int K, int flags);
void gemm_profile_end(cudaStream_t st);

namespace {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = 128 bytes = one SWIZZLE_128B row
constexpr int WG_K = 16;
constexpr int GEMM_THREADS = 384;

struct GemmParams {
  int M, N, K;
  int num_kb;        // total k-blocks (ceil(K / BK))
  int kb_per_split;  // k-blocks handled by one split
  int tiles_n;       // ceil(N / BN)
  int tiles_m;       // M units of one CTA (CL = 1) or one cluster (CL = 2): ceil(ceil(M / BM) / CL)
  int splits;
  int tma_store;     // output through shared memory + TMA: 1 = bf16 store, 2 = fp32 store, 3 = fp32 reduce-add
  mmae_gemm_epilogue ep;
};

// ~192 KB of stages (BN = 64: 8 x 24 KB, 128: 6 x 32 KB, 192: 4 x 40 KB, 256: 4 x 48 KB) + 32 KB of TMA-store staging
// (per consumer warpgroup 16 KB: two 64 x 32 fp32 boxes or four bf16 boxes, used in turn).  One CTA per SM.
template <int BN>
struct GemmCfg {
  static constexpr int STAGES = BN == 256 ? 4 : (BN == 192 ? 4 : (BN == 128 ? 6 : 8));
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int EPI_BOX_BYTES = 64 * 32 * 4;
  static constexpr int EPI_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int BAR_OFFSET = EPI_OFFSET + 2 * 2 * EPI_BOX_BYTES;
  static constexpr int TOTAL = BAR_OFFSET + 256 + 1024;  // + barriers + alignment slack
  static_assert(TOTAL <= 232448, "GEMM exceeds the 227 KB shared-memory limit");
};

struct WorkItem {
  int m0, n0, split, kb_begin, nkb;
};

template <int BN, int CL>
__device__ __forceinline__ WorkItem decode_item(int item, const GemmParams& p, int rank) {
  WorkItem w;
  const int rest = item / p.tiles_n;
  w.n0 = (item - rest * p.tiles_n) * BN;
  w.split = rest / p.tiles_m;
  w.m0 = ((rest - w.split * p.tiles_m) * CL + rank) * BM;
  w.kb_begin = w.split * p.kb_per_split;
  w.nkb = min(p.kb_per_split, p.num_kb - w.kb_begin);   // >= 1: the host never makes an empty split
  return w;
}

__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

// Fused epilogue of two adjacent accumulator columns (n, n + 1) of one output row.
__device__ __forceinline__ void epilogue_pair(float v0, float v1, int row, int n, const GemmParams& p, bool first_split,
                                              bool atomic_out) {
  const mmae_gemm_epilogue& ep = p.ep;
  v0 *= ep.alpha;
  v1 *= ep.alpha;
  if (ep.bias && first_split) {
    const float2 b = __ldg(reinterpret_cast<const float2*>(ep.bias + n));
    v0 += b.x;
    v1 += b.y;
  }
  if (ep.preact_bf16)
    *reinterpret_cast<uint32_t*>(reinterpret_cast<bf16*>(ep.preact_bf16) + int64_t(row) * ep.ld_preact + n) = pack_bf16x2(v0, v1);
  if (ep.act == 1) {
    v0 = gelu_erf(v0);
    v1 = gelu_erf(v1);
  }
  if (ep.dgelu_z) {
    const uint32_t z = __ldg(reinterpret_cast<const unsigned int*>(reinterpret_cast<const bf16*>(ep.dgelu_z) +
                                                                   int64_t(row) * ep.ld_dgelu_z + n));
    const float2 zf = unpack_bf16x2(z);
    v0 *= dgelu_erf(zf.x);
    v1 *= dgelu_erf(zf.y);
  }
  if (ep.residual && first_split) {
    const float2 r = __ldg(reinterpret_cast<const float2*>(ep.residual + int64_t(row) * ep.ld_residual + n));
    v0 += r.x;
    v1 += r.y;
  }
  if (ep.out_f32) {
    float* dst = ep.out_f32 + int64_t(row) * ep.ld_out_f32 + n;
    if (atomic_out) red_add_v2(dst, v0, v1);
    else *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
  }
  if (ep.out_bf16)
    *reinterpret_cast<uint32_t*>(reinterpret_cast<bf16*>(ep.out_bf16) + int64_t(row) * ep.ld_out_bf16 + n) = pack_bf16x2(v0, v1);
}

// TMA-store staging: one dense box of 64 rows x 32 columns
template <typename T>
__device__ __forceinline__ void stage_pair(uint8_t* box, int r, int c, float v0, float v1) {
  T* b = reinterpret_cast<T*>(box);
  if constexpr (sizeof(T) == 4) *reinterpret_cast<float2*>(b + r * 32 + c) = make_float2(v0, v1);
  else *reinterpret_cast<uint32_t*>(b + r * 32 + c) = pack_bf16x2(v0, v1);
}

template <int BN, int CL, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
    gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                     const __grid_constant__ CUtensorMap tmC, const GemmParams p) {
  // the grid is never larger than what is co-resident (launch_gemm), so every item runs on a CTA that already holds its
  // SM: a dependent kernel released here can only take SMs this grid does not use
  pdl_launch_dependents();   // the wait follows the barrier setup below
  using C = GemmCfg<BN>;
  constexpr int STAGES = C::STAGES;
  constexpr int BH = BN / CL;   // B rows (output columns) this CTA loads
  static_assert(!B_MN || BH % 64 == 0, "MN-major B is loaded in 64-column chunks");

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = threadIdx.x >> 7;
  const int rank = CL > 1 ? int(cluster_ctarank()) : 0;
  const int num_items = p.tiles_n * p.tiles_m * p.splits;
  const int first_item = blockIdx.x / CL;
  const int item_stride = gridDim.x / CL;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (p.tma_store) tma_prefetch_desc(&tmC);
#pragma unroll
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2 * CL);   // one arrival per consumer warpgroup of every CTA the stage is multicast to
    }
    fence_barrier_init();
  }
  __syncthreads();
  if constexpr (CL > 1) cluster_sync_all();   // the peer's barriers exist before any multicast / remote arrival
  pdl_wait();   // the previous kernel's outputs (our operands) are complete and visible from here on

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      uint32_t it = 0;   // k-blocks loaded so far, over all items
      for (int item = first_item; item < num_items; item += item_stride) {
        const WorkItem w = decode_item<BN, CL>(item, p, rank);
        for (int kb = 0; kb < w.nkb; ++kb, ++it) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1u);
          mbar_expect_tx(&full_bar[s], C::STAGE_BYTES);
          uint8_t* sA = smem + s * C::STAGE_BYTES;
          uint8_t* sB = sA + C::A_BYTES;
          const int k0 = (w.kb_begin + kb) * BK;
          if constexpr (!A_MN) {
            tma_load_2d(sA, &tmA, &full_bar[s], k0, w.m0);
          } else {
#pragma unroll
            for (int c = 0; c < BM / 64; ++c) tma_load_2d(sA + c * (64 * BK * 2), &tmA, &full_bar[s], w.m0 + c * 64, k0);
          }
          if constexpr (CL == 1) {
            if constexpr (!B_MN) {
              tma_load_2d(sB, &tmB, &full_bar[s], k0, w.n0);
            } else {
#pragma unroll
              for (int c = 0; c < BN / 64; ++c) tma_load_2d(sB + c * (64 * BK * 2), &tmB, &full_bar[s], w.n0 + c * 64, k0);
            }
          } else {
            if constexpr (!B_MN) {
              tma_load_2d_multicast(sB + rank * BH * 128, &tmB, &full_bar[s], k0, w.n0 + rank * BH, 0x3);
            } else {
#pragma unroll
              for (int c = 0; c < BH / 64; ++c)
                tma_load_2d_multicast(sB + (rank * (BH / 64) + c) * (64 * BK * 2), &tmB, &full_bar[s],
                                      w.n0 + rank * BH + c * 64, k0, 0x3);
            }
          }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers (warpgroups 1, 2)
    setmaxnreg_inc<232>();
    const int cw = wg - 1;                 // rows [64 cw, 64 cw + 64) of the tile
    const int t = threadIdx.x & 127;
    const int rl = (t >> 5) * 16 + ((t & 31) >> 2);       // this thread's first row within the warpgroup's 64
    uint8_t* epi = smem + C::EPI_OFFSET + cw * (2 * C::EPI_BOX_BYTES);
    const bool atomic_out = p.ep.accumulate != 0 || p.splits > 1;
    uint32_t it = 0;       // k-blocks consumed so far, over all items
    uint32_t boxes = 0;    // TMA-store boxes issued so far by this warpgroup
    // frees ring stage `s` in this CTA and, for a cluster, in the peer whose multicast also fills it
    auto release = [&](int s) {
      if (t == 0) {
        if constexpr (CL == 1) mbar_arrive(&empty_bar[s]);
        else
          for (int r = 0; r < CL; ++r) mbar_arrive_cluster(mapa_u32(smem_u32(&empty_bar[s]), uint32_t(r)));
      }
    };
    float acc[BN / 2];   // written by each item's first wgmma (scale-d = 0)

    for (int item = first_item; item < num_items; item += item_stride) {
      const WorkItem w = decode_item<BN, CL>(item, p, rank);
      for (int kb = 0; kb < w.nkb; ++kb, ++it) {
        const int s = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1;
        mbar_wait(&full_bar[s], ph);
        const uint32_t a_addr = smem_u32(smem + s * C::STAGE_BYTES) + cw * (64 * BK * 2);
        const uint32_t b_addr = smem_u32(smem + s * C::STAGE_BYTES) + C::A_BYTES;
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) reg_fence(acc[i]);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < BK / WG_K; ++j) {
          const uint32_t sd = (kb | j) != 0 ? 1u : 0u;
          // K-major : advance 16 elements (32 B) inside the 128 B swizzle row; this warpgroup's 64 rows start 8 KB in
          // MN-major: advance 16 k-rows of 128 B; 64-element M/N chunks are (64 * BK * 2) bytes apart
          const uint64_t da = A_MN ? gmma_desc_sw128(a_addr + j * (WG_K * 128), 64 * BK * 2, 1024)
                                   : gmma_desc_sw128(a_addr + j * (WG_K * 2), 16, 1024);
          const uint64_t db = B_MN ? gmma_desc_sw128(b_addr + j * (WG_K * 128), 64 * BK * 2, 1024)
                                   : gmma_desc_sw128(b_addr + j * (WG_K * 2), 16, 1024);
          if constexpr (BN == 256) wgmma_m64n256k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, sd);
          else if constexpr (BN == 192) wgmma_m64n192k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, sd);
          else if constexpr (BN == 128) wgmma_m64n128k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, sd);
          else wgmma_m64n64k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, sd);
        }
        wgmma_commit();
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) reg_fence(acc[i]);
        wgmma_wait<1>();   // the previous k-block's MMAs have retired: its stage may be refilled
        if (kb > 0) release((it - 1) % STAGES);
      }
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) reg_fence(acc[i]);
      release((it - 1) % STAGES);   // the producer refills it with the next item's operands during the epilogue

      const int row_a = w.m0 + cw * 64 + rl;
      const int row_b = row_a + 8;
      const bool first_split = w.split == 0;
      if (p.tma_store) {
        // -------------------------------------------------------------- epilogue through shared memory + TMA, one
        // 64 x 32 box at a time through the warpgroup's staging area: 4 bf16 or 2 fp32 boxes in turn
        const float* bias = first_split ? p.ep.bias : nullptr;
        const bool bf16_out = p.tma_store == 1;
#pragma unroll
        for (int b = 0; b < BN / 32; ++b) {
          if (w.n0 + b * 32 >= p.N) break;   // whole boxes right of N are neither staged nor stored
          uint8_t* box = bf16_out ? epi + (boxes & 3) * (C::EPI_BOX_BYTES / 2) : epi + (boxes & 1) * C::EPI_BOX_BYTES;
          if (t == 0) {   // the store that used this buffer last has read it
            if (bf16_out) bulk_wait_read<3>();
            else bulk_wait_read<1>();
          }
          asm volatile("bar.sync %0, 128;" ::"r"(2 + cw) : "memory");
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int j = 4 * b + jj;
            const int c = jj * 8 + 2 * (t & 3);   // column within the box
            float v[4] = {acc[4 * j] * p.ep.alpha, acc[4 * j + 1] * p.ep.alpha, acc[4 * j + 2] * p.ep.alpha,
                          acc[4 * j + 3] * p.ep.alpha};
            if (bias && w.n0 + b * 32 + c < p.N) {
              const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + w.n0 + b * 32 + c));
              v[0] += bb.x; v[1] += bb.y; v[2] += bb.x; v[3] += bb.y;
            }
            if (p.ep.act == 1) {
#pragma unroll
              for (int i = 0; i < 4; ++i) v[i] = gelu_erf(v[i]);
            }
            if (bf16_out) {
              stage_pair<bf16>(box, rl, c, v[0], v[1]);
              stage_pair<bf16>(box, rl + 8, c, v[2], v[3]);
            } else {
              stage_pair<float>(box, rl, c, v[0], v[1]);
              stage_pair<float>(box, rl + 8, c, v[2], v[3]);
            }
          }
          fence_proxy_async_smem();
          asm volatile("bar.sync %0, 128;" ::"r"(2 + cw) : "memory");
          if (t == 0) {
            if (p.tma_store == 3) tma_reduce_add_2d(&tmC, box, w.n0 + b * 32, w.m0 + cw * 64);
            else tma_store_2d(&tmC, box, w.n0 + b * 32, w.m0 + cw * 64);
            bulk_commit_group();
          }
          ++boxes;
        }
      } else {
        // -------------------------------------------------------------- epilogue straight from the accumulator registers
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          if (w.n0 + j * 8 >= p.N) break;   // N % 8 == 0: a column pair is either fully inside or fully outside
          const int n = w.n0 + j * 8 + 2 * (t & 3);
          if (row_a < p.M) epilogue_pair(acc[4 * j], acc[4 * j + 1], row_a, n, p, first_split, atomic_out);
          if (row_b < p.M) epilogue_pair(acc[4 * j + 2], acc[4 * j + 3], row_b, n, p, first_split, atomic_out);
        }
      }
    }
    if (t == 0 && p.tma_store) bulk_wait_all();   // the stores are complete before the CTA's shared memory goes away
  }
  // no CTA of a cluster may leave while its peer can still arrive on its barriers
  if constexpr (CL > 1) cluster_sync_all();
}

template <int BN, int CL, bool A_MN, bool B_MN>
int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const GemmParams& p,
                cudaStream_t stream) {
  using C = GemmCfg<BN>;
  auto kern = gemm_bf16_kernel<BN, CL, A_MN, B_MN>;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = C::TOTAL;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  // CTAs (CL = 1) or clusters (CL = 2) of this kernel the device can hold at once
  static int resident = 0;
  if (resident == 0) {
    MMAE_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::TOTAL));
    if constexpr (CL > 1) {
      cfg.gridDim = dim3(CL);
      MMAE_CUDA_OK(cudaOccupancyMaxActiveClusters(&resident, kern, &cfg));
    } else {
      int dev = 0, sms = 0;
      MMAE_CUDA_OK(cudaGetDevice(&dev));
      MMAE_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
      resident = sms;
    }
    MMAE_CHECK(resident > 0, MMAE_ERR_CUDA, "mmae_gemm_bf16: the GEMM kernel does not fit on an SM");
  }
  const int items = p.tiles_n * p.tiles_m * p.splits;
  const int slots = std::min(resident, std::max(1, sm_count() / CL));
  cfg.gridDim = dim3(std::min(items, slots) * CL);
  const bool prof = gemm_profile_begin(stream, 2.0 * p.M * p.N * p.K, p.M, p.N, p.K,
                                       (A_MN ? 1 : 0) | (B_MN ? 2 : 0) | (p.splits << 8));
  if constexpr (CL == 1) {
    cfg.attrs = attr + 1;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
  } else {
    cfg.numAttrs = pdl_enabled() ? 2 : 1;
  }
  MMAE_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, tmA, tmB, tmC, p));
  if (prof) gemm_profile_end(stream);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

}  // namespace
}  // namespace mmae

using namespace mmae;

// MMAE_GEMM_VARIANT / MMAE_GEMM_TMA_STORE set the initial values of the two switches below
static int g_gemm_variant = []() {
  const char* e = getenv("MMAE_GEMM_VARIANT");
  const int v = e ? atoi(e) : -1;
  return v >= -1 && v <= 6 ? v : -1;
}();
static int g_gemm_tma_store = []() {
  const char* e = getenv("MMAE_GEMM_TMA_STORE");
  return e ? (atoi(e) != 0) : 1;
}();

extern "C" int mmae_gemm_set_variant(int variant) {
  MMAE_CHECK(variant >= -1 && variant <= 6, MMAE_ERR_ARG, "mmae_gemm_set_variant: %d (-1 .. 6)", variant);
  g_gemm_variant = variant;
  return MMAE_OK;
}

extern "C" int mmae_gemm_set_tma_store(int enable) {
  g_gemm_tma_store = enable != 0;
  return MMAE_OK;
}

// variant -> tile: 0 / 1 / 3 / 2 = one CTA, BN = 64 / 128 / 192 / 256; 6 / 5 / 4 = two-CTA cluster (256-row tile, B shared
// by multicast), BN = 128 / 192 / 256
static int variant_bn(int v) { return v == 0 ? 64 : (v == 1 || v == 6) ? 128 : (v == 3 || v == 5) ? 192 : 256; }

// Fixed cost of one work item in the persistent kernel, in k-block times of its tile: its epilogue and the hand-over to
// the next item.  scripts/gpu_time_gemm.py --fixed-cost measured 13.4, 14.0, 10.0 and 5.0 us per extra 128 x 256 fp32
// reduce-add item at 2, 4, 8 and 12 items per SM, against 0.9 us per k-block (H100 SXM, 700 W power limit): 15 falling to
// 5.5 k-block times as items per SM grow.  The model takes 4, near the low end, where the long-K weight gradients run;
// 5 or more would cut fc1 / fc2's weight gradient to 5 splits of 40 k-blocks in 3 rounds, 4 keeps 9 splits of 22 in 5.
constexpr int KB_PER_ITEM_FIXED = 4;
// Split-K never cuts an item below this many k-blocks, which bounds the fp32 reduce-add traffic it adds
constexpr int MIN_KB_PER_SPLIT = 16;

extern "C" int mmae_gemm_bf16(const void* A, int64_t lda, int a_mn_major, const void* B, int64_t ldb,
                              int b_mn_major, int M, int N, int K, int split_k, const mmae_gemm_epilogue* ep,
                              void* stream) {
  MMAE_CHECK(A && B && ep, MMAE_ERR_ARG, "mmae_gemm_bf16: null operand");
  MMAE_CHECK(M > 0 && N > 0 && K > 0, MMAE_ERR_ARG, "mmae_gemm_bf16: bad shape M=%d N=%d K=%d", M, N, K);
  MMAE_CHECK(N % 8 == 0, MMAE_ERR_ARG, "mmae_gemm_bf16: N=%d must be a multiple of 8", N);
  MMAE_CHECK(lda % 8 == 0 && ldb % 8 == 0, MMAE_ERR_ARG, "mmae_gemm_bf16: lda/ldb must be multiples of 8");
  MMAE_CHECK((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0,
             MMAE_ERR_ARG, "mmae_gemm_bf16: operands must be 16-byte aligned");
  MMAE_CHECK(ep->out_f32 || ep->out_bf16, MMAE_ERR_ARG, "mmae_gemm_bf16: no output");
  const int num_kb = ceil_div(K, BK);
  const int sms = sm_count();
  const int tm = ceil_div(M, BM);
  if (split_k <= 0 && !(ep->out_f32 && !ep->out_bf16 && !ep->preact_bf16 && !ep->dgelu_z && ep->act == 0)) split_k = 1;

  // Tile width and split count from one model of the persistent grid: it runs sm_count() items at a time (clusters:
  // sm_count() / 2 items of 256 rows), so a launch lasts ceil(items / slots) rounds of one item, and an item costs
  // ~(k-blocks + KB_PER_ITEM_FIXED) k-block times.  A k-block of a 128 x BN tile costs ~(BN + 40): the A tile's loads
  // and MMA issue do not shrink with BN, which makes BN = 256 the better tile whenever its rounds are as full.  The
  // automatic split (split_k
  // <= 0) fills the last round of the long-K weight gradients instead of leaving it mostly idle.  An explicit variant
  // fixes the tile, an explicit split_k the split.
  int variant = g_gemm_variant;
  {
    const int cand_var[2] = {1, 2};
    const int nvar = variant >= 0 ? 1 : 2;
    long best_cost = -1;
    int best_split = 1, best_var = variant >= 0 ? variant : 1;
    for (int i = 0; i < nvar; ++i) {
      const int v = variant >= 0 ? variant : cand_var[i];
      const int bn = variant_bn(v), cl = v >= 4 ? 2 : 1;
      if (variant < 0 && bn > 128 && N < bn) continue;
      const long tiles = long(ceil_div(tm, cl)) * ceil_div(N, bn);
      const int slots = std::max(1, sms / cl);
      const int s_lo = split_k > 0 ? split_k : 1;
      const int s_hi = split_k > 0 ? split_k : std::max(1, num_kb / MIN_KB_PER_SPLIT);
      for (int s = s_lo; s <= s_hi; ++s) {
        const int kbps = ceil_div(num_kb, std::min(s, num_kb));
        const long rounds = (tiles * ceil_div(num_kb, kbps) + slots - 1) / slots;
        const long cost = rounds * (bn + 40) * cl * (kbps + KB_PER_ITEM_FIXED);
        if (best_cost < 0 || cost < best_cost) {
          best_cost = cost;
          best_split = s;
          best_var = v;
        }
      }
    }
    split_k = best_split;
    variant = best_var;
  }
  if (split_k > num_kb) split_k = num_kb;
  const int kb_per_split = ceil_div(num_kb, split_k);
  split_k = ceil_div(num_kb, kb_per_split);  // no empty splits
  if (split_k > 1 || ep->accumulate) {
    MMAE_CHECK(ep->out_f32 && !ep->out_bf16 && !ep->preact_bf16 && !ep->dgelu_z && ep->act == 0, MMAE_ERR_ARG,
               "mmae_gemm_bf16: split-K / accumulate supports only a linear fp32 epilogue");
  }
#define MMAE_LD_OK(ptr, ld) (!(ptr) || ((ld) % 8 == 0 && (reinterpret_cast<uintptr_t>(ptr) & 15) == 0))
  MMAE_CHECK(MMAE_LD_OK(ep->residual, ep->ld_residual) && MMAE_LD_OK(ep->dgelu_z, ep->ld_dgelu_z) &&
                 MMAE_LD_OK(ep->preact_bf16, ep->ld_preact) && MMAE_LD_OK(ep->out_f32, ep->ld_out_f32) &&
                 MMAE_LD_OK(ep->out_bf16, ep->ld_out_bf16) &&
                 (!ep->bias || (reinterpret_cast<uintptr_t>(ep->bias) & 15) == 0),
             MMAE_ERR_ARG, "mmae_gemm_bf16: epilogue tensors need 16-byte alignment and ld %% 8 == 0");
#undef MMAE_LD_OK

  if (variant == 5 && b_mn_major) variant = 4;   // an MN-major B half must be whole 64-column chunks
  const int BNsel = variant_bn(variant);
  const int CLsel = variant >= 4 ? 2 : 1;

  CUtensorMap tmA, tmB;
  int rc;
  if (!a_mn_major) {
    rc = make_tmap_2d_bf16(&tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, BK, BM);
  } else {
    MMAE_CHECK(M % 8 == 0, MMAE_ERR_ARG, "mmae_gemm_bf16: MN-major A needs M %% 8 == 0");
    rc = make_tmap_2d_bf16(&tmA, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, 64, BK);
  }
  if (rc) return rc;
  if (!b_mn_major) {
    rc = make_tmap_2d_bf16(&tmB, B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, BK, BNsel / CLsel);
  } else {
    rc = make_tmap_2d_bf16(&tmB, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb, 64, BK);
  }
  if (rc) return rc;

  GemmParams p;
  p.M = M; p.N = N; p.K = K;
  p.num_kb = num_kb;
  p.kb_per_split = kb_per_split;
  p.tiles_n = ceil_div(N, BNsel);
  p.tiles_m = ceil_div(tm, CLsel);
  p.splits = split_k;
  p.ep = *ep;
  // plain bf16 / fp32 outputs (optionally with bias / GELU) leave through shared memory and TMA tile stores; fp32
  // accumulation (split-K, accumulate) through TMA reduce-add tiles
  p.tma_store = 0;
  CUtensorMap tmC = tmA;
  if (g_gemm_tma_store && !ep->preact_bf16 && !ep->dgelu_z && !ep->residual) {
    if (ep->out_bf16 && !ep->out_f32 && split_k == 1 && !ep->accumulate) {
      p.tma_store = 1;
      rc = make_tmap_2d_store(&tmC, ep->out_bf16, 2, (uint64_t)M, (uint64_t)N, (uint64_t)ep->ld_out_bf16);
      if (rc) return rc;
    } else if (ep->out_f32 && !ep->out_bf16 && ep->act == 0) {
      p.tma_store = (split_k > 1 || ep->accumulate) ? 3 : 2;
      rc = make_tmap_2d_store(&tmC, ep->out_f32, 4, (uint64_t)M, (uint64_t)N, (uint64_t)ep->ld_out_f32);
      if (rc) return rc;
    }
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
#define MMAE_DISPATCH(BN_, CL_)                                                                      \
  do {                                                                                               \
    if (!a_mn_major && !b_mn_major) return launch_gemm<BN_, CL_, false, false>(tmA, tmB, tmC, p, st); \
    if (!a_mn_major && b_mn_major) return launch_gemm<BN_, CL_, false, true>(tmA, tmB, tmC, p, st);   \
    if (a_mn_major && !b_mn_major) return launch_gemm<BN_, CL_, true, false>(tmA, tmB, tmC, p, st);   \
    return launch_gemm<BN_, CL_, true, true>(tmA, tmB, tmC, p, st);                                  \
  } while (0)
  if (variant == 4) MMAE_DISPATCH(256, 2);
  if (variant == 6) MMAE_DISPATCH(128, 2);
  if (variant == 5) {
    if (!a_mn_major) return launch_gemm<192, 2, false, false>(tmA, tmB, tmC, p, st);
    return launch_gemm<192, 2, true, false>(tmA, tmB, tmC, p, st);
  }
  if (variant == 0) MMAE_DISPATCH(64, 1);
  if (variant == 3) MMAE_DISPATCH(192, 1);
  if (variant == 2) MMAE_DISPATCH(256, 1);
  MMAE_DISPATCH(128, 1);
#undef MMAE_DISPATCH
}
