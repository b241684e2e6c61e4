// wgmma / TMA GEMM for sm_90a:  C[M,N] = epilogue(alpha * A * B^T), bf16 operands, fp32 accumulate in registers.
//
// Persistent: the grid holds at most one CTA per SM, and each walks a fixed sequence of work items.  A work item is one
// 128 x BN output tile (BN = 128 / 192 / 256) over one K range (split-K).  CTA c of a grid of g takes items c, c + g,
// c + 2g, ...; items are ordered n-tile fastest, then m-tile, then split, so the CTAs running at the same time share
// their A rows (the large, token-sized operand) and the whole of B stays in L2.  Three warpgroups:
//   warpgroup 0    : TMA producer (one thread: cp.async.bulk.tensor -> 128B-swizzled shared-memory ring, mbarrier
//                    complete_tx); gives its registers to the consumers (setmaxnreg).  Ring slot and phase follow a
//                    k-block count that runs across work items, so the next item's stages load during an epilogue.
//   warpgroups 1-2 : consumers: both work on every item, 64 rows each, with wgmma 64 x BN x 16 straight from the ring
//                    (K-major or MN-major operands through the descriptor's transpose bit).  Two schemes:
//     cooperative (gemm_bf16_kernel): the two run the item's fused epilogue together while the tensor cores idle:
//                    from the accumulator registers (bias / GELU / dGELU / residual, bf16 and fp32 outputs, red.global
//                    adds for split-K), or for plain bf16 / fp32 outputs through a staging area of their own and TMA
//                    tile stores / reduce-adds.
//     asynchronous epilogue (gemm_async_epi_kernel, unsplit plain bf16 / fp32 outputs): each stages its whole slab and
//                    goes on to the next item's MMAs while the TMA stores drain.
//
#include <algorithm>
#include <cstdlib>

#include "common.cuh"
#include "../../include/multimae_b200.h"

namespace mmae {

void count_launch();
float* colred_scratch(size_t floats, cudaStream_t st);   // the per-stream workspace pool (elementwise.cu)
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
  int tiles_m;       // ceil(M / BM)
  int splits;
  int tma_store;     // output through shared memory + TMA: 1 = bf16 store, 2 = fp32 store, 3 = fp32 reduce-add
  mmae_gemm_epilogue ep;
};

// ~192 KB of stages (BN = 128: 6 x 32 KB, 192: 4 x 40 KB, 256: 4 x 48 KB) + 32 KB of TMA-store staging (per consumer
// warpgroup 16 KB: two 64 x 32 fp32 boxes or four bf16 boxes, used in turn).  One CTA per SM.
template <int BN>
struct GemmCfg {
  static constexpr int STAGES = BN == 128 ? 6 : 4;
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

template <int BN>
__device__ __forceinline__ WorkItem decode_item(int item, const GemmParams& p) {
  WorkItem w;
  const int rest = item / p.tiles_n;
  w.n0 = (item - rest * p.tiles_n) * BN;
  w.split = rest / p.tiles_m;
  w.m0 = (rest - w.split * p.tiles_m) * BM;
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

// TMA producer (one thread): walks the CTA's items in order and fills the ring; slot and phase follow a k-block count
// that runs across items, so the next item's stages load while the consumers finish the current one.  STAGES: the
// ring's depth (the stage layout is GemmCfg<BN>'s whatever the depth)
template <int BN, bool A_MN, bool B_MN, int STAGES = GemmCfg<BN>::STAGES>
__device__ __forceinline__ void produce(uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, const CUtensorMap* tmA,
                                        const CUtensorMap* tmB, const GemmParams& p, int first_item, int item_stride,
                                        int num_items) {
  using C = GemmCfg<BN>;
  uint32_t it = 0;   // k-blocks loaded so far, over all items
  for (int item = first_item; item < num_items; item += item_stride) {
    const WorkItem w = decode_item<BN>(item, p);
    for (int kb = 0; kb < w.nkb; ++kb, ++it) {
      const int s = it % STAGES;
      const uint32_t ph = (it / STAGES) & 1;
      mbar_wait(&empty_bar[s], ph ^ 1u);
      mbar_expect_tx(&full_bar[s], C::STAGE_BYTES);
      uint8_t* sA = smem + s * C::STAGE_BYTES;
      uint8_t* sB = sA + C::A_BYTES;
      const int k0 = (w.kb_begin + kb) * BK;
      if constexpr (!A_MN) {
        tma_load_2d(sA, tmA, &full_bar[s], k0, w.m0);
      } else {
#pragma unroll
        for (int c = 0; c < BM / 64; ++c) tma_load_2d(sA + c * (64 * BK * 2), tmA, &full_bar[s], w.m0 + c * 64, k0);
      }
      if constexpr (!B_MN) {
        tma_load_2d(sB, tmB, &full_bar[s], k0, w.n0);
      } else {
#pragma unroll
        for (int c = 0; c < BN / 64; ++c) tma_load_2d(sB + c * (64 * BK * 2), tmB, &full_bar[s], w.n0 + c * 64, k0);
      }
    }
  }
}

// One k-block of MMAs for 64 rows of the tile: BK / 16 wgmma 64 x BN x 16 straight from ring stage `stage`, the rows
// starting `slab` x 64 into its A tile.  `first`: the item's first k-block, whose first wgmma overwrites the accumulators.
template <int BN, bool A_MN, bool B_MN>
__device__ __forceinline__ void mma_kblock(float (&acc)[BN / 2], const uint8_t* stage, int slab, bool first) {
  const uint32_t a_addr = smem_u32(stage) + slab * (64 * BK * 2);
  const uint32_t b_addr = smem_u32(stage) + GemmCfg<BN>::A_BYTES;
#pragma unroll
  for (int j = 0; j < BK / WG_K; ++j) {
    const uint32_t sd = (first && j == 0) ? 0u : 1u;
    // K-major : advance 16 elements (32 B) inside the 128 B swizzle row; a 64-row slab starts 8 KB in
    // MN-major: advance 16 k-rows of 128 B; 64-element M/N chunks are (64 * BK * 2) bytes apart
    const uint64_t da = A_MN ? gmma_desc_sw128(a_addr + j * (WG_K * 128), 64 * BK * 2, 1024)
                             : gmma_desc_sw128(a_addr + j * (WG_K * 2), 16, 1024);
    const uint64_t db = B_MN ? gmma_desc_sw128(b_addr + j * (WG_K * 128), 64 * BK * 2, 1024)
                             : gmma_desc_sw128(b_addr + j * (WG_K * 2), 16, 1024);
    if constexpr (BN == 256) wgmma_m64n256k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, sd);
    else if constexpr (BN == 192) wgmma_m64n192k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, sd);
    else wgmma_m64n128k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, sd);
  }
}

// Fused epilogue of 64 rows x BN columns of an item's output, rows [row0, row0 + 64) and columns [n0, n0 + BN), from
// the accumulators of one consumer warpgroup (thread t of 128).  With p.tma_store, one 64 x 32 box at a time through the
// warpgroup's staging area `epi` (16 KB: four bf16 or two fp32 boxes in turn, `boxes` counts the boxes it issued) and
// named barrier `bar`; otherwise straight from the registers.
template <int BN>
__device__ __forceinline__ void epilogue_slab(const float (&acc)[BN / 2], int row0, int n0, bool first_split,
                                              const GemmParams& p, const CUtensorMap* tmC, uint8_t* epi,
                                              uint32_t& boxes, int bar, int t) {
  constexpr int EPI_BOX_BYTES = GemmCfg<BN>::EPI_BOX_BYTES;
  const int rl = (t >> 5) * 16 + ((t & 31) >> 2);       // this thread's first row within the 64
  if (p.tma_store) {
    const float* bias = first_split ? p.ep.bias : nullptr;
    const bool bf16_out = p.tma_store == 1;
    // The bias of box b + 1 is loaded while box b is staged, so its latency is paid once per item rather than once per
    // box behind the two named barriers.  Loaded inside the box, it made the encoder's fc1 forward (12672 x 3072 x 768,
    // 128 x 256 tiles) take 129 us against 110 us for the fc2 dgrad of the same shape without a bias; loaded ahead, 113
    // us (scripts/gpu_time_gemm.py, H100 SXM, 700 W power limit).
    float2 bias_cur[4] = {}, bias_next[4] = {};
    auto load_bias = [&](int b, float2 (&dst)[4]) {
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int col = n0 + b * 32 + jj * 8 + 2 * (t & 3);
        if (bias && col < p.N) dst[jj] = __ldg(reinterpret_cast<const float2*>(bias + col));
      }
    };
    load_bias(0, bias_cur);
#pragma unroll
    for (int b = 0; b < BN / 32; ++b) {
      if (n0 + b * 32 >= p.N) break;   // whole boxes right of N are neither staged nor stored
      if (b + 1 < BN / 32) load_bias(b + 1, bias_next);
      uint8_t* box = bf16_out ? epi + (boxes & 3) * (EPI_BOX_BYTES / 2) : epi + (boxes & 1) * EPI_BOX_BYTES;
      if (t == 0) {   // the store that used this buffer last has read it
        if (bf16_out) bulk_wait_read<3>();
        else bulk_wait_read<1>();
      }
      asm volatile("bar.sync %0, 128;" ::"r"(bar) : "memory");
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = 4 * b + jj;
        const int c = jj * 8 + 2 * (t & 3);   // column within the box
        float v[4] = {acc[4 * j] * p.ep.alpha, acc[4 * j + 1] * p.ep.alpha, acc[4 * j + 2] * p.ep.alpha,
                      acc[4 * j + 3] * p.ep.alpha};
        if (bias && n0 + b * 32 + c < p.N) {
          const float2 bb = bias_cur[jj];
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
      asm volatile("bar.sync %0, 128;" ::"r"(bar) : "memory");
      if (t == 0) {
        if (p.tma_store == 3) tma_reduce_add_2d(tmC, box, n0 + b * 32, row0);
        else tma_store_2d(tmC, box, n0 + b * 32, row0);
        bulk_commit_group();
      }
      ++boxes;
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) bias_cur[jj] = bias_next[jj];
    }
  } else {
    const bool atomic_out = p.ep.accumulate != 0 || p.splits > 1;
    const int row_a = row0 + rl;
    const int row_b = row_a + 8;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      if (n0 + j * 8 >= p.N) break;   // N % 8 == 0: a column pair is either fully inside or fully outside
      const int n = n0 + j * 8 + 2 * (t & 3);
      if (row_a < p.M) epilogue_pair(acc[4 * j], acc[4 * j + 1], row_a, n, p, first_split, atomic_out);
      if (row_b < p.M) epilogue_pair(acc[4 * j + 2], acc[4 * j + 3], row_b, n, p, first_split, atomic_out);
    }
  }
}

// Cooperative consumers: both warpgroups work on the same item, 64 rows each, and run its epilogue together.
// ORD (ordered split-K, deterministic mode; p.tma_store = 2): split s stores its tile into rows
// [s * tiles_m * BM, (s + 1) * tiles_m * BM) of the workspace map tmC, and splitk_reduce_kernel adds the slices in order.
template <int BN, bool A_MN, bool B_MN, bool ORD = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
    gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                     const __grid_constant__ CUtensorMap tmC, const GemmParams p) {
  // the grid is never larger than what is co-resident (launch_gemm), so every item runs on a CTA that already holds its
  // SM: a dependent kernel released here can only take SMs this grid does not use
  pdl_launch_dependents();   // the wait follows the barrier setup below
  using C = GemmCfg<BN>;
  constexpr int STAGES = C::STAGES;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = threadIdx.x >> 7;
  const int num_items = p.tiles_n * p.tiles_m * p.splits;
  const int first_item = blockIdx.x;
  const int item_stride = gridDim.x;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (p.tma_store) tma_prefetch_desc(&tmC);
#pragma unroll
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);   // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();   // the previous kernel's outputs (our operands) are complete and visible from here on

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) produce<BN, A_MN, B_MN>(smem, full_bar, empty_bar, &tmA, &tmB, p, first_item, item_stride,
                                                  num_items);
  } else {
    // ------------------------------------------------------------------ consumers (warpgroups 1, 2)
    setmaxnreg_inc<232>();
    const int cw = wg - 1;                 // rows [64 cw, 64 cw + 64) of the tile
    const int t = threadIdx.x & 127;
    uint8_t* epi = smem + C::EPI_OFFSET + cw * (2 * C::EPI_BOX_BYTES);
    uint32_t it = 0;       // k-blocks consumed so far, over all items
    uint32_t boxes = 0;    // TMA-store boxes issued so far by this warpgroup
    float acc[BN / 2];   // written by each item's first wgmma (scale-d = 0)

    for (int item = first_item; item < num_items; item += item_stride) {
      const WorkItem w = decode_item<BN>(item, p);
      for (int kb = 0; kb < w.nkb; ++kb, ++it) {
        const int s = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1;
        mbar_wait(&full_bar[s], ph);
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) reg_fence(acc[i]);
        wgmma_fence();
        mma_kblock<BN, A_MN, B_MN>(acc, smem + s * C::STAGE_BYTES, cw, kb == 0);
        wgmma_commit();
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) reg_fence(acc[i]);
        wgmma_wait<1>();   // the previous k-block's MMAs have retired: its stage may be refilled
        if (kb > 0 && t == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
      }
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) reg_fence(acc[i]);
      // the producer refills the stage with the next item's operands during the epilogue
      if (t == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
      const int slice_row = ORD ? w.split * p.tiles_m * BM : 0;
      epilogue_slab<BN>(acc, slice_row + w.m0 + cw * 64, w.n0, w.split == 0, p, &tmC, epi, boxes, 2 + cw, t);
    }
    if (t == 0 && p.tma_store) bulk_wait_all();   // the stores are complete before the CTA's shared memory goes away
  }
}

// Asynchronous-epilogue kernel (gemm_async_epi_kernel): the cooperative kernel's items, ring and MMAs, for the
// outputs that leave through a plain TMA store (p.tma_store 1 = bf16 or 2 = fp32; no split, accumulate, GELU or
// residual).  Each consumer warpgroup stages its whole 64 x BN slab at once in a region of its own and hands it to the
// TMA unit as one bulk group, then goes straight on to its next item's MMAs: the stores drain during that mainloop, and
// the warpgroup waits for them to have read the region only when it stages the next slab.  Stages: BN = 128: 6 x 32 KB
// + 2 x 16 KB of staging; 192: 4 x 40 KB + 2 x 24 KB; 256: 3 x 48 KB + 2 x 32 KB; fp32 (BN = 128): 5 x 32 KB + 2 x 32 KB.
template <int BN, bool F32>
struct AsyncEpiCfg {
  static_assert(!F32 || BN == 128, "an fp32 slab wider than 128 columns does not fit next to the ring");
  static constexpr int STAGES = F32 ? 5 : (BN == 256 ? 3 : (BN == 192 ? 4 : 6));
  static constexpr int STAGE_BYTES = GemmCfg<BN>::STAGE_BYTES;
  static constexpr int BOX_COLS = F32 ? 32 : 64;           // one 128-byte swizzle row of the output type
  static constexpr int BOX_BYTES = 64 * 128;               // 64 rows x 128 bytes
  static constexpr int SLAB_BYTES = (BN / BOX_COLS) * BOX_BYTES;
  static constexpr int EPI_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int BAR_OFFSET = EPI_OFFSET + 2 * SLAB_BYTES;
  static constexpr int TOTAL = BAR_OFFSET + 256 + 1024;   // + barriers + alignment slack
  static_assert(TOTAL <= 232448, "GEMM exceeds the 227 KB shared-memory limit");
};

// Whole-slab epilogue of gemm_async_epi_kernel: v = alpha * acc (+ bias), rows [row0, row0 + 64), columns [n0, n0 + BN),
// the values and their order of operations those of epilogue_slab's TMA path.  The slab is BN / BOX_COLS boxes of
// 64 rows x 128 bytes, each in the 128B-swizzle layout of the store map (16-byte chunk c of row r at chunk c ^ (r & 7)),
// so the 8 rows a warp writes per store land in 8 different chunks: no bank conflicts.  fp32: of each thread's column
// pair, threads whose pair lies in the odd chunk write the second element first, which keeps the two threads of each
// bank pair apart.  `bar`: the warpgroup's named barrier; thread t of 128.
template <int BN, bool F32>
__device__ __forceinline__ void epilogue_slab_async(const float (&acc)[BN / 2], int row0, int n0, const GemmParams& p,
                                                    const CUtensorMap* tmC, uint8_t* slab, int bar, int t) {
  using C = AsyncEpiCfg<BN, F32>;
  const int lane = t & 31;
  const int rl = (t >> 5) * 16 + (lane >> 2);   // this thread's first row within the 64; its second is rl + 8
  const int sw = lane >> 2;                     // (rl & 7) == ((rl + 8) & 7)
  const float* bias = p.ep.bias;
  if (t == 0) bulk_wait_read_all();   // the slab this region held one item ago has been read by its stores
  asm volatile("bar.sync %0, 128;" ::"r"(bar) : "memory");
  uint8_t* row_a = slab + rl * 128;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = n0 + j * 8 + 2 * (t & 3);
    float v[4] = {acc[4 * j] * p.ep.alpha, acc[4 * j + 1] * p.ep.alpha, acc[4 * j + 2] * p.ep.alpha,
                  acc[4 * j + 3] * p.ep.alpha};
    if (bias && col < p.N) {
      const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + col));
      v[0] += bb.x; v[1] += bb.y; v[2] += bb.x; v[3] += bb.y;
    }
    if constexpr (!F32) {
      // 8 columns = one 16-byte chunk of a 64-column box
      uint8_t* a = row_a + (j >> 3) * C::BOX_BYTES + ((((j & 7) ^ sw) << 4) | ((t & 3) << 2));
      *reinterpret_cast<uint32_t*>(a) = pack_bf16x2(v[0], v[1]);
      *reinterpret_cast<uint32_t*>(a + 8 * 128) = pack_bf16x2(v[2], v[3]);
    } else {
      // 8 columns = two 16-byte chunks of a 32-column box; the pair of thread t is in chunk 2 (j & 3) + ((t & 3) >> 1)
      const int h = (t >> 1) & 1;
      uint8_t* a = row_a + (j >> 2) * C::BOX_BYTES + ((((2 * (j & 3) + h) ^ sw) << 4) | ((t & 1) << 3));
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int f = e ^ h;
        *reinterpret_cast<float*>(a + 4 * f) = f ? v[1] : v[0];
        *reinterpret_cast<float*>(a + 8 * 128 + 4 * f) = f ? v[3] : v[2];
      }
    }
  }
  fence_proxy_async_smem();
  asm volatile("bar.sync %0, 128;" ::"r"(bar) : "memory");
  if (t == 0) {
#pragma unroll
    for (int b = 0; b < BN / C::BOX_COLS; ++b)
      if (n0 + b * C::BOX_COLS < p.N) tma_store_2d(tmC, slab + b * C::BOX_BYTES, n0 + b * C::BOX_COLS, row0);
    bulk_commit_group();
  }
}

// The cooperative kernel (no split) with epilogue_slab_async: both consumer warpgroups work on every item, 64 rows
// each, with the same produce / mma_kblock sequence, so its output bits are those of gemm_bf16_kernel<BN, ...>.
template <int BN, bool F32, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
    gemm_async_epi_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                          const __grid_constant__ CUtensorMap tmC, const GemmParams p) {
  pdl_launch_dependents();   // as in gemm_bf16_kernel
  using C = AsyncEpiCfg<BN, F32>;
  constexpr int STAGES = C::STAGES;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = threadIdx.x >> 7;
  const int num_items = p.tiles_n * p.tiles_m;
  const int first_item = blockIdx.x;
  const int item_stride = gridDim.x;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmC);
#pragma unroll
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);   // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) produce<BN, A_MN, B_MN, STAGES>(smem, full_bar, empty_bar, &tmA, &tmB, p, first_item,
                                                          item_stride, num_items);
  } else {
    setmaxnreg_inc<232>();
    const int cw = wg - 1;                 // rows [64 cw, 64 cw + 64) of the tile
    const int t = threadIdx.x & 127;
    uint8_t* slab = smem + C::EPI_OFFSET + cw * C::SLAB_BYTES;
    uint32_t it = 0;       // k-blocks consumed so far, over all items
    float acc[BN / 2];     // written by each item's first wgmma (scale-d = 0)

    for (int item = first_item; item < num_items; item += item_stride) {
      const WorkItem w = decode_item<BN>(item, p);
      for (int kb = 0; kb < w.nkb; ++kb, ++it) {
        const int s = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1;
        mbar_wait(&full_bar[s], ph);
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) reg_fence(acc[i]);
        wgmma_fence();
        mma_kblock<BN, A_MN, B_MN>(acc, smem + s * C::STAGE_BYTES, cw, kb == 0);
        wgmma_commit();
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) reg_fence(acc[i]);
        wgmma_wait<1>();   // the previous k-block's MMAs have retired: its stage may be refilled
        if (kb > 0 && t == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
      }
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) reg_fence(acc[i]);
      if (t == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
      epilogue_slab_async<BN, F32>(acc, w.m0 + cw * 64, w.n0, p, &tmC, slab, 2 + cw, t);
    }
    if (t == 0) bulk_wait_all();   // the stores are complete before the CTA's shared memory goes away
  }
}

// ORD: the cooperative kernel's ordered split-K form; AE = 1 / 2: the asynchronous-epilogue kernel for a bf16 / fp32
// TMA-stored output (one split)
template <int BN, bool A_MN, bool B_MN, bool ORD = false, int AE = 0>
int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const GemmParams& p,
                cudaStream_t stream) {
  static_assert(!AE || !ORD, "the asynchronous-epilogue kernel runs unsplit");
  constexpr int TOTAL = AE ? AsyncEpiCfg<BN, AE == 2>::TOTAL : GemmCfg<BN>::TOTAL;
  auto kern = [] {
    if constexpr (AE) return gemm_async_epi_kernel<BN, AE == 2, A_MN, B_MN>;
    else return gemm_bf16_kernel<BN, A_MN, B_MN, ORD>;
  }();
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = TOTAL;
  cfg.stream = stream;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr.val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  // CTAs of this kernel the device can hold at once: one per SM
  static int resident = 0;
  if (resident == 0) {
    MMAE_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, TOTAL));
    int dev = 0;
    MMAE_CUDA_OK(cudaGetDevice(&dev));
    MMAE_CUDA_OK(cudaDeviceGetAttribute(&resident, cudaDevAttrMultiProcessorCount, dev));
    MMAE_CHECK(resident > 0, MMAE_ERR_CUDA, "mmae_gemm_bf16: the GEMM kernel does not fit on an SM");
  }
  const int items = p.tiles_n * p.tiles_m * p.splits;
  const int slots = std::min(resident, std::max(1, sm_count()));
  cfg.gridDim = dim3(std::min(items, slots));
  const bool prof = gemm_profile_begin(stream, 2.0 * p.M * p.N * p.K, p.M, p.N, p.K,
                                       (A_MN ? 1 : 0) | (B_MN ? 2 : 0) | (ORD ? 8 : 0) | (AE ? 16 : 0) |
                                           (p.splits << 8));
  MMAE_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, tmA, tmB, tmC, p));
  if (prof) gemm_profile_end(stream);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

// Second pass of ordered split-K: out += ((ws[0] + ws[1]) + ... + ws[S - 1]) (+ residual), four columns per thread.
// Like the unordered split-K, which reduce-adds every split onto out, it adds onto out whether or not accumulate is set
// (the ABI: a split-K destination is zeroed or holds the value to accumulate onto).  Slice s of the workspace holds rows
// [s * slice_rows, ...) of a [*, N] fp32 matrix.  Each output element has one writer: a single plain add.
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ ws, int S, int slice_rows, int M,
                                                             int N, const float* __restrict__ residual,
                                                             int64_t ld_residual, float* __restrict__ out,
                                                             int64_t ld_out) {
  pdl_prologue();
  const int n4 = N / 4;
  const int64_t total = int64_t(M) * n4;
  const int64_t slice = int64_t(slice_rows) * N;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
    const int m = int(i / n4), c = int(i - int64_t(m) * n4) * 4;
    const float* src = ws + int64_t(m) * N + c;
    float4 v = __ldcg(reinterpret_cast<const float4*>(src));
    for (int s = 1; s < S; ++s) {
      const float4 u = __ldcg(reinterpret_cast<const float4*>(src + s * slice));
      v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w;
    }
    if (residual) {
      const float4 r = __ldg(reinterpret_cast<const float4*>(residual + int64_t(m) * ld_residual + c));
      v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
    }
    float4* dst = reinterpret_cast<float4*>(out + int64_t(m) * ld_out + c);
    const float4 o = *dst;
    *dst = make_float4(o.x + v.x, o.y + v.y, o.z + v.z, o.w + v.w);
  }
}

}  // namespace
}  // namespace mmae

using namespace mmae;

// -1 (the cost model) or a variant below
static bool variant_valid(int v) { return v == -1 || (v >= 1 && v <= 3) || (v >= 8 && v <= 10); }

// MMAE_GEMM_VARIANT / MMAE_GEMM_TMA_STORE set the initial values of the two switches below
static int g_gemm_variant = []() {
  const char* e = getenv("MMAE_GEMM_VARIANT");
  const int v = e ? atoi(e) : -1;
  return variant_valid(v) ? v : -1;
}();
static int g_gemm_tma_store = []() {
  const char* e = getenv("MMAE_GEMM_TMA_STORE");
  return e ? (atoi(e) != 0) : 1;
}();

extern "C" int mmae_gemm_set_variant(int variant) {
  MMAE_CHECK(variant_valid(variant), MMAE_ERR_ARG, "mmae_gemm_set_variant: %d (-1, 1, 2, 3, 8, 9 or 10)", variant);
  g_gemm_variant = variant;
  return MMAE_OK;
}

extern "C" int mmae_gemm_set_tma_store(int enable) {
  g_gemm_tma_store = enable != 0;
  return MMAE_OK;
}

// variant -> tile: 1 / 3 / 2 = the cooperative kernel, BN = 128 / 192 / 256; 8 / 9 / 10 = the asynchronous whole-slab
// epilogue, BN = 128 / 192 / 256 (a call it cannot take runs variant 1 / 3 / 2)
static int variant_bn(int v) { return (v == 1 || v == 8) ? 128 : (v == 3 || v == 9) ? 192 : 256; }
static bool variant_async(int v) { return v >= 8; }
// the cooperative single-CTA variant of an asynchronous-epilogue variant's tile
static int variant_coop(int v) { return v == 8 ? 1 : (v == 9 ? 3 : (v == 10 ? 2 : v)); }

// Fixed cost of one work item in the persistent kernel, in k-block times of its tile: its epilogue and the hand-over to
// the next item.  scripts/gpu_time_gemm.py --fixed-cost measured 13.4, 14.0, 10.0 and 5.0 us per extra 128 x 256 fp32
// reduce-add item at 2, 4, 8 and 12 items per SM, against 0.9 us per k-block (H100 SXM, 700 W power limit): 15 falling to
// 5.5 k-block times as items per SM grow.  The model takes 4, near the low end, where the long-K weight gradients run;
// 5 or more would cut fc1 / fc2's weight gradient to 5 splits of 40 k-blocks in 3 rounds, 4 keeps 9 splits of 22 in 5.
// bf16-output items with a bias (N = 768, 3 to 12 items per SM, same card and limit) cost more: 128 x 128 tiles 9.5
// (K = 256) and 10.3 (K = 768) k-block times of 0.353 us, 128 x 256 tiles 11.0 and 8.4 of 0.686 us.  (Measured while the
// TMA epilogue still loaded the bias inside each staged box: see epilogue_slab.)
constexpr int KB_PER_ITEM_FIXED = 4;
// The asynchronous-epilogue kernel (variants 8-10) leaves little of that: measured as the bf16 items above (N = 768, a
// bias), 128 x 128 items cost 2.1 (K = 256) and 2.5 (K = 768) k-block times of 0.392 us, 128 x 192 3.6 and 5.1 of
// 0.516 us, 128 x 256 2.8 and 1.5 of 0.752 us; fp32 128 x 128 items without a bias 2.1 and 5.6 of 0.349 us, against
// 5.6 and 4.5 for the cooperative kernel's (same card and limit).  The model takes 2.  Its unsplit candidates all
// share the constant, so for bf16 outputs it picks the tile width the cooperative kernel had.
constexpr int ASYNC_KB_PER_ITEM_FIXED = 2;
// Split-K never cuts an item below this many k-blocks, which bounds the fp32 reduce-add traffic it adds
constexpr int MIN_KB_PER_SPLIT = 16;
// Deterministic mode: the automatic split makes ceil(k-blocks / DET_KB_PER_SPLIT) splits of equal k-block counts, so
// the split count, and with it the summation order, follows from K alone.  The bench step's long-K weight gradients
// (K = tokens, 198 k-blocks) get 7 splits of 29 k-blocks.
constexpr int DET_KB_PER_SPLIT = 32;

// Ordered split-K (deterministic mode): each split stores its fp32 partial tile with the plain TMA-store epilogue into
// its own slice of a [splits, tiles_m * BM, N] workspace from the per-stream pool, and splitk_reduce_kernel adds the
// slices in split order (then residual), and adds the sum onto the output.
template <int BN, bool A_MN, bool B_MN>
int launch_ordered(const CUtensorMap& tmA, const CUtensorMap& tmB, GemmParams p, cudaStream_t st) {
  const int slice_rows = p.tiles_m * BM;
  const size_t floats = size_t(p.splits) * slice_rows * p.N;
  float* ws = colred_scratch(floats, st);
  if (!ws) {
    set_last_error("mmae_gemm_bf16: the ordered split-K workspace of deterministic mode (mmae_set_deterministic) needs "
                   "%zu bytes, which must be allocated outside stream capture: run the step once eagerly first",
                   floats * sizeof(float));
    return MMAE_ERR_CUDA;
  }
  CUtensorMap tmC;
  const int rc = make_tmap_2d_store(&tmC, ws, 4, uint64_t(p.splits) * slice_rows, (uint64_t)p.N, (uint64_t)p.N);
  if (rc) return rc;
  const mmae_gemm_epilogue ep = p.ep;
  p.tma_store = 2;
  const int lrc = launch_gemm<BN, A_MN, B_MN, true>(tmA, tmB, tmC, p, st);
  if (lrc) return lrc;
  const int64_t total = int64_t(p.M) * (p.N / 4);
  const unsigned blocks = (unsigned)std::max<int64_t>(1, std::min<int64_t>((total + 255) / 256, int64_t(sm_count()) * 16));
  launch_k(splitk_reduce_kernel, blocks, 256, 0, st, ws, p.splits, slice_rows, p.M, p.N, ep.residual, ep.ld_residual,
           ep.out_f32, ep.ld_out_f32);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

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
  const bool det = deterministic();
  const int sms = det ? DET_SM_COUNT : sm_count();   // deterministic mode: the tile choice follows the shape alone
  const int tm = ceil_div(M, BM);
  if (split_k <= 0 && !(ep->out_f32 && !ep->out_bf16 && !ep->preact_bf16 && !ep->dgelu_z && ep->act == 0)) split_k = 1;
  if (det && split_k <= 0) split_k = ceil_div(num_kb, DET_KB_PER_SPLIT);
  // unsplit, the output leaves through a plain TMA store: the asynchronous-epilogue kernel can take the call (bf16 at
  // every width it has, fp32 at BN = 128)
  const bool async_ok = g_gemm_tma_store && split_k <= 1 && !ep->accumulate && ep->act == 0 && !ep->residual &&
                        !ep->preact_bf16 && !ep->dgelu_z && (!ep->out_bf16 != !ep->out_f32);
  const bool async_f32 = ep->out_f32 != nullptr;

  // Tile width and split count from one model of the persistent grid: it runs sm_count() items at a time, so a launch
  // lasts ceil(items / slots) rounds of one item, and an item costs ~(k-blocks + KB_PER_ITEM_FIXED) k-block times.  A
  // k-block of a 128 x BN tile costs ~(BN + 40): the A tile's loads and MMA issue do not shrink with BN, which makes wide
  // tiles the better choice whenever their rounds are as full.
  // 128 x 192 wins where its rounds are fuller: the encoder's N = 768 GEMMs make 99 x 4 = 396 tiles, exactly three
  // rounds of 132 SMs, against 297 of 128 x 256 in 2.25.  The automatic split (split_k <= 0) fills the last round of the
  // long-K weight gradients instead of leaving it mostly idle.  An explicit variant fixes the tile, an explicit split_k
  // the split.
  // The asynchronous-epilogue kernel replaces the cooperative one of its width among the candidates wherever it can
  // take the call; its items, unsplit, cost ASYNC_KB_PER_ITEM_FIXED.
  int variant = g_gemm_variant;
  {
    int cand_var[4] = {1, 2, 3, -1};
    if (async_ok) {
      cand_var[0] = 8;
      if (!async_f32) {
        cand_var[1] = 10;
        cand_var[2] = 9;
      } else if (split_k <= 0) {
        cand_var[3] = 1;   // the split forms of the 128-column tile stay open
      }
    }
    const int nvar = variant >= 0 ? 1 : (cand_var[3] >= 0 ? 4 : 3);
    long best_cost = -1;
    int best_split = 1, best_var = variant >= 0 ? variant : cand_var[0];
    for (int i = 0; i < nvar; ++i) {
      const int v = variant >= 0 ? variant : cand_var[i];
      const int bn = variant_bn(v);
      if (variant < 0 && bn > 128 && N < bn) continue;
      const long tiles = long(tm) * ceil_div(N, bn);
      const int slots = std::max(1, sms);
      const bool ae = variant_async(v) && async_ok;
      const int fixed = ae ? ASYNC_KB_PER_ITEM_FIXED : KB_PER_ITEM_FIXED;
      const int s_lo = split_k > 0 ? split_k : 1;
      const int s_hi = split_k > 0 || ae ? s_lo : std::max(1, num_kb / MIN_KB_PER_SPLIT);
      for (int s = s_lo; s <= s_hi; ++s) {
        const int kbps = ceil_div(num_kb, std::min(s, num_kb));
        const long rounds = (tiles * ceil_div(num_kb, kbps) + slots - 1) / slots;
        const long cost = rounds * (bn + 40) * (kbps + fixed);
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

  const bool ordered = det && split_k > 1;
  // a call the asynchronous-epilogue kernel cannot take (split, or an fp32 output wider than 128 columns) runs the
  // cooperative kernel of the same width
  if (variant_async(variant) && (!async_ok || split_k > 1 || (async_f32 && variant != 8))) variant = variant_coop(variant);
  const int BNsel = variant_bn(variant);

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
    rc = make_tmap_2d_bf16(&tmB, B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, BK, BNsel);
  } else {
    rc = make_tmap_2d_bf16(&tmB, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb, 64, BK);
  }
  if (rc) return rc;

  GemmParams p;
  p.M = M; p.N = N; p.K = K;
  p.num_kb = num_kb;
  p.kb_per_split = kb_per_split;
  p.tiles_n = ceil_div(N, BNsel);
  p.tiles_m = tm;
  p.splits = split_k;
  p.ep = *ep;
  // plain bf16 / fp32 outputs (optionally with bias / GELU) leave through shared memory and TMA tile stores; fp32
  // accumulation (split-K, accumulate) through TMA reduce-add tiles
  p.tma_store = 0;
  CUtensorMap tmC = tmA;
  if (variant_async(variant)) {
    p.tma_store = async_f32 ? 2 : 1;
    rc = async_f32 ? make_tmap_2d_store_sw128(&tmC, ep->out_f32, 4, (uint64_t)M, (uint64_t)N, (uint64_t)ep->ld_out_f32)
                   : make_tmap_2d_store_sw128(&tmC, ep->out_bf16, 2, (uint64_t)M, (uint64_t)N, (uint64_t)ep->ld_out_bf16);
    if (rc) return rc;
  } else if (g_gemm_tma_store && !ep->preact_bf16 && !ep->dgelu_z && !ep->residual) {
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
  if (ordered) {
#define MMAE_DISPATCH_ORD(BN_)                                                                  \
  do {                                                                                          \
    if (!a_mn_major && !b_mn_major) return launch_ordered<BN_, false, false>(tmA, tmB, p, st);  \
    if (!a_mn_major && b_mn_major) return launch_ordered<BN_, false, true>(tmA, tmB, p, st);    \
    if (a_mn_major && !b_mn_major) return launch_ordered<BN_, true, false>(tmA, tmB, p, st);    \
    return launch_ordered<BN_, true, true>(tmA, tmB, p, st);                                    \
  } while (0)
    if (BNsel == 192) MMAE_DISPATCH_ORD(192);
    if (BNsel == 256) MMAE_DISPATCH_ORD(256);
    MMAE_DISPATCH_ORD(128);
#undef MMAE_DISPATCH_ORD
  }
#define MMAE_DISPATCH(BN_, AE_)                                                                       \
  do {                                                                                                \
    if (!a_mn_major && !b_mn_major) return launch_gemm<BN_, false, false, false, AE_>(tmA, tmB, tmC, p, st); \
    if (!a_mn_major && b_mn_major) return launch_gemm<BN_, false, true, false, AE_>(tmA, tmB, tmC, p, st);   \
    if (a_mn_major && !b_mn_major) return launch_gemm<BN_, true, false, false, AE_>(tmA, tmB, tmC, p, st);   \
    return launch_gemm<BN_, true, true, false, AE_>(tmA, tmB, tmC, p, st);                                  \
  } while (0)
  if (variant == 8 && p.tma_store == 2) MMAE_DISPATCH(128, 2);
  if (variant == 8) MMAE_DISPATCH(128, 1);
  if (variant == 9) MMAE_DISPATCH(192, 1);
  if (variant == 10) MMAE_DISPATCH(256, 1);
  if (variant == 3) MMAE_DISPATCH(192, 0);
  if (variant == 2) MMAE_DISPATCH(256, 0);
  MMAE_DISPATCH(128, 0);
#undef MMAE_DISPATCH
}
