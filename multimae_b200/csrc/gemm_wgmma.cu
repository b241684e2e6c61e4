// wgmma / TMA GEMM for sm_90a:  C[M,N] = epilogue(alpha * A * B^T), bf16 operands, fp32 accumulate in registers.
//
// One CTA computes one 128 x BN output tile (BN = 64 / 128 / 192 / 256) over a K range (split-K along gridDim.z); three
// warpgroups:
//   warpgroup 0    : TMA producer (one thread: cp.async.bulk.tensor -> 128B-swizzled shared-memory ring, mbarrier
//                    complete_tx); gives its registers to the consumers (setmaxnreg)
//   warpgroups 1-2 : consumers, 64 rows of the tile each: wgmma 64 x BN x 16 straight from the ring (K-major or MN-major
//                    operands through the descriptor's transpose bit), then the fused epilogue from the accumulator
//                    registers (bias / GELU / dGELU / residual, bf16 and fp32 outputs, red.global adds for split-K), or
//                    for plain bf16 / fp32 outputs through shared memory and TMA tile stores / reduce-adds
// CL = 2: a cluster of two CTAs along M shares the B tile - each CTA loads half of it and multicasts it to both, so a
// 256 x BN output tile reads B from L2 once.  A stage is refilled only after the consumers of BOTH CTAs released it.
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
  int tma_store;     // output through shared memory + TMA: 1 = bf16 store, 2 = fp32 store, 3 = fp32 reduce-add
  mmae_gemm_epilogue ep;
};

// ~192 KB of stages (BN = 64: 8 x 24 KB, 128: 6 x 32 KB, 192: 5 x 40 KB, 256: 4 x 48 KB).  One CTA per SM.
template <int BN>
struct GemmCfg {
  static constexpr int STAGES = BN == 256 ? 4 : (BN == 192 ? 5 : (BN == 128 ? 6 : 8));
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int TOTAL = BAR_OFFSET + 256 + 1024;  // + barriers + alignment slack
  static_assert(TOTAL <= 232448, "GEMM exceeds the 227 KB shared-memory limit");
};

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

// TMA-store staging: per consumer warpgroup, BN / 32 dense boxes of 64 rows x 32 columns
template <typename T>
__device__ __forceinline__ void stage_pair(uint8_t* stage, int r, int c, float v0, float v1) {
  T* box = reinterpret_cast<T*>(stage + (c >> 5) * (64 * 32 * sizeof(T)));
  if constexpr (sizeof(T) == 4) *reinterpret_cast<float2*>(box + r * 32 + (c & 31)) = make_float2(v0, v1);
  else *reinterpret_cast<uint32_t*>(box + r * 32 + (c & 31)) = pack_bf16x2(v0, v1);
}

template <int BN, int CL, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
    gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                     const __grid_constant__ CUtensorMap tmC, const GemmParams p) {
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
  const int n0 = blockIdx.x * BN;
  const int m0 = blockIdx.y * BM;
  const int kb_begin = blockIdx.z * p.kb_per_split;
  int nkb = p.num_kb - kb_begin;
  if (nkb > p.kb_per_split) nkb = p.kb_per_split;
  if (nkb < 0) nkb = 0;

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
      for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % STAGES;
        const uint32_t ph = (kb / STAGES) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1u);
        mbar_expect_tx(&full_bar[s], C::STAGE_BYTES);
        uint8_t* sA = smem + s * C::STAGE_BYTES;
        uint8_t* sB = sA + C::A_BYTES;
        const int k0 = (kb_begin + kb) * BK;
        if constexpr (!A_MN) {
          tma_load_2d(sA, &tmA, &full_bar[s], k0, m0);
        } else {
#pragma unroll
          for (int c = 0; c < BM / 64; ++c) tma_load_2d(sA + c * (64 * BK * 2), &tmA, &full_bar[s], m0 + c * 64, k0);
        }
        if constexpr (CL == 1) {
          if constexpr (!B_MN) {
            tma_load_2d(sB, &tmB, &full_bar[s], k0, n0);
          } else {
#pragma unroll
            for (int c = 0; c < BN / 64; ++c) tma_load_2d(sB + c * (64 * BK * 2), &tmB, &full_bar[s], n0 + c * 64, k0);
          }
        } else {
          if constexpr (!B_MN) {
            tma_load_2d_multicast(sB + rank * BH * 128, &tmB, &full_bar[s], k0, n0 + rank * BH, 0x3);
          } else {
#pragma unroll
            for (int c = 0; c < BH / 64; ++c)
              tma_load_2d_multicast(sB + (rank * (BH / 64) + c) * (64 * BK * 2), &tmB, &full_bar[s], n0 + rank * BH + c * 64,
                                    k0, 0x3);
          }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers (warpgroups 1, 2)
    setmaxnreg_inc<232>();
    const int cw = wg - 1;                 // rows [64 cw, 64 cw + 64) of the tile
    float acc[BN / 2];   // written by the first wgmma (scale-d = 0); read only when nkb > 0

    for (int kb = 0; kb < nkb; ++kb) {
      const int s = kb % STAGES;
      const uint32_t ph = (kb / STAGES) & 1;
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
      if (kb > 0 && (threadIdx.x & 127) == 0) {
        const int rs = (kb - 1) % STAGES;
        if constexpr (CL == 1) mbar_arrive(&empty_bar[rs]);
        else
          for (int r = 0; r < CL; ++r) mbar_arrive_cluster(mapa_u32(smem_u32(&empty_bar[rs]), uint32_t(r)));
      }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) reg_fence(acc[i]);

    const int t = threadIdx.x & 127;
    const int rl = (t >> 5) * 16 + ((t & 31) >> 2);       // this thread's first row within the warpgroup's 64
    const int row_a = m0 + cw * 64 + rl;
    const int row_b = row_a + 8;
    const bool first_split = blockIdx.z == 0;
    if (nkb > 0 && p.tma_store) {
      // ---------------------------------------------------------------- epilogue through shared memory + TMA
      // both warpgroups have retired their last MMA before the ring is reused as the staging area
      asm volatile("bar.sync 1, 256;" ::: "memory");
      uint8_t* stage = smem + cw * (64 * BN * (p.tma_store == 1 ? 2 : 4));
      const float* bias = first_split ? p.ep.bias : nullptr;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = j * 8 + 2 * (t & 3);
        float v[4] = {acc[4 * j] * p.ep.alpha, acc[4 * j + 1] * p.ep.alpha, acc[4 * j + 2] * p.ep.alpha,
                      acc[4 * j + 3] * p.ep.alpha};
        if (bias && n0 + c < p.N) {
          const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + n0 + c));
          v[0] += bb.x; v[1] += bb.y; v[2] += bb.x; v[3] += bb.y;
        }
        if (p.ep.act == 1) {
#pragma unroll
          for (int i = 0; i < 4; ++i) v[i] = gelu_erf(v[i]);
        }
        if (p.tma_store == 1) {
          stage_pair<bf16>(stage, rl, c, v[0], v[1]);
          stage_pair<bf16>(stage, rl + 8, c, v[2], v[3]);
        } else {
          stage_pair<float>(stage, rl, c, v[0], v[1]);
          stage_pair<float>(stage, rl + 8, c, v[2], v[3]);
        }
      }
      fence_proxy_async_smem();
      asm volatile("bar.sync %0, 128;" ::"r"(2 + cw) : "memory");
      if (t == 0) {
        const int box_bytes = 64 * 32 * (p.tma_store == 1 ? 2 : 4);
        for (int b = 0; b < BN / 32 && n0 + b * 32 < p.N; ++b) {
          if (p.tma_store == 3) tma_reduce_add_2d(&tmC, stage + b * box_bytes, n0 + b * 32, m0 + cw * 64);
          else tma_store_2d(&tmC, stage + b * box_bytes, n0 + b * 32, m0 + cw * 64);
        }
        bulk_commit_group();
        bulk_wait_all();   // the stores have read the staging area before the CTA's shared memory goes away
      }
    } else if (nkb > 0) {
      // ---------------------------------------------------------------- epilogue straight from the accumulator registers
      const bool atomic_out = p.ep.accumulate != 0 || gridDim.z > 1;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        if (n0 + j * 8 >= p.N) break;   // N % 8 == 0: a column pair is either fully inside or fully outside
        const int n = n0 + j * 8 + 2 * (t & 3);
        if (row_a < p.M) epilogue_pair(acc[4 * j], acc[4 * j + 1], row_a, n, p, first_split, atomic_out);
        if (row_b < p.M) epilogue_pair(acc[4 * j + 2], acc[4 * j + 3], row_b, n, p, first_split, atomic_out);
      }
    }
  }
  // no CTA of a cluster may leave while its peer can still arrive on its barriers
  if constexpr (CL > 1) cluster_sync_all();
}

template <int BN, int CL, bool A_MN, bool B_MN>
int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const GemmParams& p, int split_k,
                cudaStream_t stream) {
  using C = GemmCfg<BN>;
  auto kern = gemm_bf16_kernel<BN, CL, A_MN, B_MN>;
  static bool configured = false;
  if (!configured) {
    MMAE_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::TOTAL));
    configured = true;
  }
  dim3 grid(ceil_div(p.N, BN), ceil_div(ceil_div(p.M, BM), CL) * CL, split_k);
  const bool prof = gemm_profile_begin(stream, 2.0 * p.M * p.N * p.K, p.M, p.N, p.K, (A_MN ? 1 : 0) | (B_MN ? 2 : 0) | (split_k << 8));
  if constexpr (CL == 1) {
    launch_k(kern, grid, GEMM_THREADS, C::TOTAL, stream, tmA, tmB, tmC, p);
  } else {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = dim3(GEMM_THREADS);
    cfg.dynamicSmemBytes = C::TOTAL;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 1;
    attr[0].val.clusterDim.y = CL;
    attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 2 : 1;
    MMAE_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, tmA, tmB, tmC, p));
  }
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
  int variant = g_gemm_variant;
  const int sms = sm_count();
  const int tm = ceil_div(M, BM);
  if (split_k <= 0 && !(ep->out_f32 && !ep->out_bf16 && !ep->preact_bf16 && !ep->dgelu_z && ep->act == 0)) split_k = 1;
  if (split_k <= 0) {
    // auto split-K (weight gradients: small M x N, long K).  Joint choice of tile width and split count: one wave of
    // ~SM-count work items; an item costs ~BN * (k-blocks + 6), the 6 standing for the fp32 reduce-add epilogue.
    const int cand_var[2] = {1, 2};
    long best_cost = -1;
    int best_split = 1, best_var = variant >= 0 ? variant : 1;
    for (int i = 0; i < (variant >= 0 ? 1 : 2); ++i) {
      const int v = variant >= 0 ? variant : cand_var[i];
      const int bn = variant_bn(v);
      if (variant < 0 && bn > 128 && N < bn) continue;
      const int tiles = tm * ceil_div(N, bn);
      int s_ = std::max(1, sms / tiles);
      s_ = std::min(s_, std::max(1, num_kb / 4));
      const int kbps = ceil_div(num_kb, s_);
      s_ = ceil_div(num_kb, kbps);
      const long rounds = (long(tiles) * s_ + sms - 1) / sms;
      const long cost = rounds * bn * (kbps + 6);
      if (best_cost < 0 || cost < best_cost) {
        best_cost = cost;
        best_split = s_;
        best_var = v;
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

  if (variant < 0) {
    // tile-quantisation model: ceil(tiles / SMs) waves; a wave costs ~(BN + c), c standing for the per-tile fixed work
    // (pipeline fill, epilogue).  Pick the cheaper of BN = 128 / 256.
    const int cand_var[2] = {1, 2};
    long best_cost = -1;
    variant = 1;
    for (int i = 0; i < 2; ++i) {
      const int bn = variant_bn(cand_var[i]);
      if (bn > 128 && N < bn) continue;
      const long items = long(tm) * ceil_div(N, bn) * split_k;
      const long rounds = (items + sms - 1) / sms;
      const long cost = rounds * (bn + 40);
      if (best_cost < 0 || cost < best_cost) {
        best_cost = cost;
        variant = cand_var[i];
      }
    }
  }
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
#define MMAE_DISPATCH(BN_, CL_)                                                                               \
  do {                                                                                                        \
    if (!a_mn_major && !b_mn_major) return launch_gemm<BN_, CL_, false, false>(tmA, tmB, tmC, p, split_k, st); \
    if (!a_mn_major && b_mn_major) return launch_gemm<BN_, CL_, false, true>(tmA, tmB, tmC, p, split_k, st);   \
    if (a_mn_major && !b_mn_major) return launch_gemm<BN_, CL_, true, false>(tmA, tmB, tmC, p, split_k, st);   \
    return launch_gemm<BN_, CL_, true, true>(tmA, tmB, tmC, p, split_k, st);                                  \
  } while (0)
  if (variant == 4) MMAE_DISPATCH(256, 2);
  if (variant == 6) MMAE_DISPATCH(128, 2);
  if (variant == 5) {
    if (!a_mn_major) return launch_gemm<192, 2, false, false>(tmA, tmB, tmC, p, split_k, st);
    return launch_gemm<192, 2, true, false>(tmA, tmB, tmC, p, split_k, st);
  }
  if (variant == 0) MMAE_DISPATCH(64, 1);
  if (variant == 3) MMAE_DISPATCH(192, 1);
  if (variant == 2) MMAE_DISPATCH(256, 1);
  MMAE_DISPATCH(128, 1);
#undef MMAE_DISPATCH
}
