// Truncated depth standardisation, second version - the default since round 2 (mmae_standardize_depth_set_variant(1) /
// MMAE_DEPTH_STD_VARIANT=1 select the kernel of depth_standardize.cu), checked against the oracle fixtures
// (tests/test_cuda_kernels.py).  Both variants are latency-bound shared-memory selects well below the 8 B/pixel HBM figure.
//
// Variant 1's first radix-select pass funnels 32 warps into a handful of shared-memory histogram bins (depth maps use
// few exponent values; warp aggregation removes only the intra-warp conflicts), and maps that do not fit one CTA's
// shared memory (448^2) fall back to seven passes over L2 on only B CTAs.  This version
//   * keeps 16 histogram copies (pass 0: one selection, 2 warps per copy; later passes: 2 selections x 8 copies);
//   * splits a map that exceeds one CTA's shared memory over a thread-block cluster of 2 / 4 / 8 CTAs, each caching its
//     slice as order-preserving keys; the per-CTA histograms and partial sums are combined through distributed shared
//     memory (every CTA reads every peer's 2 x 256 counters and makes the same selection decision), so the map is still
//     read from HBM once and written once.
// Same arithmetic as variant 1: exact order statistics, fp32 per-thread partial sums, fp64 across threads and CTAs (in
// rank order, so every CTA of a cluster holds bit-identical mean / variance).
#include <cstdlib>

#include "internal.h"

namespace mmae {
namespace {

constexpr int DS2_THREADS = 1024;
constexpr int DS2_COPIES = 16;

__device__ __forceinline__ uint32_t f2key2(float f) {
  const uint32_t b = __float_as_uint(f);
  return (b >> 31) ? ~b : (b ^ 0x80000000u);
}
__device__ __forceinline__ float key2f2(uint32_t k) { return __uint_as_float((k >> 31) ? (k ^ 0x80000000u) : ~k); }

__device__ __forceinline__ uint32_t ld_cluster_u32(uint32_t cluster_addr) {
  uint32_t v;
  asm volatile("ld.shared::cluster.u32 %0, [%1];" : "=r"(v) : "r"(cluster_addr) : "memory");
  return v;
}
__device__ __forceinline__ double ld_cluster_f64(uint32_t cluster_addr) {
  double v;
  asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(cluster_addr) : "memory");
  return v;
}

__device__ __forceinline__ double block_sum2(double v, double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) red[warp] = v;
  __syncthreads();
  if (warp == 0) {
    double t = lane < DS2_THREADS / 32 ? red[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (lane == 0) red[0] = t;
  }
  __syncthreads();
  const double r = red[0];
  __syncthreads();
  return r;
}

// CS = CTAs per sample (cluster size); blockIdx.x = sample * CS + rank.  Dynamic shared memory: `chunk` keys.
template <int CS>
__global__ void __launch_bounds__(DS2_THREADS, 1)
depth_standardize_v2_kernel(const float* x, float* y, int n, int chunk, int lo, int hi, float eps, float* stats) {
  pdl_prologue();
  extern __shared__ __align__(16) uint8_t ds2_smem[];
  uint32_t* keys = reinterpret_cast<uint32_t*>(ds2_smem);
  __shared__ uint32_t hist[DS2_COPIES][256];
  __shared__ uint32_t merged[2][256];          // this CTA's counters per selection (read by the peers)
  __shared__ double part[2];                   // this CTA's partial sums (read by the peers)
  __shared__ uint32_t sel_key[2], sel_rank[2], sel_eq[2];
  __shared__ double red[DS2_THREADS / 32];

  const int sample = blockIdx.x / CS;
  const uint32_t rank = CS > 1 ? cluster_ctarank() : 0u;
  const int begin = min(n, int(rank) * chunk), end = min(n, begin + chunk);
  const int cnt = end - begin;
  const float* xs = x + int64_t(sample) * n + begin;
  float* ys = y + int64_t(sample) * n + begin;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // chunk is a multiple of 4, so a slice starts 16-byte aligned whenever the sample does
  const bool vec4 = (n % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) % 16 == 0);

  if (vec4) {
    for (int i = tid; i < cnt / 4; i += DS2_THREADS) {
      const float4 v = reinterpret_cast<const float4*>(xs)[i];
      reinterpret_cast<uint4*>(keys)[i] = make_uint4(f2key2(v.x), f2key2(v.y), f2key2(v.z), f2key2(v.w));
    }
  } else {
    for (int i = tid; i < cnt; i += DS2_THREADS) keys[i] = f2key2(xs[i]);
  }
  if (tid < 2) {
    sel_key[tid] = 0u;
    sel_rank[tid] = tid == 0 ? uint32_t(lo) : uint32_t(hi - 1);
    sel_eq[tid] = 0u;
  }
  __syncthreads();

  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    const uint32_t pmask = pass == 0 ? 0u : (0xFFFFFFFFu << (shift + 8));
    for (int i = tid; i < DS2_COPIES * 256; i += DS2_THREADS) (&hist[0][0])[i] = 0u;
    __syncthreads();
    const uint32_t p0 = sel_key[0], p1 = sel_key[1];
    // pass 0: every element is a candidate of both selections -> one histogram over all 16 copies
    // later : selection s counts into copies [8 s, 8 s + 8)
    const int copy0 = pass == 0 ? (warp & (DS2_COPIES - 1)) : (warp & 7);
    const int copy1 = pass == 0 ? copy0 : 8 + (warp & 7);
    for (int i0 = 0; i0 < cnt; i0 += DS2_THREADS) {       // uniform trip count per CTA: whole warps reach the votes
      const int i = i0 + tid;
      const bool valid = i < cnt;
      const uint32_t k = valid ? keys[i] : 0u;
      const uint32_t d = (k >> shift) & 255u;
      const bool m0 = valid && ((k & pmask) == p0);
      const bool m1 = valid && ((k & pmask) == p1) && pass != 0;
      const uint32_t code = d | (m0 ? 256u : 0u) | (m1 ? 512u : 0u);
      const uint32_t peers = __match_any_sync(0xffffffffu, code);
      if ((m0 || m1) && lane == __ffs(peers) - 1) {
        const uint32_t c = __popc(peers);
        if (m0) atomicAdd(&hist[copy0][d], c);
        if (m1) atomicAdd(&hist[copy1][d], c);
      }
    }
    __syncthreads();
    if (tid < 512) {                                      // merge the copies: merged[s][bin]
      const int s = tid >> 8, bin = tid & 255;
      uint32_t c = 0u;
      if (pass == 0) {
#pragma unroll
        for (int q = 0; q < DS2_COPIES; ++q) c += hist[q][bin];
      } else {
#pragma unroll
        for (int q = 0; q < 8; ++q) c += hist[8 * s + q][bin];
      }
      merged[s][bin] = c;
    }
    __syncthreads();
    if (CS > 1) cluster_sync_all();                       // every CTA's `merged` is complete and visible
    if (tid < 64) {                                       // warp s resolves selection s over the whole sample
      const int s = tid >> 5;
      uint32_t c[8], tot = 0u;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (CS > 1) {
          uint32_t a = 0u;
          const uint32_t local = smem_u32(&merged[s][lane * 8 + j]);
#pragma unroll
          for (int r = 0; r < CS; ++r) a += ld_cluster_u32(mapa_u32(local, uint32_t(r)));
          c[j] = a;
        } else {
          c[j] = merged[s][lane * 8 + j];
        }
        tot += c[j];
      }
      uint32_t incl = tot;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      const uint32_t excl = incl - tot;
      const uint32_t r = sel_rank[s];
      __syncwarp();
      if (r >= excl && r < incl) {
        uint32_t acc = excl;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (r >= acc && r < acc + c[j]) {
            sel_key[s] = (s == 0 ? p0 : p1) | (uint32_t(lane * 8 + j) << shift);
            sel_rank[s] = r - acc;
            sel_eq[s] = c[j];
          }
          acc += c[j];
        }
      }
    }
    __syncthreads();
    if (CS > 1) cluster_sync_all();                       // the peers have read `merged` before the next pass rewrites it
  }

  const uint32_t L = sel_key[0], H = sel_key[1];
  const float vL = key2f2(L), vH = key2f2(H);
  const int m = hi - lo;
  double nL, nH;
  if (L == H) {
    nL = double(m);
    nH = 0.0;
  } else {
    nL = double(sel_eq[0] - sel_rank[0]);
    nH = double(sel_rank[1] + 1u);
  }

  // sum over the whole sample of f(key) for keys strictly between L and H, identical in every CTA of the cluster
  auto cluster_total = [&](double local, int slot) -> double {
    if (CS == 1) return local;
    if (tid == 0) part[slot] = local;
    __syncthreads();
    cluster_sync_all();
    double t = 0.0;
    const uint32_t addr = smem_u32(&part[slot]);
#pragma unroll
    for (int r = 0; r < CS; ++r) t += ld_cluster_f64(mapa_u32(addr, uint32_t(r)));   // rank order: same value everywhere
    return t;
  };

  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  int it = 0;
  for (int i = tid; i < cnt; i += DS2_THREADS, ++it) {
    const uint32_t k = keys[i];
    const float v = (k > L && k < H) ? key2f2(k) : 0.f;
    switch (it & 3) {
      case 0: a0 += v; break;
      case 1: a1 += v; break;
      case 2: a2 += v; break;
      default: a3 += v; break;
    }
  }
  const double sum_mid = cluster_total(block_sum2(double(a0) + double(a1) + double(a2) + double(a3), red), 0);
  const double mean_d = (sum_mid + nL * double(vL) + nH * double(vH)) / double(m);
  const float mean = float(mean_d);

  a0 = a1 = a2 = a3 = 0.f;
  it = 0;
  for (int i = tid; i < cnt; i += DS2_THREADS, ++it) {
    const uint32_t k = keys[i];
    const float dlt = key2f2(k) - mean;
    const float v = (k > L && k < H) ? dlt * dlt : 0.f;
    switch (it & 3) {
      case 0: a0 += v; break;
      case 1: a1 += v; break;
      case 2: a2 += v; break;
      default: a3 += v; break;
    }
  }
  const double ss_mid = cluster_total(block_sum2(double(a0) + double(a1) + double(a2) + double(a3), red), 1);
  const double dL = double(vL) - mean_d, dH = double(vH) - mean_d;
  const double ss = ss_mid + nL * dL * dL + nH * dH * dH;
  const float var = float(ss / double(m - 1));
  const float sd = __fsqrt_rn(var + eps);
  if (stats != nullptr && tid == 0 && rank == 0) {
    stats[2 * sample + 0] = mean;
    stats[2 * sample + 1] = var;
  }

  if (vec4) {
    for (int i = tid; i < cnt / 4; i += DS2_THREADS) {
      const uint4 k = reinterpret_cast<const uint4*>(keys)[i];
      float4 v = make_float4(key2f2(k.x), key2f2(k.y), key2f2(k.z), key2f2(k.w));
      v.x = __fdiv_rn(v.x - mean, sd);
      v.y = __fdiv_rn(v.y - mean, sd);
      v.z = __fdiv_rn(v.z - mean, sd);
      v.w = __fdiv_rn(v.w - mean, sd);
      reinterpret_cast<float4*>(ys)[i] = v;
    }
  } else {
    for (int i = tid; i < cnt; i += DS2_THREADS) ys[i] = __fdiv_rn(key2f2(keys[i]) - mean, sd);
  }
  if (CS > 1) cluster_sync_all();                         // no CTA leaves while a peer may still read its shared memory
}

template <int CS>
int launch_v2(const float* depth, float* out, int B, int n, int chunk, int lo, int hi, float eps, float* stats,
              cudaStream_t st) {
  auto kern = depth_standardize_v2_kernel<CS>;
  const size_t smem = size_t(chunk) * sizeof(uint32_t);
  static size_t configured = 0;
  if (smem > configured) {
    MMAE_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = smem;
  }
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(B * CS);
  cfg.blockDim = dim3(DS2_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (CS > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = CS;
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
  if (pdl_enabled()) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  MMAE_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, depth, out, n, chunk, lo, hi, eps, stats));
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

}  // namespace

// MMAE_ERR_UNSUPPORTED: the map needs more than 8 CTAs' worth of shared memory (the caller falls back to variant 1)
int launch_depth_standardize_v2(const float* depth, float* out, int B, int n, int lo, int hi, float eps, float* stats,
                                cudaStream_t st) {
  // static shared memory of the kernel: 16 KB histogram copies + 2 KB merged + ~0.4 KB; keep 1 KB of slack
  const size_t budget = size_t(227) * 1024 - (DS2_COPIES * 256 * 4 + 2 * 256 * 4 + 2048);
  // smallest cluster tried first; MMAE_DEPTH_STD_MIN_CLUSTER (1 | 2 | 4 | 8) raises it: more, smaller CTAs per map
  static const int min_cs = []() {
    const char* e = getenv("MMAE_DEPTH_STD_MIN_CLUSTER");
    const int v = e ? atoi(e) : 1;
    return (v == 2 || v == 4 || v == 8) ? v : 1;
  }();
  for (int cs = min_cs; cs <= 8; cs *= 2) {
    const int chunk = (ceil_div(n, cs) + 3) / 4 * 4;
    if (size_t(chunk) * 4 > budget) continue;
    switch (cs) {
      case 1: return launch_v2<1>(depth, out, B, n, chunk, lo, hi, eps, stats, st);
      case 2: return launch_v2<2>(depth, out, B, n, chunk, lo, hi, eps, stats, st);
      case 4: return launch_v2<4>(depth, out, B, n, chunk, lo, hi, eps, stats, st);
      default: return launch_v2<8>(depth, out, B, n, chunk, lo, hi, eps, stats, st);
    }
  }
  return MMAE_ERR_UNSUPPORTED;
}

}  // namespace mmae
