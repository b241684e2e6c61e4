// Truncated depth standardisation — run_pretraining_multimae.py:487-492 (SURVEY.md §8f row n2).
//
// The reference sorts every depth map (torch.sort over [B, H*W]), drops the bottom and top 10 % of the values and
// standardises the WHOLE map with the mean / unbiased variance of the kept middle:
//     trunc = sort(x_b)[int(0.1 n) : int(0.9 n)];   y_b = (x_b - mean(trunc)) / sqrt(var(trunc) + 1e-6)
// Only two order statistics are needed for that, not the sorted array: the values at ranks lo and hi-1.  One CTA per
// sample keeps the sample in shared memory as order-preserving 32-bit keys (224^2 floats = 196 KB, inside the 227 KB a
// CTA may use), finds both order statistics at once with a 4-pass most-significant-digit radix select (8 bits per pass,
// warp-aggregated shared-memory histograms), and then sums / normalises out of shared memory: the map is read from HBM
// once and written once (8 B per pixel against the ~40 B per pixel of a radix sort + gather + two reductions).
// Samples that do not fit (448^2) run the same passes over global memory (L2-resident: 0.8 MB per sample).
//
// Ties: every element equal to a boundary value is interchangeable, so the kept multiset is
//     {x : L < x < H}  +  (copies of L with rank >= lo)  +  (copies of H with rank <= hi-1)
// which equals the reference's slice of the sorted array exactly; the sums differ from torch only by fp32 summation
// order (per-thread fp32 partials, fp64 across threads).
#include <cstdlib>

#include "internal.h"

namespace mmae {
namespace {

constexpr int DS_THREADS = 1024;

// order-preserving float <-> uint32 (ascending keys == ascending floats; NaNs of positive sign sort last like torch.sort)
__device__ __forceinline__ uint32_t f2key(float f) {
  const uint32_t b = __float_as_uint(f);
  return (b >> 31) ? ~b : (b ^ 0x80000000u);
}
__device__ __forceinline__ float key2f(uint32_t k) {
  return __uint_as_float((k >> 31) ? (k ^ 0x80000000u) : ~k);
}

__device__ __forceinline__ double block_sum(double v, double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) red[warp] = v;
  __syncthreads();
  if (warp == 0) {
    double t = lane < DS_THREADS / 32 ? red[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (lane == 0) red[0] = t;
  }
  __syncthreads();
  const double r = red[0];
  __syncthreads();
  return r;
}

template <bool CACHED>
__global__ void __launch_bounds__(DS_THREADS, 1)
depth_standardize_kernel(const float* x, float* y, int n, int lo, int hi, float eps, float* stats) {
  pdl_prologue();
  extern __shared__ __align__(16) uint8_t ds_smem[];
  uint32_t* keys = reinterpret_cast<uint32_t*>(ds_smem);   // [n] when CACHED
  __shared__ uint32_t hist[2][256];
  __shared__ uint32_t sel_key[2], sel_rank[2], sel_eq[2];
  __shared__ double red[DS_THREADS / 32];
  const float* xs = x + int64_t(blockIdx.x) * n;
  float* ys = y + int64_t(blockIdx.x) * n;
  const int tid = threadIdx.x, lane = tid & 31;
  const bool vec4 = (n % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) % 16 == 0);

  if (CACHED) {
    if (vec4) {
      for (int i = tid; i < n / 4; i += DS_THREADS) {
        const float4 v = reinterpret_cast<const float4*>(xs)[i];
        reinterpret_cast<uint4*>(keys)[i] = make_uint4(f2key(v.x), f2key(v.y), f2key(v.z), f2key(v.w));
      }
    } else {
      for (int i = tid; i < n; i += DS_THREADS) keys[i] = f2key(xs[i]);
    }
  }
  if (tid < 2) {
    sel_key[tid] = 0u;
    sel_rank[tid] = tid == 0 ? uint32_t(lo) : uint32_t(hi - 1);
    sel_eq[tid] = 0u;
  }
  __syncthreads();

  // ---- radix select of the keys at ranks lo (selection 0) and hi-1 (selection 1), most significant byte first ----
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    const uint32_t pmask = pass == 0 ? 0u : (0xFFFFFFFFu << (shift + 8));
    for (int i = tid; i < 512; i += DS_THREADS) (&hist[0][0])[i] = 0u;
    __syncthreads();
    const uint32_t p0 = sel_key[0], p1 = sel_key[1];
    for (int i0 = 0; i0 < n; i0 += DS_THREADS) {          // uniform trip count: whole warps reach the warp votes
      const int i = i0 + tid;
      const bool valid = i < n;
      uint32_t k = 0u;
      if (valid) k = CACHED ? keys[i] : f2key(xs[i]);
      const uint32_t d = (k >> shift) & 255u;
      const bool m0 = valid && ((k & pmask) == p0);
      const bool m1 = valid && ((k & pmask) == p1);
      // warp-aggregated histogram update: real depth maps put most pixels into a handful of exponent bins, which would
      // serialise per-lane shared-memory atomics 32 ways
      const uint32_t code = d | (m0 ? 256u : 0u) | (m1 ? 512u : 0u);
      const uint32_t peers = __match_any_sync(0xffffffffu, code);
      if ((m0 || m1) && lane == __ffs(peers) - 1) {
        const uint32_t c = __popc(peers);
        if (m0) atomicAdd(&hist[0][d], c);
        if (m1) atomicAdd(&hist[1][d], c);
      }
    }
    __syncthreads();
    if (tid < 64) {                                       // warp s resolves selection s: 8 bins per lane + lane scan
      const int s = tid >> 5;
      uint32_t c[8], tot = 0u;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        c[j] = hist[s][lane * 8 + j];
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
      if (r >= excl && r < incl) {                        // exactly one lane: the candidates always number > r
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
  }

  const uint32_t L = sel_key[0], H = sel_key[1];
  const float vL = key2f(L), vH = key2f(H);
  const int m = hi - lo;
  // copies of the boundary values inside the kept rank range [lo, hi)
  double nL, nH;
  if (L == H) {
    nL = double(m);
    nH = 0.0;
  } else {
    nL = double(sel_eq[0] - sel_rank[0]);                 // ranks lo .. end of L's run
    nH = double(sel_rank[1] + 1u);                        // start of H's run .. hi-1
  }

  // ---- mean of the kept values ----
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  int it = 0;
  for (int i = tid; i < n; i += DS_THREADS, ++it) {
    const uint32_t k = CACHED ? keys[i] : f2key(xs[i]);
    const float v = (k > L && k < H) ? key2f(k) : 0.f;
    switch (it & 3) {
      case 0: a0 += v; break;
      case 1: a1 += v; break;
      case 2: a2 += v; break;
      default: a3 += v; break;
    }
  }
  const double sum_mid = block_sum(double(a0) + double(a1) + double(a2) + double(a3), red);
  const double mean_d = (sum_mid + nL * double(vL) + nH * double(vH)) / double(m);
  const float mean = float(mean_d);

  // ---- unbiased variance of the kept values around that mean ----
  a0 = a1 = a2 = a3 = 0.f;
  it = 0;
  for (int i = tid; i < n; i += DS_THREADS, ++it) {
    const uint32_t k = CACHED ? keys[i] : f2key(xs[i]);
    const float dlt = key2f(k) - mean;
    const float v = (k > L && k < H) ? dlt * dlt : 0.f;
    switch (it & 3) {
      case 0: a0 += v; break;
      case 1: a1 += v; break;
      case 2: a2 += v; break;
      default: a3 += v; break;
    }
  }
  const double ss_mid = block_sum(double(a0) + double(a1) + double(a2) + double(a3), red);
  const double dL = double(vL) - mean_d, dH = double(vH) - mean_d;
  const double ss = ss_mid + nL * dL * dL + nH * dH * dH;
  const float var = float(ss / double(m - 1));            // m == 1: 0/0 = NaN like torch.var of a single element
  const float sd = __fsqrt_rn(var + eps);
  if (stats != nullptr && tid == 0) {
    stats[2 * blockIdx.x + 0] = mean;
    stats[2 * blockIdx.x + 1] = var;
  }

  // ---- y = (x - mean) / sqrt(var + eps) over the whole map ----
  if (vec4) {
    for (int i = tid; i < n / 4; i += DS_THREADS) {
      float4 v;
      if (CACHED) {
        const uint4 k = reinterpret_cast<const uint4*>(keys)[i];
        v = make_float4(key2f(k.x), key2f(k.y), key2f(k.z), key2f(k.w));
      } else {
        v = reinterpret_cast<const float4*>(xs)[i];
      }
      v.x = __fdiv_rn(v.x - mean, sd);
      v.y = __fdiv_rn(v.y - mean, sd);
      v.z = __fdiv_rn(v.z - mean, sd);
      v.w = __fdiv_rn(v.w - mean, sd);
      reinterpret_cast<float4*>(ys)[i] = v;
    }
  } else {
    for (int i = tid; i < n; i += DS_THREADS) {
      const float v = CACHED ? key2f(keys[i]) : xs[i];
      ys[i] = __fdiv_rn(v - mean, sd);
    }
  }
}

}  // namespace
}  // namespace mmae

using namespace mmae;

namespace {
// 2 (default): depth_standardize_v2.cu - 16 histogram copies per CTA and a cluster split for large maps, checked against the
// oracle fixtures (tests/test_cuda_kernels.py).  1: the single-CTA kernel of this file (also the fallback for maps beyond 8
// CTAs' shared memory).
int depth_std_variant() {
  static int v = [] {
    const char* e = getenv("MMAE_DEPTH_STD_VARIANT");
    return (e != nullptr && atoi(e) == 1) ? 1 : 2;
  }();
  return v;
}
int g_depth_std_variant = 0;   // 0: not set through the API -> environment / default
}  // namespace

extern "C" int mmae_standardize_depth_set_variant(int variant) {
  MMAE_CHECK(variant == 1 || variant == 2, MMAE_ERR_ARG, "mmae_standardize_depth_set_variant: 1 or 2");
  g_depth_std_variant = variant;
  return MMAE_OK;
}

extern "C" int mmae_standardize_depth(const float* depth, float* out, int B, int n, int lo, int hi, float eps,
                                      float* stats, void* stream) {
  MMAE_CHECK(depth && out && B > 0 && n > 0, MMAE_ERR_ARG, "mmae_standardize_depth: bad args");
  MMAE_CHECK(lo >= 0 && lo < hi && hi <= n, MMAE_ERR_ARG, "mmae_standardize_depth: need 0 <= lo < hi <= n (lo %d, hi %d, n %d)",
             lo, hi, n);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if ((g_depth_std_variant != 0 ? g_depth_std_variant : depth_std_variant()) == 2) {
    const int rc = launch_depth_standardize_v2(depth, out, B, n, lo, hi, eps, stats, st);
    if (rc != MMAE_ERR_UNSUPPORTED) return rc;            // maps beyond 8 CTAs' shared memory: the kernel below
  }
  const size_t cache = size_t(n) * sizeof(uint32_t);
  if (cache + 4096 <= size_t(227) * 1024) {
    static size_t configured = 0;
    if (cache > configured) {
      MMAE_CUDA_OK(cudaFuncSetAttribute(depth_standardize_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cache));
      configured = cache;
    }
    launch_k(depth_standardize_kernel<true>, B, DS_THREADS, cache, st, depth, out, n, lo, hi, eps, stats);
  } else {
    launch_k(depth_standardize_kernel<false>, B, DS_THREADS, 0, st, depth, out, n, lo, hi, eps, stats);
  }
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}
