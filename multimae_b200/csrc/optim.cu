// Flat-buffer gradient post-processing and optimizer update (HBM-bound, single pass each).
//
// mmae_grad_unscale_norm replaces GradScaler.unscale_ + get_grad_norm_ (utils/native_scaler.py:34-35, 49-62): the
// reference launches ~344 per-tensor norm kernels + a stack + a norm; the L2 norm of per-tensor L2 norms equals the
// L2 norm of the concatenation, so one pass over the flat gradient buffer suffices.
// mmae_adamw_step is torch.optim.AdamW's update (utils/optim_factory.py:155-174 builds it) over flat buffers.
// mmae_ema_update is ModelEma.update (utils/model_ema.py:72-84) over a list of separately allocated tensor pairs: one
// launch instead of four torch kernels per state_dict entry.  ema_kernel: 256 threads, 64 registers (4 blocks per SM),
// no spills (ptxas -v, sm_90a); its segment table travels as a by-value kernel parameter (EmaSegments, 7,176 bytes).
// mmae_adamw_step_groups is torch.optim.AdamW with parameter groups (the fine-tuning scripts' layer-decay groups) over a
// list of segments, each with its group's lr / weight decay: one launch for the whole model.  adamw_groups_kernel: 256
// threads, 86 registers (2 blocks per SM), no spills (ptxas -v, sm_90a); segment table by value (AdamwSegments, 28,680
// bytes).  step_advance_kernel: 8 registers, no spills.
#include <climits>

#include "common.cuh"
#include "../../include/multimae_b200.h"
#include "internal.h"

namespace mmae {
void count_launch();
namespace {

// out[0] += sum(g^2) after unscaling, out[1] = 1.0 if any non-finite value was seen (left untouched otherwise).  With
// `partial` (deterministic mode) block b writes its sum to partial[b] instead, for an ordered second pass.
__global__ void __launch_bounds__(256) unscale_norm_kernel(float* __restrict__ g, int64_t n, const float* __restrict__ inv_scale_ptr,
                                                           float inv_scale_imm, float post_scale, float* __restrict__ out,
                                                           float* __restrict__ partial) {
  pdl_prologue();
  __shared__ float red[8];
  const float inv = (inv_scale_ptr ? inv_scale_ptr[0] : inv_scale_imm) * post_scale;
  float acc = 0.f;
  bool bad = false;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x * 4;
  constexpr int U = 4;   // independent 16-byte loads in flight per thread
  for (int64_t i0 = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) * 4; i0 < n; i0 += stride * U) {
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + u * stride;
      if (i + 4 <= n) v[u] = *reinterpret_cast<const float4*>(g + i);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + u * stride;
      if (i + 4 <= n) {
        float4 w = v[u];
        w.x *= inv; w.y *= inv; w.z *= inv; w.w *= inv;
        if (inv != 1.0f) *reinterpret_cast<float4*>(g + i) = w;
        acc += w.x * w.x + w.y * w.y + w.z * w.z + w.w * w.w;
        bad |= !(isfinite(w.x) && isfinite(w.y) && isfinite(w.z) && isfinite(w.w));
      } else if (i < n) {
        for (int64_t j = i; j < n; ++j) {
          const float w = g[j] * inv;
          if (inv != 1.0f) g[j] = w;
          acc += w * w;
          bad |= !isfinite(w);
        }
      }
    }
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 8) {
    float t = red[threadIdx.x];
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) t += __shfl_xor_sync(0xffu, t, o);
    if (threadIdx.x == 0) {
      if (partial) partial[blockIdx.x] = t;
      else atomicAdd(out, t);
    }
  }
  if (__syncthreads_or(bad ? 1 : 0) && threadIdx.x == 0) out[1] = 1.0f;
}

__global__ void sqrt_kernel(const float* __restrict__ in, float* __restrict__ norm_out) {
  pdl_prologue(); norm_out[0] = sqrtf(in[0]); }

// device-side step counter: dyn[1] advances by one unless the step is skipped (non-finite gradients), like GradScaler.step,
// which does not call optimizer.step() at all in that case - the bias correction must not see skipped steps
__global__ void adamw_advance_kernel(float* __restrict__ dyn, const float* __restrict__ found_inf) {
  pdl_prologue();
  if (found_inf == nullptr || found_inf[0] == 0.f) dyn[1] += 1.0f;
}

// decoupled weight decay AdamW, skipping the whole update when found_inf[0] != 0 (GradScaler.step semantics)
__global__ void __launch_bounds__(256) adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                    float* __restrict__ v, int64_t n, float lr, float beta1, float beta2,
                                                    float eps, float wd, float bc1, float bc2_sqrt,
                                                    const float* __restrict__ found_inf, const float* __restrict__ dyn,
                                                    bf16* __restrict__ mirror) {
  pdl_prologue();
  if (found_inf != nullptr && found_inf[0] != 0.f) return;
  if (dyn != nullptr) {   // learning rate and step count live on the device (CUDA-graph replay): dyn = {lr, step}
    lr = dyn[0];
    const float step = dyn[1];
    bc1 = 1.0f - powf(beta1, step);
    bc2_sqrt = sqrtf(1.0f - powf(beta2, step));
  }
  const int64_t stride = int64_t(gridDim.x) * blockDim.x * 4;
  for (int64_t i = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) * 4; i < n; i += stride) {
    if (i + 4 <= n) {
      float4 pp = *reinterpret_cast<float4*>(p + i);
      const float4 gg = *reinterpret_cast<const float4*>(g + i);
      float4 mm = *reinterpret_cast<float4*>(m + i);
      float4 vv = *reinterpret_cast<float4*>(v + i);
#define MMAE_ADAM1(P, G, M, V)                                     \
  P *= (1.f - lr * wd);                                            \
  M = beta1 * M + (1.f - beta1) * G;                               \
  V = beta2 * V + (1.f - beta2) * G * G;                           \
  P -= (lr / bc1) * M / (sqrtf(V) / bc2_sqrt + eps);
      MMAE_ADAM1(pp.x, gg.x, mm.x, vv.x)
      MMAE_ADAM1(pp.y, gg.y, mm.y, vv.y)
      MMAE_ADAM1(pp.z, gg.z, mm.z, vv.z)
      MMAE_ADAM1(pp.w, gg.w, mm.w, vv.w)
      *reinterpret_cast<float4*>(p + i) = pp;
      *reinterpret_cast<float4*>(m + i) = mm;
      *reinterpret_cast<float4*>(v + i) = vv;
      if (mirror != nullptr) {   // bf16 twin of the parameters: the GEMM weight operands of the next step
        uint2 pk;
        pk.x = pack_bf16x2(pp.x, pp.y);
        pk.y = pack_bf16x2(pp.z, pp.w);
        *reinterpret_cast<uint2*>(mirror + i) = pk;
      }
    } else {
      for (int64_t j = i; j < n; ++j) {
        float P = p[j], M = m[j], V = v[j];
        const float G = g[j];
        MMAE_ADAM1(P, G, M, V)
        p[j] = P; m[j] = M; v[j] = V;
        if (mirror != nullptr) mirror[j] = __float2bfloat16_rn(P);
      }
    }
  }
#undef MMAE_ADAM1
}

// ---- model EMA: e = e * d + omd * v over a list of (dst, src, n) segments
constexpr int EMA_MAX_SEGMENTS = 256;
constexpr int EMA_THREADS = 256;
constexpr int EMA_UNROLL = 4;                                              // independent 16-byte loads per operand
constexpr int64_t EMA_CHUNK = int64_t(EMA_THREADS) * 4 * EMA_UNROLL;      // elements of one segment per block iteration

// by-value kernel argument (7,176 bytes; kernel parameters may be up to 32,764 bytes from CUDA 12.1 on sm_70+): nothing
// to allocate or upload, so a launch is stream-ordered like any other and can be captured in a graph
struct EmaSegments {
  int count;
  int chunk_off[EMA_MAX_SEGMENTS + 1];   // prefix sum of ceil(n / EMA_CHUNK) per segment
  float* dst[EMA_MAX_SEGMENTS];
  const float* src[EMA_MAX_SEGMENTS];
  int64_t n[EMA_MAX_SEGMENTS];
};

// `ema_v * decay + (1. - decay) * model_v` as torch evaluates it in fp32: two rounded products, one rounded sum, no FMA
__device__ __forceinline__ float ema1(float e, float v, float d, float omd) {
  return __fadd_rn(__fmul_rn(e, d), __fmul_rn(omd, v));
}

__global__ void __launch_bounds__(EMA_THREADS) ema_kernel(const __grid_constant__ EmaSegments segs, float d, float omd) {
  pdl_prologue();
  const int total = segs.chunk_off[segs.count];
  for (int c = blockIdx.x; c < total; c += gridDim.x) {
    int s = 0, hi = segs.count - 1;        // the segment with chunk_off[s] <= c < chunk_off[s + 1] (block-uniform search)
    while (s < hi) {
      const int mid = (s + hi + 1) >> 1;
      if (segs.chunk_off[mid] <= c) s = mid; else hi = mid - 1;
    }
    float* __restrict__ e = segs.dst[s];
    const float* __restrict__ v = segs.src[s];
    const int64_t base = int64_t(c - segs.chunk_off[s]) * EMA_CHUNK;
    const int64_t end = min(base + EMA_CHUNK, segs.n[s]);
    if (((reinterpret_cast<uintptr_t>(e) | reinterpret_cast<uintptr_t>(v)) & 15) == 0) {
      uint4 ev[EMA_UNROLL], vv[EMA_UNROLL];
#pragma unroll
      for (int u = 0; u < EMA_UNROLL; ++u) {
        const int64_t i = base + int64_t(u * EMA_THREADS + threadIdx.x) * 4;
        if (i + 4 <= end) {
          ev[u] = ld_stream_16_rw(e + i);
          vv[u] = ld_stream_16(v + i);
        }
      }
#pragma unroll
      for (int u = 0; u < EMA_UNROLL; ++u) {
        const int64_t i = base + int64_t(u * EMA_THREADS + threadIdx.x) * 4;
        if (i + 4 <= end) {
          float4 r;
          r.x = ema1(__uint_as_float(ev[u].x), __uint_as_float(vv[u].x), d, omd);
          r.y = ema1(__uint_as_float(ev[u].y), __uint_as_float(vv[u].y), d, omd);
          r.z = ema1(__uint_as_float(ev[u].z), __uint_as_float(vv[u].z), d, omd);
          r.w = ema1(__uint_as_float(ev[u].w), __uint_as_float(vv[u].w), d, omd);
          *reinterpret_cast<float4*>(e + i) = r;
        } else if (i < end) {
          for (int64_t j = i; j < end; ++j) e[j] = ema1(e[j], v[j], d, omd);
        }
      }
    } else {                               // a view whose data does not start on a 16-byte boundary
      for (int64_t j = base + threadIdx.x; j < end; j += EMA_THREADS) e[j] = ema1(e[j], v[j], d, omd);
    }
  }
}

// ---- grouped AdamW: torch.optim.AdamW over a list of (param, grad, exp_avg, exp_avg_sq, bf16 twin, n) segments, each
// with its parameter group's learning rate and weight decay (layer-decay groups of the fine-tuning scripts)
constexpr int ADAMW_MAX_SEGMENTS = 448;
constexpr int ADAMW_THREADS = 256;
constexpr int ADAMW_UNROLL = 2;                                            // independent 16-byte loads per operand
constexpr int64_t ADAMW_CHUNK = int64_t(ADAMW_THREADS) * 4 * ADAMW_UNROLL;

// by-value kernel argument, like EmaSegments: the launch allocates and uploads nothing
struct AdamwSegments {
  int count;
  int chunk_off[ADAMW_MAX_SEGMENTS + 1];   // prefix sum of ceil(n / ADAMW_CHUNK) per segment
  float* p[ADAMW_MAX_SEGMENTS];
  const float* g[ADAMW_MAX_SEGMENTS];
  float* m[ADAMW_MAX_SEGMENTS];
  float* v[ADAMW_MAX_SEGMENTS];
  bf16* mirror[ADAMW_MAX_SEGMENTS];       // NULL: no twin
  int64_t n[ADAMW_MAX_SEGMENTS];
  double lr[ADAMW_MAX_SEGMENTS];          // the segment's group learning rate
  float decay[ADAMW_MAX_SEGMENTS];        // float(1 - lr * weight_decay), evaluated in double
};
// the struct plus the eight scalar / pointer arguments of adamw_groups_kernel stay within the 32,764-byte limit
static_assert(sizeof(AdamwSegments) + 64 <= 32764, "AdamwSegments exceeds the kernel parameter limit");

__global__ void step_advance_kernel(float* __restrict__ step, const float* __restrict__ found_inf) {
  pdl_prologue();
  if (found_inf == nullptr || found_inf[0] == 0.f) step[0] += 1.0f;
}

// torch's _multi_tensor_adam (decoupled weight decay) order of operations, in fp32 with the scalars rounded from double:
//   p *= 1 - lr*wd;  m = lerp(m, g, 1 - b1);  v = v*b2 + (1 - b2)*g*g;  p += -(lr/bc1) * m / (sqrt(v)/sqrt(bc2) + eps)
__device__ __forceinline__ void adamw1(float& p, float g, float& m, float& v, float decay, float omb1, float b2, float omb2,
                                       float bc2s, float eps, float step_size) {
  p = __fmul_rn(p, decay);
  m = __fmaf_rn(omb1, __fsub_rn(g, m), m);
  v = __fmaf_rn(omb2, __fmul_rn(g, g), __fmul_rn(v, b2));
  const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2s), eps);
  p = __fmaf_rn(step_size, __fdiv_rn(m, denom), p);
}

__global__ void __launch_bounds__(ADAMW_THREADS) adamw_groups_kernel(const __grid_constant__ AdamwSegments segs, double beta1,
                                                                     double beta2, float omb1, float b2, float omb2,
                                                                     float eps, const float* __restrict__ found_inf,
                                                                     const float* __restrict__ step_dev) {
  pdl_prologue();
  if (found_inf != nullptr && found_inf[0] != 0.f) return;
  // bias corrections in double from the device step count (already advanced for this step), as torch computes them
  const double step = double(step_dev[0]);
  const double bc1 = 1.0 - pow(beta1, step);
  const float bc2s = float(sqrt(1.0 - pow(beta2, step)));
  const int total = segs.chunk_off[segs.count];
  for (int c = blockIdx.x; c < total; c += gridDim.x) {
    int s = 0, hi = segs.count - 1;        // the segment with chunk_off[s] <= c < chunk_off[s + 1] (block-uniform search)
    while (s < hi) {
      const int mid = (s + hi + 1) >> 1;
      if (segs.chunk_off[mid] <= c) s = mid; else hi = mid - 1;
    }
    float* __restrict__ p = segs.p[s];
    const float* __restrict__ g = segs.g[s];
    float* __restrict__ m = segs.m[s];
    float* __restrict__ v = segs.v[s];
    bf16* __restrict__ tw = segs.mirror[s];
    const float decay = segs.decay[s];
    const float step_size = float(-(segs.lr[s] / bc1));
    const int64_t base = int64_t(c - segs.chunk_off[s]) * ADAMW_CHUNK;
    const int64_t end = min(base + ADAMW_CHUNK, segs.n[s]);
    uint4 pv[ADAMW_UNROLL], gv[ADAMW_UNROLL], mv[ADAMW_UNROLL], vv[ADAMW_UNROLL];
#pragma unroll
    for (int u = 0; u < ADAMW_UNROLL; ++u) {
      const int64_t i = base + int64_t(u * ADAMW_THREADS + threadIdx.x) * 4;
      if (i + 4 <= end) {
        pv[u] = ld_stream_16_rw(p + i);
        gv[u] = ld_stream_16(g + i);
        mv[u] = ld_stream_16_rw(m + i);
        vv[u] = ld_stream_16_rw(v + i);
      }
    }
#pragma unroll
    for (int u = 0; u < ADAMW_UNROLL; ++u) {
      const int64_t i = base + int64_t(u * ADAMW_THREADS + threadIdx.x) * 4;
      if (i + 4 <= end) {
        float4 P = make_float4(__uint_as_float(pv[u].x), __uint_as_float(pv[u].y), __uint_as_float(pv[u].z),
                               __uint_as_float(pv[u].w));
        float4 M = make_float4(__uint_as_float(mv[u].x), __uint_as_float(mv[u].y), __uint_as_float(mv[u].z),
                               __uint_as_float(mv[u].w));
        float4 V = make_float4(__uint_as_float(vv[u].x), __uint_as_float(vv[u].y), __uint_as_float(vv[u].z),
                               __uint_as_float(vv[u].w));
        adamw1(P.x, __uint_as_float(gv[u].x), M.x, V.x, decay, omb1, b2, omb2, bc2s, eps, step_size);
        adamw1(P.y, __uint_as_float(gv[u].y), M.y, V.y, decay, omb1, b2, omb2, bc2s, eps, step_size);
        adamw1(P.z, __uint_as_float(gv[u].z), M.z, V.z, decay, omb1, b2, omb2, bc2s, eps, step_size);
        adamw1(P.w, __uint_as_float(gv[u].w), M.w, V.w, decay, omb1, b2, omb2, bc2s, eps, step_size);
        *reinterpret_cast<float4*>(p + i) = P;
        *reinterpret_cast<float4*>(m + i) = M;
        *reinterpret_cast<float4*>(v + i) = V;
        if (tw != nullptr) {
          uint2 pk;
          pk.x = pack_bf16x2(P.x, P.y);
          pk.y = pack_bf16x2(P.z, P.w);
          *reinterpret_cast<uint2*>(tw + i) = pk;
        }
      } else if (i < end) {                // the last 1-3 elements of a segment whose size is not a multiple of 4
        for (int64_t j = i; j < end; ++j) {
          float P = p[j], M = m[j], V = v[j];
          adamw1(P, g[j], M, V, decay, omb1, b2, omb2, bc2s, eps, step_size);
          p[j] = P; m[j] = M; v[j] = V;
          if (tw != nullptr) tw[j] = __float2bfloat16_rn(P);
        }
      }
    }
  }
}

}  // namespace
}  // namespace mmae

using namespace mmae;

extern "C" int mmae_grad_unscale_norm(float* grads, int64_t n, const float* inv_scale_dev, float inv_scale,
                                      float post_scale, float* out2, float* norm_out, void* stream) {
  MMAE_CHECK(grads && out2 && n >= 0 && (reinterpret_cast<uintptr_t>(grads) & 15) == 0, MMAE_ERR_ARG,
             "mmae_grad_unscale_norm: bad args");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  MMAE_CUDA_OK(cudaMemsetAsync(out2, 0, 2 * sizeof(float), st));
  if (n > 0) {
    int64_t blocks = (n / 4 + 255) / 256;
    const int64_t cap = int64_t(reduce_sm_count()) * 8;   // the grid-stride sums follow the grid
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    float* partial = nullptr;
    if (deterministic()) {
      partial = colred_scratch(size_t(blocks), st);
      if (!partial) return MMAE_ERR_CUDA;
    }
    launch_k(unscale_norm_kernel, (unsigned)blocks, 256, 0, st, grads, n, inv_scale_dev, inv_scale, post_scale, out2, partial);
    count_launch();
    MMAE_LAUNCH_OK();
    if (partial) {
      const int rc = colred_finalize(partial, int(blocks), 1, 1, out2, nullptr, nullptr, st);
      if (rc) return rc;
    }
  }
  if (norm_out) {
    launch_k(sqrt_kernel, 1, 1, 0, st, out2, norm_out);
    count_launch();
    MMAE_LAUNCH_OK();
  }
  return MMAE_OK;
}

extern "C" int mmae_adamw_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                               float beta1, float beta2, float eps, float weight_decay, int step,
                               const float* found_inf_dev, const float* dyn_lr_step_dev, void* stream) {
  MMAE_CHECK(params && grads && exp_avg && exp_avg_sq && n >= 0 && step >= 1, MMAE_ERR_ARG, "mmae_adamw_step: bad args");
  if (n == 0) return MMAE_OK;
  const float bc1 = 1.0f - powf(beta1, (float)step);
  const float bc2_sqrt = sqrtf(1.0f - powf(beta2, (float)step));
  int64_t blocks = (n / 4 + 255) / 256;
  const int64_t cap = int64_t(sm_count()) * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  if (dyn_lr_step_dev != nullptr) {
    launch_k(adamw_advance_kernel, 1, 1, 0, reinterpret_cast<cudaStream_t>(stream), const_cast<float*>(dyn_lr_step_dev), found_inf_dev);
    count_launch();
    MMAE_LAUNCH_OK();
  }
  launch_k(adamw_kernel, (unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream), params, grads, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, bc1, bc2_sqrt, found_inf_dev, dyn_lr_step_dev,
      const_cast<bf16*>(mirror_lookup(params)));
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

extern "C" int mmae_ema_update(float* const* dst_host, const float* const* src_host, const int64_t* n_host, int count,
                               float decay, float one_minus_decay, void* stream) {
  MMAE_CHECK(count >= 0 && (count == 0 || (dst_host && src_host && n_host)), MMAE_ERR_ARG,
             "mmae_ema_update: bad args (count %d)", count);
  MMAE_CHECK(isfinite(decay) && isfinite(one_minus_decay), MMAE_ERR_ARG, "mmae_ema_update: non-finite decay");
  for (int i = 0; i < count; ++i) {
    MMAE_CHECK(n_host[i] >= 0, MMAE_ERR_ARG, "mmae_ema_update: segment %d: negative size", i);
    MMAE_CHECK(n_host[i] == 0 || (dst_host[i] && src_host[i]), MMAE_ERR_ARG, "mmae_ema_update: segment %d: null pointer",
               i);
    MMAE_CHECK((n_host[i] + EMA_CHUNK - 1) / EMA_CHUNK <= INT_MAX / 2, MMAE_ERR_ARG,
               "mmae_ema_update: segment %d is too large", i);
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  EmaSegments segs;
  int i = 0;
  while (i < count) {
    // pack the next non-empty segments: as many as one launch holds, with a chunk count that stays within an int
    segs.count = 0;
    segs.chunk_off[0] = 0;
    for (; i < count && segs.count < EMA_MAX_SEGMENTS; ++i) {
      if (n_host[i] == 0) continue;
      const int64_t chunks = (n_host[i] + EMA_CHUNK - 1) / EMA_CHUNK;
      if (segs.count > 0 && segs.chunk_off[segs.count] + chunks > INT_MAX / 2) break;
      segs.dst[segs.count] = dst_host[i];
      segs.src[segs.count] = src_host[i];
      segs.n[segs.count] = n_host[i];
      segs.chunk_off[segs.count + 1] = segs.chunk_off[segs.count] + int(chunks);
      ++segs.count;
    }
    if (segs.count == 0) break;
    int64_t blocks = segs.chunk_off[segs.count];
    const int64_t cap = int64_t(sm_count()) * 8;
    if (blocks > cap) blocks = cap;
    launch_k(ema_kernel, (unsigned)blocks, EMA_THREADS, 0, st, segs, decay, one_minus_decay);
    count_launch();
    MMAE_LAUNCH_OK();
  }
  return MMAE_OK;
}

extern "C" int mmae_adamw_step_groups(const MmaeAdamwSegment* segs_host, int count, const double* lr_host,
                                      const double* weight_decay_host, int num_groups, double beta1, double beta2,
                                      double eps, const float* found_inf_dev, float* step_dev, void* stream) {
  MMAE_CHECK(count >= 0 && num_groups >= 0 && (count == 0 || (segs_host && num_groups > 0)), MMAE_ERR_ARG,
             "mmae_adamw_step_groups: bad args (count %d, num_groups %d)", count, num_groups);
  MMAE_CHECK(num_groups == 0 || (lr_host && weight_decay_host), MMAE_ERR_ARG,
             "mmae_adamw_step_groups: null group arrays");
  MMAE_CHECK(step_dev != nullptr, MMAE_ERR_ARG, "mmae_adamw_step_groups: null step counter");
  MMAE_CHECK(isfinite(beta1) && isfinite(beta2) && isfinite(eps) && beta1 >= 0.0 && beta1 < 1.0 && beta2 >= 0.0 &&
                 beta2 < 1.0 && eps >= 0.0,
             MMAE_ERR_ARG, "mmae_adamw_step_groups: bad betas / eps (%g, %g, %g)", beta1, beta2, eps);
  for (int k = 0; k < num_groups; ++k)
    MMAE_CHECK(isfinite(lr_host[k]) && isfinite(weight_decay_host[k]), MMAE_ERR_ARG,
               "mmae_adamw_step_groups: group %d: non-finite lr / weight_decay", k);
  for (int i = 0; i < count; ++i) {
    const MmaeAdamwSegment& sg = segs_host[i];
    MMAE_CHECK(sg.n >= 0, MMAE_ERR_ARG, "mmae_adamw_step_groups: segment %d: negative size", i);
    MMAE_CHECK(sg.group >= 0 && sg.group < num_groups, MMAE_ERR_ARG,
               "mmae_adamw_step_groups: segment %d: group %d out of range", i, sg.group);
    if (sg.n == 0) continue;
    MMAE_CHECK(sg.param && sg.grad && sg.exp_avg && sg.exp_avg_sq, MMAE_ERR_ARG,
               "mmae_adamw_step_groups: segment %d: null pointer", i);
    MMAE_CHECK(((reinterpret_cast<uintptr_t>(sg.param) | reinterpret_cast<uintptr_t>(sg.grad) |
                 reinterpret_cast<uintptr_t>(sg.exp_avg) | reinterpret_cast<uintptr_t>(sg.exp_avg_sq) |
                 reinterpret_cast<uintptr_t>(sg.mirror_bf16)) & 15) == 0,
               MMAE_ERR_ARG, "mmae_adamw_step_groups: segment %d: pointers must be 16-byte aligned", i);
    MMAE_CHECK((sg.n + ADAMW_CHUNK - 1) / ADAMW_CHUNK <= INT_MAX / 2, MMAE_ERR_ARG,
               "mmae_adamw_step_groups: segment %d is too large", i);
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // the step count advances (on the device, only for a step that is taken) before the update reads it
  launch_k(step_advance_kernel, 1, 1, 0, st, step_dev, found_inf_dev);
  count_launch();
  MMAE_LAUNCH_OK();
  AdamwSegments segs;
  int i = 0;
  while (i < count) {
    segs.count = 0;
    segs.chunk_off[0] = 0;
    for (; i < count && segs.count < ADAMW_MAX_SEGMENTS; ++i) {
      const MmaeAdamwSegment& sg = segs_host[i];
      if (sg.n == 0) continue;
      const int64_t chunks = (sg.n + ADAMW_CHUNK - 1) / ADAMW_CHUNK;
      if (segs.count > 0 && segs.chunk_off[segs.count] + chunks > INT_MAX / 2) break;
      const int k = segs.count;
      segs.p[k] = sg.param;
      segs.g[k] = sg.grad;
      segs.m[k] = sg.exp_avg;
      segs.v[k] = sg.exp_avg_sq;
      segs.mirror[k] = reinterpret_cast<bf16*>(sg.mirror_bf16);
      segs.n[k] = sg.n;
      segs.lr[k] = lr_host[sg.group];
      segs.decay[k] = float(1.0 - lr_host[sg.group] * weight_decay_host[sg.group]);
      segs.chunk_off[k + 1] = segs.chunk_off[k] + int(chunks);
      ++segs.count;
    }
    if (segs.count == 0) break;
    int64_t blocks = segs.chunk_off[segs.count];
    const int64_t cap = int64_t(sm_count()) * 8;
    if (blocks > cap) blocks = cap;
    launch_k(adamw_groups_kernel, (unsigned)blocks, ADAMW_THREADS, 0, st, segs, beta1, beta2, float(1.0 - beta1),
             float(beta2), float(1.0 - beta2), float(eps), found_inf_dev, static_cast<const float*>(step_dev));
    count_launch();
    MMAE_LAUNCH_OK();
  }
  return MMAE_OK;
}
