// Fused masked reconstruction losses, forward + backward (fp32, HBM-bound, no host synchronisation).
//
// Replaces multimae/criterion.py:37-57 (MaskedCrossEntropyLoss), :84-114 (MaskedMSELoss, norm_pix) and :141-171
// (MaskedL1Loss): element loss -> mean over channels -> x nearest-upsampled patch mask -> per-sample sum / mask.sum ->
// nanmean over the batch; `mask.sum() == 0` -> 0 is decided on the device.
// Work is organised in strips: one CTA per (sample, patch row) = P image rows, only masked patches are touched.
#include "common.cuh"
#include "../../include/multimae_b200.h"
#include "internal.h"

namespace mmae {
void count_launch();
namespace {

constexpr int LOSS_THREADS = 256;
constexpr int MAX_NW = 64;  // patches per strip for the CE kernel's mask cache (224/16 = 14, 448/16 = 28, 56/4 = 14 ...)

__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  float t = 0.f;
  if (threadIdx.x < LOSS_THREADS / 32) t = red[threadIdx.x];
  if (w == 0) t = warp_sum(t);
  return t;  // valid on warp 0
}

// MSE / L1 with optional norm_pix: one CTA per (sample, patch row), one WARP per patch (patches pw = warp, warp+8, ...).
// A patch is C*P rows of P contiguous floats; lane l of the warp owns float4 #(l % (P/4)) of row (l / (P/4)) + k*rows_per_it.
// kind: 0 = MSE, 1 = L1.  BWD = false: accumulate sample_sum[b];  BWD = true: write dpred (zeros for unmasked patches).
template <bool BWD>
__global__ void __launch_bounds__(LOSS_THREADS) regr_loss_kernel(int kind, int norm_pix, const float* __restrict__ pred,
                                                                 const float* __restrict__ tgt,
                                                                 const int64_t* __restrict__ mask, int C, int H, int W,
                                                                 int P, float* __restrict__ sample_sum,
                                                                 float* __restrict__ partial,
                                                                 const float* __restrict__ coef,
                                                                 const float* __restrict__ grad_out,
                                                                 float* __restrict__ dpred) {
  pdl_prologue();
  __shared__ float red[LOSS_THREADS / 32];
  const int nh = H / P, nw = W / P;
  const int b = blockIdx.x / nh, ph = blockIdx.x % nh;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int vec_per_row = P / 4;                    // float4 per patch row (P = 16 -> 4, P = 4 -> 1)
  const int rows_per_it = 32 / vec_per_row;         // patch rows covered by one warp iteration
  const int prow = lane / vec_per_row, pvec = lane % vec_per_row;
  const int nrows = C * P;                          // rows of one patch, ordered (c, py)
  const int n = C * P * P;
  const int64_t img_off = int64_t(b) * C * H * W;
  float gscale = 0.f;
  if constexpr (BWD) gscale = grad_out[0] * coef[b];
  float acc = 0.f;

  for (int pw = warp; pw < nw; pw += LOSS_THREADS / 32) {
    const bool masked = mask == nullptr ? true : (mask[(int64_t(b) * nh + ph) * nw + pw] != 0);
    if (!masked && !BWD) continue;
    float mean = 0.f, rstd = 1.f;
    if (masked && norm_pix) {                        // unbiased variance over the C*P*P target values of the patch
      float s = 0.f;
      for (int r = prow; r < nrows; r += rows_per_it) {
        const int c = r / P, py = r % P;
        const float4 t = __ldg(reinterpret_cast<const float4*>(tgt + img_off + (int64_t(c) * H + ph * P + py) * W + pw * P + pvec * 4));
        s += t.x + t.y + t.z + t.w;
      }
      mean = warp_sum(s) / n;
      float q = 0.f;
      for (int r = prow; r < nrows; r += rows_per_it) {
        const int c = r / P, py = r % P;
        const float4 t = __ldg(reinterpret_cast<const float4*>(tgt + img_off + (int64_t(c) * H + ph * P + py) * W + pw * P + pvec * 4));
        const float a = t.x - mean, bb = t.y - mean, cc = t.z - mean, d = t.w - mean;
        q += a * a + bb * bb + cc * cc + d * d;
      }
      rstd = rsqrtf(warp_sum(q) / (n - 1) + 1e-6f);
    }
    for (int r = prow; r < nrows; r += rows_per_it) {
      const int c = r / P, py = r % P;
      const int64_t off = img_off + (int64_t(c) * H + ph * P + py) * W + pw * P + pvec * 4;
      if (!masked) {
        if constexpr (BWD) *reinterpret_cast<float4*>(dpred + off) = make_float4(0.f, 0.f, 0.f, 0.f);
        continue;
      }
      float4 t = __ldg(reinterpret_cast<const float4*>(tgt + off));
      const float4 pr = __ldg(reinterpret_cast<const float4*>(pred + off));
      if (norm_pix) {
        t.x = (t.x - mean) * rstd; t.y = (t.y - mean) * rstd; t.z = (t.z - mean) * rstd; t.w = (t.w - mean) * rstd;
      }
      const float d0 = pr.x - t.x, d1 = pr.y - t.y, d2 = pr.z - t.z, d3 = pr.w - t.w;
      if constexpr (BWD) {
        float4 g;
        if (kind == 0) {
          g = make_float4(2.f * d0, 2.f * d1, 2.f * d2, 2.f * d3);
        } else {
          g = make_float4(d0 > 0.f ? 1.f : (d0 < 0.f ? -1.f : 0.f), d1 > 0.f ? 1.f : (d1 < 0.f ? -1.f : 0.f),
                          d2 > 0.f ? 1.f : (d2 < 0.f ? -1.f : 0.f), d3 > 0.f ? 1.f : (d3 < 0.f ? -1.f : 0.f));
        }
        *reinterpret_cast<float4*>(dpred + off) = make_float4(g.x * gscale, g.y * gscale, g.z * gscale, g.w * gscale);
      } else {
        acc += kind == 0 ? d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3 : fabsf(d0) + fabsf(d1) + fabsf(d2) + fabsf(d3);
      }
    }
  }
  if constexpr (!BWD) {
    const float tot = block_sum(acc, red);
    if (partial) {   // deterministic mode: one partial per (patch row, sample), added in patch-row order
      if (threadIdx.x == 0) partial[int64_t(ph) * gridDim.x / nh + b] = tot;
    } else if (threadIdx.x == 0 && tot != 0.f) {
      atomicAdd(sample_sum + b, tot);
    }
  }
}

// cross entropy over C classes at every pixel of masked patches; one thread per pixel of the strip
template <bool BWD>
__global__ void __launch_bounds__(LOSS_THREADS) ce_loss_kernel(const float* __restrict__ logits,
                                                               const int64_t* __restrict__ target,
                                                               const int64_t* __restrict__ mask, int C, int H, int W,
                                                               int P, float smoothing, float* __restrict__ sample_sum,
                                                               float* __restrict__ partial,
                                                               const float* __restrict__ coef,
                                                               const float* __restrict__ grad_out,
                                                               float* __restrict__ dlogits) {
  pdl_prologue();
  __shared__ unsigned char pmask[MAX_NW];
  __shared__ float red[LOSS_THREADS / 32];
  const int nh = H / P, nw = W / P;
  const int b = blockIdx.x / nh, ph = blockIdx.x % nh;
  for (int i = threadIdx.x; i < nw; i += blockDim.x)
    pmask[i] = mask == nullptr ? 1 : (mask[(int64_t(b) * nh + ph) * nw + i] != 0);
  __syncthreads();
  const int64_t HW = int64_t(H) * W;
  const float* lb = logits + int64_t(b) * C * HW;
  float acc = 0.f;
  float gscale = 0.f;
  if constexpr (BWD) gscale = grad_out[0] * coef[b];
  for (int pix = threadIdx.x; pix < P * W; pix += blockDim.x) {
    const int x = pix % W, py = pix / W;
    const int64_t off = int64_t(ph * P + py) * W + x;
    if (!pmask[x / P]) {
      if constexpr (BWD)
        for (int c = 0; c < C; ++c) dlogits[int64_t(b) * C * HW + c * HW + off] = 0.f;
      continue;
    }
    // one pass for max, sum of exponentials and sum of logits: 8 independent loads in flight, running maximum with
    // rescaling (the three-pass version walked the C-strided column three times with one load in flight each)
    float m = -INFINITY, s = 0.f, sum_logits = 0.f;
    for (int c0 = 0; c0 < C; c0 += 8) {
      float v[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = c0 + i < C ? __ldg(lb + int64_t(c0 + i) * HW + off) : -INFINITY;
      float cm = v[0];
#pragma unroll
      for (int i = 1; i < 8; ++i) cm = fmaxf(cm, v[i]);
      const float m_new = fmaxf(m, cm);
      float part = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (c0 + i < C) {
          part += __expf(v[i] - m_new);
          sum_logits += v[i];
        }
      }
      s = s * __expf(m - m_new) + part;
      m = m_new;
    }
    const float lse = m + logf(s);
    const int64_t tcls = target[int64_t(b) * HW + off];
    // F.cross_entropy's ignore_index (-100 by default, multimae/criterion.py:52): a label outside [0, C) contributes no
    // loss and no gradient (the pixel still counts in the mask denominator, as in the reference)
    const bool ignored = tcls < 0 || tcls >= C;
    if constexpr (BWD) {
      const float inv = 1.0f / s;
#pragma unroll 8
      for (int c = 0; c < C; ++c) {
        const float p = __expf(__ldg(lb + int64_t(c) * HW + off) - m) * inv;
        const float y = (c == tcls ? 1.f - smoothing : 0.f) + smoothing / C;
        dlogits[int64_t(b) * C * HW + c * HW + off] = ignored ? 0.f : (p - y) * gscale;
      }
    } else if (!ignored) {
      const float nll = lse - lb[tcls * HW + off];
      acc += (1.f - smoothing) * nll + smoothing * (lse - sum_logits / C);
    }
  }
  if constexpr (!BWD) {
    const float tot = block_sum(acc, red);
    if (partial) {
      if (threadIdx.x == 0) partial[int64_t(ph) * gridDim.x / nh + b] = tot;
    } else if (threadIdx.x == 0 && tot != 0.f) {
      atomicAdd(sample_sum + b, tot);
    }
  }
}

// loss = nanmean_b(sum_b / count_b); coef[b] = 1 / (valid * count_b * chan_div)  (0 for empty samples)
__global__ void __launch_bounds__(256) loss_finalize_kernel(const float* __restrict__ sample_sum,
                                                            const int64_t* __restrict__ mask, int B, int npatch,
                                                            float pix_per_patch, float chan_div, float* __restrict__ coef,
                                                            float* __restrict__ loss) {
  pdl_prologue();
  __shared__ float s_acc[256], s_valid[256];
  float acc = 0.f, valid = 0.f;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    float cnt;
    if (mask == nullptr) {
      cnt = float(npatch) * pix_per_patch;
    } else {
      int m = 0;
      for (int i = 0; i < npatch; ++i) m += mask[int64_t(b) * npatch + i] != 0;
      cnt = float(m) * pix_per_patch;
    }
    coef[b] = cnt;  // temporarily the count
    if (cnt > 0.f) {
      acc += sample_sum[b] / (cnt * chan_div);
      valid += 1.f;
    }
  }
  s_acc[threadIdx.x] = acc;
  s_valid[threadIdx.x] = valid;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      s_acc[threadIdx.x] += s_acc[threadIdx.x + o];
      s_valid[threadIdx.x] += s_valid[threadIdx.x + o];
    }
    __syncthreads();
  }
  const float nvalid = s_valid[0];
  if (threadIdx.x == 0) loss[0] = nvalid > 0.f ? s_acc[0] / nvalid : 0.f;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const float cnt = coef[b];
    coef[b] = (cnt > 0.f && nvalid > 0.f) ? 1.0f / (nvalid * cnt * chan_div) : 0.f;
  }
}

}  // namespace
}  // namespace mmae

using namespace mmae;

// kind: 0 MSE, 1 L1, 2 cross-entropy.  ws: [2*B] floats (sample sums, then backward coefficients).
extern "C" int mmae_masked_loss_forward(int kind, int norm_pix, float label_smoothing, const float* pred,
                                        const void* target, const int64_t* mask, int B, int C, int H, int W, int scale,
                                        float* ws, float* loss_out, void* stream) {
  MMAE_CHECK(pred && target && ws && loss_out && B > 0 && C > 0 && scale > 0 && H % scale == 0 && W % scale == 0,
             MMAE_ERR_ARG, "mmae_masked_loss_forward: bad args");
  MMAE_CHECK(kind >= 0 && kind <= 2 && W / scale <= MAX_NW, MMAE_ERR_UNSUPPORTED, "mmae_masked_loss_forward: kind/width");
  MMAE_CHECK(kind == 2 || (scale % 4 == 0 && 32 % (scale / 4) == 0 && W % 4 == 0), MMAE_ERR_UNSUPPORTED,
             "mmae_masked_loss_forward: patch scale %d unsupported (multiple of 4, <= 128)", scale);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  float* sample_sum = ws;
  float* coef = ws + B;
  MMAE_CUDA_OK(cudaMemsetAsync(sample_sum, 0, sizeof(float) * B, st));
  const int nh = H / scale, nw = W / scale;
  float* partial = nullptr;   // deterministic mode: [nh, B] per-block sums instead of atomics
  if (deterministic()) {
    partial = colred_scratch(size_t(nh) * B, st);
    if (!partial) return MMAE_ERR_CUDA;
  }
  if (kind == 2) {
    launch_k(ce_loss_kernel<false>, B * nh, LOSS_THREADS, 0, st, pred, reinterpret_cast<const int64_t*>(target), mask, C, H, W,
                                                           scale, label_smoothing, sample_sum, partial, nullptr, nullptr, nullptr);
  } else {
    launch_k(regr_loss_kernel<false>, B * nh, LOSS_THREADS, 0, st, kind, norm_pix, pred, reinterpret_cast<const float*>(target),
                                                             mask, C, H, W, scale, sample_sum, partial, nullptr, nullptr, nullptr);
  }
  count_launch();
  MMAE_LAUNCH_OK();
  if (partial) {
    const int rc = colred_finalize(partial, nh, B, B, sample_sum, nullptr, nullptr, st);
    if (rc) return rc;
  }
  // mask == NULL ("loss on unmasked"): plain mean over every element == per-sample means averaged (equal counts)
  launch_k(loss_finalize_kernel, 1, 256, 0, st, sample_sum, mask, B, nh * nw, float(scale) * scale, kind == 2 ? 1.f : float(C),
                                          coef, loss_out);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

extern "C" int mmae_masked_loss_backward(int kind, int norm_pix, float label_smoothing, const float* pred,
                                         const void* target, const int64_t* mask, int B, int C, int H, int W, int scale,
                                         const float* ws, const float* grad_out, float* dpred, void* stream) {
  MMAE_CHECK(pred && target && ws && grad_out && dpred && B > 0 && C > 0 && scale > 0, MMAE_ERR_ARG,
             "mmae_masked_loss_backward: bad args");
  MMAE_CHECK(kind >= 0 && kind <= 2 && W / scale <= MAX_NW, MMAE_ERR_UNSUPPORTED, "mmae_masked_loss_backward: kind/width");
  MMAE_CHECK(kind == 2 || (scale % 4 == 0 && 32 % (scale / 4) == 0 && W % 4 == 0), MMAE_ERR_UNSUPPORTED,
             "mmae_masked_loss_backward: patch scale %d unsupported (multiple of 4, <= 128)", scale);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const float* coef = ws + B;
  const int nh = H / scale;
  if (kind == 2) {
    launch_k(ce_loss_kernel<true>, B * nh, LOSS_THREADS, 0, st, pred, reinterpret_cast<const int64_t*>(target), mask, C, H, W,
                                                          scale, label_smoothing, nullptr, nullptr, coef, grad_out, dpred);
  } else {
    launch_k(regr_loss_kernel<true>, B * nh, LOSS_THREADS, 0, st, kind, norm_pix, pred, reinterpret_cast<const float*>(target),
                                                            mask, C, H, W, scale, nullptr, nullptr, coef, grad_out, dpred);
  }
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}
