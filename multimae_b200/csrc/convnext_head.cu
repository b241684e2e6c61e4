// Semantic-segmentation head of fine-tuning: ConvNeXtAdapter.forward (multimae/output_adapters.py:481-573, ConvNeXtBlock in
// multimae/output_adapter_utils.py:19-57):
//   x = proj_dec(cat_t encoder_tokens[:, task t])                     Linear [B, n, D*T] -> [B, n, E]
//   x = rearrange(x, "b (nh nw) (ph pw c) -> b c (nh ph) (nw pw)")    s = ph = pw = sqrt(preds_per_patch), C = E / (s*s)
//   x = x + pwconv2(GELU(pwconv1(LN(dwconv7x7(x)))))  x depth           depthwise 7x7 (pad 3, bias), LN over channels
//   x = final_layer(x)                                                1x1 conv -> K classes
//   out = interpolate(x, (H, W), bilinear, align_corners=False)
//
// Layout.  The proj_dec output [B*n, s*s*C] already is a channels-last image whose pixels are stored patch by patch: row
//   r = (b*n + t)*s*s + a*s + c'   of its [P, C] view (P = B*n*s*s)  holds pixel  (y, x) = ((t / nw)*s + a, (t % nw)*s + c')
// of the (Hf, Wf) = (nh*s, nw*s) feature map of sample b.  The whole residual stream stays fp32 in that [P, C] view, so the
// LayerNorm, pwconv1 / pwconv2 and final_layer are plain row-wise operations on it (no rearrange copy is ever made) and only
// the depthwise convolution and the final upsample map (y, x) to a row (pix_row below).
//
// Entry points (module-level, like the SpatialOutputAdapter split head -> blocks -> tail):
//   proj : cnx_gather_kernel (bf16 A operand [B*n, D*T]) + GEMM with bias, fp32 out = the residual stream
//          backward: bias column sums + bf16 cast, weight-gradient GEMM, input-gradient GEMM (fp32, unsplit) and
//          cnx_scatter_kernel, which writes every row of dx [B, N, D] (zeros outside the main tasks' tokens)
//   block: dwconv_kernel<false> (fp32, FFMA, bias; its output d is kept for the LayerNorm backward) -> mmae_layernorm_forward
//          (bf16 out) -> pwconv1 + GELU -> pwconv2 + bias + residual in the GEMM epilogue (fp32 out)
//          backward: cast + fc2 bias sums, fc2 wgrad, fc2 dgrad * GELU' + fc1 bias sums, fc1 wgrad, fc1 dgrad,
//          mmae_layernorm_backward (fp32 dd), dwconv_kernel<true> (dx_in = dx_out + conv_transpose(dd)),
//          dwconv_wgrad_kernel (per-column-of-tiles partial rows) summed by mmae_cast_colsum_f32, bias = colsum(dd)
//   tail : bf16 cast of x, final_layer GEMM on a class width padded to Kp = round_up(K, 8) (zero weight rows), fp32 class
//          map [P, Kp] in the workspace, upsample_fwd_kernel -> caller's [B, K, H, W]
//          backward: upsample_bwd_kernel (gather form: each low-resolution pixel sums the output gradients that reference
//          it) -> [P, Kp] (zero pad columns), bias column sums + bf16 cast, weight-gradient GEMM, input-gradient GEMM
// The activation-gradient chain has no split-K and no atomics, so repeated calls give bitwise-equal input gradients and
// depthwise-conv parameter gradients; only the weight-gradient GEMMs and the LayerNorm parameter gradients accumulate with
// atomics, as everywhere else in the library.  Nothing outside the caller's tensors is read or written for any K.
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

// feature-map geometry: nh x nw patches of s x s pixels, C channels
struct Geo {
  int nh, nw, s, C;
};

// row of the [P, C] view that holds pixel (y, x) of sample b (see the layout note above)
__device__ __forceinline__ int64_t pix_row(int b, int y, int x, const Geo& g) {
  const int t = (y / g.s) * g.nw + x / g.s;
  return ((int64_t(b) * g.nh * g.nw + t) * g.s + y % g.s) * g.s + x % g.s;
}

// ------------------------------------------------------------------------------------------------ token gather / scatter
struct TaskStarts {
  int v[MMAE_MAX_TASKS];
};

// A[b*n + t, k*D + col] = bf16(enc[b, start_k + t, col])   (multimae/output_adapters.py:545-553)
__global__ void __launch_bounds__(256) cnx_gather_kernel(const float* __restrict__ enc, int N, int D, int n, int T,
                                                         TaskStarts st, bf16* __restrict__ A) {
  pdl_prologue();
  const int row = blockIdx.x, b = row / n, t = row % n;
  const int K8 = T * D / 8;
  for (int i = threadIdx.x; i < K8; i += blockDim.x) {
    const int k = (i * 8) / D, col = i * 8 - k * D;
    const float* src = enc + (int64_t(b) * N + st.v[k] + t) * D + col;
    const uint4 lo = ld_stream_16(src), hi = ld_stream_16(src + 4);
    uint4 o;
    o.x = pack_bf16x2(__uint_as_float(lo.x), __uint_as_float(lo.y));
    o.y = pack_bf16x2(__uint_as_float(lo.z), __uint_as_float(lo.w));
    o.z = pack_bf16x2(__uint_as_float(hi.x), __uint_as_float(hi.y));
    o.w = pack_bf16x2(__uint_as_float(hi.z), __uint_as_float(hi.w));
    *reinterpret_cast<uint4*>(A + int64_t(row) * T * D + i * 8) = o;
  }
}

// dx[b, tok, :] = dA[b*n + tok - start_k, k*D : (k+1)*D] for the main task k whose tokens hold tok, else 0
__global__ void __launch_bounds__(256) cnx_scatter_kernel(const float* __restrict__ dA, int N, int D, int n, int T,
                                                          TaskStarts st, float* __restrict__ dx) {
  pdl_prologue();
  const int row = blockIdx.x, b = row / N, tok = row % N;
  int k = -1;
  for (int j = 0; j < T; ++j)
    if (tok >= st.v[j] && tok < st.v[j] + n) k = j;
  float4* out = reinterpret_cast<float4*>(dx + int64_t(row) * D);
  const float4* src = k >= 0 ? reinterpret_cast<const float4*>(dA + (int64_t(b) * n + tok - st.v[k]) * T * D + k * D) : nullptr;
  for (int c = threadIdx.x; c < D / 4; c += blockDim.x) __stcs(out + c, src ? __ldg(src + c) : make_float4(0.f, 0.f, 0.f, 0.f));
}

// ------------------------------------------------------------------------------------------------ depthwise 7x7 conv
// One CTA: a DW_TH x DW_TW pixel tile of one sample over a slice of DW_CS channels.  The tile plus its 3-pixel halo is staged
// in shared memory as [pixel][channel] (each pixel's slice is one 128-byte run of its row in global memory); warp w computes
// output row w of the tile, lane c channel c, 16 pixels per thread with a sliding window of 22 inputs per kernel row.
constexpr int DW_TW = 16, DW_TH = 8, DW_CS = 32, DW_HW = DW_TW + 6, DW_HH = DW_TH + 6;
constexpr int DW_THREADS = 32 * DW_TH;

// BWD = false: dst = dwconv(src) + bias                            (nn.Conv2d(C, C, 7, padding=3, groups=C))
// BWD = true : dst = resid + conv_transpose(src) = resid + the same conv with the kernel flipped, no bias
template <bool BWD>
__global__ void __launch_bounds__(DW_THREADS) dwconv_kernel(const float* __restrict__ src, const float* __restrict__ w,
                                                            const float* __restrict__ bias, const float* __restrict__ resid,
                                                            float* __restrict__ dst, Geo g, int tiles_x) {
  pdl_prologue();
  __shared__ float tile[DW_HH * DW_HW][DW_CS];
  __shared__ float wt[49][DW_CS];
  const int tx0 = (blockIdx.x % tiles_x) * DW_TW, ty0 = (blockIdx.x / tiles_x) * DW_TH;
  const int c0 = blockIdx.y * DW_CS, b = blockIdx.z, C = g.C;
  const int Hf = g.nh * g.s, Wf = g.nw * g.s;
  for (int i = threadIdx.x; i < 49 * DW_CS; i += DW_THREADS) {
    const int c = i / 49, tap = i % 49;
    wt[BWD ? 48 - tap : tap][c] = __ldg(w + (c0 + c) * 49 + tap);
  }
  for (int i = threadIdx.x; i < DW_HH * DW_HW * (DW_CS / 4); i += DW_THREADS) {
    const int q = i % (DW_CS / 4), pix = i / (DW_CS / 4);
    const int y = ty0 + pix / DW_HW - 3, x = tx0 + pix % DW_HW - 3;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (y >= 0 && y < Hf && x >= 0 && x < Wf) v = __ldg(reinterpret_cast<const float4*>(src + pix_row(b, y, x, g) * C + c0) + q);
    *reinterpret_cast<float4*>(&tile[pix][4 * q]) = v;
  }
  __syncthreads();
  const int c = threadIdx.x & 31, ry = threadIdx.x >> 5;
  float acc[DW_TW];
#pragma unroll
  for (int j = 0; j < DW_TW; ++j) acc[j] = 0.f;
#pragma unroll
  for (int ky = 0; ky < 7; ++ky) {
    float v[DW_HW];
#pragma unroll
    for (int j = 0; j < DW_HW; ++j) v[j] = tile[(ry + ky) * DW_HW + j][c];
#pragma unroll
    for (int kx = 0; kx < 7; ++kx) {
      const float wk = wt[ky * 7 + kx][c];
#pragma unroll
      for (int j = 0; j < DW_TW; ++j) acc[j] = fmaf(v[j + kx], wk, acc[j]);
    }
  }
  const int y = ty0 + ry;
  if (y >= Hf) return;
  const float add_b = BWD ? 0.f : __ldg(bias + c0 + c);
#pragma unroll
  for (int j = 0; j < DW_TW; ++j) {
    const int x = tx0 + j;
    if (x < Wf) {
      const int64_t o = pix_row(b, y, x, g) * C + c0 + c;
      dst[o] = acc[j] + (BWD ? __ldg(resid + o) : add_b);
    }
  }
}

// Weight gradient dW[c, ky, kx] = sum over pixels of dd(y, x) * x(y + ky - 3, x + kx - 3).  One CTA per (column of tiles,
// channel slice, sample): it walks the column's tiles accumulating all 49 taps in registers, then adds its 8 warps in a
// fixed order and writes one partial row [C*49] (its slice) of partial[b * tiles_x + column]; mmae_cast_colsum_f32 sums the
// rows.  No atomics.
__global__ void __launch_bounds__(DW_THREADS) dwconv_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dd,
                                                                  Geo g, int tiles_x, int tiles_y, float* __restrict__ partial) {
  pdl_prologue();
  __shared__ float tile[DW_HH * DW_HW][DW_CS];
  const int tx0 = blockIdx.x * DW_TW, c0 = blockIdx.y * DW_CS, b = blockIdx.z, C = g.C;
  const int Hf = g.nh * g.s, Wf = g.nw * g.s;
  const int c = threadIdx.x & 31, ry = threadIdx.x >> 5;
  float acc[49];
#pragma unroll
  for (int t = 0; t < 49; ++t) acc[t] = 0.f;
  for (int ty = 0; ty < tiles_y; ++ty) {
    const int ty0 = ty * DW_TH;
    __syncthreads();                         // the previous tile's reads are done
    for (int i = threadIdx.x; i < DW_HH * DW_HW * (DW_CS / 4); i += DW_THREADS) {
      const int q = i % (DW_CS / 4), pix = i / (DW_CS / 4);
      const int yy = ty0 + pix / DW_HW - 3, xx = tx0 + pix % DW_HW - 3;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (yy >= 0 && yy < Hf && xx >= 0 && xx < Wf)
        v = __ldg(reinterpret_cast<const float4*>(x + pix_row(b, yy, xx, g) * C + c0) + q);
      *reinterpret_cast<float4*>(&tile[pix][4 * q]) = v;
    }
    float d[DW_TW];
    const int y = ty0 + ry;
#pragma unroll
    for (int j = 0; j < DW_TW; ++j) {
      const int xx = tx0 + j;
      d[j] = (y < Hf && xx < Wf) ? __ldg(dd + pix_row(b, y, xx, g) * C + c0 + c) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int ky = 0; ky < 7; ++ky) {
      float v[DW_HW];
#pragma unroll
      for (int j = 0; j < DW_HW; ++j) v[j] = tile[(ry + ky) * DW_HW + j][c];
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) {
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < DW_TW; ++j) s = fmaf(d[j], v[j + kx], s);
        acc[ky * 7 + kx] += s;
      }
    }
  }
  float* red = &tile[0][0];                  // [DW_TH warps][7 taps][32 channels]
  float* out = partial + (int64_t(b) * tiles_x + blockIdx.x) * C * 49;
#pragma unroll
  for (int ky = 0; ky < 7; ++ky) {
    __syncthreads();
#pragma unroll
    for (int kx = 0; kx < 7; ++kx) red[(ry * 7 + kx) * 32 + c] = acc[ky * 7 + kx];
    __syncthreads();
    if (threadIdx.x < 7 * 32) {
      const int kx = threadIdx.x >> 5, cc = threadIdx.x & 31;
      float s = 0.f;
      for (int wv = 0; wv < DW_TH; ++wv) s += red[(wv * 7 + kx) * 32 + cc];
      out[(c0 + cc) * 49 + ky * 7 + kx] = s;
    }
  }
}

// ------------------------------------------------------------------------------------------------ bilinear upsample
// F.interpolate(mode="bilinear", align_corners=False) from (Hf, Wf) to (H, W), as ATen computes it: scale = in / out,
// src = max(0, (dst + 0.5) * scale - 0.5), i0 = floor(src), i1 = i0 + (i0 < in - 1), lambda = src - i0.  A source coordinate
// below 0 is clamped to 0, so the full weight goes to pixel 0.
struct Tap {
  int i0, i1;
  float l0, l1;
};
__device__ __forceinline__ Tap src_tap(int dst, float scale, int in) {
  const float s = fmaxf((dst + 0.5f) * scale - 0.5f, 0.f);
  Tap t;
  t.i0 = (int)s;
  t.i1 = t.i0 + (t.i0 < in - 1 ? 1 : 0);
  t.l1 = s - t.i0;
  t.l0 = 1.f - t.l1;
  return t;
}
constexpr int UP_THREADS = 256;
constexpr int UP_SMEM_FLOATS = 12288;        // 48 KB of dynamic shared memory

// grid (H, B, class chunks): one output row Y of one sample for kc classes.  The two source rows are staged as
// [row][x][class] (stride kc + 1 against bank conflicts), then each class's output row is written with coalesced stores.
__global__ void __launch_bounds__(UP_THREADS) upsample_fwd_kernel(const float* __restrict__ cmap, int Kp, int K, int KC, Geo g,
                                                                  int H, int W, float* __restrict__ out) {
  pdl_prologue();
  extern __shared__ float sm[];
  const int Y = blockIdx.x, b = blockIdx.y, k0 = blockIdx.z * KC, kc = min(KC, K - k0), ld = kc + 1;
  const int Hf = g.nh * g.s, Wf = g.nw * g.s;
  const float sh = (float)Hf / (float)H, sw = (float)Wf / (float)W;
  const Tap ty = src_tap(Y, sh, Hf);
  for (int i = threadIdx.x; i < 2 * Wf * kc; i += UP_THREADS) {
    const int kk = i % kc, rest = i / kc, x = rest % Wf, r = rest / Wf;
    sm[(r * Wf + x) * ld + kk] = __ldg(cmap + pix_row(b, r ? ty.i1 : ty.i0, x, g) * Kp + k0 + kk);
  }
  __syncthreads();
  for (int kk = 0; kk < kc; ++kk) {
    float* orow = out + ((int64_t(b) * K + k0 + kk) * H + Y) * W;
    for (int X = threadIdx.x; X < W; X += UP_THREADS) {
      const Tap tx = src_tap(X, sw, Wf);
      const float* r0 = sm + kk;
      const float* r1 = sm + Wf * ld + kk;
      const float v = ty.l0 * (tx.l0 * r0[tx.i0 * ld] + tx.l1 * r0[tx.i1 * ld]) +
                      ty.l1 * (tx.l0 * r1[tx.i0 * ld] + tx.l1 * r1[tx.i1 * ld]);
      __stcs(orow + X, v);
    }
  }
}

// weight of output index `dst` on source index `src` (0 when dst does not reference src)
__device__ __forceinline__ float tap_weight(int dst, int src, float scale, int in) {
  const Tap t = src_tap(dst, scale, in);
  return (t.i0 == src ? t.l0 : 0.f) + (t.i1 == src ? t.l1 : 0.f);
}

// Gather-form backward, grid (Hf, B, class chunks): source row y of one sample for kc classes of the padded width Kp.
// Pass 1: racc[kk][X] = sum over the output rows Y that reference y of wy(Y) * dout[b, k, Y, X]  (coalesced row reads).
// Pass 2: dcmap[pixel (y, x), k] = sum over the output columns X that reference x of wx(X) * racc[kk][X], written
// class-contiguous; classes K..Kp-1 get zeros.  Integer ratios r = H / Hf, rx = W / Wf: output rows (y-1)*r .. (y+2)*r - 1
// cover every row that can reference y.  Fixed summation order, no atomics.
__global__ void __launch_bounds__(UP_THREADS) upsample_bwd_kernel(const float* __restrict__ dout, int Kp, int K, int KC, Geo g,
                                                                  int H, int W, float* __restrict__ dcmap) {
  pdl_prologue();
  extern __shared__ float sm[];
  const int y = blockIdx.x, b = blockIdx.y, k0 = blockIdx.z * KC, kc = min(KC, Kp - k0), ld = W + 1;
  const int Hf = g.nh * g.s, Wf = g.nw * g.s, r = H / Hf, rx = W / Wf;
  const float sh = (float)Hf / (float)H, sw = (float)Wf / (float)W;
  const int Y0 = max(0, (y - 1) * r), Y1 = min(H, (y + 2) * r);
  for (int i = threadIdx.x; i < kc * W; i += UP_THREADS) {
    const int kk = i / W, X = i % W, k = k0 + kk;
    float s = 0.f;
    if (k < K) {
      const float* col = dout + (int64_t(b) * K + k) * H * W + X;
      for (int Y = Y0; Y < Y1; ++Y) {
        const float wy = tap_weight(Y, y, sh, Hf);
        if (wy != 0.f) s = fmaf(wy, __ldg(col + int64_t(Y) * W), s);
      }
    }
    sm[kk * ld + X] = s;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < Wf * kc; i += UP_THREADS) {
    const int kk = i % kc, x = i / kc;
    const int X0 = max(0, (x - 1) * rx), X1 = min(W, (x + 2) * rx);
    float s = 0.f;
    for (int X = X0; X < X1; ++X) {
      const float wx = tap_weight(X, x, sw, Wf);
      if (wx != 0.f) s = fmaf(wx, sm[kk * ld + X], s);
    }
    dcmap[pix_row(b, y, x, g) * Kp + k0 + kk] = s;
  }
}

// ------------------------------------------------------------------------------------------------ saved / workspace
struct ProjSaved {
  bf16 *A, *w_b;
  size_t bytes;
};
ProjSaved proj_saved(void* base, int rows, int Kin, int E) {
  Carve c{reinterpret_cast<uint8_t*>(base)};
  ProjSaved s;
  s.A = c.take<bf16>(size_t(rows) * Kin);
  s.w_b = c.take<bf16>(size_t(E) * Kin);
  s.bytes = align_up(c.off, 256);
  return s;
}
struct ProjWs {
  bf16* g;
  float* dA;
  size_t bytes;
};
ProjWs proj_ws(void* base, int rows, int Kin, int E) {
  Carve c{reinterpret_cast<uint8_t*>(base)};
  ProjWs w;
  w.g = c.take<bf16>(size_t(rows) * E);
  w.dA = c.take<float>(size_t(rows) * Kin);
  w.bytes = align_up(c.off, 256);
  return w;
}

int tiles_x_of(const Geo& g) { return ceil_div(g.nw * g.s, DW_TW); }
int tiles_y_of(const Geo& g) { return ceil_div(g.nh * g.s, DW_TH); }

struct BlockSaved {
  bf16 *w1, *w2, *h, *z, *a;
  float *d, *mean, *rstd;
  size_t bytes;
};
BlockSaved blk_saved(void* base, int64_t P, int C) {
  Carve c{reinterpret_cast<uint8_t*>(base)};
  BlockSaved s;
  s.w1 = c.take<bf16>(size_t(4) * C * C);
  s.w2 = c.take<bf16>(size_t(4) * C * C);
  s.d = c.take<float>(size_t(P) * C);
  s.mean = c.take<float>(P);
  s.rstd = c.take<float>(P);
  s.h = c.take<bf16>(size_t(P) * C);
  s.z = c.take<bf16>(size_t(P) * 4 * C);
  s.a = c.take<bf16>(size_t(P) * 4 * C);
  s.bytes = align_up(c.off, 256);
  return s;
}
struct BlockWs {
  bf16 *g, *dz, *dh;
  float *dd, *wpart;
  size_t bytes;
};
BlockWs blk_ws(void* base, int B, const Geo& geo, int64_t P) {
  Carve c{reinterpret_cast<uint8_t*>(base)};
  const int C = geo.C;
  BlockWs w;
  w.g = c.take<bf16>(size_t(P) * C);
  w.dz = c.take<bf16>(size_t(P) * 4 * C);
  w.dh = c.take<bf16>(size_t(P) * C);
  w.dd = c.take<float>(size_t(P) * C);
  w.wpart = c.take<float>(size_t(B) * tiles_x_of(geo) * C * 49);
  w.bytes = align_up(c.off, 256);
  return w;
}

struct TailSaved {
  bf16 *x_b, *w_b;
  size_t bytes;
};
TailSaved tl_saved(void* base, int64_t P, int C, int K) {
  Carve c{reinterpret_cast<uint8_t*>(base)};
  TailSaved s;
  s.x_b = c.take<bf16>(size_t(P) * C);
  s.w_b = c.take<bf16>(size_t(round8(K)) * C);
  s.bytes = align_up(c.off, 256);
  return s;
}
struct TailWs {
  float *cmap, *bias_p, *db_p, *dw_p;   // cmap: the [P, Kp] class map (forward) or its gradient (backward)
  bf16* g;
  size_t bytes;
};
TailWs tl_ws(void* base, int64_t P, int C, int K) {
  Carve c{reinterpret_cast<uint8_t*>(base)};
  const int Kp = round8(K);
  TailWs w;
  w.cmap = c.take<float>(size_t(P) * Kp);
  w.bias_p = c.take<float>(Kp);
  w.db_p = c.take<float>(Kp);
  w.dw_p = c.take<float>(size_t(Kp) * C);
  w.g = c.take<bf16>(size_t(P) * Kp);
  w.bytes = align_up(c.off, 256);
  return w;
}

int check_geo(const char* what, int B, int nh, int nw, int s, int C) {
  MMAE_CHECK(B > 0 && nh > 0 && nw > 0 && s > 0, MMAE_ERR_ARG, "%s: bad shape B=%d nh=%d nw=%d s=%d", what, B, nh, nw, s);
  MMAE_CHECK(C % 128 == 0 && C > 0 && C <= 1024, MMAE_ERR_UNSUPPORTED,
             "%s: C=%d channels per pixel must be a multiple of 128, at most 1024 (the LayerNorm kernels)", what, C);
  MMAE_CHECK(int64_t(B) * nh * nw * s * s < (int64_t(1) << 31), MMAE_ERR_UNSUPPORTED, "%s: too many pixels", what);
  return MMAE_OK;
}

int check_proj(const char* what, int B, int N, int D, int n, int T, const int* start_host, int E) {
  MMAE_CHECK(B > 0 && N > 0 && n > 0 && T >= 1 && T <= MMAE_MAX_TASKS && start_host && E > 0 && E % 8 == 0,
             MMAE_ERR_ARG, "%s: bad args (B=%d N=%d n=%d tasks=%d E=%d)", what, B, N, n, T, E);
  MMAE_CHECK(D > 0 && D % 8 == 0, MMAE_ERR_UNSUPPORTED, "%s: D=%d must be a multiple of 8", what, D);
  for (int k = 0; k < T; ++k)
    MMAE_CHECK(start_host[k] >= 0 && start_host[k] + n <= N, MMAE_ERR_ARG, "%s: task %d tokens [%d, %d) outside [0, %d)",
               what, k, start_host[k], start_host[k] + n, N);
  return MMAE_OK;
}

template <typename K, typename... A>
int launch(K kernel, dim3 grid, dim3 block, size_t smem, void* st, A... args) {
  launch_k(kernel, grid, block, smem, reinterpret_cast<cudaStream_t>(st), args...);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

}  // namespace
}  // namespace mmae

using namespace mmae;

// ====================================================================================================== proj
extern "C" int64_t mmae_convnext_proj_saved_bytes(int B, int n, int D_in, int E) {
  return (int64_t)proj_saved(nullptr, B * n, D_in, E).bytes;
}
extern "C" int64_t mmae_convnext_proj_workspace_bytes(int B, int n, int D_in, int E) {
  return (int64_t)proj_ws(nullptr, B * n, D_in, E).bytes;
}

extern "C" int mmae_convnext_proj_forward(const float* enc, int B, int N, int D, int n, int num_tasks, const int* start_host,
                                          int E, const float* w, const float* bias, float* x_out, void* saved, void* ws,
                                          void* stream) {
  RUN(check_proj("mmae_convnext_proj_forward", B, N, D, n, num_tasks, start_host, E));
  MMAE_CHECK(enc && w && bias && x_out && saved && aligned16(enc) && aligned16(x_out), MMAE_ERR_ARG,
             "mmae_convnext_proj_forward: bad args (tensors must be 16-byte aligned)");
  (void)ws;
  const int rows = B * n, Kin = num_tasks * D;
  ProjSaved s = proj_saved(saved, rows, Kin, E);
  TaskStarts ts{};
  for (int k = 0; k < num_tasks; ++k) ts.v[k] = start_host[k];
  RUN(launch(cnx_gather_kernel, dim3(rows), dim3(256), 0, stream, enc, N, D, n, num_tasks, ts, s.A));
  RUN(weight_operand(w, &s.w_b, int64_t(E) * Kin, true, stream));
  return linear_f32(s.A, s.w_b, bias, nullptr, x_out, rows, E, Kin, stream);     // output_adapters.py:562
}

extern "C" int mmae_convnext_proj_backward(const float* dx_out, int B, int N, int D, int n, int num_tasks,
                                           const int* start_host, int E, const float* w, float* d_w, float* d_b, float* denc,
                                           const void* saved, void* ws, void* stream) {
  RUN(check_proj("mmae_convnext_proj_backward", B, N, D, n, num_tasks, start_host, E));
  MMAE_CHECK(dx_out && w && d_w && d_b && denc && saved && ws && aligned16(dx_out) && aligned16(denc), MMAE_ERR_ARG,
             "mmae_convnext_proj_backward: bad args (tensors must be 16-byte aligned)");
  const int rows = B * n, Kin = num_tasks * D;
  ProjSaved s = proj_saved(const_cast<void*>(saved), rows, Kin, E);
  ProjWs wk = proj_ws(ws, rows, Kin, E);
  RUN(weight_operand(w, &s.w_b, 0, false, stream));
  RUN(mmae_cast_colsum_f32(dx_out, E, wk.g, E, d_b, rows, E, stream));
  RUN(wgrad(wk.g, E, s.A, Kin, d_w, rows, E, Kin, stream));
  mmae_gemm_epilogue ep = ep_zero();
  ep.out_f32 = wk.dA;
  ep.ld_out_f32 = Kin;
  RUN(mmae_gemm_bf16(wk.g, E, 0, s.w_b, Kin, 1, rows, Kin, E, 1, &ep, stream));
  TaskStarts ts{};
  for (int k = 0; k < num_tasks; ++k) ts.v[k] = start_host[k];
  return launch(cnx_scatter_kernel, dim3(B * N), dim3(std::min(256, std::max(32, D / 4))), 0, stream, (const float*)wk.dA,
                N, D, n, num_tasks, ts, denc);
}

// ====================================================================================================== block
extern "C" int64_t mmae_convnext_block_saved_bytes(int B, int nh, int nw, int s, int C) {
  return (int64_t)blk_saved(nullptr, int64_t(B) * nh * nw * s * s, C).bytes;
}
extern "C" int64_t mmae_convnext_block_workspace_bytes(int B, int nh, int nw, int s, int C) {
  return (int64_t)blk_ws(nullptr, B, Geo{nh, nw, s, C}, int64_t(B) * nh * nw * s * s).bytes;
}

// order of the parameter / gradient pointer arrays of the block entry points
enum { DW_W, DW_B, NORM_W, NORM_B, PW1_W, PW1_B, PW2_W, PW2_B, NUM_BLOCK_PARAMS };

extern "C" int mmae_convnext_block_forward(const float* x_in, float* x_out, int B, int nh, int nw, int s, int C, float eps,
                                           const float* const* p, void* saved, void* ws, void* stream) {
  RUN(check_geo("mmae_convnext_block_forward", B, nh, nw, s, C));
  MMAE_CHECK(x_in && x_out && p && saved && aligned16(x_in) && aligned16(x_out), MMAE_ERR_ARG,
             "mmae_convnext_block_forward: bad args");
  (void)ws;
  const Geo g{nh, nw, s, C};
  const int P = B * nh * nw * s * s;
  BlockSaved sv = blk_saved(saved, P, C);
  RUN(weight_operand(p[PW1_W], &sv.w1, int64_t(4) * C * C, true, stream));
  RUN(weight_operand(p[PW2_W], &sv.w2, int64_t(4) * C * C, true, stream));
  // dwconv (output_adapter_utils.py:50)
  const int tx = tiles_x_of(g), ty = tiles_y_of(g);
  RUN(launch(dwconv_kernel<false>, dim3(tx * ty, C / DW_CS, B), dim3(DW_THREADS), 0, stream, x_in, p[DW_W], p[DW_B],
             (const float*)nullptr, sv.d, g, tx));
  // norm -> pwconv1 -> GELU -> pwconv2, input + x (:52-59)
  RUN(mmae_layernorm_forward(sv.d, C, p[NORM_W], p[NORM_B], sv.h, C, nullptr, 0, sv.mean, sv.rstd, P, C, eps, stream));
  RUN(linear_gelu(sv.h, sv.w1, p[PW1_B], sv.z, sv.a, P, 4 * C, C, stream));
  return linear_f32(sv.a, sv.w2, p[PW2_B], x_in, x_out, P, C, 4 * C, stream);
}

extern "C" int mmae_convnext_block_backward(const float* x_in, const float* dx_out, float* dx_in, int B, int nh, int nw,
                                            int s, int C, const float* const* p, float* const* gr,
                                            const void* saved, void* ws, void* stream) {
  RUN(check_geo("mmae_convnext_block_backward", B, nh, nw, s, C));
  MMAE_CHECK(x_in && dx_out && dx_in && p && gr && saved && ws && aligned16(dx_out) && aligned16(dx_in), MMAE_ERR_ARG,
             "mmae_convnext_block_backward: bad args");
  const Geo g{nh, nw, s, C};
  const int P = B * nh * nw * s * s;
  BlockSaved sv = blk_saved(const_cast<void*>(saved), P, C);
  BlockWs w = blk_ws(ws, B, g, P);
  RUN(weight_operand(p[PW1_W], &sv.w1, 0, false, stream));
  RUN(weight_operand(p[PW2_W], &sv.w2, 0, false, stream));
  RUN(mmae_cast_colsum_f32(dx_out, C, w.g, C, gr[PW2_B], P, C, stream));
  RUN(wgrad(w.g, C, sv.a, 4 * C, gr[PW2_W], P, C, 4 * C, stream));
  RUN(dgrad_dgelu_colsum(w.g, C, sv.w2, sv.z, w.dz, gr[PW1_B], P, C, 4 * C, stream));
  RUN(wgrad(w.dz, 4 * C, sv.h, C, gr[PW1_W], P, 4 * C, C, stream));
  RUN(dgrad_bf16(w.dz, 4 * C, sv.w1, nullptr, w.dh, P, 4 * C, C, stream));
  RUN(mmae_layernorm_backward(w.dh, 1, C, sv.d, C, sv.mean, sv.rstd, p[NORM_W], nullptr, 0, w.dd, C, gr[NORM_W], gr[NORM_B],
                              P, C, stream));
  const int tx = tiles_x_of(g), ty = tiles_y_of(g);
  RUN(launch(dwconv_kernel<true>, dim3(tx * ty, C / DW_CS, B), dim3(DW_THREADS), 0, stream, (const float*)w.dd, p[DW_W],
             (const float*)nullptr, dx_out, dx_in, g, tx));
  RUN(launch(dwconv_wgrad_kernel, dim3(tx, C / DW_CS, B), dim3(DW_THREADS), 0, stream, x_in, (const float*)w.dd, g, tx, ty,
             w.wpart));
  RUN(mmae_cast_colsum_f32(w.wpart, int64_t(C) * 49, nullptr, 0, gr[DW_W], B * tx, C * 49, stream));
  return mmae_cast_colsum_f32(w.dd, C, nullptr, 0, gr[DW_B], P, C, stream);
}

// ====================================================================================================== tail
extern "C" int64_t mmae_convnext_tail_saved_bytes(int B, int nh, int nw, int s, int C, int K) {
  return (int64_t)tl_saved(nullptr, int64_t(B) * nh * nw * s * s, C, K).bytes;
}
extern "C" int64_t mmae_convnext_tail_workspace_bytes(int B, int nh, int nw, int s, int C, int K) {
  return (int64_t)tl_ws(nullptr, int64_t(B) * nh * nw * s * s, C, K).bytes;
}

namespace mmae {
int upsample_check(const char* what, int nh, int nw, int s, int K, int H, int W) {
  const int Hf = nh * s, Wf = nw * s;
  MMAE_CHECK(K > 0 && H > 0 && W > 0 && H % Hf == 0 && W % Wf == 0, MMAE_ERR_UNSUPPORTED,
             "%s: the upsample needs K > 0 and integer ratios, got (%d, %d) -> (%d, %d)", what, Hf, Wf, H, W);
  MMAE_CHECK(2 * Wf * 2 <= UP_SMEM_FLOATS && 2 * (W + 1) <= UP_SMEM_FLOATS, MMAE_ERR_UNSUPPORTED,
             "%s: rows of %d / %d pixels are too wide for the upsample kernels", what, Wf, W);
  return MMAE_OK;
}

int launch_upsample_fwd(const float* cmap, int Kp, int K, int B, int nh, int nw, int s, int H, int W, float* out, void* stream) {
  const Geo g{nh, nw, s, 0};
  const int Wf = nw * s, KC = std::min(K, UP_SMEM_FLOATS / (2 * Wf) - 1);
  return launch(upsample_fwd_kernel, dim3(H, B, ceil_div(K, KC)), dim3(UP_THREADS), size_t(2) * Wf * (KC + 1) * sizeof(float),
                stream, cmap, Kp, K, KC, g, H, W, out);
}

int launch_upsample_bwd(const float* dout, int Kp, int K, int B, int nh, int nw, int s, int H, int W, float* dcmap,
                        void* stream) {
  const Geo g{nh, nw, s, 0};
  const int KC = std::min(Kp, UP_SMEM_FLOATS / (W + 1));
  return launch(upsample_bwd_kernel, dim3(nh * s, B, ceil_div(Kp, KC)), dim3(UP_THREADS), size_t(KC) * (W + 1) * sizeof(float),
                stream, dout, Kp, K, KC, g, H, W, dcmap);
}
}  // namespace mmae

extern "C" int mmae_convnext_tail_forward(const float* x, int B, int nh, int nw, int s, int C, int K, int H, int W,
                                          const float* w, const float* bias, float* out, void* saved, void* ws, void* stream) {
  RUN(check_geo("mmae_convnext_tail_forward", B, nh, nw, s, C));
  RUN(upsample_check("mmae_convnext_tail_forward", nh, nw, s, K, H, W));
  MMAE_CHECK(x && w && bias && out && saved && ws && aligned16(x), MMAE_ERR_ARG, "mmae_convnext_tail_forward: bad args");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int P = B * nh * nw * s * s, Kp = round8(K);
  TailSaved sv = tl_saved(saved, P, C, K);
  TailWs wk = tl_ws(ws, P, C, K);
  RUN(mmae_cast_f32_to_bf16(x, sv.x_b, int64_t(P) * C, stream));
  // final_layer (output_adapters.py:570) on the padded width: zero weight rows / bias entries K..Kp-1
  const bf16* m = mirror_lookup(w);
  if (m != nullptr)
    MMAE_CUDA_OK(cudaMemcpyAsync(sv.w_b, m, size_t(K) * C * sizeof(bf16), cudaMemcpyDeviceToDevice, st));
  else
    RUN(mmae_cast_f32_to_bf16(w, sv.w_b, int64_t(K) * C, stream));
  if (Kp != K) MMAE_CUDA_OK(cudaMemsetAsync(sv.w_b + size_t(K) * C, 0, size_t(Kp - K) * C * sizeof(bf16), st));
  MMAE_CUDA_OK(cudaMemsetAsync(wk.bias_p, 0, Kp * sizeof(float), st));
  MMAE_CUDA_OK(cudaMemcpyAsync(wk.bias_p, bias, K * sizeof(float), cudaMemcpyDeviceToDevice, st));
  RUN(linear_f32(sv.x_b, sv.w_b, wk.bias_p, nullptr, wk.cmap, P, Kp, C, stream));
  // F.interpolate(size=(H, W), mode="bilinear") (:573)
  return launch_upsample_fwd(wk.cmap, Kp, K, B, nh, nw, s, H, W, out, stream);
}

extern "C" int mmae_convnext_tail_backward(const float* dout, int B, int nh, int nw, int s, int C, int K, int H, int W,
                                           const float* w, float* d_w, float* d_b, float* dx, const void* saved, void* ws,
                                           void* stream) {
  RUN(check_geo("mmae_convnext_tail_backward", B, nh, nw, s, C));
  RUN(upsample_check("mmae_convnext_tail_backward", nh, nw, s, K, H, W));
  MMAE_CHECK(dout && w && d_w && d_b && dx && saved && ws && aligned16(dx), MMAE_ERR_ARG,
             "mmae_convnext_tail_backward: bad args");
  (void)w;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int P = B * nh * nw * s * s, Kp = round8(K);
  TailSaved sv = tl_saved(const_cast<void*>(saved), P, C, K);
  TailWs wk = tl_ws(ws, P, C, K);
  RUN(launch_upsample_bwd(dout, Kp, K, B, nh, nw, s, H, W, wk.cmap, stream));
  const bool pad = Kp != K;
  if (pad) {
    MMAE_CUDA_OK(cudaMemsetAsync(wk.db_p, 0, Kp * sizeof(float), st));
    MMAE_CUDA_OK(cudaMemsetAsync(wk.dw_p, 0, size_t(Kp) * C * sizeof(float), st));
  }
  RUN(mmae_cast_colsum_f32(wk.cmap, Kp, wk.g, Kp, pad ? wk.db_p : d_b, P, Kp, stream));
  RUN(wgrad(wk.g, Kp, sv.x_b, C, pad ? wk.dw_p : d_w, P, Kp, C, stream));
  mmae_gemm_epilogue ep = ep_zero();
  ep.out_f32 = dx;
  ep.ld_out_f32 = C;
  RUN(mmae_gemm_bf16(wk.g, Kp, 0, sv.w_b, C, 1, P, C, Kp, 1, &ep, stream));
  if (pad) {
    RUN(add_f32(d_b, wk.db_p, K, st));
    RUN(add_f32(d_w, wk.dw_p, int64_t(K) * C, st));
  }
  return MMAE_OK;
}
