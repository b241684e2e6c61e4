// Module-level entry points of the C ABI: each one is the forward or backward of one reference nn.Module on the hot
// path, expressed as a fixed sequence of the kernels in this library (wgmma GEMMs with fused epilogues, LayerNorm,
// fused attention, index kernels).  The host passes raw device pointers; all scratch ("ws") and saved-for-backward
// ("saved") memory is caller-provided, sized by the *_bytes queries, so nothing here allocates.
#include <cstdlib>

#include "internal.h"

namespace mmae {
namespace {

struct Carver {
  uint8_t* base;
  size_t off = 0;
  explicit Carver(void* b) : base(reinterpret_cast<uint8_t*>(b)) {}
  template <typename T>
  T* take(size_t n) {
    off = align_up(off, 256);
    T* p = reinterpret_cast<T*>(base + off);
    off += n * sizeof(T);
    return p;
  }
};

}  // namespace

// ---------------------------------------------------------------------------------------------- GEMM helpers
// Shared with the other module-level entry points (declared in internal.h).

// split-K count of the weight-gradient GEMMs: 0 = chosen by mmae_gemm_bf16 together with the tile width
int pick_split(int, int, int) { return 0; }

// bf16 operand of a weight: the registered mirror of the fp32 parameter buffer (no cast, refreshed by the optimizer
// kernel), else the per-call saved slot (cast now in forward; already cast in backward).
int weight_operand(const float* w, bf16** slot, int64_t n, bool cast_now, void* st) {
  if (const bf16* m = mirror_lookup(w)) {
    *slot = const_cast<bf16*>(m);
    return MMAE_OK;
  }
  return cast_now ? mmae_cast_f32_to_bf16(w, *slot, n, st) : MMAE_OK;
}

mmae_gemm_epilogue ep_zero() {
  mmae_gemm_epilogue ep;
  memset(&ep, 0, sizeof(ep));
  ep.alpha = 1.0f;
  return ep;
}

// y = x W^T + b  (bf16 out), W: [N, K]
int linear_bf16(const bf16* x, const bf16* W, const float* b, bf16* y, int M, int N, int K, void* st) {
  mmae_gemm_epilogue ep = ep_zero();
  ep.bias = b;
  ep.out_bf16 = y;
  ep.ld_out_bf16 = N;
  return mmae_gemm_bf16(x, K, 0, W, K, 0, M, N, K, 1, &ep, st);
}
// y = x W^T + b (+ residual) (fp32 out)
int linear_f32(const bf16* x, const bf16* W, const float* b, const float* resid, float* y, int M, int N, int K,
               void* st) {
  mmae_gemm_epilogue ep = ep_zero();
  ep.bias = b;
  ep.residual = resid;
  ep.ld_residual = N;
  ep.out_f32 = y;
  ep.ld_out_f32 = N;
  return mmae_gemm_bf16(x, K, 0, W, K, 0, M, N, K, 1, &ep, st);
}
// 1: GELU / GELU' applied in the GEMM epilogue; 0: GEMM writes the pre-activation and a streaming kernel applies it.
// Default 0: on one H100 80GB HBM3 capped at 400 W the MultiMAE-B bs 128 step takes 44.5 ms with it, 53.4 ms fused.
int g_fuse_gelu = []() {
  const char* e = getenv("MMAE_FUSE_GELU");
  return e ? atoi(e) : 0;
}();

// z = x W^T + b (bf16, saved), a = gelu(z) (bf16)
int linear_gelu(const bf16* x, const bf16* W, const float* b, bf16* z, bf16* a, int M, int N, int K, void* st) {
  mmae_gemm_epilogue ep = ep_zero();
  ep.bias = b;
  if (g_fuse_gelu) {
    ep.act = 1;
    ep.preact_bf16 = z;
    ep.ld_preact = N;
    ep.out_bf16 = a;
    ep.ld_out_bf16 = N;
    return mmae_gemm_bf16(x, K, 0, W, K, 0, M, N, K, 1, &ep, st);
  }
  ep.out_bf16 = z;
  ep.ld_out_bf16 = N;
  int rc = mmae_gemm_bf16(x, K, 0, W, K, 0, M, N, K, 1, &ep, st);
  if (rc != MMAE_OK) return rc;
  return mmae_gelu_bf16(z, a, int64_t(M) * N, 0, st);
}
// dx[M, Kin] = dy[M, Nout] W[Nout, Kin]  (bf16 out; optional * gelu'(z))
int dgrad_bf16(const bf16* dy, int64_t lddy, const bf16* W, const bf16* dgelu_z, bf16* dx, int M, int Nout, int Kin,
               void* st) {
  mmae_gemm_epilogue ep = ep_zero();
  const bool fused = dgelu_z != nullptr && g_fuse_gelu;
  ep.dgelu_z = fused ? dgelu_z : nullptr;
  ep.ld_dgelu_z = Kin;
  ep.out_bf16 = dx;
  ep.ld_out_bf16 = Kin;
  int rc = mmae_gemm_bf16(dy, lddy, 0, W, Kin, 1, M, Kin, Nout, 1, &ep, st);
  if (rc != MMAE_OK || dgelu_z == nullptr || fused) return rc;
  return mmae_gelu_bf16(dgelu_z, dx, int64_t(M) * Kin, 1, st);
}
// dz = (dy W) * gelu'(z)  and  db1 += colsum(dz)   (fc2 dgrad + GELU backward + fc1 bias gradient)
int dgrad_dgelu_colsum(const bf16* dy, int64_t lddy, const bf16* W, const bf16* z, bf16* dz, float* db, int M, int Nout,
                       int Kin, void* st) {
  if (g_fuse_gelu) {
    int rc = dgrad_bf16(dy, lddy, W, z, dz, M, Nout, Kin, st);
    if (rc != MMAE_OK) return rc;
    return mmae_colsum_bf16(dz, Kin, db, M, Kin, st);
  }
  int rc = dgrad_bf16(dy, lddy, W, nullptr, dz, M, Nout, Kin, st);
  if (rc != MMAE_OK) return rc;
  return mmae_dgelu_colsum_bf16(z, dz, Kin, db, M, Kin, st);
}
// dW[Nout, Kin] += dy[M, Nout]^T x[M, Kin]
int wgrad(const bf16* dy, int64_t lddy, const bf16* x, int64_t ldx, float* dW, int M, int Nout, int Kin, void* st) {
  mmae_gemm_epilogue ep = ep_zero();
  ep.accumulate = 1;
  ep.out_f32 = dW;
  ep.ld_out_f32 = Kin;
  return mmae_gemm_bf16(dy, lddy, 1, x, ldx, 1, Nout, Kin, M, pick_split(Nout, Kin, M), &ep, st);
}

namespace {

#define RUN(expr)             \
  do {                        \
    int _rc = (expr);         \
    if (_rc != MMAE_OK) return _rc; \
  } while (0)

// ------------------------------------------------------------------------------------------------------ block
struct BlockSaved {
  bf16 *wqkv, *wproj, *w1, *w2, *h1, *qkv, *o, *h2, *z, *a;
  float *mean1, *rstd1, *mean2, *rstd2, *lse, *x_mid;
  size_t bytes;
};
BlockSaved block_saved(void* base, int B, int N, int D, int H, int hid) {
  Carver c(base);
  const size_t M = size_t(B) * N;
  BlockSaved s;
  s.wqkv = c.take<bf16>(size_t(3) * D * D);
  s.wproj = c.take<bf16>(size_t(D) * D);
  s.w1 = c.take<bf16>(size_t(hid) * D);
  s.w2 = c.take<bf16>(size_t(D) * hid);
  s.mean1 = c.take<float>(M);
  s.rstd1 = c.take<float>(M);
  s.mean2 = c.take<float>(M);
  s.rstd2 = c.take<float>(M);
  s.h1 = c.take<bf16>(M * D);
  s.qkv = c.take<bf16>(M * 3 * D);
  s.lse = c.take<float>(size_t(B) * H * N);
  s.o = c.take<bf16>(M * D);
  s.x_mid = c.take<float>(M * D);
  s.h2 = c.take<bf16>(M * D);
  s.z = c.take<bf16>(M * hid);
  s.a = c.take<bf16>(M * hid);
  s.bytes = align_up(c.off, 256);
  return s;
}
struct BlockWs {
  bf16 *g, *big, *dh, *d_o;
  bf16 *g2, *big2;   // second copies so the weight-gradient GEMMs on the side stream keep reading g / big undisturbed
  float *dx_mid, *delta;
  size_t bytes;
};
BlockWs block_ws(void* base, int B, int N, int D, int H, int hid) {
  Carver c(base);
  const size_t M = size_t(B) * N;
  BlockWs w;
  w.g = c.take<bf16>(M * D);
  w.big = c.take<bf16>(M * std::max(hid, 3 * D));
  w.dh = c.take<bf16>(M * D);
  w.d_o = c.take<bf16>(M * D);
  w.g2 = c.take<bf16>(M * D);
  w.big2 = c.take<bf16>(M * 3 * D);
  w.dx_mid = c.take<float>(M * D);
  w.delta = c.take<float>(size_t(B) * H * N);
  w.bytes = align_up(c.off, 256);
  return w;
}

// Weight-gradient side stream.  In a block's backward only the dgrad chain is on the critical path; the four weight
// gradient GEMMs hang off it.  They run on a library-owned stream, forked after the kernel that produces their dY operand
// and joined before the function returns, so they could fill the tensor cores while the main stream runs the HBM-bound
// GELU' / LayerNorm / softmax kernels.  A GEMM CTA claims most of an SM's shared memory, so the two streams mostly
// alternate.  OFF by default;
// MMAE_WGRAD_STREAM=1 / mmae_set_wgrad_stream(1) turns it on for experiments on other shapes.
struct SideStream {
  cudaStream_t stream = nullptr;
  cudaEvent_t fork[4] = {nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t join = nullptr;
  bool ok = false;
};
SideStream g_side;
int g_wgrad_stream = []() {
  const char* e = getenv("MMAE_WGRAD_STREAM");
  return e ? atoi(e) : 0;
}();

bool side_ready() {
  if (!g_wgrad_stream) return false;
  if (g_side.ok) return true;
  if (cudaStreamCreateWithFlags(&g_side.stream, cudaStreamNonBlocking) != cudaSuccess) return false;
  for (int i = 0; i < 4; ++i)
    if (cudaEventCreateWithFlags(&g_side.fork[i], cudaEventDisableTiming) != cudaSuccess) return false;
  if (cudaEventCreateWithFlags(&g_side.join, cudaEventDisableTiming) != cudaSuccess) return false;
  g_side.ok = true;
  return true;
}
// everything enqueued on `main` so far happens before what is enqueued on the side stream from now on
int side_fork(void* main, int idx) {
  MMAE_CUDA_OK(cudaEventRecord(g_side.fork[idx], reinterpret_cast<cudaStream_t>(main)));
  MMAE_CUDA_OK(cudaStreamWaitEvent(g_side.stream, g_side.fork[idx], 0));
  return MMAE_OK;
}
int side_join(void* main) {
  MMAE_CUDA_OK(cudaEventRecord(g_side.join, g_side.stream));
  MMAE_CUDA_OK(cudaStreamWaitEvent(reinterpret_cast<cudaStream_t>(main), g_side.join, 0));
  return MMAE_OK;
}

// --------------------------------------------------------------------------------------------------- decoder head
struct HeadSaved {
  bf16 *enc_b, *wpc, *wq, *wkv, *wproj, *w1, *w2, *qn, *cn, *q, *kv, *o, *h, *z, *a;
  float *queries, *context, *qmean, *qrstd, *cmean, *crstd, *omean, *orstd, *lse, *x0;
  size_t bytes;
};
HeadSaved head_saved(void* base, const mmae_decoder_index& ix, int De, int H, int hid) {
  Carver c(base);
  const size_t Dd = ix.dim, Mq = size_t(ix.batch) * ix.num_queries,
               Mc = size_t(ix.batch) * (ix.num_visible + ix.num_global);
  HeadSaved s;
  s.enc_b = c.take<bf16>(Mc * De);
  s.wpc = c.take<bf16>(Dd * De);
  s.wq = c.take<bf16>(Dd * Dd);
  s.wkv = c.take<bf16>(2 * Dd * Dd);
  s.wproj = c.take<bf16>(Dd * Dd);
  s.w1 = c.take<bf16>(size_t(hid) * Dd);
  s.w2 = c.take<bf16>(Dd * hid);
  s.queries = c.take<float>(Mq * Dd);
  s.context = c.take<float>(Mc * Dd);
  s.qmean = c.take<float>(Mq);
  s.qrstd = c.take<float>(Mq);
  s.cmean = c.take<float>(Mc);
  s.crstd = c.take<float>(Mc);
  s.omean = c.take<float>(Mq);
  s.orstd = c.take<float>(Mq);
  s.qn = c.take<bf16>(Mq * Dd);
  s.cn = c.take<bf16>(Mc * Dd);
  s.q = c.take<bf16>(Mq * Dd);
  s.kv = c.take<bf16>(Mc * 2 * Dd);
  s.lse = c.take<float>(size_t(ix.batch) * H * ix.num_queries);
  s.o = c.take<bf16>(Mq * Dd);
  s.x0 = c.take<float>(Mq * Dd);
  s.h = c.take<bf16>(Mq * Dd);
  s.z = c.take<bf16>(Mq * hid);
  s.a = c.take<bf16>(Mq * hid);
  s.bytes = align_up(c.off, 256);
  return s;
}
struct HeadWs {
  float *ctx, *dx0, *dqueries, *dcontext, *dctx, *delta;
  bf16 *g, *dz, *dh, *d_o, *dq, *dkv, *dqn, *dcn, *dctx_b;
  size_t bytes;
};
HeadWs head_ws(void* base, const mmae_decoder_index& ix, int De, int H, int hid) {
  Carver c(base);
  const size_t Dd = ix.dim, Mq = size_t(ix.batch) * ix.num_queries,
               Mc = size_t(ix.batch) * (ix.num_visible + ix.num_global);
  HeadWs w;
  w.ctx = c.take<float>(Mc * Dd);
  w.dx0 = c.take<float>(Mq * Dd);
  w.dqueries = c.take<float>(Mq * Dd);
  w.dcontext = c.take<float>(Mc * Dd);
  w.dctx = c.take<float>(Mc * Dd);
  w.delta = c.take<float>(size_t(ix.batch) * H * ix.num_queries);
  w.g = c.take<bf16>(Mq * Dd);
  w.dz = c.take<bf16>(Mq * hid);
  w.dh = c.take<bf16>(Mq * Dd);
  w.d_o = c.take<bf16>(Mq * Dd);
  w.dq = c.take<bf16>(Mq * Dd);
  w.dkv = c.take<bf16>(Mc * 2 * Dd);
  w.dqn = c.take<bf16>(Mq * Dd);
  w.dcn = c.take<bf16>(Mc * Dd);
  w.dctx_b = c.take<bf16>(Mc * Dd);
  w.bytes = align_up(c.off, 256);
  return w;
}

// ------------------------------------------------------------------------------------------------------ embed
struct EmbedSaved {
  bf16* A;
  int *row_task, *row_patch;
  size_t bytes;
};
EmbedSaved embed_saved(void* base, const mmae_embed_layout& L, int B, int T) {
  Carver c(base);
  EmbedSaved s;
  s.A = c.take<bf16>(size_t(B) * T * L.k_offset[L.num_tasks]);
  s.row_task = c.take<int>(size_t(B) * T);
  s.row_patch = c.take<int>(size_t(B) * T);
  s.bytes = align_up(c.off, 256);
  return s;
}
struct EmbedWs {
  bf16 *Wcat, *dC, *dA;
  float* Cmat;
  size_t bytes;
};
EmbedWs embed_ws(void* base, const mmae_embed_layout& L, int B, int T, int D) {
  Carver c(base);
  EmbedWs w;
  const size_t Kcat = L.k_offset[L.num_tasks];
  size_t kmax = 0;
  for (int t = 0; t < L.num_tasks; ++t) kmax = std::max<size_t>(kmax, L.k_offset[t + 1] - L.k_offset[t]);
  w.Wcat = c.take<bf16>(size_t(D) * Kcat);
  w.Cmat = c.take<float>(size_t(B) * T * D);
  w.dC = c.take<bf16>(size_t(B) * T * D);
  w.dA = c.take<bf16>(size_t(B) * T * kmax);
  w.bytes = align_up(c.off, 256);
  return w;
}

}  // namespace
}  // namespace mmae

using namespace mmae;

// ====================================================================================================== block
extern "C" int64_t mmae_block_saved_bytes(int B, int N, int D, int H, int hidden) {
  return (int64_t)block_saved(nullptr, B, N, D, H, hidden).bytes;
}
extern "C" int64_t mmae_block_workspace_bytes(int B, int N, int D, int H, int hidden) {
  return (int64_t)block_ws(nullptr, B, N, D, H, hidden).bytes;
}

// Chained form (mmae_block_forward_chain): consecutive blocks hand the last residual add over instead of running it as a
// pass of its own.  `x_add` (bf16) != null: the block input is x_in + x_add, formed inside the first LayerNorm kernel and
// written to `x_sum` (what backward gets as x_in).  `y_out` (bf16) != null: the MLP branch output goes there, x_out is not
// written, and the block's output is x_mid (mmae_block_saved_x_mid) + y_out - the next block's (x_in, x_add).
// Stochastic depth (mmae_block_forward_dp): s_attn / s_mlp [B] multiply the attention / MLP branch of each sample inside the
// residual adds, s_prev [B] multiplies x_add (the previous block's MLP branch).  Null: factor 1, the plain block.
static int block_forward_impl(const float* x_in, const bf16* x_add, float* x_sum, float* x_out, bf16* y_out, int B, int N,
                              int D, int H, int hidden, float eps, const float* s_attn, const float* s_mlp,
                              const float* s_prev, const mmae_block_params* p, void* saved, void* ws, void* st) {
  MMAE_CHECK(x_in && (x_out || y_out) && (!x_add || x_sum) && p && saved && ws && B > 0 && N > 0 && H > 0 && D % H == 0,
             MMAE_ERR_ARG, "mmae_block_forward: bad args");
  MMAE_CHECK(!s_prev || x_add, MMAE_ERR_ARG, "mmae_block_forward_dp: the previous block's scale needs x_add");
  const int M = B * N, dh = D / H;
  BlockSaved s = block_saved(saved, B, N, D, H, hidden);
  RUN(weight_operand(p->qkv_w, &s.wqkv, int64_t(3) * D * D, true, st));
  RUN(weight_operand(p->proj_w, &s.wproj, int64_t(D) * D, true, st));
  RUN(weight_operand(p->fc1_w, &s.w1, int64_t(hidden) * D, true, st));
  RUN(weight_operand(p->fc2_w, &s.w2, int64_t(D) * hidden, true, st));
  // Residual adds are not done in the GEMM epilogues: the branch output is stored as bf16 (what the reference's autocast
  // Linear produces, and half the bytes of an fp32 read-modify-write) and the add is fused into the next streaming kernel.
  BlockWs w = block_ws(ws, B, N, D, H, hidden);
  bf16* y = w.g;   // [M, D] bf16 scratch (forward only)
  // x = x + attn(norm1(x))                                       multimae_utils.py:230
  if (x_add) {   // the previous block's `x = x + mlp(..)` (multimae_utils.py:231) fused in front of this block's norm1
    RUN(add_layernorm_forward_scaled(x_in, D, x_add, D, s_prev, N, x_sum, D, p->norm1_w, p->norm1_b, s.h1, D, s.mean1, s.rstd1,
                                     M, D, eps, st));
    x_in = x_sum;
  } else {
    RUN(mmae_layernorm_forward(x_in, D, p->norm1_w, p->norm1_b, s.h1, D, nullptr, 0, s.mean1, s.rstd1, M, D, eps, st));
  }
  RUN(linear_bf16(s.h1, s.wqkv, p->qkv_b, s.qkv, M, 3 * D, D, st));
  RUN(mmae_attention_forward(s.qkv, 3 * D, s.qkv + D, 3 * D, s.qkv + 2 * D, 3 * D, s.o, D, s.lse, B, H, N, N, dh,
                             1.0f / sqrtf((float)dh), st));
  RUN(linear_bf16(s.o, s.wproj, p->proj_b, y, M, D, D, st));
  // x = x + mlp(norm2(x))                                        multimae_utils.py:231  (add fused in front of norm2)
  RUN(add_layernorm_forward_scaled(x_in, D, y, D, s_attn, N, s.x_mid, D, p->norm2_w, p->norm2_b, s.h2, D, s.mean2, s.rstd2, M,
                                   D, eps, st));
  RUN(linear_gelu(s.h2, s.w1, p->fc1_b, s.z, s.a, M, hidden, D, st));
  if (y_out) return linear_bf16(s.a, s.w2, p->fc2_b, y_out, M, D, hidden, st);   // the add is the next block's first kernel
  RUN(linear_bf16(s.a, s.w2, p->fc2_b, y, M, D, hidden, st));
  RUN(add_scaled_f32(s.x_mid, y, 1, s_mlp, int64_t(N) * D, x_out, int64_t(M) * D, st));
  return MMAE_OK;
}

extern "C" int mmae_block_forward(const float* x_in, float* x_out, int B, int N, int D, int H, int hidden, float eps,
                                  const mmae_block_params* p, void* saved, void* ws, void* st) {
  MMAE_CHECK(x_out, MMAE_ERR_ARG, "mmae_block_forward: bad args");
  return block_forward_impl(x_in, nullptr, nullptr, x_out, nullptr, B, N, D, H, hidden, eps, nullptr, nullptr, nullptr, p,
                            saved, ws, st);
}
extern "C" int mmae_block_forward_chain(const float* x_in, const void* x_add_bf16, float* x_sum, float* x_out,
                                        void* y_out_bf16, int B, int N, int D, int H, int hidden, float eps,
                                        const mmae_block_params* p, void* saved, void* ws, void* st) {
  return block_forward_impl(x_in, reinterpret_cast<const bf16*>(x_add_bf16), x_sum, x_out, reinterpret_cast<bf16*>(y_out_bf16),
                            B, N, D, H, hidden, eps, nullptr, nullptr, nullptr, p, saved, ws, st);
}
extern "C" int mmae_block_forward_dp(const float* x_in, const void* x_add_bf16, float* x_sum, float* x_out, void* y_out_bf16,
                                     int B, int N, int D, int H, int hidden, float eps, const float* scale_attn,
                                     const float* scale_mlp, const float* scale_prev, const mmae_block_params* p, void* saved,
                                     void* ws, void* st) {
  return block_forward_impl(x_in, reinterpret_cast<const bf16*>(x_add_bf16), x_sum, x_out, reinterpret_cast<bf16*>(y_out_bf16),
                            B, N, D, H, hidden, eps, scale_attn, scale_mlp, scale_prev, p, saved, ws, st);
}
extern "C" float* mmae_block_saved_x_mid(void* saved, int B, int N, int D, int H, int hidden) {
  return saved ? block_saved(saved, B, N, D, H, hidden).x_mid : nullptr;
}

// Chained form (mmae_block_backward_chain).  `dx_out_b` (bf16) != null: bf16(dx_out) made by the NEXT block's backward,
// which also added its column sums to this block's fc2 bias gradient: the cast + column-sum pass is skipped.
// `dx_in_b` (bf16) != null: the first LayerNorm's backward also writes bf16(dx_in) there and adds colsum(dx_in) to
// `dx_in_colsum` - the PREVIOUS block's fc2 bias gradient - for that block's backward to start from.
// Stochastic depth: the gradient entering a branch is s * (gradient of the residual stream), so s_mlp scales the MLP branch's
// bf16 operand and fc2 bias gradient, s_attn the proj operand and bias gradient that LN2's backward emits, s_prev what LN1's
// backward hands to the previous block.  The fp32 residual-path gradients (dx_mid, dx_in) are never scaled.
static int block_backward_impl(const float* x_in, const float* dx_out, const bf16* dx_out_b, float* dx_in, bf16* dx_in_b,
                               float* dx_in_colsum, int B, int N, int D, int H, int hidden, const float* s_attn,
                               const float* s_mlp, const float* s_prev, const mmae_block_params* p,
                               const mmae_block_grads* g, const void* saved, void* ws, void* st) {
  MMAE_CHECK(x_in && dx_out && dx_in && (!dx_in_b || dx_in_colsum) && p && g && saved && ws, MMAE_ERR_ARG,
             "mmae_block_backward: bad args");
  MMAE_CHECK(!s_prev || dx_in_b, MMAE_ERR_ARG, "mmae_block_backward_dp: the previous block's scale needs dx_in_bf16");
  const int M = B * N, dh = D / H;
  BlockSaved s = block_saved(const_cast<void*>(saved), B, N, D, H, hidden);
  RUN(weight_operand(p->qkv_w, &s.wqkv, 0, false, st));
  RUN(weight_operand(p->proj_w, &s.wproj, 0, false, st));
  RUN(weight_operand(p->fc1_w, &s.w1, 0, false, st));
  RUN(weight_operand(p->fc2_w, &s.w2, 0, false, st));
  BlockWs w = block_ws(ws, B, N, D, H, hidden);
  const bool side = side_ready();
  void* ws_st = side ? static_cast<void*>(g_side.stream) : st;   // stream of the weight-gradient GEMMs
  bf16* g2 = side ? w.g2 : w.g;
  bf16* dqkv = side ? w.big2 : w.big;
  // ---- MLP branch
  const bf16* gout = dx_out_b;
  if (!gout) {
    RUN(cast_colsum_f32_scaled(dx_out, D, w.g, D, g->fc2_b, s_mlp, N, M, D, st));
    gout = w.g;
  }
  if (side) RUN(side_fork(st, 0));
  RUN(wgrad(gout, D, s.a, hidden, g->fc2_w, M, D, hidden, ws_st));
  RUN(dgrad_dgelu_colsum(gout, D, s.w2, s.z, w.big, g->fc1_b, M, D, hidden, st));   // dz = (g W2) * gelu'(z); db1
  if (side) RUN(side_fork(st, 1));
  RUN(wgrad(w.big, hidden, s.h2, D, g->fc1_w, M, hidden, D, ws_st));
  RUN(dgrad_bf16(w.big, hidden, s.w1, nullptr, w.dh, M, hidden, D, st));
  // LN2 backward also emits bf16(dx_mid) and its column sums = operand and bias gradient of the proj backward
  RUN(layernorm_backward_ex_scaled(w.dh, 1, D, s.x_mid, D, s.mean2, s.rstd2, p->norm2_w, dx_out, D, w.dx_mid, D, g->norm2_w,
                                   g->norm2_b, g2, D, g->proj_b, s_attn, N, M, D, st));
  // ---- attention branch
  if (side) RUN(side_fork(st, 2));
  RUN(wgrad(g2, D, s.o, D, g->proj_w, M, D, D, ws_st));
  RUN(dgrad_bf16(g2, D, s.wproj, nullptr, w.d_o, M, D, D, st));
  RUN(mmae_attention_backward(s.qkv, 3 * D, s.qkv + D, 3 * D, s.qkv + 2 * D, 3 * D, s.o, D, w.d_o, D, s.lse, w.delta,
                              dqkv, 3 * D, dqkv + D, 3 * D, dqkv + 2 * D, 3 * D, B, H, N, N, dh,
                              1.0f / sqrtf((float)dh), st));
  RUN(mmae_colsum_bf16(dqkv, 3 * D, g->qkv_b, M, 3 * D, st));
  if (side) RUN(side_fork(st, 3));
  RUN(wgrad(dqkv, 3 * D, s.h1, D, g->qkv_w, M, 3 * D, D, ws_st));
  RUN(dgrad_bf16(dqkv, 3 * D, s.wqkv, nullptr, w.dh, M, 3 * D, D, st));
  if (dx_in_b)
    RUN(layernorm_backward_ex_scaled(w.dh, 1, D, x_in, D, s.mean1, s.rstd1, p->norm1_w, w.dx_mid, D, dx_in, D, g->norm1_w,
                                     g->norm1_b, dx_in_b, D, dx_in_colsum, s_prev, N, M, D, st));
  else
    RUN(mmae_layernorm_backward(w.dh, 1, D, x_in, D, s.mean1, s.rstd1, p->norm1_w, w.dx_mid, D, dx_in, D, g->norm1_w,
                                g->norm1_b, M, D, st));
  if (side) RUN(side_join(st));   // the caller sees every gradient of this block in stream order
  return MMAE_OK;
}

extern "C" int mmae_block_backward(const float* x_in, const float* dx_out, float* dx_in, int B, int N, int D, int H,
                                   int hidden, const mmae_block_params* p, const mmae_block_grads* g, const void* saved,
                                   void* ws, void* st) {
  return block_backward_impl(x_in, dx_out, nullptr, dx_in, nullptr, nullptr, B, N, D, H, hidden, nullptr, nullptr, nullptr, p,
                             g, saved, ws, st);
}
extern "C" int mmae_block_backward_chain(const float* x_in, const float* dx_out, const void* dx_out_bf16, float* dx_in,
                                         void* dx_in_bf16, float* dx_in_colsum, int B, int N, int D, int H, int hidden,
                                         const mmae_block_params* p, const mmae_block_grads* g, const void* saved, void* ws,
                                         void* st) {
  return block_backward_impl(x_in, dx_out, reinterpret_cast<const bf16*>(dx_out_bf16), dx_in,
                             reinterpret_cast<bf16*>(dx_in_bf16), dx_in_colsum, B, N, D, H, hidden, nullptr, nullptr, nullptr,
                             p, g, saved, ws, st);
}
extern "C" int mmae_block_backward_dp(const float* x_in, const float* dx_out, const void* dx_out_bf16, float* dx_in,
                                      void* dx_in_bf16, float* dx_in_colsum, int B, int N, int D, int H, int hidden,
                                      const float* scale_attn, const float* scale_mlp, const float* scale_prev,
                                      const mmae_block_params* p, const mmae_block_grads* g, const void* saved, void* ws,
                                      void* st) {
  return block_backward_impl(x_in, dx_out, reinterpret_cast<const bf16*>(dx_out_bf16), dx_in,
                             reinterpret_cast<bf16*>(dx_in_bf16), dx_in_colsum, B, N, D, H, hidden, scale_attn, scale_mlp,
                             scale_prev, p, g, saved, ws, st);
}

extern "C" int mmae_set_wgrad_stream(int enable) {
  g_wgrad_stream = enable != 0;
  return MMAE_OK;
}

// ================================================================================================ decoder head
extern "C" int64_t mmae_dechead_saved_bytes(const mmae_decoder_index* ix, int D_enc, int H, int hidden) {
  return (int64_t)head_saved(nullptr, *ix, D_enc, H, hidden).bytes;
}
extern "C" int64_t mmae_dechead_workspace_bytes(const mmae_decoder_index* ix, int D_enc, int H, int hidden) {
  return (int64_t)head_ws(nullptr, *ix, D_enc, H, hidden).bytes;
}

// `ctx_ext` != null: the context projection was done by mmae_ctxproj_forward for all adapters at once; this head reads
// its [Mc, Dd] column segment (row stride ld_ctx floats) and De is 0 (no enc_b / proj_context operand slots in `saved`).
static int dechead_forward_impl(const float* enc, const float* ctx_ext, int64_t ld_ctx, int De,
                                const mmae_decoder_index* ixp, int H, int hidden, float eps, const mmae_dechead_params* p,
                                float* x_out, void* saved, void* ws, void* st) {
  MMAE_CHECK((enc || ctx_ext) && ixp && p && x_out && saved && ws, MMAE_ERR_ARG, "mmae_dechead_forward: bad args");
  MMAE_CHECK(!ctx_ext || (ld_ctx % 4 == 0 && (reinterpret_cast<uintptr_t>(ctx_ext) & 15) == 0), MMAE_ERR_ARG,
             "mmae_dechead_forward_ctx: the context segment must be 16-byte aligned with a row stride that is a multiple of 4");
  const mmae_decoder_index& ix = *ixp;
  const int Dd = ix.dim, B = ix.batch, P = ix.num_queries, Nc = ix.num_visible + ix.num_global;
  MMAE_CHECK(Dd % H == 0 && ix.num_tasks <= MMAE_MAX_TASKS &&
                 ((ix.query_mode == 0 && ix.own_task >= 0 && ix.own_task < ix.num_tasks) ||
                  (ix.query_mode == 1 && ix.own_task >= -1 && ix.own_task <= ix.num_tasks && ix.own_task < MMAE_MAX_TASKS)),
             MMAE_ERR_ARG, "mmae_dechead_forward: bad decoder index");
  MMAE_CHECK(ix.own_task < 0 || p->task_emb[ix.own_task] != nullptr || ix.query_mode == 0, MMAE_ERR_ARG,
             "mmae_dechead_forward: query task embedding slot %d is empty", ix.own_task);
  const int Mq = B * P, Mc = B * Nc, dh = Dd / H;
  HeadSaved s = head_saved(saved, ix, De, H, hidden);
  HeadWs w = head_ws(ws, ix, De, H, hidden);
  cudaStream_t cst = reinterpret_cast<cudaStream_t>(st);
  if (!ctx_ext) {
    RUN(mmae_cast_f32_to_bf16(enc, s.enc_b, int64_t(Mc) * De, st));
    RUN(weight_operand(p->proj_context_w, &s.wpc, int64_t(Dd) * De, true, st));
  }
  RUN(weight_operand(p->q_w, &s.wq, int64_t(Dd) * Dd, true, st));
  RUN(weight_operand(p->kv_w, &s.wkv, int64_t(2) * Dd * Dd, true, st));
  RUN(weight_operand(p->proj_w, &s.wproj, int64_t(Dd) * Dd, true, st));
  RUN(weight_operand(p->fc1_w, &s.w1, int64_t(hidden) * Dd, true, st));
  RUN(weight_operand(p->fc2_w, &s.w2, int64_t(Dd) * hidden, true, st));
  // proj_context                                                   output_adapters.py:258
  if (!ctx_ext) RUN(linear_f32(s.enc_b, s.wpc, p->proj_context_b, nullptr, w.ctx, Mc, Dd, De, st));
  // queries / context                                              output_adapters.py:183-234
  TaskEmbPtrs te;
  for (int t = 0; t < MMAE_MAX_TASKS; ++t) te.p[t] = p->task_emb[t];
  RUN(launch_dec_build(ctx_ext ? ctx_ext : w.ctx, ctx_ext ? ld_ctx : int64_t(Dd), ix, p->mask_token, te, p->pos, s.queries,
                       s.context, cst));
  // decoder(query_norm(q), context_norm(c))                        output_adapters.py:265
  RUN(mmae_layernorm_forward(s.queries, Dd, p->query_norm_w, p->query_norm_b, s.qn, Dd, nullptr, 0, s.qmean, s.qrstd, Mq,
                             Dd, eps, st));
  RUN(mmae_layernorm_forward(s.context, Dd, p->context_norm_w, p->context_norm_b, s.cn, Dd, nullptr, 0, s.cmean, s.crstd,
                             Mc, Dd, eps, st));
  RUN(linear_bf16(s.qn, s.wq, p->q_b, s.q, Mq, Dd, Dd, st));
  RUN(linear_bf16(s.cn, s.wkv, p->kv_b, s.kv, Mc, 2 * Dd, Dd, st));
  RUN(mmae_attention_forward(s.q, Dd, s.kv, 2 * Dd, s.kv + Dd, 2 * Dd, s.o, Dd, s.lse, B, H, P, Nc, dh,
                             1.0f / sqrtf((float)dh), st));
  RUN(linear_f32(s.o, s.wproj, p->proj_b, nullptr, s.x0, Mq, Dd, Dd, st));
  // x = x + mlp(out_norm(x))                                       output_adapters.py:266
  RUN(mmae_layernorm_forward(s.x0, Dd, p->out_norm_w, p->out_norm_b, s.h, Dd, nullptr, 0, s.omean, s.orstd, Mq, Dd, eps,
                             st));
  RUN(linear_gelu(s.h, s.w1, p->fc1_b, s.z, s.a, Mq, hidden, Dd, st));
  RUN(linear_bf16(s.a, s.w2, p->fc2_b, w.g, Mq, Dd, hidden, st));          // bf16 branch output, add outside the epilogue
  RUN(mmae_add_bf16_f32(s.x0, w.g, x_out, int64_t(Mq) * Dd, st));
  return MMAE_OK;
}

extern "C" int mmae_dechead_forward(const float* enc, int De, const mmae_decoder_index* ixp, int H, int hidden, float eps,
                                    const mmae_dechead_params* p, float* x_out, void* saved, void* ws, void* st) {
  MMAE_CHECK(enc && De > 0, MMAE_ERR_ARG, "mmae_dechead_forward: bad args");
  return dechead_forward_impl(enc, nullptr, 0, De, ixp, H, hidden, eps, p, x_out, saved, ws, st);
}
extern "C" int mmae_dechead_forward_ctx(const float* ctx, int64_t ld_ctx, const mmae_decoder_index* ixp, int H, int hidden,
                                        float eps, const mmae_dechead_params* p, float* x_out, void* saved, void* ws,
                                        void* st) {
  MMAE_CHECK(ctx, MMAE_ERR_ARG, "mmae_dechead_forward_ctx: bad args");
  return dechead_forward_impl(nullptr, ctx, ld_ctx, 0, ixp, H, hidden, eps, p, x_out, saved, ws, st);
}

// `dctx_ext` != null: the bf16 context gradient goes to the adapter's column segment of the shared [Mc, sum Dd] matrix
// (row stride ld_dctx) and the proj_context weight / encoder-output gradients are left to mmae_ctxproj_backward.
static int dechead_backward_impl(int De, const mmae_decoder_index* ixp, int H, int hidden, const mmae_dechead_params* p,
                                 const mmae_dechead_grads* g, const float* dx_out, float* denc, void* dctx_ext,
                                 int64_t ld_dctx, const void* saved, void* ws, void* st) {
  MMAE_CHECK(ixp && p && g && dx_out && (denc || dctx_ext) && saved && ws, MMAE_ERR_ARG, "mmae_dechead_backward: bad args");
  MMAE_CHECK(!dctx_ext || (ld_dctx % 8 == 0 && (reinterpret_cast<uintptr_t>(dctx_ext) & 15) == 0), MMAE_ERR_ARG,
             "mmae_dechead_backward_ctx: the gradient segment must be 16-byte aligned with a row stride that is a multiple of 8");
  const mmae_decoder_index& ix = *ixp;
  const int Dd = ix.dim, B = ix.batch, P = ix.num_queries, Nc = ix.num_visible + ix.num_global;
  const int Mq = B * P, Mc = B * Nc, dh = Dd / H;
  HeadSaved s = head_saved(const_cast<void*>(saved), ix, De, H, hidden);
  if (!dctx_ext) RUN(weight_operand(p->proj_context_w, &s.wpc, 0, false, st));
  RUN(weight_operand(p->q_w, &s.wq, 0, false, st));
  RUN(weight_operand(p->kv_w, &s.wkv, 0, false, st));
  RUN(weight_operand(p->proj_w, &s.wproj, 0, false, st));
  RUN(weight_operand(p->fc1_w, &s.w1, 0, false, st));
  RUN(weight_operand(p->fc2_w, &s.w2, 0, false, st));
  HeadWs w = head_ws(ws, ix, De, H, hidden);
  cudaStream_t cst = reinterpret_cast<cudaStream_t>(st);
  // ---- MLP
  RUN(mmae_cast_colsum_f32(dx_out, Dd, w.g, Dd, g->fc2_b, Mq, Dd, st));
  RUN(dgrad_dgelu_colsum(w.g, Dd, s.w2, s.z, w.dz, g->fc1_b, Mq, Dd, hidden, st));
  RUN(wgrad(w.g, Dd, s.a, hidden, g->fc2_w, Mq, Dd, hidden, st));
  RUN(wgrad(w.dz, hidden, s.h, Dd, g->fc1_w, Mq, hidden, Dd, st));
  RUN(dgrad_bf16(w.dz, hidden, s.w1, nullptr, w.dh, Mq, hidden, Dd, st));
  RUN(mmae_layernorm_backward_ex(w.dh, 1, Dd, s.x0, Dd, s.omean, s.orstd, p->out_norm_w, dx_out, Dd, w.dx0, Dd,
                                 g->out_norm_w, g->out_norm_b, w.g, Dd, g->proj_b, Mq, Dd, st));
  // ---- cross attention (no residual around it)
  RUN(wgrad(w.g, Dd, s.o, Dd, g->proj_w, Mq, Dd, Dd, st));
  RUN(dgrad_bf16(w.g, Dd, s.wproj, nullptr, w.d_o, Mq, Dd, Dd, st));
  RUN(mmae_attention_backward(s.q, Dd, s.kv, 2 * Dd, s.kv + Dd, 2 * Dd, s.o, Dd, w.d_o, Dd, s.lse, w.delta, w.dq, Dd,
                              w.dkv, 2 * Dd, w.dkv + Dd, 2 * Dd, B, H, P, Nc, dh, 1.0f / sqrtf((float)dh), st));
  RUN(mmae_colsum_bf16(w.dq, Dd, g->q_b, Mq, Dd, st));
  RUN(wgrad(w.dq, Dd, s.qn, Dd, g->q_w, Mq, Dd, Dd, st));
  RUN(dgrad_bf16(w.dq, Dd, s.wq, nullptr, w.dqn, Mq, Dd, Dd, st));
  RUN(mmae_colsum_bf16(w.dkv, 2 * Dd, g->kv_b, Mc, 2 * Dd, st));
  RUN(wgrad(w.dkv, 2 * Dd, s.cn, Dd, g->kv_w, Mc, 2 * Dd, Dd, st));
  RUN(dgrad_bf16(w.dkv, 2 * Dd, s.wkv, nullptr, w.dcn, Mc, 2 * Dd, Dd, st));
  RUN(mmae_layernorm_backward(w.dqn, 1, Dd, s.queries, Dd, s.qmean, s.qrstd, p->query_norm_w, nullptr, 0, w.dqueries, Dd,
                              g->query_norm_w, g->query_norm_b, Mq, Dd, st));
  RUN(mmae_layernorm_backward(w.dcn, 1, Dd, s.context, Dd, s.cmean, s.crstd, p->context_norm_w, nullptr, 0, w.dcontext,
                              Dd, g->context_norm_w, g->context_norm_b, Mc, Dd, st));
  // ---- queries / context construction
  TaskEmbGradPtrs dte;
  for (int t = 0; t < MMAE_MAX_TASKS; ++t) dte.p[t] = g->task_emb[t];
  RUN(launch_dec_build_bwd(w.dqueries, w.dcontext, ix, w.dctx, g->mask_token, dte, cst));
  // ---- proj_context
  if (dctx_ext)   // bf16 cast into the shared matrix + the bias gradient; weight / encoder gradients: mmae_ctxproj_backward
    return mmae_cast_colsum_f32(w.dctx, Dd, dctx_ext, ld_dctx, g->proj_context_b, Mc, Dd, st);
  RUN(mmae_cast_colsum_f32(w.dctx, Dd, w.dctx_b, Dd, g->proj_context_b, Mc, Dd, st));
  RUN(wgrad(w.dctx_b, Dd, s.enc_b, De, g->proj_context_w, Mc, Dd, De, st));
  {
    mmae_gemm_epilogue ep = ep_zero();
    ep.accumulate = 1;
    ep.out_f32 = denc;
    ep.ld_out_f32 = De;
    RUN(mmae_gemm_bf16(w.dctx_b, Dd, 0, s.wpc, De, 1, Mc, De, Dd, 1, &ep, st));
  }
  return MMAE_OK;
}

extern "C" int mmae_dechead_backward(const float* enc, int De, const mmae_decoder_index* ixp, int H, int hidden,
                                     const mmae_dechead_params* p, const mmae_dechead_grads* g, const float* dx_out,
                                     float* denc, const void* saved, void* ws, void* st) {
  (void)enc;
  MMAE_CHECK(denc && De > 0, MMAE_ERR_ARG, "mmae_dechead_backward: bad args");
  return dechead_backward_impl(De, ixp, H, hidden, p, g, dx_out, denc, nullptr, 0, saved, ws, st);
}
extern "C" int mmae_dechead_backward_ctx(const mmae_decoder_index* ixp, int H, int hidden, const mmae_dechead_params* p,
                                         const mmae_dechead_grads* g, const float* dx_out, void* dctx_bf16,
                                         int64_t ld_dctx, const void* saved, void* ws, void* st) {
  MMAE_CHECK(dctx_bf16, MMAE_ERR_ARG, "mmae_dechead_backward_ctx: bad args");
  return dechead_backward_impl(0, ixp, H, hidden, p, g, dx_out, nullptr, dctx_bf16, ld_dctx, saved, ws, st);
}

// ============================================================================== shared context projection
// MultiMAE.forward hands the SAME encoder output to every output adapter (multimae/multimae.py:357-366) and each adapter
// starts with its own proj_context Linear (multimae/output_adapters.py:258).  Here the n Linears are one GEMM
//   ctx[rows, sum_i Dd_i] = bf16(enc)[rows, De] x Wcat[sum_i Dd_i, De]^T + bcat
// (one bf16 cast of enc instead of n; N = 1024 instead of four 256-column problems), and in backward
//   dWcat += dctx^T enc_b  (one K = rows GEMM)      denc = dctx Wcat  (one K = sum Dd GEMM, written - not n accumulated
// fp32 read-modify-write passes plus n zero fills and n-1 adds on the autograd side).
// Wcat / bcat / dWcat are used IN PLACE when the adapters' parameters (and their bf16 mirror, and their gradient slots)
// lie back to back - the flat arena orders them that way (functional.GradArena) - and are gathered otherwise.
namespace {
struct CtxSaved {
  bf16 *enc_b, *wcat;
  float* bcat;
  size_t bytes;
};
CtxSaved ctx_saved(void* base, int rows, int De, int Dsum) {
  Carver c(base);
  CtxSaved s;
  s.enc_b = c.take<bf16>(size_t(rows) * De);
  s.wcat = c.take<bf16>(size_t(Dsum) * De);
  s.bcat = c.take<float>(Dsum);
  s.bytes = align_up(c.off, 256);
  return s;
}
int ctx_dims_ok(const mmae_ctxproj_params* p, int* dsum) {
  if (!p || p->num < 1 || p->num > MMAE_MAX_TASKS) return 0;
  int tot = 0;
  for (int i = 0; i < p->num; ++i) {
    if (p->dim[i] <= 0 || p->dim[i] % 8 != 0 || !p->weight[i] || !p->bias[i]) return 0;
    tot += p->dim[i];
  }
  *dsum = tot;
  return 1;
}
// bf16 [Dsum, De] operand: the mirror in place when the n twins are adjacent, else gathered into s.wcat (fill = forward)
int ctx_weight_operand(const mmae_ctxproj_params* p, int De, const CtxSaved& s, bool fill, const bf16** out, void* st) {
  const bf16* m0 = mirror_lookup(p->weight[0]);
  bool inplace = m0 != nullptr;
  int64_t off = 0;
  for (int i = 0; i < p->num && inplace; ++i) {
    inplace = mirror_lookup(p->weight[i]) == m0 + off * De;
    off += p->dim[i];
  }
  if (inplace) {
    *out = m0;
    return MMAE_OK;
  }
  *out = s.wcat;
  if (!fill) return MMAE_OK;
  off = 0;
  for (int i = 0; i < p->num; ++i) {
    const int64_t n = int64_t(p->dim[i]) * De;
    if (const bf16* m = mirror_lookup(p->weight[i]))
      MMAE_CUDA_OK(cudaMemcpyAsync(s.wcat + off * De, m, n * sizeof(bf16), cudaMemcpyDeviceToDevice,
                                   reinterpret_cast<cudaStream_t>(st)));
    else
      RUN(mmae_cast_f32_to_bf16(p->weight[i], s.wcat + off * De, n, st));
    off += p->dim[i];
  }
  return MMAE_OK;
}
}  // namespace

extern "C" int64_t mmae_ctxproj_saved_bytes(int rows, int D_enc, int dim_total) {
  return (int64_t)ctx_saved(nullptr, rows, D_enc, dim_total).bytes;
}

extern "C" int mmae_ctxproj_forward(const float* enc, int rows, int De, const mmae_ctxproj_params* p, float* ctx,
                                    void* saved, void* st) {
  int Dsum = 0;
  MMAE_CHECK(enc && ctx && saved && rows > 0 && De > 0 && De % 8 == 0 && ctx_dims_ok(p, &Dsum), MMAE_ERR_ARG,
             "mmae_ctxproj_forward: bad args (1..%d adapters, dims multiples of 8)", MMAE_MAX_TASKS);
  CtxSaved s = ctx_saved(saved, rows, De, Dsum);
  RUN(mmae_cast_f32_to_bf16(enc, s.enc_b, int64_t(rows) * De, st));
  const bf16* W = nullptr;
  RUN(ctx_weight_operand(p, De, s, true, &W, st));
  const float* bias = p->bias[0];
  bool adjacent = true;
  int64_t off = 0;
  for (int i = 0; i < p->num; ++i) {
    adjacent = adjacent && p->bias[i] == p->bias[0] + off;
    off += p->dim[i];
  }
  if (!adjacent) {
    off = 0;
    for (int i = 0; i < p->num; ++i) {
      MMAE_CUDA_OK(cudaMemcpyAsync(s.bcat + off, p->bias[i], size_t(p->dim[i]) * sizeof(float), cudaMemcpyDeviceToDevice,
                                   reinterpret_cast<cudaStream_t>(st)));
      off += p->dim[i];
    }
    bias = s.bcat;
  }
  return linear_f32(s.enc_b, W, bias, nullptr, ctx, rows, Dsum, De, st);
}

extern "C" int mmae_ctxproj_backward(int rows, int De, const mmae_ctxproj_params* p, const mmae_ctxproj_grads* g,
                                     const void* dctx_bf16, float* denc, const void* saved, void* st) {
  int Dsum = 0;
  MMAE_CHECK(g && dctx_bf16 && denc && saved && rows > 0 && De > 0 && ctx_dims_ok(p, &Dsum), MMAE_ERR_ARG,
             "mmae_ctxproj_backward: bad args");
  for (int i = 0; i < p->num; ++i) MMAE_CHECK(g->weight[i], MMAE_ERR_ARG, "mmae_ctxproj_backward: null gradient slot %d", i);
  CtxSaved s = ctx_saved(const_cast<void*>(saved), rows, De, Dsum);
  const bf16* W = nullptr;
  RUN(ctx_weight_operand(p, De, s, false, &W, st));
  const bf16* dctx = reinterpret_cast<const bf16*>(dctx_bf16);
  bool adjacent = true;
  int64_t off = 0;
  for (int i = 0; i < p->num; ++i) {
    adjacent = adjacent && g->weight[i] == g->weight[0] + off * De;
    off += p->dim[i];
  }
  if (adjacent) {
    RUN(wgrad(dctx, Dsum, s.enc_b, De, g->weight[0], rows, Dsum, De, st));
  } else {
    off = 0;
    for (int i = 0; i < p->num; ++i) {
      RUN(wgrad(dctx + off, Dsum, s.enc_b, De, g->weight[i], rows, p->dim[i], De, st));
      off += p->dim[i];
    }
  }
  mmae_gemm_epilogue ep = ep_zero();
  ep.out_f32 = denc;
  ep.ld_out_f32 = De;
  return mmae_gemm_bf16(dctx, Dsum, 0, W, De, 1, rows, De, Dsum, 1, &ep, st);
}

// ================================================================================================ decoder tail
namespace {
struct TailSaved {
  bf16 *x_b, *w_b;
  size_t bytes;
};
TailSaved tail_saved(void* base, int B, int nh, int nw, int Dd, int C, int P) {
  Carver c(base);
  TailSaved s;
  s.x_b = c.take<bf16>(size_t(B) * nh * nw * Dd);
  s.w_b = c.take<bf16>(size_t(C) * P * P * Dd);
  s.bytes = align_up(c.off, 256);
  return s;
}
struct TailWs {
  bf16* y;
  bf16* dy;
  size_t bytes;
};
TailWs tail_ws(void* base, int B, int nh, int nw, int Dd, int C, int P) {
  (void)Dd;
  Carver c(base);
  TailWs w;
  w.y = c.take<bf16>(size_t(B) * nh * nw * C * P * P);
  w.dy = c.take<bf16>(size_t(B) * nh * nw * C * P * P);
  w.bytes = align_up(c.off, 256);
  return w;
}
}  // namespace

extern "C" int64_t mmae_dectail_saved_bytes(int B, int nh, int nw, int Dd, int C, int P) {
  return (int64_t)tail_saved(nullptr, B, nh, nw, Dd, C, P).bytes;
}
extern "C" int64_t mmae_dectail_workspace_bytes(int B, int nh, int nw, int Dd, int C, int P) {
  return (int64_t)tail_ws(nullptr, B, nh, nw, Dd, C, P).bytes;
}

extern "C" int mmae_dectail_forward(const float* x, int B, int nh, int nw, int Dd, int C, int P, const float* out_w,
                                    const float* out_b, float* pred, void* saved, void* ws, void* st) {
  MMAE_CHECK(x && out_w && out_b && pred && saved && ws, MMAE_ERR_ARG, "mmae_dectail_forward: bad args");
  const int M = B * nh * nw, Nout = C * P * P;
  TailSaved s = tail_saved(saved, B, nh, nw, Dd, C, P);
  TailWs w = tail_ws(ws, B, nh, nw, Dd, C, P);
  RUN(mmae_cast_f32_to_bf16(x, s.x_b, int64_t(M) * Dd, st));
  RUN(weight_operand(out_w, &s.w_b, int64_t(Nout) * Dd, true, st));
  RUN(linear_bf16(s.x_b, s.w_b, out_b, w.y, M, Nout, Dd, st));              // output_adapters.py:274 (half precision
  RUN(mmae_unpatchify_bf16(w.y, Nout, pred, B, C, nh, nw, P, st));          //  like the autocast Linear); :277-280
  return MMAE_OK;
}

extern "C" int mmae_dectail_backward(const float* dpred, int B, int nh, int nw, int Dd, int C, int P, const float* out_w,
                                     float* d_out_w, float* d_out_b, float* dx, const void* saved, void* ws, void* st) {
  MMAE_CHECK(dpred && out_w && d_out_w && d_out_b && dx && saved && ws, MMAE_ERR_ARG, "mmae_dectail_backward: bad args");
  const int M = B * nh * nw, Nout = C * P * P;
  TailSaved s = tail_saved(const_cast<void*>(saved), B, nh, nw, Dd, C, P);
  RUN(weight_operand(out_w, &s.w_b, 0, false, st));
  TailWs w = tail_ws(ws, B, nh, nw, Dd, C, P);
  RUN(mmae_patchify_bf16(dpred, w.dy, Nout, B, C, nh, nw, P, st));
  RUN(mmae_colsum_bf16(w.dy, Nout, d_out_b, M, Nout, st));
  RUN(wgrad(w.dy, Nout, s.x_b, Dd, d_out_w, M, Nout, Dd, st));
  {
    mmae_gemm_epilogue ep = ep_zero();
    ep.out_f32 = dx;
    ep.ld_out_f32 = Dd;
    RUN(mmae_gemm_bf16(w.dy, Nout, 0, s.w_b, Dd, 1, M, Dd, Nout, 1, &ep, st));
  }
  return MMAE_OK;
}

// ====================================================================================================== embed
extern "C" int64_t mmae_embed_saved_bytes(const mmae_embed_layout* L, int B, int T, int D) {
  (void)D;
  return (int64_t)embed_saved(nullptr, *L, B, T).bytes;
}
extern "C" int64_t mmae_embed_workspace_bytes(const mmae_embed_layout* L, int B, int T, int D) {
  return (int64_t)embed_ws(nullptr, *L, B, T, D).bytes;
}

extern "C" int mmae_embed_forward(const mmae_embed_layout* Lp, const mmae_embed_inputs* in, const mmae_embed_params* prm,
                                  const int64_t* ids_keep, int B, int T, int G, int D, float* x_out, void* saved, void* ws,
                                  void* st) {
  MMAE_CHECK(Lp && in && prm && ids_keep && x_out && saved && ws && B > 0 && T > 0 && G >= 0 && D % 8 == 0, MMAE_ERR_ARG,
             "mmae_embed_forward: bad args");
  const mmae_embed_layout& L = *Lp;
  MMAE_CHECK(L.num_tasks >= 1 && L.num_tasks <= MMAE_MAX_TASKS, MMAE_ERR_ARG, "mmae_embed_forward: bad task count");
  const int Kcat = L.k_offset[L.num_tasks];
  MMAE_CHECK(Kcat % 8 == 0, MMAE_ERR_UNSUPPORTED, "mmae_embed_forward: K segments must be multiples of 8");
  EmbedSaved s = embed_saved(saved, L, B, T);
  EmbedWs w = embed_ws(ws, L, B, T, D);
  cudaStream_t cst = reinterpret_cast<cudaStream_t>(st);
  for (int t = 0; t < L.num_tasks; ++t) {
    const int Kt = L.k_offset[t + 1] - L.k_offset[t];
    MMAE_CHECK(Kt % 8 == 0 && L.k_offset[t] % 8 == 0, MMAE_ERR_UNSUPPORTED, "mmae_embed_forward: K_t %% 8 != 0");
    RUN(launch_cast2d(prm->weight[t], Kt, w.Wcat + L.k_offset[t], Kcat, D, Kt, cst));
  }
  RUN(launch_embed_gather(L, *in, ids_keep, B, T, s.A, s.row_task, s.row_patch, cst));
  {
    mmae_gemm_epilogue ep = ep_zero();
    ep.out_f32 = w.Cmat;
    ep.ld_out_f32 = D;
    RUN(mmae_gemm_bf16(s.A, Kcat, 0, w.Wcat, Kcat, 0, B * T, D, Kcat, 1, &ep, st));
  }
  RUN(launch_embed_assemble(w.Cmat, *prm, s.row_task, s.row_patch, B, T, G, D, x_out, cst));
  return MMAE_OK;
}

extern "C" int mmae_embed_backward(const mmae_embed_layout* Lp, const mmae_embed_inputs* in, const mmae_embed_params* prm,
                                   const mmae_embed_grads* g, const int64_t* ids_keep, int B, int T, int G, int D,
                                   const float* dx, const void* saved, void* ws, void* st) {
  MMAE_CHECK(Lp && in && prm && g && ids_keep && dx && saved && ws, MMAE_ERR_ARG, "mmae_embed_backward: bad args");
  const mmae_embed_layout& L = *Lp;
  const int Kcat = L.k_offset[L.num_tasks];
  EmbedSaved s = embed_saved(const_cast<void*>(saved), L, B, T);
  EmbedWs w = embed_ws(ws, L, B, T, D);
  cudaStream_t cst = reinterpret_cast<cudaStream_t>(st);
  RUN(launch_embed_assemble_bwd(dx, B, T, G, D, s.row_task, w.dC, *g, L.num_tasks, cst));
  for (int t = 0; t < L.num_tasks; ++t) {
    const int Kt = L.k_offset[t + 1] - L.k_offset[t];
    // dW_t[D, K_t] += dC^T A_cat[:, segment t]      (rows of other tasks are zero in this segment)
    RUN(wgrad(w.dC, D, s.A + L.k_offset[t], Kcat, g->weight[t], B * T, D, Kt, st));
    if (L.is_semseg[t] && g->class_emb[t] != nullptr) {
      // dA = dC W_t  ->  scatter-add into the class-embedding table      input_adapters.py:229
      bf16* Wt = w.Wcat;  // reuse: [D, K_t] contiguous
      RUN(mmae_cast_f32_to_bf16(prm->weight[t], Wt, int64_t(D) * Kt, st));
      RUN(dgrad_bf16(w.dC, D, Wt, nullptr, w.dA, B * T, D, Kt, st));
      RUN(launch_semseg_emb_bwd(w.dA, Kt, reinterpret_cast<const int64_t*>(in->data[t]), ids_keep, s.row_task,
                                s.row_patch, t, T, B * T, L.grid_w[t], L.grid_h[t], L.patch[t], L.channels[t],
                                L.num_classes[t], g->class_emb[t], cst));
    }
  }
  return MMAE_OK;
}

extern "C" int mmae_set_fuse_gelu(int enable) {
  mmae::g_fuse_gelu = enable;
  return MMAE_OK;
}
