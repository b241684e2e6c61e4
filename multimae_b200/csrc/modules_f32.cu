// fp32 tier of the module-level entry points (Block, SpatialOutputAdapter head / tail) for the adapters listed in
// `fp32_output_adapters` (multimae/multimae.py:367-377 runs them outside autocast).  Same call sequence as modules.cu with
// every activation kept in fp32: Linear layers through the 3 x bf16 split GEMM (fp32_ops.cu), attention / GELU in fp32
// CUDA-core kernels, LayerNorm / index kernels are the fp32 ones both tiers share.  Roughly 3x the tensor-core work of the
// bf16 tier plus fp32 activations: an accuracy tier (1e-3 relative to the fp32 reference), not a fast path.
#include <cstdlib>

#include "internal.h"

namespace mmae {
int linear_f32x3_forward(const float* x, const float* W, const float* bias, const float* resid, float* y, int M, int N, int K,
                         bf16* wsA, bf16* wsB, void* st);
int linear_f32x3_dgrad(const float* dy, const float* W, float* dx, int M, int N, int K, int accumulate, bf16* wsA, bf16* wsB,
                       void* st);
int linear_f32x3_wgrad(const float* dy, const float* x, float* dW, float* db, int M, int N, int K, bf16* wsA, bf16* wsB, void* st);
int gelu_f32(const float* z, float* io, int64_t n, int backward, void* st);

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

#define RUN(expr)                    \
  do {                               \
    int _rc = (expr);                \
    if (_rc != MMAE_OK) return _rc;  \
  } while (0)

// split-operand scratch shared by every Linear of one module call: rows x widest feature dimension, three pieces
struct SplitWs {
  bf16 *A, *B;
};
size_t split_elems(size_t rows, size_t maxdim) { return 3 * std::max(rows, maxdim) * maxdim; }

// ------------------------------------------------------------------------------------------------------ block
struct BlockSavedF {
  float *h1, *qkv, *o, *x_mid, *h2, *z, *a, *mean1, *rstd1, *mean2, *rstd2, *lse;
  size_t bytes;
};
BlockSavedF block_saved_f(void* base, int B, int N, int D, int H, int hid) {
  Carver c(base);
  const size_t M = size_t(B) * N;
  BlockSavedF s;
  s.mean1 = c.take<float>(M);
  s.rstd1 = c.take<float>(M);
  s.mean2 = c.take<float>(M);
  s.rstd2 = c.take<float>(M);
  s.lse = c.take<float>(size_t(B) * H * N);
  s.h1 = c.take<float>(M * D);
  s.qkv = c.take<float>(M * 3 * D);
  s.o = c.take<float>(M * D);
  s.x_mid = c.take<float>(M * D);
  s.h2 = c.take<float>(M * D);
  s.z = c.take<float>(M * hid);
  s.a = c.take<float>(M * hid);
  s.bytes = align_up(c.off, 256);
  return s;
}
struct BlockWsF {
  SplitWs sp;
  float *big, *g, *dh, *d_o, *dx_mid, *delta;
  size_t bytes;
};
BlockWsF block_ws_f(void* base, int B, int N, int D, int H, int hid) {
  Carver c(base);
  const size_t M = size_t(B) * N, wide = std::max(hid, 3 * D);
  BlockWsF w;
  w.sp.A = c.take<bf16>(split_elems(M, wide));
  w.sp.B = c.take<bf16>(split_elems(M, wide));
  w.big = c.take<float>(M * wide);
  w.g = c.take<float>(M * D);
  w.dh = c.take<float>(M * D);
  w.d_o = c.take<float>(M * D);
  w.dx_mid = c.take<float>(M * D);
  w.delta = c.take<float>(size_t(B) * H * N);
  w.bytes = align_up(c.off, 256);
  return w;
}

// --------------------------------------------------------------------------------------------------- decoder head
struct HeadSavedF {
  float *queries, *context, *qn, *cn, *q, *kv, *o, *x0, *h, *z, *a;
  float *qmean, *qrstd, *cmean, *crstd, *omean, *orstd, *lse;
  size_t bytes;
};
HeadSavedF head_saved_f(void* base, const mmae_decoder_index& ix, int H, int hid) {
  Carver c(base);
  const size_t Dd = ix.dim, Mq = size_t(ix.batch) * ix.num_queries, Mc = size_t(ix.batch) * (ix.num_visible + ix.num_global);
  HeadSavedF s;
  s.qmean = c.take<float>(Mq);
  s.qrstd = c.take<float>(Mq);
  s.cmean = c.take<float>(Mc);
  s.crstd = c.take<float>(Mc);
  s.omean = c.take<float>(Mq);
  s.orstd = c.take<float>(Mq);
  s.lse = c.take<float>(size_t(ix.batch) * H * ix.num_queries);
  s.queries = c.take<float>(Mq * Dd);
  s.context = c.take<float>(Mc * Dd);
  s.qn = c.take<float>(Mq * Dd);
  s.cn = c.take<float>(Mc * Dd);
  s.q = c.take<float>(Mq * Dd);
  s.kv = c.take<float>(Mc * 2 * Dd);
  s.o = c.take<float>(Mq * Dd);
  s.x0 = c.take<float>(Mq * Dd);
  s.h = c.take<float>(Mq * Dd);
  s.z = c.take<float>(Mq * hid);
  s.a = c.take<float>(Mq * hid);
  s.bytes = align_up(c.off, 256);
  return s;
}
struct HeadWsF {
  SplitWs sp;
  float *ctx, *dz, *dh, *dx0, *d_o, *dq, *dkv, *dqn, *dcn, *dqueries, *dcontext, *dctx, *delta;
  size_t bytes;
};
HeadWsF head_ws_f(void* base, const mmae_decoder_index& ix, int De, int H, int hid) {
  Carver c(base);
  const size_t Dd = ix.dim, Mq = size_t(ix.batch) * ix.num_queries, Mc = size_t(ix.batch) * (ix.num_visible + ix.num_global);
  const size_t wide = std::max<size_t>(std::max<size_t>(hid, De), 2 * Dd), rows = std::max(Mq, Mc);
  HeadWsF w;
  w.sp.A = c.take<bf16>(split_elems(rows, wide));
  w.sp.B = c.take<bf16>(split_elems(rows, wide));
  w.ctx = c.take<float>(Mc * Dd);
  w.dz = c.take<float>(Mq * hid);
  w.dh = c.take<float>(Mq * Dd);
  w.dx0 = c.take<float>(Mq * Dd);
  w.d_o = c.take<float>(Mq * Dd);
  w.dq = c.take<float>(Mq * Dd);
  w.dkv = c.take<float>(Mc * 2 * Dd);
  w.dqn = c.take<float>(Mq * Dd);
  w.dcn = c.take<float>(Mc * Dd);
  w.dqueries = c.take<float>(Mq * Dd);
  w.dcontext = c.take<float>(Mc * Dd);
  w.dctx = c.take<float>(Mc * Dd);
  w.delta = c.take<float>(size_t(ix.batch) * H * ix.num_queries);
  w.bytes = align_up(c.off, 256);
  return w;
}

struct TailWsF {
  SplitWs sp;
  float *y, *dy;
  size_t bytes;
};
TailWsF tail_ws_f(void* base, int B, int nh, int nw, int Dd, int C, int P) {
  Carver c(base);
  const size_t M = size_t(B) * nh * nw, Nout = size_t(C) * P * P, wide = std::max<size_t>(Nout, Dd);
  TailWsF w;
  w.sp.A = c.take<bf16>(split_elems(M, wide));
  w.sp.B = c.take<bf16>(split_elems(M, wide));
  w.y = c.take<float>(M * Nout);
  w.dy = c.take<float>(M * Nout);
  w.bytes = align_up(c.off, 256);
  return w;
}

}  // namespace
}  // namespace mmae

using namespace mmae;

// ====================================================================================================== block
extern "C" int64_t mmae_block_f32_saved_bytes(int B, int N, int D, int H, int hidden) {
  return (int64_t)block_saved_f(nullptr, B, N, D, H, hidden).bytes;
}
extern "C" int64_t mmae_block_f32_workspace_bytes(int B, int N, int D, int H, int hidden) {
  return (int64_t)block_ws_f(nullptr, B, N, D, H, hidden).bytes;
}

// Stochastic depth: s_attn / s_mlp [B] (null: factor 1) multiply each sample's attention / MLP branch.  With a factor the
// branch GEMM writes the branch alone (w.g, unused otherwise in forward) and a row-scaled add forms the residual sum.
extern "C" int mmae_block_f32_forward(const float* x_in, float* x_out, int B, int N, int D, int H, int hidden, float eps,
                                      const float* s_attn, const float* s_mlp, const mmae_block_params* p, void* saved,
                                      void* ws, void* st) {
  MMAE_CHECK(x_in && x_out && p && saved && ws && B > 0 && N > 0 && H > 0 && D % H == 0, MMAE_ERR_ARG, "mmae_block_f32_forward: bad args");
  const int M = B * N, dh = D / H;
  const int64_t MD = int64_t(M) * D, ND = int64_t(N) * D;
  BlockSavedF s = block_saved_f(saved, B, N, D, H, hidden);
  BlockWsF w = block_ws_f(ws, B, N, D, H, hidden);
  // x = x + attn(norm1(x))                                        multimae_utils.py:230
  RUN(mmae_layernorm_forward(x_in, D, p->norm1_w, p->norm1_b, nullptr, 0, s.h1, D, s.mean1, s.rstd1, M, D, eps, st));
  RUN(linear_f32x3_forward(s.h1, p->qkv_w, p->qkv_b, nullptr, s.qkv, M, 3 * D, D, w.sp.A, w.sp.B, st));
  RUN(mmae_attention_f32_forward(s.qkv, 3 * D, s.qkv + D, 3 * D, s.qkv + 2 * D, 3 * D, s.o, D, s.lse, B, H, N, N, dh,
                                 1.0f / sqrtf((float)dh), st));
  if (s_attn) {
    RUN(linear_f32x3_forward(s.o, p->proj_w, p->proj_b, nullptr, w.g, M, D, D, w.sp.A, w.sp.B, st));
    RUN(add_scaled_f32(x_in, w.g, 0, s_attn, ND, s.x_mid, MD, st));
  } else {
    RUN(linear_f32x3_forward(s.o, p->proj_w, p->proj_b, x_in, s.x_mid, M, D, D, w.sp.A, w.sp.B, st));
  }
  // x = x + mlp(norm2(x))                                         multimae_utils.py:231
  RUN(mmae_layernorm_forward(s.x_mid, D, p->norm2_w, p->norm2_b, nullptr, 0, s.h2, D, s.mean2, s.rstd2, M, D, eps, st));
  RUN(linear_f32x3_forward(s.h2, p->fc1_w, p->fc1_b, nullptr, s.z, M, hidden, D, w.sp.A, w.sp.B, st));
  RUN(gelu_f32(s.z, s.a, int64_t(M) * hidden, 0, st));
  if (s_mlp) {
    RUN(linear_f32x3_forward(s.a, p->fc2_w, p->fc2_b, nullptr, w.g, M, D, hidden, w.sp.A, w.sp.B, st));
    return add_scaled_f32(s.x_mid, w.g, 0, s_mlp, ND, x_out, MD, st);
  }
  RUN(linear_f32x3_forward(s.a, p->fc2_w, p->fc2_b, s.x_mid, x_out, M, D, hidden, w.sp.A, w.sp.B, st));
  return MMAE_OK;
}

// Backward with factors: the branch's weight / input gradients are taken from a row-scaled copy of the residual-stream
// gradient (w.g, unused otherwise in backward); the residual path itself carries the unscaled gradient.
extern "C" int mmae_block_f32_backward(const float* x_in, const float* dx_out, float* dx_in, int B, int N, int D, int H,
                                       int hidden, const float* s_attn, const float* s_mlp, const mmae_block_params* p,
                                       const mmae_block_grads* g, const void* saved, void* ws, void* st) {
  MMAE_CHECK(x_in && dx_out && dx_in && p && g && saved && ws, MMAE_ERR_ARG, "mmae_block_f32_backward: bad args");
  const int M = B * N, dh = D / H;
  const int64_t MD = int64_t(M) * D, ND = int64_t(N) * D;
  BlockSavedF s = block_saved_f(const_cast<void*>(saved), B, N, D, H, hidden);
  BlockWsF w = block_ws_f(ws, B, N, D, H, hidden);
  // ---- MLP branch
  const float* g_mlp = dx_out;
  if (s_mlp) {
    RUN(add_scaled_f32(nullptr, dx_out, 0, s_mlp, ND, w.g, MD, st));
    g_mlp = w.g;
  }
  RUN(linear_f32x3_wgrad(g_mlp, s.a, g->fc2_w, g->fc2_b, M, D, hidden, w.sp.A, w.sp.B, st));
  RUN(linear_f32x3_dgrad(g_mlp, p->fc2_w, w.big, M, D, hidden, 0, w.sp.A, w.sp.B, st));         // d a  [M, hidden]
  RUN(gelu_f32(s.z, w.big, int64_t(M) * hidden, 1, st));                                          // dz = da * gelu'(z)
  RUN(linear_f32x3_wgrad(w.big, s.h2, g->fc1_w, g->fc1_b, M, hidden, D, w.sp.A, w.sp.B, st));
  RUN(linear_f32x3_dgrad(w.big, p->fc1_w, w.dh, M, hidden, D, 0, w.sp.A, w.sp.B, st));
  RUN(mmae_layernorm_backward(w.dh, 0, D, s.x_mid, D, s.mean2, s.rstd2, p->norm2_w, dx_out, D, w.dx_mid, D, g->norm2_w,
                              g->norm2_b, M, D, st));
  // ---- attention branch
  const float* g_attn = w.dx_mid;
  if (s_attn) {
    RUN(add_scaled_f32(nullptr, w.dx_mid, 0, s_attn, ND, w.g, MD, st));
    g_attn = w.g;
  }
  RUN(linear_f32x3_wgrad(g_attn, s.o, g->proj_w, g->proj_b, M, D, D, w.sp.A, w.sp.B, st));
  RUN(linear_f32x3_dgrad(g_attn, p->proj_w, w.d_o, M, D, D, 0, w.sp.A, w.sp.B, st));
  RUN(mmae_attention_f32_backward(s.qkv, 3 * D, s.qkv + D, 3 * D, s.qkv + 2 * D, 3 * D, s.o, D, w.d_o, D, s.lse, w.delta, w.big,
                                  3 * D, w.big + D, 3 * D, w.big + 2 * D, 3 * D, B, H, N, N, dh, 1.0f / sqrtf((float)dh), st));
  RUN(linear_f32x3_wgrad(w.big, s.h1, g->qkv_w, g->qkv_b, M, 3 * D, D, w.sp.A, w.sp.B, st));
  RUN(linear_f32x3_dgrad(w.big, p->qkv_w, w.dh, M, 3 * D, D, 0, w.sp.A, w.sp.B, st));
  RUN(mmae_layernorm_backward(w.dh, 0, D, x_in, D, s.mean1, s.rstd1, p->norm1_w, w.dx_mid, D, dx_in, D, g->norm1_w,
                              g->norm1_b, M, D, st));
  return MMAE_OK;
}

// ================================================================================================ decoder head
extern "C" int64_t mmae_dechead_f32_saved_bytes(const mmae_decoder_index* ix, int D_enc, int H, int hidden) {
  (void)D_enc;
  return (int64_t)head_saved_f(nullptr, *ix, H, hidden).bytes;
}
extern "C" int64_t mmae_dechead_f32_workspace_bytes(const mmae_decoder_index* ix, int D_enc, int H, int hidden) {
  return (int64_t)head_ws_f(nullptr, *ix, D_enc, H, hidden).bytes;
}

extern "C" int mmae_dechead_f32_forward(const float* enc, int De, const mmae_decoder_index* ixp, int H, int hidden, float eps,
                                        const mmae_dechead_params* p, float* x_out, void* saved, void* ws, void* st) {
  MMAE_CHECK(enc && ixp && p && x_out && saved && ws, MMAE_ERR_ARG, "mmae_dechead_f32_forward: bad args");
  const mmae_decoder_index& ix = *ixp;
  const int Dd = ix.dim, B = ix.batch, P = ix.num_queries, Nc = ix.num_visible + ix.num_global;
  MMAE_CHECK(Dd % H == 0 && ix.num_tasks <= MMAE_MAX_TASKS, MMAE_ERR_ARG, "mmae_dechead_f32_forward: bad decoder index");
  const int Mq = B * P, Mc = B * Nc, dh = Dd / H;
  HeadSavedF s = head_saved_f(saved, ix, H, hidden);
  HeadWsF w = head_ws_f(ws, ix, De, H, hidden);
  cudaStream_t cst = reinterpret_cast<cudaStream_t>(st);
  RUN(linear_f32x3_forward(enc, p->proj_context_w, p->proj_context_b, nullptr, w.ctx, Mc, Dd, De, w.sp.A, w.sp.B, st));   // output_adapters.py:258
  TaskEmbPtrs te;
  for (int t = 0; t < MMAE_MAX_TASKS; ++t) te.p[t] = p->task_emb[t];
  RUN(launch_dec_build(w.ctx, ix.dim, ix, p->mask_token, te, p->pos, s.queries, s.context, cst));                               // :183-234
  RUN(mmae_layernorm_forward(s.queries, Dd, p->query_norm_w, p->query_norm_b, nullptr, 0, s.qn, Dd, s.qmean, s.qrstd, Mq, Dd, eps, st));
  RUN(mmae_layernorm_forward(s.context, Dd, p->context_norm_w, p->context_norm_b, nullptr, 0, s.cn, Dd, s.cmean, s.crstd, Mc, Dd, eps, st));
  RUN(linear_f32x3_forward(s.qn, p->q_w, p->q_b, nullptr, s.q, Mq, Dd, Dd, w.sp.A, w.sp.B, st));
  RUN(linear_f32x3_forward(s.cn, p->kv_w, p->kv_b, nullptr, s.kv, Mc, 2 * Dd, Dd, w.sp.A, w.sp.B, st));
  RUN(mmae_attention_f32_forward(s.q, Dd, s.kv, 2 * Dd, s.kv + Dd, 2 * Dd, s.o, Dd, s.lse, B, H, P, Nc, dh, 1.0f / sqrtf((float)dh), st));
  RUN(linear_f32x3_forward(s.o, p->proj_w, p->proj_b, nullptr, s.x0, Mq, Dd, Dd, w.sp.A, w.sp.B, st));                       // :265
  RUN(mmae_layernorm_forward(s.x0, Dd, p->out_norm_w, p->out_norm_b, nullptr, 0, s.h, Dd, s.omean, s.orstd, Mq, Dd, eps, st));
  RUN(linear_f32x3_forward(s.h, p->fc1_w, p->fc1_b, nullptr, s.z, Mq, hidden, Dd, w.sp.A, w.sp.B, st));
  RUN(gelu_f32(s.z, s.a, int64_t(Mq) * hidden, 0, st));
  RUN(linear_f32x3_forward(s.a, p->fc2_w, p->fc2_b, s.x0, x_out, Mq, Dd, hidden, w.sp.A, w.sp.B, st));                      // :266
  return MMAE_OK;
}

extern "C" int mmae_dechead_f32_backward(const float* enc, int De, const mmae_decoder_index* ixp, int H, int hidden,
                                         const mmae_dechead_params* p, const mmae_dechead_grads* g, const float* dx_out, float* denc,
                                         const void* saved, void* ws, void* st) {
  MMAE_CHECK(enc && ixp && p && g && dx_out && denc && saved && ws, MMAE_ERR_ARG, "mmae_dechead_f32_backward: bad args");
  const mmae_decoder_index& ix = *ixp;
  const int Dd = ix.dim, B = ix.batch, P = ix.num_queries, Nc = ix.num_visible + ix.num_global;
  const int Mq = B * P, Mc = B * Nc, dh = Dd / H;
  HeadSavedF s = head_saved_f(const_cast<void*>(saved), ix, H, hidden);
  HeadWsF w = head_ws_f(ws, ix, De, H, hidden);
  cudaStream_t cst = reinterpret_cast<cudaStream_t>(st);
  // ---- MLP
  RUN(linear_f32x3_wgrad(dx_out, s.a, g->fc2_w, g->fc2_b, Mq, Dd, hidden, w.sp.A, w.sp.B, st));
  RUN(linear_f32x3_dgrad(dx_out, p->fc2_w, w.dz, Mq, Dd, hidden, 0, w.sp.A, w.sp.B, st));
  RUN(gelu_f32(s.z, w.dz, int64_t(Mq) * hidden, 1, st));
  RUN(linear_f32x3_wgrad(w.dz, s.h, g->fc1_w, g->fc1_b, Mq, hidden, Dd, w.sp.A, w.sp.B, st));
  RUN(linear_f32x3_dgrad(w.dz, p->fc1_w, w.dh, Mq, hidden, Dd, 0, w.sp.A, w.sp.B, st));
  RUN(mmae_layernorm_backward(w.dh, 0, Dd, s.x0, Dd, s.omean, s.orstd, p->out_norm_w, dx_out, Dd, w.dx0, Dd, g->out_norm_w,
                              g->out_norm_b, Mq, Dd, st));
  // ---- cross attention (no residual around it)
  RUN(linear_f32x3_wgrad(w.dx0, s.o, g->proj_w, g->proj_b, Mq, Dd, Dd, w.sp.A, w.sp.B, st));
  RUN(linear_f32x3_dgrad(w.dx0, p->proj_w, w.d_o, Mq, Dd, Dd, 0, w.sp.A, w.sp.B, st));
  RUN(mmae_attention_f32_backward(s.q, Dd, s.kv, 2 * Dd, s.kv + Dd, 2 * Dd, s.o, Dd, w.d_o, Dd, s.lse, w.delta, w.dq, Dd, w.dkv,
                                  2 * Dd, w.dkv + Dd, 2 * Dd, B, H, P, Nc, dh, 1.0f / sqrtf((float)dh), st));
  RUN(linear_f32x3_wgrad(w.dq, s.qn, g->q_w, g->q_b, Mq, Dd, Dd, w.sp.A, w.sp.B, st));
  RUN(linear_f32x3_dgrad(w.dq, p->q_w, w.dqn, Mq, Dd, Dd, 0, w.sp.A, w.sp.B, st));
  RUN(linear_f32x3_wgrad(w.dkv, s.cn, g->kv_w, g->kv_b, Mc, 2 * Dd, Dd, w.sp.A, w.sp.B, st));
  RUN(linear_f32x3_dgrad(w.dkv, p->kv_w, w.dcn, Mc, 2 * Dd, Dd, 0, w.sp.A, w.sp.B, st));
  RUN(mmae_layernorm_backward(w.dqn, 0, Dd, s.queries, Dd, s.qmean, s.qrstd, p->query_norm_w, nullptr, 0, w.dqueries, Dd,
                              g->query_norm_w, g->query_norm_b, Mq, Dd, st));
  RUN(mmae_layernorm_backward(w.dcn, 0, Dd, s.context, Dd, s.cmean, s.crstd, p->context_norm_w, nullptr, 0, w.dcontext, Dd,
                              g->context_norm_w, g->context_norm_b, Mc, Dd, st));
  // ---- queries / context construction
  TaskEmbGradPtrs dte;
  for (int t = 0; t < MMAE_MAX_TASKS; ++t) dte.p[t] = g->task_emb[t];
  RUN(launch_dec_build_bwd(w.dqueries, w.dcontext, ix, w.dctx, g->mask_token, dte, cst));
  // ---- proj_context: denc is accumulated (the adapters share the encoder-output gradient)
  RUN(linear_f32x3_wgrad(w.dctx, enc, g->proj_context_w, g->proj_context_b, Mc, Dd, De, w.sp.A, w.sp.B, st));
  RUN(linear_f32x3_dgrad(w.dctx, p->proj_context_w, denc, Mc, Dd, De, 1, w.sp.A, w.sp.B, st));
  return MMAE_OK;
}

// ================================================================================================ decoder tail
extern "C" int64_t mmae_dectail_f32_workspace_bytes(int B, int nh, int nw, int Dd, int C, int P) {
  return (int64_t)tail_ws_f(nullptr, B, nh, nw, Dd, C, P).bytes;
}

extern "C" int mmae_dectail_f32_forward(const float* x, int B, int nh, int nw, int Dd, int C, int P, const float* out_w,
                                        const float* out_b, float* pred, void* ws, void* st) {
  MMAE_CHECK(x && out_w && out_b && pred && ws, MMAE_ERR_ARG, "mmae_dectail_f32_forward: bad args");
  const int M = B * nh * nw, Nout = C * P * P;
  TailWsF w = tail_ws_f(ws, B, nh, nw, Dd, C, P);
  RUN(linear_f32x3_forward(x, out_w, out_b, nullptr, w.y, M, Nout, Dd, w.sp.A, w.sp.B, st));     // output_adapters.py:274
  RUN(mmae_unpatchify(w.y, Nout, pred, B, C, nh, nw, P, st));                                    // :277-280
  return MMAE_OK;
}

extern "C" int mmae_dectail_f32_backward(const float* x, const float* dpred, int B, int nh, int nw, int Dd, int C, int P,
                                         const float* out_w, float* d_out_w, float* d_out_b, float* dx, void* ws, void* st) {
  MMAE_CHECK(x && dpred && out_w && d_out_w && d_out_b && dx && ws, MMAE_ERR_ARG, "mmae_dectail_f32_backward: bad args");
  const int M = B * nh * nw, Nout = C * P * P;
  TailWsF w = tail_ws_f(ws, B, nh, nw, Dd, C, P);
  RUN(mmae_patchify(dpred, w.dy, Nout, B, C, nh, nw, P, st));
  RUN(linear_f32x3_wgrad(w.dy, x, d_out_w, d_out_b, M, Nout, Dd, w.sp.A, w.sp.B, st));
  RUN(linear_f32x3_dgrad(w.dy, out_w, dx, M, Nout, Dd, 0, w.sp.A, w.sp.B, st));
  return MMAE_OK;
}
