// Internal (non-ABI) declarations shared between the kernel files and modules.cu.
#pragma once
#include <algorithm>

#include "common.cuh"
#include "../../include/multimae_b200.h"

namespace mmae {

struct TaskEmbPtrs {
  const float* p[MMAE_MAX_TASKS];
};
struct TaskEmbGradPtrs {
  float* p[MMAE_MAX_TASKS];
};

void count_launch();

// Column-partial reduction (elementwise.cu).  Kernels that reduce over rows write one partial row per block into the
// library's scratch buffer and colred_finalize adds the column totals to up to three destinations of `seg` columns each
// (dst[k] covers partial columns [k*seg, (k+1)*seg) of rows `ld` floats apart; trailing null destinations are skipped).  No atomics: Y x C scalar atomics on a
// few cache lines serialise in one or two L2 slices, and the result is deterministic.
float* colred_scratch(size_t floats, cudaStream_t st);   // nullptr + last error if it cannot be provided
// the scratch buffers carry a zeroed header of ticket counters in front of the partial rows ("last block adds up")
constexpr size_t COLRED_HEADER_FLOATS = 1024;
inline unsigned int* colred_counters(float* partial) {
  return partial ? reinterpret_cast<unsigned int*>(partial - COLRED_HEADER_FLOATS) : nullptr;
}
int colred_finalize(const float* partial, int Y, int ld, int seg, float* dst0, float* dst1, float* dst2, cudaStream_t st);

// same with up to 9 destinations of `seg` columns each (null entries are skipped)
struct ColredDst {
  float* p[9];
};
int colred_finalize_n(const float* partial, int Y, int ld, int seg, const ColredDst& dst, int nseg, cudaStream_t st);

// bf16 weight mirror registry (runtime.cu): the bf16 twin of a registered fp32 parameter buffer, or nullptr
const bf16* mirror_lookup(const float* w);

int launch_embed_gather(const mmae_embed_layout& L, const mmae_embed_inputs& in, const int64_t* ids_keep, int B, int T,
                        bf16* A, int* row_task, int* row_patch, cudaStream_t st);
int launch_embed_assemble(const float* Cmat, const mmae_embed_params& prm, const int* row_task, const int* row_patch,
                          int B, int T, int G, int D, float* x, cudaStream_t st);
int launch_embed_assemble_bwd(const float* dx, int B, int T, int G, int D, const int* row_task, bf16* dC,
                              const mmae_embed_grads& grads, int num_tasks, cudaStream_t st);
int launch_semseg_emb_bwd(const bf16* dA, int64_t ld_dA, const int64_t* labels, const int64_t* ids_keep,
                          const int* row_task, const int* row_patch, int task, int T, int rows, int grid_w, int grid_h,
                          int P, int E, int num_classes, float* dtable, cudaStream_t st);
int launch_dec_build(const float* ctx, int64_t ld_ctx, const mmae_decoder_index& ix, const float* mask_token,
                     const TaskEmbPtrs& task_emb, const float* pos, float* queries, float* context, cudaStream_t st);
int launch_dec_build_bwd(const float* dqueries, const float* dcontext, const mmae_decoder_index& ix, float* dctx,
                         float* dmask_token, const TaskEmbGradPtrs& dtask_emb, cudaStream_t st);
// depth_standardize_v2.cu (experimental variant 2); MMAE_ERR_UNSUPPORTED when the map exceeds 8 CTAs' shared memory
int launch_depth_standardize_v2(const float* depth, float* out, int B, int n, int lo, int hi, float eps, float* stats,
                                cudaStream_t st);
int launch_cast2d(const float* src, int64_t ld_src, bf16* dst, int64_t ld_dst, int rows, int cols, cudaStream_t st);

// Row-scaled forms of the streaming kernels behind stochastic depth (drop path).  `row_scale` is one fp32 factor per sample,
// row r of the [M, D] activation belonging to sample r / rows_per_sample; a null row_scale gives the plain kernel.
// layernorm.cu: x_sum = x + s * addend, then LayerNorm
int add_layernorm_forward_scaled(const float* x, int64_t ldx, const bf16* addend, int64_t ldadd, const float* row_scale,
                                 int rows_per_sample, float* x_sum, int64_t ldsum, const float* gamma, const float* beta,
                                 bf16* y_bf16, int64_t ldy, float* mean, float* rstd, int M, int D, float eps, void* stream);
// layernorm.cu: mmae_layernorm_backward_ex with bf16(dx) and colsum(dx) multiplied by s (dx itself unscaled)
int layernorm_backward_ex_scaled(const void* dy, int dy_is_bf16, int64_t lddy, const float* x, int64_t ldx, const float* mean,
                                 const float* rstd, const float* gamma, const float* dx_resid, int64_t ldr, float* dx,
                                 int64_t lddx, float* dgamma, float* dbeta, bf16* dx_bf16, int64_t lddxb, float* dx_colsum,
                                 const float* row_scale, int rows_per_sample, int M, int D, void* stream);
// elementwise.cu: dst = bf16(s * src), colsum += column sums of s * src
int cast_colsum_f32_scaled(const float* src, int64_t ld_src, bf16* dst, int64_t ld_dst, float* colsum, const float* row_scale,
                           int rows_per_sample, int M, int N, void* stream);
// elementwise.cu: out = x + s * y over n contiguous elements, `per_sample` elements per sample; y is bf16 (y_is_bf16) or
// fp32; x may be null (out = s * y, a scaled copy)
int add_scaled_f32(const float* x, const void* y, int y_is_bf16, const float* row_scale, int64_t per_sample, float* out,
                   int64_t n, void* stream);
// cls_head.cu: dst[i] += src[i] over n contiguous fp32 elements (any n)
int add_f32(float* dst, const float* src, int64_t n, cudaStream_t st);

// GEMM helpers of the module-level entry points (modules.cu): bf16 operands, fp32 accumulation through mmae_gemm_bf16.
// bf16 operand of a weight: the registered mirror of the fp32 parameter buffer, else the per-call slot *slot (cast now when
// cast_now; in backward the forward already cast it there)
int weight_operand(const float* w, bf16** slot, int64_t n, bool cast_now, void* st);
mmae_gemm_epilogue ep_zero();
// y = x W^T + b (bf16 out), W: [N, K]
int linear_bf16(const bf16* x, const bf16* W, const float* b, bf16* y, int M, int N, int K, void* st);
// y = x W^T + b (+ resid) (fp32 out)
int linear_f32(const bf16* x, const bf16* W, const float* b, const float* resid, float* y, int M, int N, int K, void* st);
// z = x W^T + b (bf16, kept for backward), a = gelu(z) (bf16)
int linear_gelu(const bf16* x, const bf16* W, const float* b, bf16* z, bf16* a, int M, int N, int K, void* st);
// dx[M, Kin] = dy[M, Nout] W[Nout, Kin] (bf16 out, unsplit; optional * gelu'(z))
int dgrad_bf16(const bf16* dy, int64_t lddy, const bf16* W, const bf16* dgelu_z, bf16* dx, int M, int Nout, int Kin, void* st);
// dz = (dy W) * gelu'(z) and db += colsum(dz)
int dgrad_dgelu_colsum(const bf16* dy, int64_t lddy, const bf16* W, const bf16* z, bf16* dz, float* db, int M, int Nout,
                       int Kin, void* st);
// dW[Nout, Kin] += dy[M, Nout]^T x[M, Kin]  (split-K chosen by mmae_gemm_bf16: fp32 atomics)
int wgrad(const bf16* dy, int64_t lddy, const bf16* x, int64_t ldx, float* dW, int M, int Nout, int Kin, void* st);

}  // namespace mmae
