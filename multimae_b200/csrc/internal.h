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

}  // namespace mmae
