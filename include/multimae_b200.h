/*
 * multimae_b200 — C ABI of the H100-native (sm_90a) MultiMAE pre-training hot path.
 *
 * The reference (EPFL-VILAB/MultiMAE) is pure Python on top of PyTorch: it has no FFI layer of its own.
 * The "plugin boundary" of the hot path is the Python module API consumed by run_pretraining_multimae.py
 * (SURVEY.md §8b).  This header is what the Python host side (multimae_b200/*.py, loaded with ctypes)
 * binds; every entry point names the reference code it replaces (path:line in the EPFL-VILAB/MultiMAE tree).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host; no PyTorch types cross this ABI;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *   - functions return 0 on success, non-zero on error; mmae_last_error() returns a message for the
 *     calling thread's last failure;  nothing here falls back to a CPU path;
 *   - matrices are row-major; "bf16" is __nv_bfloat16; leading dimensions are in elements;
 *   - all leading dimensions must be multiples of 8 elements and base pointers 16-byte aligned.
 */
#ifndef MULTIMAE_B200_H_
#define MULTIMAE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MMAE_ABI_VERSION 17

int mmae_abi_version(void);
const char* mmae_last_error(void);
/* number of kernel launches issued through this library by the calling process so far */
int64_t mmae_launch_count(void);

/* Optional device timing of every GEMM launch (cudaEvent pair on the launch stream); used by bench.py to report the
 * achieved TFLOP/s of the dominant kernel.  mmae_profile_gemm(1) starts/resets, (0) stops; _read synchronises the
 * recorded events and returns the summed algorithmic FLOPs (2*M*N*K), summed kernel milliseconds and launch count. */
int mmae_profile_gemm(int enable);
int mmae_profile_gemm_read(double* flops, double* ms, int64_t* launches);
/* text dump, one line per recorded launch: "M N K flags ms" (flags: bit0 A MN-major, bit1 B MN-major, bits 8+ split_k) */
int64_t mmae_profile_gemm_dump(char* buf_host, int64_t capacity);

/* ------------------------------------------------------------------------------------------------
 * GEMM on the Hopper tensor cores (wgmma, bf16 x bf16 -> fp32 accumulate in registers), TMA-fed.
 * Replaces every nn.Linear / nn.Conv2d(k=s=P) matmul of the path:
 *   multimae/multimae_utils.py:149,153,172,180,203-204,212 ; multimae/input_adapters.py:110,232 ;
 *   multimae/output_adapters.py:258,274 and their autograd backward (dgrad / wgrad).
 *
 *   C[M,N] = epilogue( alpha * sum_k A(m,k) * B(n,k) )
 *   a_mn_major = 0 : A is stored [M,K] (K contiguous),  lda = row pitch
 *   a_mn_major = 1 : A is stored [K,M] (M contiguous),  lda = row pitch      (used by wgrad)
 *   b_mn_major = 0 : B is stored [N,K] (K contiguous)   (nn.Linear weight as-is: forward)
 *   b_mn_major = 1 : B is stored [K,N] (N contiguous)   (nn.Linear weight as-is: dgrad; wgrad input)
 *
 * Epilogue, in this order (all optional):
 *   v = alpha*acc ; v += bias[n] ; preact_bf16[m,n] = v ; v = act(v) ; v *= gelu'(dgelu_z[m,n]) ;
 *   v += residual[m,n] ; out_f32[m,n] (=|+=) v ; out_bf16[m,n] = v
 * split_k > 1 (or accumulate != 0) accumulates into out_f32 with fp32 atomics; the destination must have
 * been zeroed (or hold the value to accumulate onto); bias/residual are applied by split 0 only; act,
 * dgelu_z, preact_bf16 and out_bf16 are not allowed with split_k > 1.
 * split_k <= 0: automatic - split count and tile width are chosen together so that one wave of ~SM-count work items
 * covers the problem (fp32-only linear epilogues; anything else runs unsplit).  The accumulation then uses TMA
 * reduce-add tiles (cp.reduce.async.bulk.tensor) unless mmae_gemm_set_tma_store(0).
 * ---------------------------------------------------------------------------------------------- */
typedef struct mmae_gemm_epilogue {
  float alpha;
  int act;                 /* 0 = identity, 1 = exact-erf GELU (nn.GELU default) */
  int accumulate;          /* 1: out_f32 += v (atomic) */
  int reserved;
  const float* bias;       /* [N] fp32 or NULL */
  const float* residual;   /* [M, ld_residual] fp32 or NULL */
  const void* dgelu_z;     /* bf16 [M, ld_dgelu_z] or NULL */
  void* preact_bf16;       /* bf16 [M, ld_preact] or NULL */
  float* out_f32;          /* [M, ld_out_f32] or NULL */
  void* out_bf16;          /* bf16 [M, ld_out_bf16] or NULL */
  int64_t ld_residual, ld_dgelu_z, ld_preact, ld_out_f32, ld_out_bf16;
} mmae_gemm_epilogue;

/* Kernel variant for measurements: -1 = heuristic (default), 0 / 1 / 3 / 2 = one CTA per 128 x 64 / 128 / 192 / 256
 * tile, 6 / 5 / 4 = two-CTA cluster per 256 x 128 / 192 / 256 tile (the B tile loaded once and multicast to both CTAs).
 * Env MMAE_GEMM_VARIANT sets the initial value. */
int mmae_gemm_set_variant(int variant);
/* 1 (default): plain bf16 / fp32 outputs (optionally with bias / GELU) leave through shared memory + TMA tile stores, fp32
 * accumulation (split-K, accumulate) through TMA reduce-add tiles; 0: per-thread global stores / red.global adds.
 * Env MMAE_GEMM_TMA_STORE sets the initial value. */
int mmae_gemm_set_tma_store(int enable);
/* 1: kernels are launched with programmatic stream serialization and start with griddepcontrol (launch_dependents +
 * wait), so the next kernel's blocks are scheduled while the previous one drains; 0 (default): plain stream order - a
 * programmatically launched dependent keeps stale L1 lines for non-coherent loads (see runtime.cu).  Env MMAE_PDL. */
int mmae_set_pdl(int enable);
/* SM budget of the SM-count-sized grids (GEMM split-K / tile choice, one-wave element-wise grids): 0 = every SM
 * (default), n = at most n.  Data-parallel runs leave NCCL's all-reduce CTAs their SMs.  Env MMAE_SM_BUDGET. */
int mmae_set_sm_budget(int sms);
/* 1: mmae_block_backward runs its four weight-gradient GEMMs on a library-owned side stream, forked behind the kernel
 * that produces their dY operand and joined before the call returns (the caller's stream order is unchanged);
 * 0 (default; no gain measured at the MultiMAE-B shapes): everything on the caller's stream.  Env MMAE_WGRAD_STREAM. */
int mmae_set_wgrad_stream(int enable);

int mmae_gemm_bf16(const void* A, int64_t lda, int a_mn_major, const void* B, int64_t ldb, int b_mn_major,
                   int M, int N, int K, int split_k, const mmae_gemm_epilogue* ep, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Element-wise / layout helpers (HBM-bound)
 * ---------------------------------------------------------------------------------------------- */
/* dst_bf16[i] = bf16(src[i])            (autocast's fp32->half cast of weights/activations) */
int mmae_cast_f32_to_bf16(const float* src, void* dst_bf16, int64_t n, void* stream);
/* dst[M,N] bf16 = bf16(src[M,N] fp32) and colsum[n] += sum_m src[m,n]  (bias gradient: autograd of
 * nn.Linear bias, multimae/multimae_utils.py:143-145,165-167); colsum may be NULL; dst may be NULL */
int mmae_cast_colsum_f32(const float* src, int64_t ld_src, void* dst_bf16, int64_t ld_dst, float* colsum,
                         int M, int N, void* stream);
/* colsum[n] += sum_m src_bf16[m,n] */
int mmae_colsum_bf16(const void* src_bf16, int64_t ld_src, float* colsum, int M, int N, void* stream);
/* exact-erf GELU over a bf16 stream (nn.GELU, multimae/multimae_utils.py:139,150): backward = 0: io[i] = gelu(z[i]);
 * backward = 1: io[i] *= gelu'(z[i]) in place.  n must be a multiple of 8. */
int mmae_gelu_bf16(const void* z, void* io, int64_t n, int backward, void* stream);
/* dz[m,n] *= gelu'(z[m,n]) in place and colsum[n] += sum_m dz[m,n] (fc1 bias gradient) in one pass */
int mmae_dgelu_colsum_bf16(const void* z, void* dz, int64_t ld, float* colsum, int M, int N, void* stream);
/* 1: the module-level entry points fuse GELU / GELU' into the GEMM epilogue; 0: streaming kernel after the GEMM.
 * Default and its measurement: modules.cu.  Env MMAE_FUSE_GELU sets the initial value. */
int mmae_set_fuse_gelu(int enable);
/* out[i] = x[i] + float(y_bf16[i]); n must be a multiple of 8 */
int mmae_add_bf16_f32(const float* x, const void* y_bf16, float* out, int64_t n, void* stream);
/* dst[N,M] = src[M,N]^T (bf16) */
int mmae_transpose_bf16(const void* src, int64_t ld_src, void* dst, int64_t ld_dst, int M, int N, void* stream);

/* ------------------------------------------------------------------------------------------------
 * LayerNorm (fp32 statistics; eps given).  nn.LayerNorm(eps=1e-6): multimae/multimae_utils.py:222,225 and
 * multimae/output_adapters.py:120-122.  D must be a multiple of 128, <= 1024.
 *   forward : y = (x-mean)*rstd*gamma+beta, written as bf16 (GEMM operand) and/or fp32; saves mean/rstd.
 *   backward: dx = dx_resid(optional) + LN'(dy); dgamma/dbeta are ACCUMULATED (+=) with fp32 atomics.
 * ---------------------------------------------------------------------------------------------- */
int mmae_layernorm_forward(const float* x, int64_t ldx, const float* gamma, const float* beta, void* y_bf16,
                           int64_t ldy, float* y_f32, int64_t ldyf, float* mean, float* rstd, int M, int D,
                           float eps, void* stream);
/* x_sum = x + addend_bf16 (fp32, written when non-NULL) followed by LayerNorm(x_sum) -> y_bf16: the residual add
 * `x = x + branch(...)` (multimae/multimae_utils.py:230-231) fused in front of the next norm. */
int mmae_add_layernorm_forward(const float* x, int64_t ldx, const void* addend_bf16, int64_t ldadd, float* x_sum,
                               int64_t ldsum, const float* gamma, const float* beta, void* y_bf16, int64_t ldy,
                               float* mean, float* rstd, int M, int D, float eps, void* stream);
int mmae_layernorm_backward(const void* dy, int dy_is_bf16, int64_t lddy, const float* x, int64_t ldx,
                            const float* mean, const float* rstd, const float* gamma, const float* dx_resid,
                            int64_t ldr, float* dx, int64_t lddx, float* dgamma, float* dbeta, int M, int D,
                            void* stream);

/* as mmae_layernorm_backward, additionally writing bf16(dx) and accumulating dx_colsum[d] += sum_rows dx[:,d] */
int mmae_layernorm_backward_ex(const void* dy, int dy_is_bf16, int64_t lddy, const float* x, int64_t ldx,
                               const float* mean, const float* rstd, const float* gamma, const float* dx_resid,
                               int64_t ldr, float* dx, int64_t lddx, float* dgamma, float* dbeta, void* dx_bf16,
                               int64_t lddxb, float* dx_colsum, int M, int D, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fused multi-head attention (scores stay on chip).  Attention / CrossAttention:
 * multimae/multimae_utils.py:172-179, 203-211.  q/k/v/o are bf16 views into row-major [B*N, ld] projection
 * buffers: head h = columns [h*head_dim, (h+1)*head_dim) from the given base pointer, batch b = rows
 * [b*N, (b+1)*N).  head_dim in {32, 64}.  lse[B,H,Nq] = log-sum-exp of the scaled scores (saved for backward).
 * backward: delta_ws is a [B,H,Nq] fp32 scratch; dq/dk/dv are written (not accumulated).
 * Kernels: wgmma forward (<= 256 keys) / backward and warp-level mma.sync forward / backward (bf16 in, fp32 accumulate).
 * ---------------------------------------------------------------------------------------------- */
/* bit mask of kernel families: 1 = wgmma forward for <= 128 keys, 2 | 8 | 32 | 128 = wgmma forward for 129..256 keys,
 * 4 | 64 = wgmma backward; otherwise the mma.sync kernels run (16: no Hopper kernel, ignored); 0 = mma.sync everywhere.
 * Default 0, the fastest measured on H100 (attention.cu); env MMAE_ATTN_TC; a negative value restores the start-up default. */
int mmae_attention_set_tc(int enable);
/* dropout_p: dropout on the softmax probabilities (site MMAE_DROP_SITE_ATTN below), its mask from *seed; seed may be NULL
 * when dropout_p is 0, which means no dropout.  With dropout_p > 0 the mma.sync kernels run whatever
 * mmae_attention_set_tc selects (the wgmma kernels have no dropout).  lse stays the log-sum-exp of the undropped scores. */
int mmae_attention_forward(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                           void* o, int64_t ldo, float* lse, int B, int H, int Nq, int Nk, int head_dim, float scale,
                           float dropout_p, const uint64_t* seed, void* stream);
int mmae_attention_backward(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                            const void* o, int64_t ldo, const void* d_o, int64_t lddo, const float* lse,
                            float* delta_ws, void* dq, int64_t lddq, void* dk, int64_t lddk, void* dv,
                            int64_t lddv, int B, int H, int Nq, int Nk, int head_dim, float scale, float dropout_p,
                            const uint64_t* seed, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Dropout in training (nn.Dropout, multimae/multimae_utils.py:154,177,181): inverted dropout, a kept element is scaled by
 * 1/(1-p), and p = 1 zeroes everything.  No mask is stored: the keep bit of element (row, col) of a site's [rows, cols]
 * matrix is word (col & 3) of Philox4x32-10 at counter {col / 4, row (64 bits, low word first), site} under the 64-bit key
 * *seed, kept iff that word < (1 - p) * 2^32.  Forward and backward regenerate the same bits.  Seeds live in device
 * memory, so a captured CUDA graph reads the value of each replay.  Sites and their matrices:
 *   MMAE_DROP_SITE_ATTN  the softmax probabilities: row (b*H + h)*Nq + i, column j (key)         Attention.attn_drop
 *   MMAE_DROP_SITE_PROJ  the attention branch output, [B*N, D]                                 Attention.proj_drop
 *   MMAE_DROP_SITE_MLP   the MLP branch output after fc2, [B*N, D]                             Mlp.drop
 * ---------------------------------------------------------------------------------------------- */
#define MMAE_DROP_SITE_ATTN 0
#define MMAE_DROP_SITE_PROJ 1
#define MMAE_DROP_SITE_MLP 2
/* out[r * cols + c] = keep bit (0 / 1 byte) of element (r, c) of `site` at rate p, from the generator the kernels use;
 * all ones at p = 0.  For tests and inspection: the training path never materialises a mask. */
int mmae_dropout_keep_mask(const uint64_t* seed, int site, int64_t rows, int cols, float p, void* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Dirichlet token-mask sampler.  MultiMAE.generate_random_masks, multimae/multimae.py:189-216, as a pure
 * function of the random draws: shares[B,T] (Dirichlet sample), noise_task[B,total] (the per-task
 * torch.rand draws concatenated in task order), noise_all[B,total].  Outputs are int64 like the reference:
 * task_masks[B,total] (0 = visible; split per task by the caller), ids_keep[B,num_encoded],
 * ids_restore[B,total].  Ties break towards the lower index.
 * ---------------------------------------------------------------------------------------------- */
int mmae_sample_masks(const float* shares, const float* noise_task, const float* noise_all, int B, int num_tasks,
                      const int* tokens_per_task_host, int num_encoded, int64_t* task_masks, int64_t* ids_keep,
                      int64_t* ids_restore, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Gather-first patch embedding (PatchedInputAdapter.forward multimae/input_adapters.py:97-119,
 * SemSegInputAdapter.forward :215-241, and the cat/gather/global-token cat of multimae/multimae.py:340-347).
 * Only the num_encoded visible patches per sample are embedded: one K-concatenated GEMM
 * [B*T, sum_t K_t] x [D, sum_t K_t]^T whose A rows are zero outside the token's own task segment.
 * ---------------------------------------------------------------------------------------------- */
#define MMAE_MAX_TASKS 8

typedef struct mmae_embed_layout {
  int num_tasks;
  int grid_h[MMAE_MAX_TASKS], grid_w[MMAE_MAX_TASKS]; /* patch grid of each task at the current image size */
  int tok_offset[MMAE_MAX_TASKS + 1];                 /* token range of each task in the concatenated sequence */
  int k_offset[MMAE_MAX_TASKS + 1];                   /* K segment of each task (K_t = channels * patch^2) */
  int patch[MMAE_MAX_TASKS];                          /* P_H = P_W in input pixels (16, 16, 4) */
  int channels[MMAE_MAX_TASKS];                       /* image channels, or dim_class_emb for semseg */
  int is_semseg[MMAE_MAX_TASKS];
  int num_classes[MMAE_MAX_TASKS];
} mmae_embed_layout;

typedef struct mmae_embed_inputs {
  const void* data[MMAE_MAX_TASKS];       /* fp32 [B,C,H,W]  or  int64 [B,H,W] class ids */
  const float* class_emb[MMAE_MAX_TASKS]; /* [num_classes, dim_class_emb] (semseg) or NULL */
} mmae_embed_inputs;

typedef struct mmae_embed_params {
  const float* weight[MMAE_MAX_TASKS]; /* proj.weight viewed as [D, C*P*P] */
  const float* bias[MMAE_MAX_TASKS];   /* proj.bias [D] */
  const float* pos[MMAE_MAX_TASKS];    /* [N_t, D] rows of the (resized) positional table */
  const float* global_tokens;          /* [G, D] */
} mmae_embed_params;

typedef struct mmae_embed_grads {      /* accumulated (+=) */
  float* weight[MMAE_MAX_TASKS];
  float* bias[MMAE_MAX_TASKS];
  float* class_emb[MMAE_MAX_TASKS];
  float* global_tokens;
} mmae_embed_grads;

int64_t mmae_embed_saved_bytes(const mmae_embed_layout* layout, int B, int T, int D);
int64_t mmae_embed_workspace_bytes(const mmae_embed_layout* layout, int B, int T, int D);
/* x_out: [B, T+G, D] fp32 packed encoder input (global tokens last) */
int mmae_embed_forward(const mmae_embed_layout* layout, const mmae_embed_inputs* in, const mmae_embed_params* prm,
                       const int64_t* ids_keep, int B, int T, int G, int D, float* x_out, void* saved, void* ws,
                       void* stream);
int mmae_embed_backward(const mmae_embed_layout* layout, const mmae_embed_inputs* in, const mmae_embed_params* prm,
                        const mmae_embed_grads* grads, const int64_t* ids_keep, int B, int T, int G, int D,
                        const float* dx, const void* saved, void* ws, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Trainable positional tables of the input adapters (learnable_pos_emb=True, or sincos_pos_emb=False:
 * multimae/input_adapters.py:76-82, 183-189).  Each forward resizes the parameter pos_emb [1, D, h, w] to the patch grid
 * (nh, nw) of the call, F.interpolate(pos_emb, (nh, nw), mode, align_corners=False) (:113 bicubic with A = -0.75 and taps
 * clamped at the border, :235 bilinear), and hands the rows [nh*nw, D] to mmae_embed_forward as prm->pos[t].  When
 * (nh, nw) == (h, w) the resize is the identity and the rows are the transposed table.  Every result here is computed in
 * gather form, without atomics: bitwise repeatable.
 * ---------------------------------------------------------------------------------------------- */
#define MMAE_POS_BICUBIC 0  /* PatchedInputAdapter */
#define MMAE_POS_BILINEAR 1 /* SemSegInputAdapter */
/* rows[p, d] = resized table at grid position (p / nw, p % nw), channel d; table: [D, h, w] fp32 read in place */
int mmae_pos_resample_forward(const float* table, int D, int h, int w, int nh, int nw, int mode, float* rows, void* stream);
/* adjoint: dtable[d, y, x] += sum over the rows p that read (y, x) of their interpolation weight times drows[p, d] */
int mmae_pos_resample_backward(const float* drows, int D, int h, int w, int nh, int nw, int mode, float* dtable,
                               void* stream);
/* Gradient of the rows prm->pos[t] of mmae_embed_forward, for the tasks whose table is trainable.  drows_host: host array
 * of layout->num_tasks device pointers, NULL for a task whose table is frozen; drows_host[t] [N_t, D] is WRITTEN:
 *   drows_t[p, :] = sum over b of dx[b, slot, :] where slot = ids_restore[b, tok_offset[t] + p] < T
 * (a patch that is masked in sample b contributes nothing from b; one masked in every sample gets 0).  ids_restore:
 * [B, tok_offset[num_tasks]] (multimae/multimae.py:205; the identity permutation when nothing is masked); dx: the
 * [B, T+G, D] gradient given to mmae_embed_backward.  D must be a multiple of 4. */
int mmae_embed_pos_backward(const mmae_embed_layout* layout, const int64_t* ids_restore, int B, int T, int G, int D,
                            const float* dx, float* const* drows_host, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Pre-LN transformer block (Block / Attention / Mlp, multimae/multimae_utils.py:138-182, 217-232); used by the
 * encoder (D=768/1024) and the decoder transformer layers (D=256).  x: [B, N, D] fp32 residual stream.
 * `saved` keeps the bf16 operands needed by backward; sizes from the *_bytes queries.  Gradients of the
 * parameters are ACCUMULATED (+=) into `grads` (zero them once per step).
 * ---------------------------------------------------------------------------------------------- */
typedef struct mmae_block_params {
  const float *norm1_w, *norm1_b, *qkv_w, *qkv_b, *proj_w, *proj_b, *norm2_w, *norm2_b, *fc1_w, *fc1_b, *fc2_w, *fc2_b;
} mmae_block_params;
typedef struct mmae_block_grads {
  float *norm1_w, *norm1_b, *qkv_w, *qkv_b, *proj_w, *proj_b, *norm2_w, *norm2_b, *fc1_w, *fc1_b, *fc2_w, *fc2_b;
} mmae_block_grads;
/* Dropout of one block (see MMAE_DROP_SITE_ATTN): attn_p on the attention probabilities, proj_p on the attention branch
 * and mlp_p on the MLP branch, each site's mask from `seed` (a device uint64_t; NULL is allowed where all three rates are
 * 0).  A branch element (r, c) of sample b enters the residual stream as scale[b] * keep(r, c) / (1 - p) times the branch
 * output, and backward applies the same factor to the gradient entering the branch (its bf16 operand and bias gradient).
 * prev_mlp_p / prev_seed are the PREVIOUS block's mlp_p / seed, for the MLP branch it hands over through x_add_bf16
 * (forward) and dx_in_bf16 (backward), as scale_prev is its scale_mlp. */
typedef struct mmae_block_dropout mmae_block_dropout;
struct mmae_block_dropout {
  float attn_p, proj_p, mlp_p;
  const uint64_t* seed;
  float prev_mlp_p;
  const uint64_t* prev_seed;
};

int64_t mmae_block_saved_bytes(int B, int N, int D, int H, int hidden);
int64_t mmae_block_workspace_bytes(int B, int N, int D, int H, int hidden);
/* One block; every pointer named below may be NULL, and with all of them NULL the calls are the plain block.  Forward
 * computes, for the rows of sample b (row r of the [B*N, D] activation belongs to sample r / N),
 *   x = x_in + scale_prev[b] * x_add_bf16,   x_mid = x + scale_attn[b] * attn(norm1(x)),
 *   x_out = x_mid + scale_mlp[b] * mlp(norm2(x_mid))
 * Hand-offs between consecutive blocks (nn.Sequential of Blocks: the encoder, multimae/multimae.py:349, and each
 * decoder_transformer, multimae/output_adapters.py:271): the residual add that ends a block, `x = x + mlp(norm2(x))`
 * (multimae/multimae_utils.py:231), runs inside the next block instead of as a pass of its own.
 *   x_add_bf16   the previous block's MLP branch (its y_out_bf16); the sum x is formed inside the first LayerNorm kernel and
 *                written to x_sum (fp32), the x_in to give the backward call.  NULL: x = x_in and x_sum is not used.
 *   y_out_bf16   the MLP branch output is written there instead of x_out; the block's output is then x_mid + y_out_bf16,
 *                x_mid = mmae_block_saved_x_mid(saved).  NULL: x_out is written.
 *   dx_out_bf16  bf16(scale_mlp * dx_out), written by the next block's backward, which also added its column sums to this
 *                block's fc2 bias gradient: this block's cast + bias-gradient pass over dx_out is skipped.  NULL: it runs.
 *   dx_in_bf16   the first LayerNorm's backward also writes bf16(scale_prev * dx_in) there and adds its column sums to
 *                dx_in_colsum (the PREVIOUS block's fc2 bias gradient).  NULL: neither is written.
 * Stochastic depth (drop path, multimae/multimae_utils.py:105-132, 230-231): scale_attn, scale_mlp and scale_prev are
 * per-sample fp32 factors, float[B]; NULL means factor 1.  scale_prev is the PREVIOUS block's scale_mlp and needs x_add_bf16
 * (forward) and dx_in_bf16 (backward).  Backward takes the same three vectors: the gradient entering a branch is scaled,
 * the residual-path gradient is not.
 * Dropout: `drop` (mmae_block_dropout above), the same struct forward and backward.  NULL, or all rates 0, means no
 * dropout: the same kernels and the same results.  With attn_p > 0 attention runs the mma.sync kernels whatever
 * mmae_attention_set_tc selects. */
int mmae_block_forward(const float* x_in, const void* x_add_bf16, float* x_sum, float* x_out, void* y_out_bf16, int B, int N,
                       int D, int H, int hidden, float eps, const float* scale_attn, const float* scale_mlp,
                       const float* scale_prev, const mmae_block_dropout* drop, const mmae_block_params* prm, void* saved,
                       void* ws, void* stream);
float* mmae_block_saved_x_mid(void* saved, int B, int N, int D, int H, int hidden);
int mmae_block_backward(const float* x_in, const float* dx_out, const void* dx_out_bf16, float* dx_in, void* dx_in_bf16,
                        float* dx_in_colsum, int B, int N, int D, int H, int hidden, const float* scale_attn,
                        const float* scale_mlp, const float* scale_prev, const mmae_block_dropout* drop,
                        const mmae_block_params* prm, const mmae_block_grads* grads, const void* saved, void* ws,
                        void* stream);

/* ------------------------------------------------------------------------------------------------
 * SpatialOutputAdapter, split at its decoder_transformer (multimae/output_adapters.py:236-282):
 *   head: proj_context -> queries/context construction (get_queries_and_context :183-234) -> LayerNorms ->
 *         CrossAttention (no residual) -> x + mlp(out_norm(x))                                   (:258-266)
 *   tail: out_proj + un-patchify to [B, C, H, W]                                                (:274-280)
 * ---------------------------------------------------------------------------------------------- */
typedef struct mmae_decoder_index {
  int batch, dim, num_visible, num_global, num_queries, total_tokens, num_tasks, own_task;
  /* query_mode 0 (output_adapters.py:209-213): the queries are the own_task rows of the restored context, own_task in
   * [0, num_tasks).  query_mode 1 (:214-221, use_task_queries=False or a task that is not among the inputs): every query
   * is mask_token + pos (+ task_emb[own_task] when own_task >= 0; the slot may be num_tasks, an embedding that belongs to
   * no input task). */
  int query_mode;
  int tok_offset[MMAE_MAX_TASKS + 1];
  const int64_t* ids_keep;    /* [B, num_visible] */
  const int64_t* ids_restore; /* [B, total_tokens] */
} mmae_decoder_index;

typedef struct mmae_dechead_params {
  const float *proj_context_w, *proj_context_b, *mask_token, *pos;  /* pos: [num_queries, Dd] resized table rows */
  const float* task_emb[MMAE_MAX_TASKS];                           /* [Dd] per context task or NULL */
  const float *context_norm_w, *context_norm_b, *query_norm_w, *query_norm_b, *out_norm_w, *out_norm_b;
  const float *q_w, *q_b, *kv_w, *kv_b, *proj_w, *proj_b, *fc1_w, *fc1_b, *fc2_w, *fc2_b;
} mmae_dechead_params;
typedef struct mmae_dechead_grads {
  float *proj_context_w, *proj_context_b, *mask_token;
  float* task_emb[MMAE_MAX_TASKS];
  float *context_norm_w, *context_norm_b, *query_norm_w, *query_norm_b, *out_norm_w, *out_norm_b;
  float *q_w, *q_b, *kv_w, *kv_b, *proj_w, *proj_b, *fc1_w, *fc1_b, *fc2_w, *fc2_b;
} mmae_dechead_grads;

int64_t mmae_dechead_saved_bytes(const mmae_decoder_index* ix, int D_enc, int H, int hidden);
int64_t mmae_dechead_workspace_bytes(const mmae_decoder_index* ix, int D_enc, int H, int hidden);
/* enc: [B, T+G, D_enc] fp32 encoder output; x_out: [B, num_queries, Dd] fp32 */
int mmae_dechead_forward(const float* enc, int D_enc, const mmae_decoder_index* ix, int H, int hidden, float eps,
                         const mmae_dechead_params* prm, float* x_out, void* saved, void* ws, void* stream);
/* denc is ACCUMULATED (+=): the four adapters share one encoder-output gradient */
int mmae_dechead_backward(const float* enc, int D_enc, const mmae_decoder_index* ix, int H, int hidden,
                          const mmae_dechead_params* prm, const mmae_dechead_grads* grads, const float* dx_out,
                          float* denc, const void* saved, void* ws, void* stream);

/* Shared context projection.  MultiMAE.forward passes the SAME encoder output to every output adapter
 * (multimae/multimae.py:357-366) and each adapter begins with its own proj_context Linear
 * (multimae/output_adapters.py:258): n Linears [rows, D_enc] -> [rows, Dd_i] on one input.  mmae_ctxproj_forward runs them
 * as ONE GEMM with N = sum_i Dd_i (one bf16 cast of enc, ctx = enc W_cat^T + b_cat, fp32 [rows, dim_total], adapter i owns
 * the column segment starting at sum(dim[0..i))); the heads then run through mmae_dechead_forward_ctx /
 * mmae_dechead_backward_ctx, which read their segment, write their bf16 context gradient into the matching segment of one
 * [rows, dim_total] matrix and produce the proj_context BIAS gradient; mmae_ctxproj_backward finishes with one weight
 * gradient GEMM (K = rows) and one input-gradient GEMM (K = dim_total) that WRITES denc.  Parameters, their bf16 mirror and
 * their gradient slots are used in place when the n tensors lie back to back in memory, gathered otherwise.
 * For the *_ctx heads, mmae_dechead_saved_bytes / _workspace_bytes are queried with D_enc = 0. */
typedef struct mmae_ctxproj_params {
  int num;                              /* adapters sharing the projection, 1..MMAE_MAX_TASKS */
  int dim[MMAE_MAX_TASKS];              /* dim_tokens of each adapter (multiples of 8) */
  const float* weight[MMAE_MAX_TASKS];  /* proj_context.weight [dim_i, D_enc] */
  const float* bias[MMAE_MAX_TASKS];    /* proj_context.bias [dim_i] */
} mmae_ctxproj_params;
typedef struct mmae_ctxproj_grads {     /* accumulated (+=) */
  float* weight[MMAE_MAX_TASKS];
} mmae_ctxproj_grads;
int64_t mmae_ctxproj_saved_bytes(int rows, int D_enc, int dim_total);
/* enc: [rows, D_enc] fp32 -> ctx: [rows, dim_total] fp32 */
int mmae_ctxproj_forward(const float* enc, int rows, int D_enc, const mmae_ctxproj_params* prm, float* ctx, void* saved,
                         void* stream);
/* dctx_bf16: [rows, dim_total] bf16 (every segment written by its head); denc: [rows, D_enc] fp32, WRITTEN */
int mmae_ctxproj_backward(int rows, int D_enc, const mmae_ctxproj_params* prm, const mmae_ctxproj_grads* grads,
                          const void* dctx_bf16, float* denc, const void* saved, void* stream);
/* ctx: this adapter's segment of the shared projection (row stride ld_ctx floats); prm->proj_context_w / _b are unused */
int mmae_dechead_forward_ctx(const float* ctx, int64_t ld_ctx, const mmae_decoder_index* ix, int H, int hidden, float eps,
                             const mmae_dechead_params* prm, float* x_out, void* saved, void* ws, void* stream);
/* dctx_bf16: this adapter's segment of the shared gradient matrix (row stride ld_dctx bf16 elements, WRITTEN);
 * grads->proj_context_b is accumulated, grads->proj_context_w is left to mmae_ctxproj_backward */
int mmae_dechead_backward_ctx(const mmae_decoder_index* ix, int H, int hidden, const mmae_dechead_params* prm,
                              const mmae_dechead_grads* grads, const float* dx_out, void* dctx_bf16, int64_t ld_dctx,
                              const void* saved, void* ws, void* stream);

int64_t mmae_dectail_saved_bytes(int B, int nh, int nw, int Dd, int C, int P);
int64_t mmae_dectail_workspace_bytes(int B, int nh, int nw, int Dd, int C, int P);
/* x: [B, nh*nw, Dd] fp32 -> pred [B, C, nh*P, nw*P] fp32 */
int mmae_dectail_forward(const float* x, int B, int nh, int nw, int Dd, int C, int P, const float* out_w,
                         const float* out_b, float* pred, void* saved, void* ws, void* stream);
int mmae_dectail_backward(const float* dpred, int B, int nh, int nw, int Dd, int C, int P, const float* out_w,
                          float* d_out_w, float* d_out_b, float* dx, const void* saved, void* ws, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Classification head of fine-tuning: LinearOutputAdapter.forward (multimae/output_adapters.py:345-356),
 *   pooled = mean_pool ? x.mean(1) : x[:, N-1]   (mean over all N tokens, global token included; or the global token)
 *   out    = LayerNorm(pooled) W^T + b           (W: [C, D] head.weight, b: [C]; fp32 LayerNorm statistics)
 * x: [B, N, D] fp32 encoder output; out: [B, C] fp32 logits, or with C = 0 (head = nn.Identity) the fp32 LayerNorm output
 * [B, D].  D must be a multiple of 8 (at most 8192); any C >= 0.  The head GEMM takes bf16 operands (the registered
 * weight mirror when there is one) and accumulates in fp32.  Backward WRITES dx ([B, N, D]: dpooled / N on every token,
 * or dpooled on token N-1 and zeros elsewhere) and ACCUMULATES (+=) the four parameter gradients.  `saved` (from
 * forward to backward) and `ws` are sized by the *_bytes queries.  head_w / d_head_w / d_head_b may be NULL when C = 0.
 * ---------------------------------------------------------------------------------------------- */
int64_t mmae_clshead_saved_bytes(int B, int N, int D, int C);
int64_t mmae_clshead_workspace_bytes(int B, int N, int D, int C);
int mmae_clshead_forward(const float* x, int B, int N, int D, int C, int mean_pool, float eps, const float* norm_w,
                         const float* norm_b, const float* head_w, const float* head_b, float* out, void* saved, void* ws,
                         void* stream);
int mmae_clshead_backward(const float* dout, int B, int N, int D, int C, int mean_pool, const float* norm_w,
                          const float* head_w, float* d_norm_w, float* d_norm_b, float* d_head_w, float* d_head_b,
                          float* dx, const void* saved, void* ws, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Semantic-segmentation head of fine-tuning: ConvNeXtAdapter (multimae/output_adapters.py:481-573, ConvNeXtBlock in
 * multimae/output_adapter_utils.py:19-57), split like SpatialOutputAdapter: proj -> block x depth -> tail.
 * The feature map (Hf, Wf) = (nh*s, nw*s), s = sqrt(preds_per_patch), is held as the fp32 [P, C] view of the proj_dec output
 * (P = B*nh*nw*s*s): row (b*n + t)*s*s + a*s + c' is pixel ((t / nw)*s + a, (t % nw)*s + c') of sample b, n = nh*nw.
 * C must be a multiple of 128, at most 1024.  GEMMs take bf16 operands (registered weight mirrors when there are any) and
 * accumulate in fp32.  Backward WRITES the activation gradient and ACCUMULATES (+=) the parameter gradients; the activation
 * gradients and the depthwise-conv parameter gradients are computed without atomics (bitwise repeatable).  `saved` (from
 * forward to backward) and `ws` are sized by the *_bytes queries.
 * ---------------------------------------------------------------------------------------------- */
/* proj: x[P, C] = cat_t(enc[:, start_t : start_t + n]) W^T + b  (enc [B, N, D] fp32, W [E, D*num_tasks], E = s*s*C).
 * Backward writes denc [B, N, D] in full: zeros on the tokens of other tasks and on the global tokens. */
int64_t mmae_convnext_proj_saved_bytes(int B, int n, int D_in, int E);
int64_t mmae_convnext_proj_workspace_bytes(int B, int n, int D_in, int E);
int mmae_convnext_proj_forward(const float* enc, int B, int N, int D, int n, int num_tasks, const int* start_host, int E,
                               const float* w, const float* b, float* x_out, void* saved, void* ws, void* stream);
int mmae_convnext_proj_backward(const float* dx_out, int B, int N, int D, int n, int num_tasks, const int* start_host, int E,
                                const float* w, float* d_w, float* d_b, float* denc, const void* saved, void* ws, void* stream);
/* block: x_out = x_in + pwconv2(GELU(pwconv1(LN(dwconv7x7(x_in)))))  (zero padding at the map borders).
 * params_host / grads_host: host arrays of 8 device pointers, in this order: dwconv.weight [C, 1, 7, 7], dwconv.bias [C],
 * norm.weight [C], norm.bias [C], pwconv1.weight [4C, C], pwconv1.bias [4C], pwconv2.weight [C, 4C], pwconv2.bias [C] */
int64_t mmae_convnext_block_saved_bytes(int B, int nh, int nw, int s, int C);
int64_t mmae_convnext_block_workspace_bytes(int B, int nh, int nw, int s, int C);
int mmae_convnext_block_forward(const float* x_in, float* x_out, int B, int nh, int nw, int s, int C, float eps,
                                const float* const* params_host, void* saved, void* ws, void* stream);
int mmae_convnext_block_backward(const float* x_in, const float* dx_out, float* dx_in, int B, int nh, int nw, int s, int C,
                                 const float* const* params_host, float* const* grads_host, const void* saved, void* ws,
                                 void* stream);
/* tail: out [B, K, H, W] fp32 = bilinear(x W^T + b) (align_corners=False; W: final_layer.weight [K, C, 1, 1]); H, W must be
 * integer multiples of Hf, Wf.  Any K >= 1. */
int64_t mmae_convnext_tail_saved_bytes(int B, int nh, int nw, int s, int C, int K);
int64_t mmae_convnext_tail_workspace_bytes(int B, int nh, int nw, int s, int C, int K);
int mmae_convnext_tail_forward(const float* x, int B, int nh, int nw, int s, int C, int K, int H, int W, const float* w,
                               const float* b, float* out, void* saved, void* ws, void* stream);
int mmae_convnext_tail_backward(const float* dout, int B, int nh, int nw, int s, int C, int K, int H, int W, const float* w,
                                float* d_w, float* d_b, float* dx, const void* saved, void* ws, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Segmenter head of semantic-segmentation fine-tuning: SegmenterMaskTransformerAdapter (multimae/output_adapters.py:359-478):
 * proj -> transformer blocks (mmae_block_*) over n + K tokens -> tail.  n = nh*nw patch tokens are followed by one token per
 * class.  E (the decoder width) must be a multiple of 128, at most 1024; 8 <= K <= 256.  GEMMs take bf16 operands and
 * accumulate in fp32.  Backward WRITES the activation gradient and ACCUMULATES (+=) the parameter gradients; the activation
 * gradient, d_cls and the mask_norm gradients are computed without atomics (bitwise repeatable).
 * ---------------------------------------------------------------------------------------------- */
/* proj: seq[b, :n] = cat_t(enc[b, start_t : start_t + n]) W^T + bias, seq[b, n:] = cls_emb  (seq [B, n + K, E] fp32,
 * W [E, D*num_tasks], cls_emb [K, E]).  Backward writes denc [B, N, D] in full and adds sum_b dseq[b, n + k] to d_cls[k]. */
int64_t mmae_segmenter_proj_saved_bytes(int B, int n, int D_in, int E);
int64_t mmae_segmenter_proj_workspace_bytes(int B, int n, int D_in, int E);
int mmae_segmenter_proj_forward(const float* enc, int B, int N, int D, int n, int num_tasks, const int* start_host, int E, int K,
                                const float* w, const float* b, const float* cls_emb, float* seq, void* saved, void* ws,
                                void* stream);
int mmae_segmenter_proj_backward(const float* dseq, int B, int N, int D, int n, int num_tasks, const int* start_host, int E,
                                 int K, const float* w, float* d_w, float* d_b, float* d_cls, float* denc, const void* saved,
                                 void* ws, void* stream);
/* The fused cosine mask + class LayerNorm on its own.  P [B*n, E], C [B*K, E] bf16; rp [B*n], rc [B*K] = 1 / max(norm, 1e-12) of
 * their rows.  forward: cmap[b*n + i, j] = LN_j(P_b[i] . C_b[j] rp rc) gamma_j + beta_j, fp32 [B*n, Kp], Kp = round_up(K, 8),
 * pad columns zero; mean / rstd [B*n] are saved for backward.  backward: dcmap [B*n, Kp] -> dP, dC (bf16, gradients of the
 * UNnormalised rows: the normalise backward is included), d_gamma / d_beta += . */
int64_t mmae_segmenter_mask_workspace_bytes(int B, int n, int K);
int mmae_segmenter_mask_forward(const void* P, const void* C, const float* rp, const float* rc, const float* gamma,
                                const float* beta, float eps, int B, int n, int K, int E, float* cmap, float* mean, float* rstd,
                                void* stream);
int mmae_segmenter_mask_backward(const void* P, const void* C, const float* rp, const float* rc, const float* gamma,
                                 const float* mean, const float* rstd, const float* dcmap, int B, int n, int K, int E, void* dP,
                                 void* dC, float* d_gamma, float* d_beta, void* ws, void* stream);
/* tail: out [B, K, H, W] fp32 = bilinear(mask_norm(normalize(patch_proj(y[:, :n])) normalize(classes_proj(y[:, n:]))^T)),
 * y = decoder_norm(x), x [B, n + K, E] fp32; H, W integer multiples of nh, nw.  params_host / grads_host: host arrays of 6
 * device pointers: decoder_norm.weight, decoder_norm.bias [E], patch_proj.weight, classes_proj.weight [E, E],
 * mask_norm.weight, mask_norm.bias [K]. */
int64_t mmae_segmenter_tail_saved_bytes(int B, int nh, int nw, int E, int K);
int64_t mmae_segmenter_tail_workspace_bytes(int B, int nh, int nw, int E, int K);
int mmae_segmenter_tail_forward(const float* x, int B, int nh, int nw, int E, int K, int H, int W, float eps_dec, float eps_mask,
                                const float* const* params_host, float* out, void* saved, void* ws, void* stream);
int mmae_segmenter_tail_backward(const float* x, const float* dout, float* dx, int B, int nh, int nw, int E, int K, int H, int W,
                                 const float* const* params_host, float* const* grads_host, const void* saved, void* ws,
                                 void* stream);

/* ------------------------------------------------------------------------------------------------
 * fp32 tier for `fp32_output_adapters` (multimae/multimae.py:367-377: the listed output adapters run outside autocast;
 * the shipped pre-training config lists ['semseg']).  Every activation stays fp32; Linear layers run as ONE bf16 wgmma
 * GEMM over 3-way split, K-concatenated operands (x_hi W_hi + x_hi W_lo + x_lo W_hi, fp32 accumulation: ~2^-16 relative),
 * attention and GELU as fp32 CUDA-core kernels.  Same argument meaning as the bf16-tier entry points of the same name;
 * the parameter / gradient structs are shared.  head_dim 32 only (the decoders').
 * ---------------------------------------------------------------------------------------------- */
int64_t mmae_linear_f32_workspace_bytes(int M, int N, int K);
/* y[M,N] = x[M,K] W[N,K]^T (+ bias[N]) (+ residual[M,N]); N, K multiples of 8 */
int mmae_linear_f32_forward(const float* x, const float* W, const float* bias, const float* residual, float* y, int M, int N,
                            int K, void* ws, void* stream);
/* dx[M,K] = dy W (when dx != NULL); dW[N,K] += dy^T x, db[N] += colsum(dy) (when dW / db != NULL); M, N, K multiples of 8 */
int mmae_linear_f32_backward(const float* x, const float* W, const float* dy, float* dx, float* dW, float* db, int M, int N, int K,
                             void* ws, void* stream);
/* io = gelu(z) (backward = 0) or io *= gelu'(z) (backward = 1); exact erf form, n multiple of 4 */
int mmae_gelu_f32(const float* z, float* io, int64_t n, int backward, void* stream);
int mmae_attention_f32_forward(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv, float* o,
                               int64_t ldo, float* lse, int B, int H, int Nq, int Nk, int head_dim, float scale, void* stream);
int mmae_attention_f32_backward(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv,
                                const float* o, int64_t ldo, const float* d_o, int64_t lddo, const float* lse, float* delta_ws,
                                float* dq, int64_t lddq, float* dk, int64_t lddk, float* dv, int64_t lddv, int B, int H, int Nq,
                                int Nk, int head_dim, float scale, void* stream);
int64_t mmae_block_f32_saved_bytes(int B, int N, int D, int H, int hidden);
int64_t mmae_block_f32_workspace_bytes(int B, int N, int D, int H, int hidden);
/* mmae_block_forward / _backward without hand-offs: scale_attn / scale_mlp as there, float[B] or NULL (factor 1) */
int mmae_block_f32_forward(const float* x_in, float* x_out, int B, int N, int D, int H, int hidden, float eps,
                           const float* scale_attn, const float* scale_mlp, const mmae_block_params* prm, void* saved,
                           void* ws, void* stream);
int mmae_block_f32_backward(const float* x_in, const float* dx_out, float* dx_in, int B, int N, int D, int H, int hidden,
                            const float* scale_attn, const float* scale_mlp, const mmae_block_params* prm,
                            const mmae_block_grads* grads, const void* saved, void* ws, void* stream);
int64_t mmae_dechead_f32_saved_bytes(const mmae_decoder_index* ix, int D_enc, int H, int hidden);
int64_t mmae_dechead_f32_workspace_bytes(const mmae_decoder_index* ix, int D_enc, int H, int hidden);
int mmae_dechead_f32_forward(const float* enc, int D_enc, const mmae_decoder_index* ix, int H, int hidden, float eps,
                             const mmae_dechead_params* prm, float* x_out, void* saved, void* ws, void* stream);
int mmae_dechead_f32_backward(const float* enc, int D_enc, const mmae_decoder_index* ix, int H, int hidden,
                              const mmae_dechead_params* prm, const mmae_dechead_grads* grads, const float* dx_out,
                              float* denc, const void* saved, void* ws, void* stream);
int64_t mmae_dectail_f32_workspace_bytes(int B, int nh, int nw, int Dd, int C, int P);
int mmae_dectail_f32_forward(const float* x, int B, int nh, int nw, int Dd, int C, int P, const float* out_w,
                             const float* out_b, float* pred, void* ws, void* stream);
int mmae_dectail_f32_backward(const float* x, const float* dpred, int B, int nh, int nw, int Dd, int C, int P,
                              const float* out_w, float* d_out_w, float* d_out_b, float* dx, void* ws, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Masked reconstruction losses (multimae/criterion.py:37-57, 84-114, 141-171).
 * kind: 0 = MSE, 1 = L1, 2 = cross-entropy (pred = logits [B,C,H,W], target = int64 [B,H,W]).
 * mask: int64 [B, (H/scale)*(W/scale)] (non-zero = contributes) or NULL (plain mean).  ws: 2*B floats kept until
 * backward.  loss_out / grad_out are device scalars.  No host synchronisation (mask.sum()==0 -> 0 on device).
 * ---------------------------------------------------------------------------------------------- */
int mmae_masked_loss_forward(int kind, int norm_pix, float label_smoothing, const float* pred, const void* target,
                             const int64_t* mask, int B, int C, int H, int W, int scale, float* ws, float* loss_out,
                             void* stream);
int mmae_masked_loss_backward(int kind, int norm_pix, float label_smoothing, const float* pred, const void* target,
                              const int64_t* mask, int B, int C, int H, int W, int scale, const float* ws,
                              const float* grad_out, float* dpred, void* stream);

/* bf16 weight mirror.  Registers a bf16 twin (same element count and layout) of a flat fp32 parameter buffer; pass
 * mirror_bf16 = NULL to unregister.  While registered: (1) the block / decoder / tail orchestrators take the bf16 GEMM
 * operand of any weight that lies inside `params_f32` (at an offset that is a multiple of 8 elements) from the twin
 * instead of casting it per call, (2) mmae_adamw_step on `params_f32` also writes the updated values to the twin.  The
 * caller keeps the twin in sync after any other modification of the parameters (mmae_cast_f32_to_bf16 over the buffer).
 * Replaces the per-Linear autocast weight casts of the reference (torch.cuda.amp.autocast, run_pretraining_multimae.py:452). */
int mmae_weight_mirror_register(const float* params_f32, void* mirror_bf16, int64_t n);

/* ------------------------------------------------------------------------------------------------
 * Flat-buffer gradient post-processing and AdamW (utils/native_scaler.py:34-36, 49-62; torch.optim.AdamW as built
 * by utils/optim_factory.py:155-174).  out2[0] = sum of squares AFTER unscaling, out2[1] = 1 if a non-finite
 * gradient was seen; grads *= inv_scale * post_scale (inv_scale read from inv_scale_dev when non-NULL).
 * ---------------------------------------------------------------------------------------------- */
int mmae_grad_unscale_norm(float* grads, int64_t n, const float* inv_scale_dev, float inv_scale, float post_scale,
                           float* out2, float* norm_out, void* stream);
/* dyn_lr_step_dev (optional): device float[2] = {learning rate, step count}; when non-NULL it overrides the host
 * `lr` / `step` arguments so that a CUDA-graph replay picks up the current schedule values, and the call itself advances
 * the step count by one on the device - unless found_inf_dev[0] != 0, in which case nothing is updated (GradScaler.step
 * does not call optimizer.step() for a non-finite gradient, so skipped steps do not advance the bias correction). */
int mmae_adamw_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                    float beta1, float beta2, float eps, float weight_decay, int step, const float* found_inf_dev,
                    const float* dyn_lr_step_dev, void* stream);

/* Model EMA (utils/model_ema.py:72-84, ModelEma.update): for each i < count, the fp32 tensors dst_host[i] (EMA copy) and
 * src_host[i] (live model) of n_host[i] elements (the three arrays are HOST arrays of device pointers / sizes) get
 *   dst = dst * decay + one_minus_decay * src
 * with two rounded products and a rounded sum, which is what the reference's torch ops compute when decay =
 * float(d) and one_minus_decay = float(1.0 - d), the subtraction done in double.  Up to 256 segments go in one launch
 * (more are split over several); nothing is allocated or copied to the device.  Every argument is checked before the
 * first launch: null pointers (allowed for n = 0), negative sizes and a non-finite decay are refused. */
int mmae_ema_update(float* const* dst_host, const float* const* src_host, const int64_t* n_host, int count, float decay,
                    float one_minus_decay, void* stream);

/* One segment of mmae_adamw_step_groups: n fp32 elements of parameters, gradients and both moments, an optional bf16
 * twin of the parameters (NULL: none), and the index of the parameter group whose lr / weight decay apply. */
typedef struct MmaeAdamwSegment {
  float* param;
  const float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  void* mirror_bf16;
  int64_t n;
  int group;
  int reserved;
} MmaeAdamwSegment;

/* torch.optim.AdamW with parameter groups (utils/optim_factory.py:49-101 builds them: per-layer lr_scale, weight decay
 * 0.05 or 0) over the HOST array segs_host[0 .. count): each segment is updated with lr_host[group] and
 * weight_decay_host[group] (HOST arrays of num_groups doubles) and the shared beta1 / beta2 / eps, in the order of torch's
 * _multi_tensor_adam: p *= 1 - lr*wd; m = lerp(m, g, 1 - beta1); v = v*beta2 + (1 - beta2)*g*g;
 * p += -(lr/bc1) * m / (sqrt(v)/sqrt(bc2) + eps), the scalars evaluated in double and rounded to fp32.  A non-NULL
 * mirror_bf16 receives bf16(p).  step_dev (device float) is the step count: the call advances it by one and derives the
 * bias corrections bc1 = 1 - beta1^step, bc2 = 1 - beta2^step from it on the device.  When found_inf_dev is non-NULL and
 * found_inf_dev[0] != 0, nothing is written: parameters, moments, twins and the step count keep their values.  Up to 448
 * segments go in one launch (more are split over several); nothing is allocated or copied to the device.  Every argument
 * is checked before the first launch: null pointers (allowed for n = 0), negative sizes, group indices outside
 * [0, num_groups), non-finite lr / weight decay / betas / eps, and pointers that are not 16-byte aligned are refused. */
int mmae_adamw_step_groups(const MmaeAdamwSegment* segs_host, int count, const double* lr_host,
                           const double* weight_decay_host, int num_groups, double beta1, double beta2, double eps,
                           const float* found_inf_dev, float* step_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Pre-training augmentation (MMAE_GPU_AUGMENT) — the resampling half of DataAugmentationForMultiMAE
 * (utils/datasets.py:66-111): Pillow-exact Image.resize of each crop to out_size x out_size (BICUBIC for rgb 'RGB' and
 * depth 'I;16', horizontal then vertical pass, rounded and clipped between the passes as Pillow does), TF.hflip, and
 * TF.normalize(TF.to_tensor(rgb)) / depth / 2**16; semseg ('P', NEAREST) is resized to out_size, then to out_size / 4.
 *
 * `packed` (device) and `packed_host` (its host copy, read for validation only) hold, 16-byte aligned:
 *   at offset 0, int32 descriptors [batch][num_tasks][8] = {kind, crop offset / 16, crop h, crop w, flip,
 *   column table offset / 16, row table offset / 16, intermediate offset / 16 in `scratch`};
 *   tables: int32 header {n_in, n_out, ksize, type}, then for type 1 (BICUBIC) int32 bounds [n_out][2] = {first tap,
 *   tap count}, int32 22-bit fixed-point weights [n_out][ksize], double weights [n_out][ksize] (8-byte aligned), and for
 *   type 2 (NEAREST) int32 source indices [n_out];
 *   crops: kind 0 (rgb) uint8 [h][w][3], kind 1 (depth) uint16 [h][w], kind 2 (semseg) uint8 [h][w].
 * rgb / depth items use BICUBIC tables crop w -> out_size (columns) and crop h -> out_size (rows) and an intermediate of
 * h x out_size pixels in `scratch`; semseg items use NEAREST tables, composed with the NEAREST table at map4_offset
 * (out_size -> out_size / 4).  out_host[t] (HOST array of num_tasks device pointers) receives task t: fp32
 * [batch, 3, S, S] (rgb), fp32 [batch, 1, S, S] (depth) or int64 [batch, S/4, S/4] (semseg); kinds_host[t] is its kind.
 * mean_host / std_host: 3 floats each (rgb).  Two launches (one per pass) for the whole batch, no atomics.  Every
 * descriptor and table is checked on the host before the first launch: kinds, crop sizes in [1, 32768], offsets and table
 * lengths inside the buffers, table sizes matching the crop, tap ranges and indices inside their input.
 * ---------------------------------------------------------------------------------------------- */
int mmae_augment_batch(const void* packed_host, const void* packed, int64_t packed_bytes, int batch, int num_tasks,
                       const int* kinds_host, int out_size, int64_t map4_offset, void* scratch, int64_t scratch_bytes,
                       void* const* out_host, const float* mean_host, const float* std_host, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Classification fine-tuning augmentation (MMAE_GPU_AUGMENT) — the pixel half of utils/datasets.py:build_transform:
 * Pillow-exact Image.resize of each crop to out_size x out_size (BILINEAR or BICUBIC, 8-bit fixed point), the horizontal
 * flip, then `num_layers` RandAugment layers on the 8-bit image, then TF.normalize(TF.to_tensor(img)).
 *
 * `packed` / `packed_host` hold, 16-byte aligned: int32 descriptors [batch][8] as mmae_augment_batch's with one rgb task
 * (kind 0); at ops_offset * 16 the op records [batch][num_layers] of 72 bytes = {int32 kind, filter, iarg, pad; double
 * factor; double m[6]} (kinds: 0 identity, 1 invert, 2 posterize iarg bits, 3 solarize threshold iarg, 4 solarize-add
 * iarg, 5 autocontrast, 6 equalize, 7 color, 8 contrast, 9 brightness, 10 sharpness (blend factor), 11 affine transform
 * with the inverse matrix m and filter 2 bilinear / 3 bicubic, 12 transpose by iarg = 90 / 180 / 270 degrees); the
 * tables (type 1 BICUBIC or 3 BILINEAR, mmae_augment_batch's layout, n_in = crop extent, n_out = out_size); the crops.
 * fill_host: the affine transforms' fill colour (3 ints in [0, 255]).  `scratch`: the horizontal pass's intermediates
 * (descriptor field 7) from offset 0; with num_layers > 0 then, each section 256-byte aligned after the end of the last
 * intermediate, two uint8 [batch][S][S][3] images and int32 [batch][1024].  out: fp32 [batch, 3, S, S].
 * 2 + 2 * num_layers launches for the whole batch.  Every descriptor, table and op record is checked on the host first.
 * ---------------------------------------------------------------------------------------------- */
int mmae_cls_augment_batch(const void* packed_host, const void* packed, int64_t packed_bytes, int batch, int num_layers,
                           int64_t ops_offset, int out_size, const int* fill_host, void* scratch, int64_t scratch_bytes,
                           float* out, const float* mean_host, const float* std_host, void* stream);

/* image <-> token layout helpers ('b (nh nw) (c ph pw) <-> b c (nh ph) (nw pw)') */
int mmae_unpatchify(const float* tokens, int64_t ld_tok, float* image, int B, int C, int nh, int nw, int P,
                    void* stream);
int mmae_patchify(const float* image, float* tokens, int64_t ld_tok, int B, int C, int nh, int nw, int P, void* stream);
int mmae_unpatchify_bf16(const void* tokens_bf16, int64_t ld_tok, float* image, int B, int C, int nh, int nw, int P,
                         void* stream);
int mmae_patchify_bf16(const float* image, void* tokens_bf16, int64_t ld_tok, int B, int C, int nh, int nw, int P,
                       void* stream);

/* ------------------------------------------------------------------------------------------------
 * Truncated depth standardisation — the caller-side step of train_one_epoch, run_pretraining_multimae.py:487-492
 * (torch.sort of every depth map, slice [int(0.1 n), int(0.9 n)), mean / unbiased var of the slice, standardise
 * the whole map).  depth, out: [B, n] fp32 (out may alias depth); lo / hi: the slice bounds as the reference
 * computes them on the host; eps: 1e-6 in the reference; stats (optional): [B, 2] = {mean, var} of the kept
 * values.  One launch: radix select of the two order statistics instead of a sort.
 * ---------------------------------------------------------------------------------------------- */
int mmae_standardize_depth(const float* depth, float* out, int B, int n, int lo, int hi, float eps, float* stats,
                           void* stream);
/* 1: the single-CTA radix-select kernel; 2 (default): histogram copies per CTA and a cluster split of large maps over
 * distributed shared memory.  Env MMAE_DEPTH_STD_VARIANT sets the initial value. */
int mmae_standardize_depth_set_variant(int variant);

#ifdef __cplusplus
}
#endif
#endif /* MULTIMAE_B200_H_ */
