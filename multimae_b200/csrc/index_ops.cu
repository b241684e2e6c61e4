// Coalesced index kernels around the GEMMs (all HBM-bound integer/byte shuffling, no tensor cores):
//   * gather-first patch embedding operand builder (+ nn.Embedding lookup for semseg)
//   * packed-sequence assembly (bias + positional embedding + global token)
//   * decoder query / context construction and its backward
//   * patch <-> image (un)patchify
// They replace the cat/gather/repeat/rearrange chains of multimae/multimae.py:340-347,
// multimae/input_adapters.py:110-117,229-239 and multimae/output_adapters.py:183-234,277-280.
#include "common.cuh"
#include "../../include/multimae_b200.h"

#include "internal.h"

namespace mmae {
void count_launch();
namespace {

__device__ __forceinline__ int task_of(const mmae_embed_layout& L, int g) {
  int t = 0;
#pragma unroll
  for (int i = 1; i < MMAE_MAX_TASKS; ++i)
    if (i < L.num_tasks && g >= L.tok_offset[i]) t = i;
  return t;
}

// ---------------------------------------------------------------------------------------------------------------------
// A_cat[r, :] for kept token r = (b, i): zeros except the K-segment of the token's task, which holds the patch pixels
// in conv-weight order (c, py, px); semseg patches hold class_emb[label, e] in (e, py, px) order.
// One CTA per kept token.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) embed_gather_kernel(mmae_embed_layout L, mmae_embed_inputs in,
                                                           const int64_t* __restrict__ ids_keep, int T,
                                                           bf16* __restrict__ A, int* __restrict__ row_task,
                                                           int* __restrict__ row_patch) {
  pdl_prologue();
  const int r = blockIdx.x;
  const int b = r / T;
  const int g = (int)ids_keep[r];
  const int t = task_of(L, g);
  const int p = g - L.tok_offset[t];
  if (threadIdx.x == 0) {
    row_task[r] = t;
    row_patch[r] = p;
  }
  const int P = L.patch[t], C = L.channels[t], Wt = L.grid_w[t] * P, Ht = L.grid_h[t] * P;
  const int ph = p / L.grid_w[t], pw = p % L.grid_w[t];
  const int k_begin = L.k_offset[t], k_end = L.k_offset[t + 1];
  bf16* Ar = A + int64_t(r) * L.k_offset[L.num_tasks];
  const bf16 zero = __float2bfloat16_rn(0.f);
  for (int k = threadIdx.x; k < L.k_offset[L.num_tasks]; k += blockDim.x) {
    bf16 v = zero;
    if (k >= k_begin && k < k_end) {
      const int kk = k - k_begin;
      const int c = kk / (P * P), py = (kk / P) % P, px = kk % P;
      const int y = ph * P + py, x = pw * P + px;
      if (L.is_semseg[t]) {
        const int64_t label = reinterpret_cast<const int64_t*>(in.data[t])[(int64_t(b) * Ht + y) * Wt + x];
        // a label outside [0, num_classes) (e.g. a 255 / -100 "ignore" label in a pseudo-label map) embeds as zeros instead
        // of reading out of bounds (nn.Embedding would raise a device-side assert, multimae/input_adapters.py:229)
        if (label >= 0 && label < L.num_classes[t]) v = __float2bfloat16_rn(__ldg(in.class_emb[t] + label * C + c));
      } else {
        v = __float2bfloat16_rn(__ldg(reinterpret_cast<const float*>(in.data[t]) + ((int64_t(b) * C + c) * Ht + y) * Wt + x));
      }
    }
    Ar[k] = v;
  }
}

// x[b, i, :] = C[b*T+i, :] + bias_t + pos_t[p]   (i < T);   x[b, T+j, :] = global_tokens[j, :]
__global__ void __launch_bounds__(256) embed_assemble_kernel(const float* __restrict__ Cmat, mmae_embed_params prm,
                                                             const int* __restrict__ row_task,
                                                             const int* __restrict__ row_patch, int T, int G, int D,
                                                             float* __restrict__ x) {
  pdl_prologue();
  const int row = blockIdx.x;  // b*(T+G) + i
  const int b = row / (T + G), i = row % (T + G);
  float4* dst = reinterpret_cast<float4*>(x + int64_t(row) * D);
  if (i >= T) {
    const float4* src = reinterpret_cast<const float4*>(prm.global_tokens + int64_t(i - T) * D);
    for (int c = threadIdx.x; c < D / 4; c += blockDim.x) dst[c] = __ldg(src + c);
    return;
  }
  const int r = b * T + i;
  const int t = row_task[r], p = row_patch[r];
  const float4* cs = reinterpret_cast<const float4*>(Cmat + int64_t(r) * D);
  const float4* bs = reinterpret_cast<const float4*>(prm.bias[t]);
  const float4* ps = reinterpret_cast<const float4*>(prm.pos[t] + int64_t(p) * D);
  for (int c = threadIdx.x; c < D / 4; c += blockDim.x) {
    const float4 a = __ldg(cs + c), bb = __ldg(bs + c), pp = __ldg(ps + c);
    dst[c] = make_float4(a.x + bb.x + pp.x, a.y + bb.y + pp.y, a.z + bb.z + pp.z, a.w + bb.w + pp.w);
  }
}

// backward of the assembly: dC (bf16 rows of kept tokens), per-task bias grads, global-token grad.  With `partial`
// (deterministic mode) block k writes its sums to row k of partial, [G global tokens | num_tasks biases] x D, for
// colred_finalize to add in block order; otherwise it adds them with atomics.
constexpr int EB_ROWS = 32;
__global__ void __launch_bounds__(256) embed_assemble_bwd_kernel(const float* __restrict__ dx, int T, int G, int D, int B,
                                                                 const int* __restrict__ row_task,
                                                                 bf16* __restrict__ dC, mmae_embed_grads grads,
                                                                 int num_tasks, float* __restrict__ partial) {
  pdl_prologue();
  // block handles EB_ROWS consecutive sequence rows; thread c handles columns c, c+256, ...
  const int row0 = blockIdx.x * EB_ROWS;
  const int rows_total = B * (T + G);
  float* prow = partial ? partial + int64_t(blockIdx.x) * (G + num_tasks) * D : nullptr;
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    if (prow)   // this thread alone owns column c of the block's row
      for (int g = 0; g < G; ++g) prow[int64_t(g) * D + c] = 0.f;
    float accb[MMAE_MAX_TASKS];
#pragma unroll
    for (int t = 0; t < MMAE_MAX_TASKS; ++t) accb[t] = 0.f;
    float accg = 0.f;
    int gidx = -1;
    for (int row = row0; row < min(row0 + EB_ROWS, rows_total); ++row) {
      const int b = row / (T + G), i = row % (T + G);
      const float v = dx[int64_t(row) * D + c];
      if (i >= T) {
        // global tokens: at most one global-token index per flush (G is tiny); flush when it changes
        if (gidx != i - T && gidx >= 0) {
          if (prow) prow[int64_t(gidx) * D + c] += accg;
          else atomicAdd(grads.global_tokens + int64_t(gidx) * D + c, accg);
          accg = 0.f;
        }
        gidx = i - T;
        accg += v;
      } else {
        const int r = b * T + i;
        dC[int64_t(r) * D + c] = __float2bfloat16_rn(v);
        const int t = row_task[r];
#pragma unroll
        for (int tt = 0; tt < MMAE_MAX_TASKS; ++tt)
          if (tt == t) accb[tt] += v;
      }
    }
    if (prow) {
      if (gidx >= 0) prow[int64_t(gidx) * D + c] += accg;
#pragma unroll
      for (int t = 0; t < MMAE_MAX_TASKS; ++t)
        if (t < num_tasks) prow[int64_t(G + t) * D + c] = accb[t];
      continue;
    }
    if (gidx >= 0) atomicAdd(grads.global_tokens + int64_t(gidx) * D + c, accg);
#pragma unroll
    for (int t = 0; t < MMAE_MAX_TASKS; ++t)
      if (t < num_tasks && accb[t] != 0.f) atomicAdd(grads.bias[t] + c, accb[t]);
  }
}

// dclass_emb[label, e] += dA[r, k_off + e*P*P + py*P + px] over the semseg rows; smem-privatised table per CTA
__global__ void __launch_bounds__(256) semseg_emb_bwd_kernel(const bf16* __restrict__ dA, int64_t ld_dA,
                                                             const int64_t* __restrict__ labels,
                                                             const int64_t* __restrict__ ids_keep,
                                                             const int* __restrict__ row_task,
                                                             const int* __restrict__ row_patch, int task, int T,
                                                             int rows, int rows_per_cta, int grid_w, int grid_h, int P,
                                                             int E, int num_classes, float* __restrict__ dtable) {
  pdl_prologue();
  extern __shared__ float tab[];  // [num_classes * E]
  for (int i = threadIdx.x; i < num_classes * E; i += blockDim.x) tab[i] = 0.f;
  __syncthreads();
  const int r0 = blockIdx.x * rows_per_cta;
  const int Wt = grid_w * P, Ht = grid_h * P;
  for (int r = r0; r < min(r0 + rows_per_cta, rows); ++r) {
    if (row_task[r] != task) continue;  // uniform per row
    const int b = r / T, p = row_patch[r];
    const int ph = p / grid_w, pw = p % grid_w;
    for (int k = threadIdx.x; k < E * P * P; k += blockDim.x) {
      const int e = k / (P * P), py = (k / P) % P, px = k % P;
      const int64_t label = labels[(int64_t(b) * Ht + ph * P + py) * Wt + pw * P + px];
      if (label >= 0 && label < num_classes) atomicAdd(&tab[label * E + e], __bfloat162float(dA[int64_t(r) * ld_dA + k]));
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < num_classes * E; i += blockDim.x)
    if (tab[i] != 0.f) atomicAdd(dtable + i, tab[i]);
}

// Deterministic form of semseg_emb_bwd_kernel: thread e owns column e of the CTA's table and adds its values in (row,
// pixel) order, so no two threads touch one entry; the CTA then writes its table to row blockIdx.x of `partial`, which
// colred_finalize adds up in CTA order.
__global__ void __launch_bounds__(256) semseg_emb_bwd_det_kernel(const bf16* __restrict__ dA, int64_t ld_dA,
                                                                 const int64_t* __restrict__ labels,
                                                                 const int* __restrict__ row_task,
                                                                 const int* __restrict__ row_patch, int task, int T,
                                                                 int rows, int rows_per_cta, int grid_w, int grid_h,
                                                                 int P, int E, int num_classes, float* __restrict__ partial) {
  pdl_prologue();
  extern __shared__ float tab[];  // [num_classes * E]
  for (int i = threadIdx.x; i < num_classes * E; i += blockDim.x) tab[i] = 0.f;
  __syncthreads();
  const int r0 = blockIdx.x * rows_per_cta;
  const int Wt = grid_w * P, Ht = grid_h * P;
  for (int r = r0; r < min(r0 + rows_per_cta, rows); ++r) {
    if (row_task[r] != task) continue;  // uniform per row
    const int b = r / T, p = row_patch[r];
    const int ph = p / grid_w, pw = p % grid_w;
    const int64_t* lrow = labels + (int64_t(b) * Ht + ph * P) * Wt + pw * P;
    const bf16* arow = dA + int64_t(r) * ld_dA;
    for (int e = threadIdx.x; e < E; e += blockDim.x) {
      for (int q = 0; q < P * P; ++q) {
        const int64_t label = lrow[int64_t(q / P) * Wt + q % P];
        if (label >= 0 && label < num_classes) tab[label * E + e] += __bfloat162float(arow[e * P * P + q]);
      }
    }
  }
  __syncthreads();
  float* prow = partial + int64_t(blockIdx.x) * num_classes * E;
  for (int i = threadIdx.x; i < num_classes * E; i += blockDim.x) prow[i] = tab[i];
}

// ---------------------------------------------------------------------------------------------------------------------
// decoder queries / context  (multimae/output_adapters.py:183-234)
//   queries[b, j]  = (visible ? ctx[b, rank] : mask_token) + task_emb[own] + pos[j]            j in own task's tokens
//   context[b, i]  = ctx[b, i] + task_emb[task(i)] + pos[patch(i)]   (i < T);   context[b, T+g] = ctx[b, T+g]
// One CTA row per output row; rows [0, B*P) are queries, rows [B*P, B*P + B*(T+G)) are context.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int DBF_ROWS = 16;   // rows per block: 4 row lanes x 4 rows in flight per thread
__global__ void __launch_bounds__(256) dec_build_kernel(const float* __restrict__ ctx, int64_t ld_ctx,  // row stride of ctx
                                                        mmae_decoder_index ix,
                                                        const float* __restrict__ mask_token, TaskEmbPtrs task_emb,
                                                        const float* __restrict__ pos,  // [P, Dd]
                                                        float* __restrict__ queries, float* __restrict__ context) {
  pdl_prologue();
  const int Dd = ix.dim, T = ix.num_visible, G = ix.num_global, P = ix.num_queries;
  const int nq_rows = ix.batch * P, n_rows = nq_rows + ix.batch * (T + G);
  const int rl = threadIdx.x >> 6, ct = threadIdx.x & 63;     // row lane, column thread (float4 columns ct, ct+64, ...)
  // resolve the 4 rows of this thread first (index loads in flight together), then move the data
  const float4 *base[4], *te[4], *pe[4];
  float4* dst[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int row = blockIdx.x * DBF_ROWS + u * 4 + rl;
    base[u] = te[u] = pe[u] = nullptr;
    dst[u] = nullptr;
    if (row >= n_rows) continue;
    if (row < nq_rows) {
      const int b = row / P, j = row % P;
      int rank = T;                                           // query_mode 1: every query starts from the mask token
      if (ix.query_mode == 0) {
        const int g = ix.tok_offset[ix.own_task] + j;
        rank = (int)ix.ids_restore[int64_t(b) * ix.total_tokens + g];
      }
      base[u] = rank < T ? reinterpret_cast<const float4*>(ctx + (int64_t(b) * (T + G) + rank) * ld_ctx)
                         : reinterpret_cast<const float4*>(mask_token);
      te[u] = ix.own_task >= 0 ? reinterpret_cast<const float4*>(task_emb.p[ix.own_task]) : nullptr;
      pe[u] = reinterpret_cast<const float4*>(pos + int64_t(j) * Dd);
      dst[u] = reinterpret_cast<float4*>(queries + int64_t(row) * Dd);
    } else {
      const int cr = row - nq_rows;
      const int b = cr / (T + G), i = cr % (T + G);
      base[u] = reinterpret_cast<const float4*>(ctx + int64_t(cr) * ld_ctx);
      dst[u] = reinterpret_cast<float4*>(context + int64_t(cr) * Dd);
      if (i < T) {
        const int g = (int)ix.ids_keep[int64_t(b) * T + i];
        int t = 0;
#pragma unroll
        for (int q = 1; q < MMAE_MAX_TASKS; ++q)
          if (q < ix.num_tasks && g >= ix.tok_offset[q]) t = q;
        te[u] = reinterpret_cast<const float4*>(task_emb.p[t]);
        pe[u] = reinterpret_cast<const float4*>(pos + int64_t(g - ix.tok_offset[t]) * Dd);
      }
    }
  }
  for (int c = ct; c < Dd / 4; c += 64) {
    float4 v[4], p4[4], a4[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (dst[u] == nullptr) continue;
      v[u] = __ldg(base[u] + c);
      p4[u] = pe[u] ? __ldg(pe[u] + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      a4[u] = te[u] ? __ldg(te[u] + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (dst[u] == nullptr) continue;
      // same association as the reference: (ctx + pos) + task_emb
      float4 o = make_float4(v[u].x + p4[u].x, v[u].y + p4[u].y, v[u].z + p4[u].z, v[u].w + p4[u].w);
      if (te[u]) o = make_float4(o.x + a4[u].x, o.y + a4[u].y, o.z + a4[u].z, o.w + a4[u].w);
      dst[u][c] = o;
    }
  }
}

// backward: dctx[b,i] = dcontext[b,i] (+ dqueries[b, g-start] if token i belongs to the own task);
// dmask_token += dqueries of masked positions; dtask_emb[t] += dcontext rows of task t (+ all dqueries for own).
// Block = 4 row lanes x 64 column threads (float4 columns), DB_ROWS rows per block, 4 rows in flight per thread.  The
// column sums (mask token, one task embedding per task) leave as one partial row per block [1 + MAX_TASKS segments of Dd]
// and are added up by colred_finalize_n: thousands of blocks x Dd x (1 + tasks) scalar atomics on ~5 KB serialise in L2.
constexpr int DB_ROWS = 64;
__global__ void __launch_bounds__(256) dec_build_bwd_kernel(const float* __restrict__ dqueries,
                                                            const float* __restrict__ dcontext, mmae_decoder_index ix,
                                                            float* __restrict__ dctx, float* __restrict__ partial) {
  pdl_prologue();
  extern __shared__ float4 dbred[];   // [4 row lanes][1 + MAX_TASKS][Dd / 4]
  const int Dd = ix.dim, T = ix.num_visible, G = ix.num_global, P = ix.num_queries;
  const int nq_rows = ix.batch * P, n_rows = nq_rows + ix.batch * (T + G);
  const int rl = threadIdx.x >> 6, ct = threadIdx.x & 63;
  const int d4 = Dd / 4;
  for (int c = ct; c < d4; c += 64) {
    float4 acc[1 + MMAE_MAX_TASKS];
#pragma unroll
    for (int k = 0; k < 1 + MMAE_MAX_TASKS; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int r0 = 0; r0 < DB_ROWS; r0 += 16) {
      // resolve 4 rows, load, then combine
      int kind[4], task[4];          // kind: -1 none, 0 query row, 1 context row of a visible token, 2 global-token row
      int64_t src_q[4], src_c[4];
      bool masked[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int row = blockIdx.x * DB_ROWS + r0 + u * 4 + rl;
        kind[u] = -1;
        task[u] = 0;
        src_q[u] = src_c[u] = -1;
        masked[u] = false;
        if (row >= n_rows) continue;
        if (row < nq_rows) {
          const int b = row / P, j = row % P;
          int rank = T;
          if (ix.query_mode == 0) {
            const int g = ix.tok_offset[ix.own_task] + j;
            rank = (int)ix.ids_restore[int64_t(b) * ix.total_tokens + g];
          }
          kind[u] = 0;
          task[u] = ix.own_task;                                // -1: no task embedding on the queries
          masked[u] = rank >= T;
          src_q[u] = int64_t(row);
        } else {
          const int cr = row - nq_rows;
          const int b = cr / (T + G), i = cr % (T + G);
          src_c[u] = int64_t(cr);
          kind[u] = 2;
          if (i < T) {
            const int g = (int)ix.ids_keep[int64_t(b) * T + i];
            int t = 0;
#pragma unroll
            for (int q = 1; q < MMAE_MAX_TASKS; ++q)
              if (q < ix.num_tasks && g >= ix.tok_offset[q]) t = q;
            kind[u] = 1;
            task[u] = t;
            if (ix.query_mode == 0 && t == ix.own_task) src_q[u] = int64_t(b) * P + (g - ix.tok_offset[t]);
          }
        }
      }
      float4 vq[4], vc[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        vq[u] = src_q[u] >= 0 ? __ldg(reinterpret_cast<const float4*>(dqueries + src_q[u] * Dd) + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        vc[u] = src_c[u] >= 0 ? __ldg(reinterpret_cast<const float4*>(dcontext + src_c[u] * Dd) + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (kind[u] < 0) continue;
        if (kind[u] == 0) {          // query row: mask token (if masked) and the own task embedding
          if (masked[u]) { acc[0].x += vq[u].x; acc[0].y += vq[u].y; acc[0].z += vq[u].z; acc[0].w += vq[u].w; }
#pragma unroll
          for (int t = 0; t < MMAE_MAX_TASKS; ++t)
            if (t == task[u]) { acc[1 + t].x += vq[u].x; acc[1 + t].y += vq[u].y; acc[1 + t].z += vq[u].z; acc[1 + t].w += vq[u].w; }
        } else {
          float4 v = vc[u];
          if (kind[u] == 1) {
#pragma unroll
            for (int t = 0; t < MMAE_MAX_TASKS; ++t)
              if (t == task[u]) { acc[1 + t].x += v.x; acc[1 + t].y += v.y; acc[1 + t].z += v.z; acc[1 + t].w += v.w; }
            if (src_q[u] >= 0) { v.x += vq[u].x; v.y += vq[u].y; v.z += vq[u].z; v.w += vq[u].w; }
          }
          reinterpret_cast<float4*>(dctx + src_c[u] * Dd)[c] = v;
        }
      }
    }
    // block reduction over the 4 row lanes, then this block's partial row
#pragma unroll
    for (int k = 0; k < 1 + MMAE_MAX_TASKS; ++k) dbred[(rl * (1 + MMAE_MAX_TASKS) + k) * d4 + c] = acc[k];
  }
  __syncthreads();
  const int nseg = 1 + MMAE_MAX_TASKS;
  for (int i = threadIdx.x; i < nseg * d4; i += blockDim.x) {
    float4 a = dbred[i];
#pragma unroll
    for (int r = 1; r < 4; ++r) {
      const float4 o = dbred[r * nseg * d4 + i];
      a.x += o.x; a.y += o.y; a.z += o.z; a.w += o.w;
    }
    reinterpret_cast<float4*>(partial + int64_t(blockIdx.x) * nseg * Dd)[i] = a;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// unpatchify: tokens [B*nh*nw, C*P*P] (c, py, px) -> image [B, C, nh*P, nw*P]   (output_adapters.py:277-280)
// One CTA per (b, patch row); one thread per (token, 4-column group): token-side accesses are contiguous across
// threads, image-side accesses are 16-byte pieces of P-pixel row segments.
// ---------------------------------------------------------------------------------------------------------------------
template <bool TO_IMAGE, typename TokT>
__global__ void __launch_bounds__(256) unpatchify_kernel(TokT* __restrict__ tok, int64_t ld_tok, float* __restrict__ img,
                                                         int B, int C, int nh, int nw, int P) {
  pdl_prologue();
  const int W = nw * P, H = nh * P;
  const int b = blockIdx.x / nh, ph = blockIdx.x % nh;
  const int groups_per_tok = C * P * P / 4;
  for (int idx = threadIdx.x; idx < nw * groups_per_tok; idx += blockDim.x) {
    const int pw = idx / groups_per_tok, gcol = (idx % groups_per_tok) * 4;
    const int c = gcol / (P * P), py = (gcol / P) % P, px = gcol % P;
    float* ip = img + ((int64_t(b) * C + c) * H + ph * P + py) * W + pw * P + px;
    TokT* tp = tok + (int64_t(b) * nh * nw + ph * nw + pw) * ld_tok + gcol;
    if constexpr (TO_IMAGE) {
      if constexpr (sizeof(TokT) == 4) {
        *reinterpret_cast<float4*>(ip) = __ldg(reinterpret_cast<const float4*>(tp));
      } else {
        const uint2 u = __ldg(reinterpret_cast<const uint2*>(tp));
        const float2 a = unpack_bf16x2(u.x), b2 = unpack_bf16x2(u.y);
        *reinterpret_cast<float4*>(ip) = make_float4(a.x, a.y, b2.x, b2.y);
      }
    } else {
      const float4 v = __ldg(reinterpret_cast<const float4*>(ip));
      if constexpr (sizeof(TokT) == 4) {
        *reinterpret_cast<float4*>(tp) = v;
      } else {
        uint2 o;
        o.x = pack_bf16x2(v.x, v.y);
        o.y = pack_bf16x2(v.z, v.w);
        *reinterpret_cast<uint2*>(tp) = o;
      }
    }
  }
}

// bf16 token rows <-> fp32 image through a shared-memory tile of one patch row (b, ph): both sides move whole lines
// (token rows with 16-byte accesses, image rows W pixels wide), instead of 64-byte image-row pieces per warp.
// smem: [nw][cols + 16] bf16 (the 32-byte row pad spreads the patch columns over the banks), cols = C * P * P.
template <bool TO_IMAGE>
__global__ void __launch_bounds__(256) unpatchify_tile_kernel(bf16* __restrict__ tok, int64_t ld_tok, float* __restrict__ img,
                                                              int B, int C, int nh, int nw, int P) {
  pdl_prologue();
  extern __shared__ __align__(16) uint8_t up_smem[];
  bf16* tile = reinterpret_cast<bf16*>(up_smem);
  const int W = nw * P, H = nh * P, cols = C * P * P, pitch = cols + 16;
  const int b = blockIdx.x / nh, ph = blockIdx.x % nh;
  bf16* trow0 = tok + (int64_t(b) * nh * nw + int64_t(ph) * nw) * ld_tok;
  const int vec_per_row = cols / 8;
  if constexpr (TO_IMAGE) {
    for (int idx = threadIdx.x; idx < nw * vec_per_row; idx += blockDim.x) {
      const int pw = idx / vec_per_row, v = idx % vec_per_row;
      *reinterpret_cast<uint4*>(tile + pw * pitch + v * 8) = ld_stream_16(trow0 + int64_t(pw) * ld_tok + v * 8);
    }
    __syncthreads();
  }
  // image side: rows (c, py), 4 consecutive pixels per thread
  const int quads = W / 4, rows = C * P;
  for (int idx = threadIdx.x; idx < rows * quads; idx += blockDim.x) {
    const int r = idx / quads, x = (idx % quads) * 4;
    const int c = r / P, py = r % P, pw = x / P, px = x % P;
    float* ip = img + ((int64_t(b) * C + c) * H + ph * P + py) * W + x;
    bf16* tp = tile + pw * pitch + (c * P + py) * P + px;
    if constexpr (TO_IMAGE) {
      const uint2 u = *reinterpret_cast<const uint2*>(tp);
      const float2 a = unpack_bf16x2(u.x), b2 = unpack_bf16x2(u.y);
      *reinterpret_cast<float4*>(ip) = make_float4(a.x, a.y, b2.x, b2.y);
    } else {
      const float4 v = __ldg(reinterpret_cast<const float4*>(ip));
      uint2 o;
      o.x = pack_bf16x2(v.x, v.y);
      o.y = pack_bf16x2(v.z, v.w);
      *reinterpret_cast<uint2*>(tp) = o;
    }
  }
  if constexpr (!TO_IMAGE) {
    __syncthreads();
    for (int idx = threadIdx.x; idx < nw * vec_per_row; idx += blockDim.x) {
      const int pw = idx / vec_per_row, v = idx % vec_per_row;
      *reinterpret_cast<uint4*>(trow0 + int64_t(pw) * ld_tok + v * 8) = *reinterpret_cast<const uint4*>(tile + pw * pitch + v * 8);
    }
  }
}

// shared-memory tile variant usable: 16-byte token vectors, 4-pixel quads inside a patch row, tile within the opt-in limit
static bool unpatchify_tile_ok(int64_t ld_tok, int C, int nw, int P, const void* tok, size_t* smem) {
  const int cols = C * P * P;
  *smem = size_t(nw) * (cols + 16) * sizeof(bf16);
  return cols % 8 == 0 && ld_tok % 8 == 0 && P % 4 == 0 && (reinterpret_cast<uintptr_t>(tok) & 15) == 0 && *smem <= 200 * 1024;
}

__global__ void cast2d_kernel(const float* __restrict__ src, int64_t ld_src, bf16* __restrict__ dst, int64_t ld_dst,
                              int rows, int cols) {
  pdl_prologue();
  const int r = blockIdx.y;
  for (int c = (blockIdx.x * blockDim.x + threadIdx.x) * 4; c < cols; c += gridDim.x * blockDim.x * 4) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(src + int64_t(r) * ld_src + c));
    uint2 o;
    o.x = pack_bf16x2(v.x, v.y);
    o.y = pack_bf16x2(v.z, v.w);
    *reinterpret_cast<uint2*>(dst + int64_t(r) * ld_dst + c) = o;
  }
}

}  // namespace

// ---- internal launchers shared with modules.cu ------------------------------------------------------------------------
int launch_embed_gather(const mmae_embed_layout& L, const mmae_embed_inputs& in, const int64_t* ids_keep, int B, int T,
                        bf16* A, int* row_task, int* row_patch, cudaStream_t st) {
  launch_k(embed_gather_kernel, B * T, 256, 0, st, L, in, ids_keep, T, A, row_task, row_patch);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

int launch_embed_assemble(const float* Cmat, const mmae_embed_params& prm, const int* row_task, const int* row_patch,
                          int B, int T, int G, int D, float* x, cudaStream_t st) {
  launch_k(embed_assemble_kernel, B * (T + G), 256, 0, st, Cmat, prm, row_task, row_patch, T, G, D, x);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

int launch_embed_assemble_bwd(const float* dx, int B, int T, int G, int D, const int* row_task, bf16* dC,
                              const mmae_embed_grads& grads, int num_tasks, cudaStream_t st) {
  const int blocks = ceil_div(B * (T + G), EB_ROWS);
  float* partial = nullptr;
  if (deterministic()) {
    MMAE_CHECK(G + num_tasks <= 9, MMAE_ERR_UNSUPPORTED,
               "embedding backward: deterministic mode adds at most 9 global-token / bias gradients (G=%d, tasks=%d)", G,
               num_tasks);
    partial = colred_scratch(size_t(blocks) * (G + num_tasks) * D, st);
    if (!partial) return MMAE_ERR_CUDA;
  }
  launch_k(embed_assemble_bwd_kernel, blocks, 256, 0, st, dx, T, G, D, B, row_task, dC, grads, num_tasks, partial);
  count_launch();
  MMAE_LAUNCH_OK();
  if (!partial || G + num_tasks == 0) return MMAE_OK;
  ColredDst dst;
  for (int k = 0; k < 9; ++k) dst.p[k] = nullptr;
  for (int g = 0; g < G; ++g) dst.p[g] = grads.global_tokens ? grads.global_tokens + int64_t(g) * D : nullptr;
  for (int t = 0; t < num_tasks; ++t) dst.p[G + t] = grads.bias[t];
  return colred_finalize_n(partial, blocks, (G + num_tasks) * D, D, dst, G + num_tasks, st);
}

int launch_semseg_emb_bwd(const bf16* dA, int64_t ld_dA, const int64_t* labels, const int64_t* ids_keep,
                          const int* row_task, const int* row_patch, int task, int T, int rows, int grid_w, int grid_h,
                          int P, int E, int num_classes, float* dtable, cudaStream_t st) {
  const size_t smem = size_t(num_classes) * E * 4;
  MMAE_CHECK(smem <= 96 * 1024, MMAE_ERR_UNSUPPORTED, "class embedding table too large for the smem-privatised scatter");
  static bool configured = false;
  if (!configured) {
    MMAE_CUDA_OK(cudaFuncSetAttribute(semseg_emb_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    configured = true;
  }
  const int ctas = std::min(rows, 2 * reduce_sm_count());
  const int rows_per_cta = ceil_div(rows, ctas);
  if (deterministic()) {
    static bool det_configured = false;
    if (!det_configured) {
      MMAE_CUDA_OK(cudaFuncSetAttribute(semseg_emb_bwd_det_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
      det_configured = true;
    }
    const int grid = ceil_div(rows, rows_per_cta);
    float* partial = colred_scratch(size_t(grid) * num_classes * E, st);
    if (!partial) return MMAE_ERR_CUDA;
    launch_k(semseg_emb_bwd_det_kernel, grid, 256, smem, st, dA, ld_dA, labels, row_task, row_patch, task, T, rows,
             rows_per_cta, grid_w, grid_h, P, E, num_classes, partial);
    count_launch();
    MMAE_LAUNCH_OK();
    return colred_finalize(partial, grid, num_classes * E, num_classes * E, dtable, nullptr, nullptr, st);
  }
  launch_k(semseg_emb_bwd_kernel, ceil_div(rows, rows_per_cta), 256, smem, st, dA, ld_dA, labels, ids_keep, row_task,
                                                                          row_patch, task, T, rows, rows_per_cta,
                                                                          grid_w, grid_h, P, E, num_classes, dtable);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

int launch_dec_build(const float* ctx, int64_t ld_ctx, const mmae_decoder_index& ix, const float* mask_token,
                     const TaskEmbPtrs& task_emb, const float* pos, float* queries, float* context, cudaStream_t st) {
  const int rows = ix.batch * ix.num_queries + ix.batch * (ix.num_visible + ix.num_global);
  launch_k(dec_build_kernel, ceil_div(rows, DBF_ROWS), 256, 0, st, ctx, ld_ctx, ix, mask_token, task_emb, pos, queries, context);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

int launch_dec_build_bwd(const float* dqueries, const float* dcontext, const mmae_decoder_index& ix, float* dctx,
                         float* dmask_token, const TaskEmbGradPtrs& dtask_emb, cudaStream_t st) {
  const int rows = ix.batch * ix.num_queries + ix.batch * (ix.num_visible + ix.num_global);
  const int blocks = ceil_div(rows, DB_ROWS);
  constexpr int NSEG = 1 + MMAE_MAX_TASKS;
  float* partial = colred_scratch(size_t(blocks) * NSEG * ix.dim, st);
  if (!partial) return MMAE_ERR_CUDA;
  const size_t smem = size_t(4) * NSEG * ix.dim * sizeof(float);
  static bool configured = false;
  if (!configured) {
    MMAE_CUDA_OK(cudaFuncSetAttribute(dec_build_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * NSEG * 1024 * 4));
    configured = true;
  }
  launch_k(dec_build_bwd_kernel, blocks, 256, smem, st, dqueries, dcontext, ix, dctx, partial);
  count_launch();
  MMAE_LAUNCH_OK();
  ColredDst dst;
  dst.p[0] = dmask_token;
  for (int t = 0; t < MMAE_MAX_TASKS; ++t) dst.p[1 + t] = dtask_emb.p[t];   // null entries are skipped
  return colred_finalize_n(partial, blocks, NSEG * ix.dim, ix.dim, dst, NSEG, st);
}

int launch_cast2d(const float* src, int64_t ld_src, bf16* dst, int64_t ld_dst, int rows, int cols, cudaStream_t st) {
  dim3 grid(std::max(1, std::min(8, ceil_div(cols, 1024))), rows);
  launch_k(cast2d_kernel, grid, 256, 0, st, src, ld_src, dst, ld_dst, rows, cols);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

}  // namespace mmae

using namespace mmae;

extern "C" int mmae_unpatchify(const float* tokens, int64_t ld_tok, float* image, int B, int C, int nh, int nw, int P,
                               void* stream) {
  MMAE_CHECK(tokens && image && B > 0 && C > 0 && nh > 0 && nw > 0 && P > 0, MMAE_ERR_ARG, "mmae_unpatchify: bad args");
  MMAE_CHECK(P % 4 == 0 && ld_tok % 4 == 0, MMAE_ERR_UNSUPPORTED, "mmae_unpatchify: P and ld must be multiples of 4");
  launch_k(unpatchify_kernel<true, const float>, B * nh, 256, 0, reinterpret_cast<cudaStream_t>(stream), tokens, ld_tok, image, B, C, nh, nw, P);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

extern "C" int mmae_patchify(const float* image, float* tokens, int64_t ld_tok, int B, int C, int nh, int nw, int P, void* stream) {
  MMAE_CHECK(tokens && image && B > 0 && C > 0 && nh > 0 && nw > 0 && P > 0, MMAE_ERR_ARG, "mmae_patchify: bad args");
  MMAE_CHECK(P % 4 == 0 && ld_tok % 4 == 0, MMAE_ERR_UNSUPPORTED, "mmae_patchify: P and ld must be multiples of 4");
  launch_k(unpatchify_kernel<false, float>, B * nh, 256, 0, reinterpret_cast<cudaStream_t>(stream), tokens, ld_tok,
           const_cast<float*>(image), B, C, nh, nw, P);
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

extern "C" int mmae_unpatchify_bf16(const void* tokens_bf16, int64_t ld_tok, float* image, int B, int C, int nh, int nw,
                                    int P, void* stream) {
  MMAE_CHECK(tokens_bf16 && image && B > 0 && C > 0 && nh > 0 && nw > 0 && P > 0, MMAE_ERR_ARG, "mmae_unpatchify_bf16: bad args");
  MMAE_CHECK(P % 4 == 0 && ld_tok % 4 == 0, MMAE_ERR_UNSUPPORTED, "mmae_unpatchify_bf16: P and ld must be multiples of 4");
  size_t smem = 0;
  if (unpatchify_tile_ok(ld_tok, C, nw, P, tokens_bf16, &smem)) {
    static size_t configured = 0;
    if (smem > configured) {
      MMAE_CUDA_OK(cudaFuncSetAttribute(unpatchify_tile_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      configured = smem;
    }
    launch_k(unpatchify_tile_kernel<true>, B * nh, 256, smem, reinterpret_cast<cudaStream_t>(stream),
             reinterpret_cast<bf16*>(const_cast<void*>(tokens_bf16)), ld_tok, image, B, C, nh, nw, P);
  } else {
    launch_k(unpatchify_kernel<true, const bf16>, B * nh, 256, 0, reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const bf16*>(tokens_bf16), ld_tok, image, B, C, nh, nw, P);
  }
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}

extern "C" int mmae_patchify_bf16(const float* image, void* tokens_bf16, int64_t ld_tok, int B, int C, int nh, int nw,
                                  int P, void* stream) {
  MMAE_CHECK(tokens_bf16 && image && B > 0 && C > 0 && nh > 0 && nw > 0 && P > 0, MMAE_ERR_ARG,
             "mmae_patchify_bf16: bad args");
  MMAE_CHECK(P % 4 == 0 && ld_tok % 4 == 0, MMAE_ERR_UNSUPPORTED, "mmae_patchify_bf16: P and ld must be multiples of 4");
  size_t smem = 0;
  if (unpatchify_tile_ok(ld_tok, C, nw, P, tokens_bf16, &smem)) {
    static size_t configured = 0;
    if (smem > configured) {
      MMAE_CUDA_OK(cudaFuncSetAttribute(unpatchify_tile_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      configured = smem;
    }
    launch_k(unpatchify_tile_kernel<false>, B * nh, 256, smem, reinterpret_cast<cudaStream_t>(stream),
             reinterpret_cast<bf16*>(tokens_bf16), ld_tok, const_cast<float*>(image), B, C, nh, nw, P);
  } else {
    launch_k(unpatchify_kernel<false, bf16>, B * nh, 256, 0, reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<bf16*>(tokens_bf16), ld_tok, const_cast<float*>(image), B, C, nh, nw, P);
  }
  count_launch();
  MMAE_LAUNCH_OK();
  return MMAE_OK;
}
