// Host-side runtime glue of the C ABI: error strings, launch accounting, TMA tensor-map encoding.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "../../include/multimae_b200.h"

namespace mmae {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

// ---- optional per-launch device timing of the GEMM kernel (bench.py roofline leg; off by default) -------------------
struct GemmProfile {
  bool on = false;
  std::vector<cudaEvent_t> begin, end;
  std::vector<double> flops;
  std::vector<long long> shape;   // packed M, N, K, flags per launch (4 entries each)
  size_t used = 0;
};
static GemmProfile g_prof;
static const size_t kProfCap = 8192;

bool gemm_profile_begin(cudaStream_t st, double flops, int M, int N, int K, int flags) {
  if (!g_prof.on || g_prof.used >= kProfCap) return false;
  if (g_prof.begin.size() <= g_prof.used) {
    cudaEvent_t a, b;
    if (cudaEventCreate(&a) != cudaSuccess || cudaEventCreate(&b) != cudaSuccess) return false;
    g_prof.begin.push_back(a);
    g_prof.end.push_back(b);
    g_prof.flops.push_back(0.0);
    for (int i = 0; i < 4; ++i) g_prof.shape.push_back(0);
  }
  g_prof.flops[g_prof.used] = flops;
  g_prof.shape[4 * g_prof.used + 0] = M;
  g_prof.shape[4 * g_prof.used + 1] = N;
  g_prof.shape[4 * g_prof.used + 2] = K;
  g_prof.shape[4 * g_prof.used + 3] = flags;
  cudaEventRecord(g_prof.begin[g_prof.used], st);
  return true;
}
void gemm_profile_end(cudaStream_t st) {
  cudaEventRecord(g_prof.end[g_prof.used], st);
  g_prof.used++;
}

// SM budget of the persistent kernels: the physical SM count, or fewer (MMAE_SM_BUDGET / mmae_set_sm_budget).  Data-parallel
// runs overlap NCCL's all-reduce CTAs with the backward: a persistent GEMM that claims every SM runs a second wave on the
// SMs NCCL holds; sized to SMs - NCCL CTAs it finishes in one.
static int g_sm_budget = []() {
  const char* e = getenv("MMAE_SM_BUDGET");
  return e ? atoi(e) : 0;
}();
int sm_count() {
  static int cached = 0;
  if (cached == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&cached, cudaDevAttrMultiProcessorCount, dev);
    if (cached <= 0) cached = 132;
  }
  return g_sm_budget > 0 && g_sm_budget < cached ? g_sm_budget : cached;
}

typedef CUresult (*encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                    CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                    CUtensorMapFloatOOBfill);

static encode_tiled_fn get_encode_fn() {
  static encode_tiled_fn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) {
      set_last_error("cuTensorMapEncodeTiled entry point unavailable (%s)", cudaGetErrorString(e));
      return nullptr;
    }
    fn = reinterpret_cast<encode_tiled_fn>(p);
  }
  return fn;
}

int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                      uint32_t box_cols, uint32_t box_rows) {
  encode_tiled_fn fn = get_encode_fn();
  if (!fn) return MMAE_ERR_CUDA;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled(2d) failed: %d (rows=%llu cols=%llu ld=%llu box=%ux%u base=%p)", (int)r,
                   (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld, box_cols, box_rows,
                   base);
    return MMAE_ERR_CUDA;
  }
  return MMAE_OK;
}

// Output-tile map for the GEMM epilogue's TMA stores / reductions: box = 64 rows x 32 columns, dense (no swizzle).
// `ld` in elements.
int make_tmap_2d_store(CUtensorMap* out, const void* base, int elem_bytes, uint64_t rows, uint64_t cols, uint64_t ld) {
  encode_tiled_fn fn = get_encode_fn();
  if (!fn) return MMAE_ERR_CUDA;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * (uint64_t)elem_bytes};
  cuuint32_t box[2] = {32, 64};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                  const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled(store) failed: %d (rows=%llu cols=%llu ld=%llu base=%p)", (int)r,
                   (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld, base);
    return MMAE_ERR_CUDA;
  }
  return MMAE_OK;
}

// Output-tile map of the GEMM's whole-slab epilogue: box = 64 rows x 128 bytes (64 bf16 or 32 fp32 columns), staged
// with the 128B swizzle so that the accumulator fragments go to shared memory without bank conflicts.
int make_tmap_2d_store_sw128(CUtensorMap* out, const void* base, int elem_bytes, uint64_t rows, uint64_t cols,
                             uint64_t ld) {
  encode_tiled_fn fn = get_encode_fn();
  if (!fn) return MMAE_ERR_CUDA;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * (uint64_t)elem_bytes};
  cuuint32_t box[2] = {128u / (uint32_t)elem_bytes, 64};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                  const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled(store, sw128) failed: %d (rows=%llu cols=%llu ld=%llu base=%p)", (int)r,
                   (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld, base);
    return MMAE_ERR_CUDA;
  }
  return MMAE_OK;
}

int make_tmap_3d_bf16(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t s1,
                      uint64_t s2, uint32_t b0, uint32_t b1, uint32_t b2) {
  encode_tiled_fn fn = get_encode_fn();
  if (!fn) return MMAE_ERR_CUDA;
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {s1 * 2, s2 * 2};
  cuuint32_t box[3] = {b0, b1, b2};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled(3d) failed: %d", (int)r);
    return MMAE_ERR_CUDA;
  }
  return MMAE_OK;
}

// 3D bf16 store map [d2][d1][d0] (element strides s1, s2): box b0 x b1 x b2 with b0 * 2 bytes = the swizzle span
// (128: SWIZZLE_128B, 64: SWIZZLE_64B); out-of-bounds parts of a stored box are clipped by the TMA unit
int make_tmap_3d_bf16_store(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t s1,
                            uint64_t s2, uint32_t b0, uint32_t b1, uint32_t b2) {
  encode_tiled_fn fn = get_encode_fn();
  if (!fn) return MMAE_ERR_CUDA;
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {s1 * 2, s2 * 2};
  cuuint32_t box[3] = {b0, b1, b2};
  cuuint32_t estr[3] = {1, 1, 1};
  const CUtensorMapSwizzle sw = b0 * 2 == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : (b0 * 2 == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE);
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled(3d store) failed: %d", (int)r);
    return MMAE_ERR_CUDA;
  }
  return MMAE_OK;
}

}  // namespace mmae

// ---------------------------------------------------------------------------------------------------------------------
// bf16 weight mirror: a flat fp32 parameter buffer (FlatAdamW's) may register a bf16 twin of the same length.  The module
// orchestrators then take GEMM weight operands straight from the twin instead of casting ~117 tensors per step, and
// mmae_adamw_step refreshes the twin in the same pass that updates the fp32 master copy.
// ---------------------------------------------------------------------------------------------------------------------
namespace mmae {
namespace {
struct MirrorEntry {
  const float* f32;
  bf16* b16;
  int64_t n;
};
constexpr int MAX_MIRRORS = 8;
MirrorEntry g_mirror[MAX_MIRRORS];
int g_num_mirrors = 0;
}  // namespace

const bf16* mirror_lookup(const float* w) {
  for (int i = 0; i < g_num_mirrors; ++i) {
    const MirrorEntry& e = g_mirror[i];
    if (w >= e.f32 && w < e.f32 + e.n) {
      const int64_t off = w - e.f32;
      if (off % 8 != 0) return nullptr;   // TMA needs a 16-byte aligned bf16 base
      return e.b16 + off;
    }
  }
  return nullptr;
}
}  // namespace mmae

extern "C" int mmae_weight_mirror_register(const float* params_f32, void* mirror_bf16, int64_t n) {
  using namespace mmae;
  MMAE_CHECK(params_f32 != nullptr, MMAE_ERR_ARG, "mmae_weight_mirror_register: null parameter buffer");
  int at = -1;
  for (int i = 0; i < g_num_mirrors; ++i)
    if (g_mirror[i].f32 == params_f32) at = i;
  if (mirror_bf16 == nullptr || n <= 0) {   // unregister
    if (at >= 0) g_mirror[at] = g_mirror[--g_num_mirrors];
    return MMAE_OK;
  }
  MMAE_CHECK((reinterpret_cast<uintptr_t>(params_f32) & 31) == 0 && (reinterpret_cast<uintptr_t>(mirror_bf16) & 15) == 0,
             MMAE_ERR_ARG, "mmae_weight_mirror_register: buffers must be 32-byte (fp32) / 16-byte (bf16) aligned");
  if (at < 0) {
    MMAE_CHECK(g_num_mirrors < MAX_MIRRORS, MMAE_ERR_UNSUPPORTED, "mmae_weight_mirror_register: too many mirrors");
    at = g_num_mirrors++;
  }
  g_mirror[at] = {params_f32, reinterpret_cast<bf16*>(mirror_bf16), n};
  return MMAE_OK;
}

namespace mmae {
// Programmatic dependent launch is OFF by default (MMAE_PDL=1 / mmae_set_pdl(1) turns it on).  Found in round 2: after
// griddepcontrol.wait a non-coherent load (ld.global.nc, i.e. __ldg / const __restrict__ / L1::no_allocate streaming loads,
// which most kernels here use for their inputs) can still hit a stale L1 line of a buffer the PREVIOUS kernel has just
// rewritten - the L1 invalidation of an ordinary kernel boundary does not happen for a programmatically launched
// dependent.  At the training shapes the lines are evicted by the ~100 MB every kernel streams, at small shapes (tests) the
// fp32 attention kernels read stale gradients.  Captured CUDA graphs never used PDL (train_step.py), so the measured step
// is unaffected; eager launches lose the ~3.5 % PDL gave them.
static int g_pdl = []() {
  const char* e = getenv("MMAE_PDL");
  return e ? atoi(e) : 0;
}();
bool pdl_enabled() { return g_pdl != 0; }
}  // namespace mmae
namespace mmae {
static int g_deterministic = 0;
bool deterministic() { return g_deterministic != 0; }
int reduce_sm_count() { return g_deterministic ? DET_SM_COUNT : sm_count(); }
}  // namespace mmae
extern "C" int mmae_set_deterministic(int enable) {
  mmae::g_deterministic = enable != 0;
  return MMAE_OK;
}
extern "C" int mmae_set_sm_budget(int sms) {
  mmae::g_sm_budget = sms;
  return MMAE_OK;
}
extern "C" int mmae_set_pdl(int enable) {
  mmae::g_pdl = enable != 0;
  return MMAE_OK;
}

extern "C" int mmae_abi_version(void) { return MMAE_ABI_VERSION; }
extern "C" const char* mmae_last_error(void) { return mmae::g_err; }
extern "C" int64_t mmae_launch_count(void) { return mmae::g_launches.load(std::memory_order_relaxed); }

extern "C" int mmae_profile_gemm(int enable) {
  mmae::g_prof.on = enable != 0;
  if (enable) mmae::g_prof.used = 0;   // (1) resets and starts, (0) stops and keeps the records for _read
  return MMAE_OK;
}
extern "C" int mmae_profile_gemm_read(double* flops, double* ms, int64_t* launches) {
  double f = 0.0, t = 0.0;
  for (size_t i = 0; i < mmae::g_prof.used; ++i) {
    if (cudaEventSynchronize(mmae::g_prof.end[i]) != cudaSuccess) return MMAE_ERR_CUDA;
    float e = 0.f;
    if (cudaEventElapsedTime(&e, mmae::g_prof.begin[i], mmae::g_prof.end[i]) != cudaSuccess) return MMAE_ERR_CUDA;
    t += e;
    f += mmae::g_prof.flops[i];
  }
  if (flops) *flops = f;
  if (ms) *ms = t;
  if (launches) *launches = (int64_t)mmae::g_prof.used;
  return MMAE_OK;
}

// one line per recorded launch: "M N K flags ms" (flags: bit0 a_mn, bit1 b_mn, bit2 unused, bit3 ordered split-K, bit4
// asynchronous epilogue, bits 8.. split_k); returns
// bytes written
extern "C" int64_t mmae_profile_gemm_dump(char* buf, int64_t cap) {
  int64_t off = 0;
  for (size_t i = 0; i < mmae::g_prof.used; ++i) {
    if (cudaEventSynchronize(mmae::g_prof.end[i]) != cudaSuccess) return -1;
    float e = 0.f;
    cudaEventElapsedTime(&e, mmae::g_prof.begin[i], mmae::g_prof.end[i]);
    const int n = snprintf(buf + off, (size_t)(cap - off), "%lld %lld %lld %lld %.6f\n", mmae::g_prof.shape[4 * i],
                           mmae::g_prof.shape[4 * i + 1], mmae::g_prof.shape[4 * i + 2], mmae::g_prof.shape[4 * i + 3], e);
    if (n <= 0 || off + n >= cap) break;
    off += n;
  }
  return off;
}
