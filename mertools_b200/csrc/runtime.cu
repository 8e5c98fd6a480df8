// runtime.cu — host-side plumbing of libmer_b200.so: error string, device checks, TMA descriptor
// encoding through the driver entry point (resolved at run time so the library links without
// libcuda and loads on a GPU-less build box), and the thin extern "C" wrappers of the kernel-level
// entry points declared in include/mer_b200.h.
#include <cuda_profiler_api.h>
#include <stdarg.h>
#include <stdlib.h>

#include <vector>

#include "mer_common.cuh"
#include "mer_kernels.h"

static thread_local char g_err[1024] = "";

void mer_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// ---- optional per-launch timing (bench.py roofline): CUDA events on the launching stream ----
namespace {
struct ProfSlot { cudaEvent_t a, b; double work; int klass; };
bool g_prof_on = false;
int g_prof_paused = 0;              // > 0: launches inside a composite op are not recorded on their own
std::vector<ProfSlot> g_prof;       // slots in use since the last enable
std::vector<ProfSlot> g_prof_pool;  // recycled event pairs
}  // namespace

void mer_prof_pause(int on) { g_prof_paused += on ? 1 : -1; }

// ---- capture windows for `ncu --profile-from-start off` (scripts/profile_kernels.sh) ----
// MER_CUPROF="klass:first:count,..." brackets launches [first, first + count) of a kernel class (the klass ids of
// mer_prof_begin) with cudaProfilerStart / cudaProfilerStop, so that ONE profiled process captures a few launches of
// every kernel of the step instead of one process per kernel.  Unset (the product): two integer compares per launch.
namespace {
struct CuprofWin { int klass, first, count, seen; };
std::vector<CuprofWin> g_cuprof;
int g_cuprof_state = 0;  // 0 = environment not parsed, 1 = no windows, 2 = windows present
bool g_cuprof_open = false;

void cuprof_parse() {
  g_cuprof_state = 1;
  const char* e = getenv("MER_CUPROF");
  if (!e) return;
  while (*e) {
    CuprofWin w = {0, 0, 0, 0};
    int used = 0;
    if (sscanf(e, "%d:%d:%d%n", &w.klass, &w.first, &w.count, &used) == 3 && w.count > 0) g_cuprof.push_back(w);
    e += used;
    while (*e && *e != ',') ++e;
    if (*e == ',') ++e;
    if (used == 0 && !*e) break;
  }
  if (!g_cuprof.empty()) g_cuprof_state = 2;
}

void cuprof_begin(int klass) {
  if (g_cuprof_state == 0) cuprof_parse();
  if (g_cuprof_state != 2) return;
  for (auto& w : g_cuprof) {
    if (w.klass != klass) continue;
    const int n = w.seen++;
    if (n >= w.first && n < w.first + w.count && !g_cuprof_open) {
      cudaProfilerStart();
      g_cuprof_open = true;
    }
  }
}

void cuprof_end() {
  if (g_cuprof_open) {
    cudaProfilerStop();
    g_cuprof_open = false;
  }
}
}  // namespace

int mer_prof_begin(int klass, double work, cudaStream_t stream) {
  if (g_prof_paused == 0) cuprof_begin(klass);
  if (!g_prof_on || g_prof_paused > 0) return -1;
  ProfSlot slot;
  if (!g_prof_pool.empty()) {
    slot = g_prof_pool.back();
    g_prof_pool.pop_back();
  } else {
    if (cudaEventCreate(&slot.a) != cudaSuccess || cudaEventCreate(&slot.b) != cudaSuccess) return -1;
  }
  slot.work = work;
  slot.klass = klass;
  cudaEventRecord(slot.a, stream);
  g_prof.push_back(slot);
  return (int)g_prof.size() - 1;
}

void mer_prof_end(int slot, cudaStream_t stream) {
  if (g_prof_paused == 0) cuprof_end();
  if (slot >= 0 && slot < (int)g_prof.size()) cudaEventRecord(g_prof[slot].b, stream);
}

extern "C" int mer_profile_enable(int on) {
  for (auto& sl : g_prof) g_prof_pool.push_back(sl);
  g_prof.clear();
  g_prof_on = on != 0;
  return 0;
}

// Sum of the event-timed durations and algorithmic work (FLOPs, or bytes for the HBM-bound classes) of the
// launches of `klass` recorded since mer_profile_enable(1).  Synchronises on the recorded events.
extern "C" int mer_profile_collect(int klass, double* total_ms, double* total_work, int* launches) {
  double ms = 0.0, wk = 0.0;
  int n = 0;
  for (auto& sl : g_prof) {
    if (sl.klass != klass) continue;
    MER_CUDA_CHECK(cudaEventSynchronize(sl.b));
    float t = 0.f;
    MER_CUDA_CHECK(cudaEventElapsedTime(&t, sl.a, sl.b));
    ms += t;
    wk += sl.work;
    ++n;
  }
  if (total_ms) *total_ms = ms;
  if (total_work) *total_work = wk;
  if (launches) *launches = n;
  return 0;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) ==
            cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

int mer_make_tmap(CUtensorMap* out, CUtensorMapDataType dtype, int rank, const void* base,
                  const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                  CUtensorMapSwizzle swizzle) {
  PFN_encodeTiled enc = get_encode();
  MER_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i + 1 < rank) gstr[i] = strides_bytes[i];
  }
  CUresult r = enc(out, dtype, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    mer_set_error(
        "cuTensorMapEncodeTiled failed (CUresult %d): rank %d dims [%llu %llu %llu %llu] strides "
        "[%llu %llu %llu] box [%u %u %u %u] base %p",
        (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
        (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0),
        (unsigned long long)(rank > 1 ? strides_bytes[0] : 0),
        (unsigned long long)(rank > 2 ? strides_bytes[1] : 0),
        (unsigned long long)(rank > 3 ? strides_bytes[2] : 0), box[0], rank > 1 ? box[1] : 0,
        rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0, base);
    return 3;
  }
  return 0;
}

int mer_num_sms() {
  static int cache[64] = {};
  const int dev = MerPerDevice::current();
  int& n = cache[dev];
  if (!n) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

static long long g_launches = 0;
void mer_count_launches(int n) { g_launches += n; }

extern "C" {

long long mer_launch_count(void) { return g_launches; }

const char* mer_last_error(void) { return g_err; }

int mer_abi_version(void) { return 4; }

int mer_check_device(void) {
  int dev = 0, major = 0, minor = 0;
  MER_CUDA_CHECK(cudaGetDevice(&dev));
  MER_CUDA_CHECK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  MER_CUDA_CHECK(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  MER_REQUIRE(major == 9 && minor == 0, "libmer_b200 needs an sm_90a device (H100), found sm_%d%d", major, minor);
  return 0;
}

int mer_gemm(const MerGemmDesc* desc, void* stream) {
  return mer_gemm_launch(desc, static_cast<cudaStream_t>(stream));
}

int mer_layernorm(const float* x, const float* gamma, const float* beta, float* y, void* y_split,
                  float* acc, long long rows, int dim, float eps, int flags, void* stream) {
  return mer_layernorm_launch(x, gamma, beta, y, y_split, acc, rows, dim, eps, flags,
                              static_cast<cudaStream_t>(stream));
}

int mer_attention(const float* qkv, const float* vt, long long vt_ld, float* ctx,
                  const int32_t* cu_seqlens, int n_seq, long long tokens, int max_seqlen, int heads,
                  int flags, void* stream) {
  return mer_attention_launch(qkv, vt, vt_ld, ctx, cu_seqlens, n_seq, tokens, max_seqlen, heads, flags,
                              static_cast<cudaStream_t>(stream));
}

}  // extern "C"
