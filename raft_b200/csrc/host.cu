// Host code every family shares: the error state, the workspace check, the tensor-map encoder, the device check and
// the profiling ring (b2d_profile_begin / b2d_profile_end).
#include <cuda.h>
#include <cuda_runtime.h>
#include <algorithm>
#include <atomic>
#include <mutex>
#include <string>
#include <vector>

#include "host.cuh"

namespace b2d {

static thread_local std::string g_err;

int fail(int code, const std::string& msg)
{
  g_err = msg;
  return code;
}

int check_workspace(const void* ws, size_t bytes, size_t need, size_t align)
{
  if (need > 0 && (!ws || bytes < need))
    return fail(B2D_ERR_WORKSPACE, "workspace too small: need " + std::to_string(need) + " bytes");
  if (reinterpret_cast<uintptr_t>(ws) % align) return fail(B2D_ERR_INVALID_ARG, "workspace must be 256-byte aligned");
  return B2D_OK;
}

// ------------------------------------------------------------------------------------------
// TMA descriptor encode through the driver entry point (no link-time libcuda dependency, so the
// library still loads -- and reports a clean error -- on a machine without a driver).
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode()
{
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

static int encode_tiled(CUtensorMap* map, CUtensorMapDataType dtype, int rank, const void* base, const cuuint64_t* dims,
                        const cuuint64_t* strides, const cuuint32_t* box, CUtensorMapSwizzle swizzle,
                        CUtensorMapL2promotion promotion, const char* tag)
{
  EncodeTiledFn enc = get_encode();
  if (!enc) return fail(B2D_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, dtype, static_cast<cuuint32_t>(rank), const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, promotion, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(B2D_ERR_CUDA, std::string("cuTensorMapEncodeTiled") + tag + " failed: " + std::to_string((int)r));
  return B2D_OK;
}

int encode_2d(CUtensorMap* map, CUtensorMapDataType dtype, const void* base, int64_t cols, int64_t rows,
              int64_t pitch_bytes, unsigned box_cols, unsigned box_rows, CUtensorMapSwizzle swizzle,
              CUtensorMapL2promotion promotion, const char* tag)
{
  const cuuint64_t dims[2]    = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(pitch_bytes)};
  const cuuint32_t box[2]     = {box_cols, box_rows};
  return encode_tiled(map, dtype, 2, base, dims, strides, box, swizzle, promotion, tag);
}

int encode_3d(CUtensorMap* map, CUtensorMapDataType dtype, const void* base, const int64_t (&dims)[3],
              const int64_t (&pitch_bytes)[2], const unsigned (&box)[3], CUtensorMapSwizzle swizzle,
              CUtensorMapL2promotion promotion, const char* tag)
{
  const cuuint64_t d[3] = {static_cast<cuuint64_t>(dims[0]), static_cast<cuuint64_t>(dims[1]), static_cast<cuuint64_t>(dims[2])};
  const cuuint64_t s[2] = {static_cast<cuuint64_t>(pitch_bytes[0]), static_cast<cuuint64_t>(pitch_bytes[1])};
  const cuuint32_t b[3] = {box[0], box[1], box[2]};
  return encode_tiled(map, dtype, 3, base, d, s, b, swizzle, promotion, tag);
}

int device_sms(int* sms)
{
  int dev = 0, cc = 0;
  B2D_CUDA(cudaGetDevice(&dev));
  B2D_CUDA(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev));
  B2D_CUDA(cudaDeviceGetAttribute(&cc, cudaDevAttrComputeCapabilityMajor, dev));
  if (cc != 9) return fail(B2D_ERR_CUDA, "raft_b200 requires an sm_90 (H100) device; found cc major " + std::to_string(cc));
  return B2D_OK;
}

// ------------------------------------------------------------------------------------------
// Optional timing of the dominant kernel (bench.py's roofline): CUDA events on the call's stream around
// the main kernel of every b2d_pairwise_distance call between b2d_profile_begin and b2d_profile_end.
// Nothing is synchronised until b2d_profile_end, so the timed region of the caller is not perturbed.
namespace {
struct ProfileRing {
  std::vector<cudaEvent_t> ev;  // pairs
  int used = 0;
  bool on  = false;
} g_prof;
std::mutex g_prof_mu;
std::atomic<bool> g_prof_armed{false};   // fast path: a call outside a profiling region touches no lock
}  // namespace

ProfileScope::ProfileScope(cudaStream_t st) : s(st)
{
  if (!g_prof_armed.load(std::memory_order_acquire)) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (g_prof.on && 2 * (g_prof.used + 1) <= static_cast<int>(g_prof.ev.size())) {
    slot = g_prof.used++;
    cudaEventRecord(g_prof.ev[2 * slot], s);
  }
}
ProfileScope::~ProfileScope()
{
  if (slot >= 0) cudaEventRecord(g_prof.ev[2 * slot + 1], s);
}

}  // namespace b2d

using namespace b2d;

int b2d_profile_begin(int capacity)
{
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (capacity < 1 || capacity > 4096) return fail(B2D_ERR_INVALID_ARG, "capacity must be in [1, 4096]");
  while (static_cast<int>(g_prof.ev.size()) < 2 * capacity) {
    cudaEvent_t e;
    B2D_CUDA(cudaEventCreate(&e));
    g_prof.ev.push_back(e);
  }
  g_prof.used = 0;
  g_prof.on   = true;
  g_prof_armed.store(true, std::memory_order_release);
  return B2D_OK;
}

int b2d_profile_end(float* ms, int max_count, int* count)
{
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof.on = false;
  g_prof_armed.store(false, std::memory_order_release);
  if (!ms || !count || max_count < 0) return fail(B2D_ERR_INVALID_ARG, "null ms / count");
  const int c = std::min(g_prof.used, max_count);
  for (int i = 0; i < c; ++i) {
    B2D_CUDA(cudaEventSynchronize(g_prof.ev[2 * i + 1]));
    B2D_CUDA(cudaEventElapsedTime(&ms[i], g_prof.ev[2 * i], g_prof.ev[2 * i + 1]));
  }
  *count = c;
  return B2D_OK;
}

int b2d_version(void) { return 200; }

const char* b2d_last_error(void) { return g_err.c_str(); }
