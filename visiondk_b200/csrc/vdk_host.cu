// vdk_host.cu — library-level C-ABI entry points and host helpers (error text, TMA descriptors).
#include "vdk_host.h"

#include <cstring>
#include <mutex>
#include <vector>

namespace vdk {

static thread_local char t_error[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(t_error, sizeof(t_error), fmt, ap);
  va_end(ap);
}

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(t_error, sizeof(t_error), fmt, ap);
  va_end(ap);
  return code;
}

// cuTensorMapEncodeTiled is a driver API; it is resolved at run time through the runtime so the library
// carries no link-time dependency on libcuda (it must load — not compute — on a machine without a driver).
using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_tiled_fn() {
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

int make_tma_2d_16bit(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                      uint32_t box_rows, uint32_t box_cols) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) return fail(VDK_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (ld * 2) % 16 != 0)
    return fail(VDK_ERR_INVALID, "TMA operand must be 16-byte aligned with a 16-byte-multiple pitch (ld=%llu)",
                (unsigned long long)ld);
  if (box_cols * 2 != 128 || box_rows > 256)
    return fail(VDK_ERR_INVALID, "TMA box must be 128 bytes wide and <= 256 rows");
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(VDK_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return VDK_OK;
}

int make_tma_nhwc_16bit(CUtensorMap* map, const void* base, int B, int H, int W, int C, int box_h, int box_w,
                        int box_c) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) return fail(VDK_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (C * 2) % 16 != 0 || (box_c * 2) % 16 != 0)
    return fail(VDK_ERR_INVALID, "NHWC TMA operand must be 16-byte aligned with C*2 a multiple of 16 (C=%d)", C);
  if (box_c > 256 || box_w > 256 || box_h > 256) return fail(VDK_ERR_INVALID, "NHWC TMA box dims must be <= 256");
  cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t gstride[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT16, 4, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(VDK_ERR_CUDA, "cuTensorMapEncodeTiled (NHWC) failed with CUresult %d", (int)r);
  return VDK_OK;
}

int make_tma_3d_16bit(CUtensorMap* map, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t pitch1, uint64_t pitch2,
                      uint32_t box_rows) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) return fail(VDK_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (pitch1 * 2) % 16 != 0 || (pitch2 * 2) % 16 != 0)
    return fail(VDK_ERR_INVALID, "3-D TMA operand must be 16-byte aligned with 16-byte-multiple pitches");
  if (box_rows > 256) return fail(VDK_ERR_INVALID, "TMA box must be <= 256 rows");
  cuuint64_t gdim[3] = {d0, d1, d2};
  cuuint64_t gstride[2] = {pitch1 * 2, pitch2 * 2};
  cuuint32_t box[3] = {64, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT16, 3, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(VDK_ERR_CUDA, "cuTensorMapEncodeTiled (3-D) failed with CUresult %d", (int)r);
  return VDK_OK;
}

// ---- live profile (see vdk_host.h) ----
struct ProfRecord {
  int category;
  double flops, bytes;
  cudaEvent_t e0, e1;
};
static bool g_prof_on = false;
static std::vector<ProfRecord> g_prof;
static std::mutex g_prof_mu;

ProfScope::ProfScope(int category, double flops, double bytes, cudaStream_t s) : slot(-1), stream(s) {
  if (!g_prof_on) return;
  std::lock_guard<std::mutex> lock(g_prof_mu);
  ProfRecord r{category, flops, bytes, nullptr, nullptr};
  if (cudaEventCreate(&r.e0) != cudaSuccess || cudaEventCreate(&r.e1) != cudaSuccess) return;
  cudaEventRecord(r.e0, s);
  g_prof.push_back(r);
  slot = static_cast<int>(g_prof.size()) - 1;
}

ProfScope::~ProfScope() {
  if (slot < 0) return;
  std::lock_guard<std::mutex> lock(g_prof_mu);
  if (slot < static_cast<int>(g_prof.size())) cudaEventRecord(g_prof[slot].e1, stream);
}

int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

}  // namespace vdk

extern "C" {

int vdk_version(void) { return 100; }  // 0.1.0

// sizeof() of every by-pointer struct of the ABI, in header order: lets a binding (ctypes mirror) check its layout
int vdk_struct_sizes(size_t* out, int n) {
  const size_t sizes[] = {sizeof(vdk_gemm_desc),        sizeof(vdk_topk_plan),  sizeof(vdk_head_desc), sizeof(vdk_convnext_net),
                          sizeof(vdk_convnext_tensors), sizeof(vdk_vit_net),   sizeof(vdk_vit_tensors)};
  const int k = static_cast<int>(sizeof(sizes) / sizeof(sizes[0]));
  for (int i = 0; i < n && i < k; ++i) out[i] = sizes[i];
  return k;
}

const char* vdk_last_error_string(void) { return vdk::t_error; }

int vdk_prof_begin(void) {
  std::lock_guard<std::mutex> lock(vdk::g_prof_mu);
  for (auto& r : vdk::g_prof) {
    cudaEventDestroy(r.e0);
    cudaEventDestroy(r.e1);
  }
  vdk::g_prof.clear();
  vdk::g_prof_on = true;
  return VDK_OK;
}

int vdk_prof_end(vdk_prof_total* totals, int n_categories) {
  VDK_REQUIRE(totals && n_categories >= 1, "vdk_prof_end: bad arguments");
  std::lock_guard<std::mutex> lock(vdk::g_prof_mu);
  vdk::g_prof_on = false;
  for (int c = 0; c < n_categories; ++c) totals[c] = vdk_prof_total{0, 0.0, 0.0, 0.0};
  int rc = VDK_OK;
  for (auto& r : vdk::g_prof) {
    float ms = 0.f;
    if (cudaEventSynchronize(r.e1) != cudaSuccess || cudaEventElapsedTime(&ms, r.e0, r.e1) != cudaSuccess)
      rc = vdk::fail(VDK_ERR_CUDA, "vdk_prof_end: event timing failed");
    if (r.category >= 0 && r.category < n_categories) {
      totals[r.category].launches += 1;
      totals[r.category].ms += ms;
      totals[r.category].flops += r.flops;
      totals[r.category].bytes += r.bytes;
    }
    cudaEventDestroy(r.e0);
    cudaEventDestroy(r.e1);
  }
  vdk::g_prof.clear();
  return rc;
}

int vdk_device_check(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0)
    return vdk::fail(VDK_ERR_CUDA, "no CUDA device: %s", e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
  int dev = 0, major = 0, minor = 0;
  VDK_CUDA_OK(cudaGetDevice(&dev));
  VDK_CUDA_OK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  VDK_CUDA_OK(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  if (major != 9 || minor != 0)
    return vdk::fail(VDK_ERR_CUDA, "device compute capability %d.%d; this library is sm_90a only", major, minor);
  return VDK_OK;
}

}  // extern "C"
