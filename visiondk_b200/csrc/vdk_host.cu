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

// cuTensorMapEncodeIm2col, resolved the same way
using EncodeIm2colFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeIm2colFn encode_im2col_fn() {
  static EncodeIm2colFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeIm2colFn>(p);
  });
  return fn;
}

int make_tma_im2col_16bit(CUtensorMap* map, const void* base, int B, int H, int W, int C, int kernel, int stride, int pad) {
  if (C % 64 != 0) return fail(VDK_ERR_INVALID, "im2col TMA operand must have C a multiple of 64 (C=%d)", C);
  const int p[2] = {pad, pad};
  return make_tma_im2col_16bit_pads(map, base, B, H, W, C, kernel, stride, p, p);
}

int make_tma_im2col_16bit_pads(CUtensorMap* map, const void* base, int B, int H, int W, int C, int kernel, int stride,
                               const int pad_h[2], const int pad_w[2]) {
  EncodeIm2colFn fn = encode_im2col_fn();
  if (!fn) return fail(VDK_ERR_CUDA, "cuTensorMapEncodeIm2col entry point unavailable (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || C % 8 != 0)
    return fail(VDK_ERR_INVALID, "im2col TMA operand must be 16-byte aligned with C a multiple of 8 (C=%d)", C);
  cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t gstride[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  // window origins run from -lo to (size - 1) + hi - (kernel - 1) in steps of `stride`: exactly the output positions
  // (the corners are ordered (w, h), like the tensor's dimensions)
  const int lower[2] = {-pad_w[0], -pad_h[0]};
  const int upper[2] = {pad_w[1] - (kernel - 1), pad_h[1] - (kernel - 1)};
  cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT16, 4, const_cast<void*>(base), gdim, gstride, lower, upper, 64, 128, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(VDK_ERR_CUDA, "cuTensorMapEncodeIm2col failed with CUresult %d", (int)r);
  return VDK_OK;
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

int make_tma_qkv_16bit(CUtensorMap* map, const void* base, int D, int H, int N, int B, uint32_t box_cols, uint32_t box_rows) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) return fail(VDK_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (D * 2) % 16 != 0)
    return fail(VDK_ERR_INVALID, "qkv TMA operand must be 16-byte aligned with head_dim * 2 a multiple of 16 (head_dim=%d)", D);
  if ((box_cols != 64 && box_cols != 16) || box_rows > 256) return fail(VDK_ERR_INVALID, "qkv TMA box must be 64 or 16 columns, <= 256 rows");
  cuuint64_t gdim[4] = {(cuuint64_t)D, 3ull * H, (cuuint64_t)N, (cuuint64_t)B};
  cuuint64_t gstride[3] = {(cuuint64_t)D * 2, 3ull * H * D * 2, 3ull * H * D * 2 * N};
  cuuint32_t box[4] = {box_cols, 1, box_rows, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT16, 4, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, box_cols == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_32B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(VDK_ERR_CUDA, "cuTensorMapEncodeTiled (qkv) failed with CUresult %d", (int)r);
  return VDK_OK;
}

int make_tma_epilogue_map(CUtensorMap* map, const void* base, int elem_bytes, uint64_t rows, uint64_t cols, uint64_t ld,
                          uint64_t depth, uint64_t depth_stride) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) return fail(VDK_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  const uint64_t eb = static_cast<uint64_t>(elem_bytes);
  // one matrix: the pitch of a single-matrix map only has to be a legal stride, so take the matrix's own size
  if (depth <= 1) depth_stride = (rows * ld * eb + 15) / 16 * 16 / eb;
  if ((elem_bytes != 2 && elem_bytes != 4) || (reinterpret_cast<uintptr_t>(base) & 15) != 0 || (ld * eb) % 16 != 0 ||
      (depth_stride * eb) % 16 != 0)
    return fail(VDK_ERR_INVALID, "epilogue TMA operand must be 16-byte aligned with 16-byte-multiple pitches (ld=%llu)",
                (unsigned long long)ld);
  cuuint64_t gdim[3] = {cols, rows, depth < 1 ? 1 : depth};
  cuuint64_t gstride[2] = {ld * eb, depth_stride * eb};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(128 / elem_bytes), 64, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(map, elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_UINT16, 3, const_cast<void*>(base),
                  gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(VDK_ERR_CUDA, "cuTensorMapEncodeTiled (epilogue) failed with CUresult %d", (int)r);
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

// the same for the structs of the ResNet surface: vdk_conv_desc, vdk_resnet_net
int vdk_resnet_struct_sizes(size_t* out, int n) {
  const size_t sizes[] = {sizeof(vdk_conv_desc), sizeof(vdk_resnet_net)};
  const int k = static_cast<int>(sizeof(sizes) / sizeof(sizes[0]));
  for (int i = 0; i < n && i < k; ++i) out[i] = sizes[i];
  return k;
}

// the same for the general Bottleneck network: vdk_bottleneck_net
int vdk_bottleneck_struct_sizes(size_t* out, int n) {
  const size_t sizes[] = {sizeof(vdk_bottleneck_net)};
  const int k = static_cast<int>(sizeof(sizes) / sizeof(sizes[0]));
  for (int i = 0; i < n && i < k; ++i) out[i] = sizes[i];
  return k;
}

// the same for the Swin V2 network: vdk_swinv2_net
int vdk_swinv2_struct_sizes(size_t* out, int n) {
  const size_t sizes[] = {sizeof(vdk_swinv2_net)};
  const int k = static_cast<int>(sizeof(sizes) / sizeof(sizes[0]));
  for (int i = 0; i < n && i < k; ++i) out[i] = sizes[i];
  return k;
}

// the same for the EfficientNetV2 surface: vdk_conv_ex_desc, vdk_effnetv2_net
int vdk_effnetv2_struct_sizes(size_t* out, int n) {
  const size_t sizes[] = {sizeof(vdk_conv_ex_desc), sizeof(vdk_effnetv2_net)};
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
