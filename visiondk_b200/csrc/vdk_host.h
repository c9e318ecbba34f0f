// vdk_host.h — host-side helpers shared by the translation units of libvdk_b200.so:
// error reporting (vdk_last_error_string), TMA descriptor encoding, device properties.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>

#include "../../include/vdk_b200.h"

namespace vdk {

// Thread-local last error text; every C-ABI entry point returns a VDK_* code and records why.
void set_error(const char* fmt, ...);
int fail(int code, const char* fmt, ...);

// Checks a CUDA runtime call inside a C-ABI entry point.
#define VDK_CUDA_OK(expr)                                                                          \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess)                                                                         \
      return ::vdk::fail(VDK_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

#define VDK_REQUIRE(cond, ...)                                       \
  do {                                                               \
    if (!(cond)) return ::vdk::fail(VDK_ERR_INVALID, __VA_ARGS__);   \
  } while (0)

// Encodes a 2-D row-major tensor map for 16-bit elements: `rows` x `cols`, row pitch `ld` elements,
// box = box_rows x box_cols, 128-byte swizzle (box_cols * 2 bytes must be 128).
// Returns VDK_OK or an error code (driver entry point missing, bad alignment...).
int make_tma_2d_16bit(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                      uint32_t box_rows, uint32_t box_cols);

// 4-D tile map over an NHWC 16-bit tensor: box = [1, box_h, box_w, box_c], no swizzle, out-of-bounds reads give 0
// (which is exactly the zero padding of a convolution).
int make_tma_nhwc_16bit(CUtensorMap* map, const void* base, int B, int H, int W, int C, int box_h, int box_w, int box_c);

// im2col map over an NHWC 16-bit tensor (C a multiple of 64) for a square kernel x kernel convolution with the given stride
// and zero padding: one load = 128 consecutive output pixels (row-major over (b, ho, wo), crossing rows and images) x 64
// channels of one filter tap, 128-byte swizzle — the K-major A stage of the GEMM.  Taps outside the image read as zero.
int make_tma_im2col_16bit(CUtensorMap* map, const void* base, int B, int H, int W, int C, int kernel, int stride, int pad);
// The same with C a multiple of 8 and separate low / high padding per axis (pad_h = {top, bottom}, pad_w = {left, right}):
// a load still takes 64 channels, those past C read as zero.
int make_tma_im2col_16bit_pads(CUtensorMap* map, const void* base, int B, int H, int W, int C, int kernel, int stride,
                               const int pad_h[2], const int pad_w[2]);

// 4-D map over the qkv Linear's output, 16-bit [B][N][3H][D] (D contiguous), seen as (D, 3H, N, B): box = [1][box_rows][1]
// [box_cols], box_cols 64 with 128-byte swizzle or 16 with 32-byte swizzle; out-of-bounds rows (past N) and columns (past D)
// read as zero.  The attention kernel's view of its input.
int make_tma_qkv_16bit(CUtensorMap* map, const void* base, int D, int H, int N, int B, uint32_t box_cols, uint32_t box_rows);

// 3-D map over `depth` row-major [rows][cols] matrices of 16-bit (elem_bytes 2) or fp32 (elem_bytes 4) elements: row pitch
// `ld` elements, matrix pitch `depth_stride` elements (ignored when depth == 1).  Box = 64 rows x 128 bytes, 128-byte
// swizzle; an fp32 map has the FLOAT32 element type so that a TMA reduce-add adds floats.  The GEMM epilogue's view of
// its output, its saved pre-activation and its residual input.
int make_tma_epilogue_map(CUtensorMap* map, const void* base, int elem_bytes, uint64_t rows, uint64_t cols, uint64_t ld,
                          uint64_t depth, uint64_t depth_stride);

int sm_count();

// Live kernel timing inside a real step (bench.py's roofline): while a profile is open (vdk_prof_begin), every launch wrapped
// in a ProfScope is bracketed by two CUDA events on its own stream; vdk_prof_end sums launch count, milliseconds and the
// algorithmic FLOPs / bytes per category.  Closed (the default), a ProfScope costs one predictable branch.
enum ProfCategory { kProfGemm = 0, kProfDepthwise = 1, kProfAttention = 2, kProfScoreFilter = 3, kProfOther = 4, kProfCategories = 5 };
struct ProfScope {
  ProfScope(int category, double flops, double bytes, cudaStream_t stream);
  ~ProfScope();
  int slot;
  cudaStream_t stream;
};

}  // namespace vdk

namespace vdk {
// Internal form of vdk_gemm used by the composite entry points (convnext forward, heads).
int gemm_run(const vdk_gemm_desc& g, cudaStream_t stream);
// Internal form of vdk_conv2d (the ResNet forward).
int conv_run(const vdk_conv_desc& c, cudaStream_t stream);
// Internal form of vdk_conv2d_grouped (the ResNeXt / SE-ResNeXt forward).
int conv_grouped_run(const vdk_conv_desc& c, int groups, cudaStream_t stream);
// Internal form of vdk_conv2d_ex (the EfficientNetV2 forward).
// allow_relu: also take VDK_EPI_RELU, which the public vdk_conv2d_ex keeps refusing (the MobileNetV3 forward's 1x1s use it)
int conv_ex_run(const vdk_conv_ex_desc& c, cudaStream_t stream, bool allow_relu = false);
// Internal form of vdk_conv2d_grouped_ex (the ResNeSt forward), and the 64-channel blocks per tap its packed weight holds.
int conv_grouped_ex_run(const vdk_conv_desc& c, int groups, cudaStream_t stream);
int conv_grouped_ex_cpb(int Cin, int Cout, int groups);
}  // namespace vdk
