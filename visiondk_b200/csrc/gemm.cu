// gemm.cu — D = epilogue(A . B^T) on sm_90a warpgroup tensor cores (wgmma), operands staged by TMA.
//
// Replaces the library GEMMs behind timm's ConvNeXt/ViT Linear layers and patchify convolutions that
// models/faceX/backbone/timm_wrapper.py:52 runs, and the neck Linear of timm_wrapper.py:36 (SURVEY K1-K5).
//
// One persistent CTA per SM, 384 threads:
//   warpgroup 0    : TMA producer (one thread; A tile 128x64, B tile BNx64 per stage, 128-byte swizzle), registers
//                    handed to the consumers with setmaxnreg; in the weight-gradient form, warps 1-2 also sum A's
//                    columns from the stages (the bias gradient, `col_sums`)
//   warpgroups 1-2 : consumers, 64 rows each: wgmma m64 x BN x 16 into registers (fp32), then the epilogue.  The
//                    epilogue math (bias / GELU / layer-scale+residual / LayerNorm / GELU') runs on the accumulator
//                    fragments; each 64-row x 128-byte box of results is written to a swizzled shared-memory ring
//                    (stmatrix for 16-bit outputs) and drained by a TMA store (a TMA reduce-add for atomic split-K), so
//                    the stores run under the next tile's MMAs.  Each warpgroup syncs only its own 128 threads.  A
//                    residual / saved pre-activation is TMA-loaded into the same ring while the tile's MMAs run and read
//                    back in fragment layout (ldmatrix).
#include "vdk_host.h"
#include "vdk_ptx.cuh"

#include <algorithm>
#include <cstdlib>

#include "train_gemm.h"

namespace vdk {

constexpr int kBM = 128;
constexpr int kBK = 64;  // 64 x 16-bit = one 128-byte swizzle row
constexpr int kGemmThreads = 384;  // producer warpgroup, two consumer warpgroups
constexpr int kBoxBytes = 64 * 128;  // epilogue box: one warpgroup's 64 rows x 128 bytes (64 16-bit or 32 fp32 columns)
// A-operand / epilogue set of a gemm_tn_kernel instantiation.  kGemmPlain: vdk_gemm (dense A, epilogues NONE..MUL_GELU_GRAD);
// the two convolution modes add the ReLU epilogues and are compiled only into vdk_conv2d's instantiations.
constexpr int kGemmPlain = 0;
constexpr int kConvDense = 1;   // 1x1 / stride-1 convolution: a plain GEMM over [B*H*W, Cin]
constexpr int kConvIm2col = 2;  // k x k / stride-s convolution: A tiles gathered from NHWC by TMA im2col loads
// grouped k x k convolution (vdk_conv2d_grouped, BN = 128): the N tile at n0 contracts over input channels n0 .. n0 + 127
// only (whole groups, block-diagonal B), so its K block kb = (tap kb / 2, channels n0 + (kb % 2) * 64)
constexpr int kConvGrouped = 3;
// vdk_conv2d_ex (TF-"same" padded MBConv convolutions): as kConvDense / kConvIm2col, plus the SiLU and hard-swish
// epilogues.  cv_pad holds
// the low padding of both axes (h | w << 8); the high padding only shapes the im2col map.  Cin a multiple of 8: a K block
// still loads 64 channels of one tap, the channels past Cin arrive as TMA zero fill and meet zero weight columns.
constexpr int kConvExDense = 4;
constexpr int kConvExIm2col = 5;
// grouped k x k convolution with any group widths (vdk_conv2d_grouped_ex, BN = 128; ResNeSt's split-attention conv,
// Cout = radix * Cin): the N tile at n0 contracts over the input channels of the groups its output channels belong to,
// from c_lo = (n0 / cv_cg_out) * cv_cg_in rounded down to a multiple of 8 on (the im2col load's channel coordinate must
// be 16-byte aligned), as cv_cpb 64-channel blocks per tap (channels past Cin are TMA zero fill; the packed weight is
// zero outside each output channel's own group)
constexpr int kConvGroupedEx = 6;
// dense dgrad (kTA = 0, kTB = 1) with the LayerNorm-backward epilogue VDK_EPI_LN_BWD (ln_bwd_tile below)
constexpr int kGemmLnBwd = 7;

// The implicit-GEMM convolution modes (kConvIm2col) overlay their geometry on fields they do not use, so that the struct —
// and with it the code of the plain GEMM instantiations — stays as it is.
struct GemmParams {
  int M, N, K;
  void* D;
  int ldd;
  const float* bias;
  union {
    struct {
      const float* gamma;  // layer-scale (SCALE_RESIDUAL) or LayerNorm weight (LAYERNORM)
      const float* beta;   // LayerNorm bias
    };
    struct {  // convolution: row m = output pixel (b, ho, wo); K blocks = (filter tap (dy, dx) row-major, 64-channel block)
      int cv_cpb;               // Cin / 64: K blocks per filter tap
      int cv_kw;                // filter width
      int cv_stride, cv_pad;
    };
  };
  const void* residual;  // SCALE_RESIDUAL: added; MUL_GELU_GRAD: the saved 16-bit pre-activation whose GELU' scales the output
  union {
    int ldr;        // host side only: the kernel reads the residual through its TMA map
    int cv_cg_out;  // kConvGroupedEx: output channels per group
  };
  int out_dtype;
  int epilogue;
  union {
    float ln_eps;
    int cv_cg_in;    // kConvGroupedEx: input channels per group
    int ln_cluster;  // kGemmLnBwd: ln_group / BN > 1: a row spans this many tiles, the CTAs of one thread-block cluster
  };
  int split_k;  // > 1: each tile's K range is split over split_k work items, fp32 partials are atomically added
  union {
    long long split_stride;  // > 0: split s writes its partial tile to D + s*split_stride with plain stores (deterministic)
    struct {
      int cv_wo, cv_howo;  // convolution: output width, output pixels per image
    };
  };
  union {
    void* aux;  // GELU only: also store the pre-activation (acc + bias) here, pitch ldd (saved for the backward)
    // split-K slabs with an MN-major A only (the weight-gradient form): split s also stores the column sums of A over
    // its K range, sum_k A[k, m], to col_sums[s * M + m] (the bias gradient, summed in the producer warpgroup)
    float* col_sums;
    float* ln_slab;  // kGemmLnBwd: one row [2][N] of dgamma / dbeta partials per group of num_n CTAs
  };
  int partial_out;  // the caller asked for split-K: raw fp32 partials are added / slab-stored even if one split remains
  // kGemmLnBwd only (appended, so that the other instantiations read every field at the offset they did)
  const float* ln_rstd;
  int ln_group, ln_wo;
};
// kGemmLnBwd: the row-sum exchange of a cluster behind the barriers, per consumer warpgroup and tile parity: one float2
// (sum g, sum g xh) per row from each of up to 4 ranks, and its mbarrier
constexpr int kLnXchBytes = 2 * 2 * 4 * 64 * 8;
constexpr int kLnSmemBytes = kLnXchBytes + 4 * 8;

template <int BN>
struct GemmCfg {
  static constexpr int kStageA = kBM * kBK * 2;
  static constexpr int kStageB = BN * kBK * 2;
  static constexpr int kStageBytes = kStageA + kStageB;
  static constexpr int kStages = (BN == 256) ? 3 : 5;
  // epilogue ring of each consumer warpgroup, in boxes; it holds a whole 16-bit residual half tile (BN / 64 boxes)
  static constexpr int kRing = (BN == 256) ? 4 : 3;
  static_assert(BN / 64 <= kRing, "a 16-bit residual half tile must fit in the ring");
  static constexpr int kRingBytes = 2 * kRing * kBoxBytes;
  static constexpr int kParFloats = 3 * BN;  // per consumer warpgroup: bias, gamma, beta of the tile's columns
  // stages + two rings + two parameter copies + full / empty / residual barriers + 1 KB align slack.  Within 227 KB:
  //   BN = 256: 3 x 48 KB + 2 x 4 x 8 KB + 6 KB + 64 B + 1 KB = 215.1 KB (a fourth 48 KB stage does not fit)
  //   BN = 128: 5 x 32 KB + 2 x 3 x 8 KB + 3 KB + 96 B + 1 KB = 212.1 KB (a fourth ring box per warpgroup does not fit)
  static constexpr int kSmemBytes = kStages * kStageBytes + kRingBytes + 2 * kParFloats * 4 + (2 * kStages + 2) * 8 + 1024;
  static_assert(kSmemBytes <= 227 * 1024, "GEMM shared memory budget");
};

__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// SiLU x / (1 + e^-x) with ex2.approx and rcp.approx (relative errors 2^-22 and 2^-23): relative error <= 1e-6 for
// |x| <= 64 before the output rounding (the fp32 product -x log2(e) adds |x| 2^-24 to the exponent); x -> -0 for x < -126.
__device__ __forceinline__ float silu_fast(float x) { return x * rcp_approx(1.f + ex2_approx(-1.4426950409f * x)); }

// erf-GELU for the forward epilogue.  The fc1 epilogue applies 4C x tokens GELUs per block, so the activation has to
// cost few issue slots and at most one SFU op per pair of elements or the epilogue, not the MMA, sets the pace.
// y = 0.5 x (1 + tanh(u)), u = x (c1 + c3 x^2) with (c1, c3) refitted to the erf form (max |dev| 3.1e-4 instead of the
// textbook tanh-GELU's 4.7e-4); u and tanh are evaluated two elements at a time in fp16x2 (tanh.approx.f16x2,
// rel. error 2^-11), the final multiply in fp32 so that y -> x exactly for large x.  Absolute error <= 6e-4 |x| before the
// output rounding (4.3e-4 |x| measured over every finite bf16 / fp16 x, tests/test_gemm_gpu.py): below one bf16 ulp.
__device__ __forceinline__ void gelu_pair(float& x0, float& x1) {
  const __half2 h = __floats2half2_rn(x0, x1);
  const __half2 t = __hmul2(h, h);
  const __half2 p = __hfma2(t, __floats2half2_rn(0.03489978f, 0.03489978f), __floats2half2_rn(0.79973199f, 0.79973199f));
  const __half2 u = __hmul2(h, p);
  uint32_t ui = *reinterpret_cast<const uint32_t*>(&u), thi;
  asm("tanh.approx.f16x2 %0, %1;" : "=r"(thi) : "r"(ui));
  const float2 th = __half22float2(*reinterpret_cast<const __half2*>(&thi));
  const float hx0 = 0.5f * x0, hx1 = 0.5f * x1;
  x0 = fmaf(hx0, th.x, hx0);
  x1 = fmaf(hx1, th.y, hx1);
}

// d/dx of the forward's GELU form 0.5 x (1 + tanh(u)), u = x (c1 + c3 x^2), two elements at a time in fp16x2 like the
// forward (the fc2 data-gradient epilogue evaluates 4C x tokens of these per block): x is clamped to [-8, 8], where
// the derivative has reached 1 / 0 to fp16 precision, so that x^2 (1 - tanh^2) cannot overflow into inf * 0.
// Absolute error <= 8e-3 before the output rounding (7.6e-3 measured over every finite bf16 / fp16 x, tests/test_gemm_gpu.py;
// 7.4e-4 of it is the fitted form's own derivative error): the worst case is near |x| = 3, where the error of
// tanh.approx.f16 in 1 - tanh^2 is multiplied by x (c1 + 3 c3 x^2) ~ 5.  About two bf16 ulps of a gradient of order 1.
__device__ __forceinline__ float2 gelu_grad_pair(float x0, float x1) {
  const __half2 lim = __floats2half2_rn(8.0f, 8.0f);
  const __half2 h = __hmax2(__hmin2(__floats2half2_rn(x0, x1), lim), __hneg2(lim));
  const __half2 t = __hmul2(h, h);
  const __half2 c1 = __floats2half2_rn(0.79973199f, 0.79973199f);
  const __half2 u = __hmul2(h, __hfma2(t, __floats2half2_rn(0.03489978f, 0.03489978f), c1));
  uint32_t ui = *reinterpret_cast<const uint32_t*>(&u), thi;
  asm("tanh.approx.f16x2 %0, %1;" : "=r"(thi) : "r"(ui));
  const __half2 th = *reinterpret_cast<const __half2*>(&thi);
  const __half2 half = __floats2half2_rn(0.5f, 0.5f);
  const __half2 du = __hfma2(t, __floats2half2_rn(3.0f * 0.03489978f, 3.0f * 0.03489978f), c1);
  const __half2 s = __hfma2(__hneg2(th), th, __floats2half2_rn(1.0f, 1.0f));  // 1 - tanh^2
  const __half2 a = __hmul2(__hmul2(h, du), s);
  return __half22float2(__hfma2(a, half, __hfma2(th, half, half)));
}

__device__ __forceinline__ uint32_t pack2(float a, float b, int out_dtype) {
  if (out_dtype == VDK_DTYPE_BF16) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  } else {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
}
__device__ __forceinline__ float2 unpack2(uint32_t u, int dtype) {
  if (dtype == VDK_DTYPE_BF16) {
    __nv_bfloat162 h = *reinterpret_cast<__nv_bfloat162*>(&u);
    return __bfloat1622float2(h);
  } else {
    __half2 h = *reinterpret_cast<__half2*>(&u);
    return __half22float2(h);
  }
}

// Epilogue arithmetic of one fragment pair: columns c, c + 1 of the tile (c even) in one row.  `par`: this warpgroup's
// copy of the tile's bias / gamma / beta ([3][BN], zero beyond N), staged once per tile so that the epilogue's critical
// path holds no global loads.  `r`: the residual / saved pre-activation pair.  The operations and their order are those
// of the row-wise form: + bias, then the epilogue (fp32 throughout, GELU and GELU' in fp16x2 pairs).
template <int BN, int kMode>
__device__ __forceinline__ void epi_pair(const GemmParams& p, float& x0, float& x1, const float* par, int c, float ln_mean,
                                         float ln_rstd, float2 r) {
  if (p.bias != nullptr && p.epilogue != VDK_EPI_LAYERNORM) {  // LayerNorm: added to the accumulator before the statistics
    const float2 b = *reinterpret_cast<const float2*>(par + c);
    x0 += b.x;
    x1 += b.y;
  }
  if (p.epilogue == VDK_EPI_MUL_GELU_GRAD) {
    const float2 g = gelu_grad_pair(r.x, r.y);
    x0 *= g.x;
    x1 *= g.y;
  } else if (p.epilogue == VDK_EPI_GELU) {
    gelu_pair(x0, x1);
  } else if (p.epilogue == VDK_EPI_LAYERNORM) {
    const float2 g = *reinterpret_cast<const float2*>(par + BN + c);
    const float2 b = *reinterpret_cast<const float2*>(par + 2 * BN + c);
    x0 = (x0 - ln_mean) * ln_rstd * g.x + b.x;
    x1 = (x1 - ln_mean) * ln_rstd * g.y + b.y;
  } else if (p.epilogue == VDK_EPI_SCALE_RESIDUAL) {
    // gamma x is rounded before the residual is added: __fmul_rn keeps the compiler from contracting the two into an FMA
    const float2 g = *reinterpret_cast<const float2*>(par + BN + c);
    x0 = __fmul_rn(x0, g.x);
    x1 = __fmul_rn(x1, g.y);
    x0 += r.x;
    x1 += r.y;
  }
  if constexpr (kMode != kGemmPlain) {
    if (p.epilogue == VDK_EPI_RELU) {
      x0 = fmaxf(x0, 0.f);
      x1 = fmaxf(x1, 0.f);
    } else if (p.epilogue == VDK_EPI_RESIDUAL_RELU) {
      x0 = fmaxf(x0 + r.x, 0.f);
      x1 = fmaxf(x1 + r.y, 0.f);
    }
  }
  if constexpr (kMode == kConvExDense || kMode == kConvExIm2col) {
    if (p.epilogue == VDK_EPI_SILU) {
      x0 = silu_fast(x0);
      x1 = silu_fast(x1);
    } else if (p.epilogue == VDK_EPI_SILU_RESIDUAL) {
      x0 = silu_fast(x0) + r.x;
      x1 = silu_fast(x1) + r.y;
    } else if (p.epilogue == VDK_EPI_HARDSWISH) {
      x0 = hardswish(x0);
      x1 = hardswish(x1);
    }
  }
}

// A warpgroup's box in ring slot `slot` is written: make it visible to the async proxy, let the leader hand it to TMA
// (store, or reduce-add into fp32) and move to the next slot.  Before the barrier the leader waits until the store that
// last read the NEXT slot is done reading, so after the barrier every thread may write that slot.
template <int kRing>
__device__ __forceinline__ void epi_publish(const CUtensorMap* map, const uint8_t* box, int& slot, bool leader, uint32_t bar_id,
                                            int c0, int c1, int c2, bool reduce) {
  fence_proxy_async_smem();
  if (leader) tma_store_wait_read<kRing - 2>();
  named_bar_sync(bar_id, 128);
  if (leader) {
    if (reduce) tma_reduce_add_3d(map, box, c0, c1, c2);
    else tma_store_3d(map, box, c0, c1, c2);
    tma_store_commit();
  }
  slot = (slot + 1 == kRing) ? 0 : slot + 1;
}

// byte offset of the 16-byte chunk `chunk` of row `row` in a 128-byte-swizzled box (the TMA SWIZZLE_128B pattern)
__device__ __forceinline__ uint32_t box_off(int row, int chunk) { return row * 128 + ((chunk ^ (row & 7)) << 4); }

// kGemmLnBwd: the LayerNorm pixel of GEMM row m, group q (the rstd index; D's row in units of ln_group elements)
__device__ __forceinline__ long long ln_pixel(const GemmParams& p, int m, int q) {
  if (p.ln_wo == 0) return m;
  const int bho = m / p.ln_wo, wo = m - bho * p.ln_wo;
  return ((static_cast<long long>(bho) * 2 + (q >> 1)) * p.ln_wo + wo) * 2 + (q & 1);
}

// Sum of v[i] over the 8 lanes that hold the same fragment columns (lane bits 2-4), by recursive halving (14 shuffles,
// not 48): afterwards v[0], v[1] hold the sums of entries 8 b4 + 4 b3 + 2 b2 + {0, 1} (b = the lane's bits).
__device__ __forceinline__ void halve_columns(float (&v)[16], int lane) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const bool up = (lane & 16) != 0;
    v[i] = (up ? v[i + 8] : v[i]) + __shfl_xor_sync(0xffffffffu, up ? v[i] : v[i + 8], 16);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const bool up = (lane & 8) != 0;
    v[i] = (up ? v[i + 4] : v[i]) + __shfl_xor_sync(0xffffffffu, up ? v[i] : v[i + 4], 8);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const bool up = (lane & 4) != 0;
    v[i] = (up ? v[i + 2] : v[i]) + __shfl_xor_sync(0xffffffffu, up ? v[i] : v[i + 2], 4);
  }
}

// st.async of a float2 into the shared memory of a CTA of the cluster, completing `bytes` on its mbarrier
__device__ __forceinline__ void st_async_f2(uint32_t local_addr, uint32_t local_bar, uint32_t rank, float a, float b) {
  uint32_t ra, rb;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(local_addr), "r"(rank));
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rb) : "r"(local_bar), "r"(rank));
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v2.f32 [%0], {%1, %2}, [%3];"
               :: "r"(ra), "f"(a), "f"(b), "r"(rb) : "memory");
}

// kGemmLnBwd epilogue of one warpgroup's 64 x BN half tile; the saved LayerNorm output y has landed in ring boxes
// 0 .. BN / 64 - 1.  ln_bwd_kernel's arithmetic (train_ops.cu) on dy = bf16(acc): pass 1 rounds dy in place and sums, per
// row and group, g = dy gamma and g xh with xh = (y - beta) (1 / gamma); pass 2 writes D = rstd (g - m1 - xh m2) through
// the ring (stmatrix, then 128-byte row pieces, so that the patch layout needs no TMA view).  colp[box][2 qty + i]
// accumulates over the CTA's tiles the column sum of dy xh (qty 0) / dy (qty 1) of box column 8 (4 b4 + 2 b3 + b2) +
// fcol + i (halve_columns).  A tile holds at most two groups (ln_group >= 128).  A group wider than the tile (ln_cluster
// > 1 CTAs, one per tile of the row) completes its row sums across the cluster: every CTA sends its partial of each row
// to every rank's `xch` slot [own rank][row] with st.async on that rank's `xbar`, and adds the ranks' partials in rank
// order, so that all of them use the same statistics.
template <int BN>
__device__ __forceinline__ void ln_bwd_tile(const GemmParams& p, float (&acc)[BN / 2], float (&colp)[BN / 64][4], const float* par,
                                            uint8_t* ring, int wrow0, int n0, int fcol, int frow, int mrow, int mcb, int wl,
                                            int lane, uint8_t* xch, uint64_t* xbar, uint32_t xphase, bool leader) {
  constexpr int kGroups = BN / 128;
  const int G = p.ln_group;
  float rs[kGroups][2], s1[kGroups][2], s2[kGroups][2];
#pragma unroll
  for (int gi = 0; gi < kGroups; ++gi)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = wrow0 + frow + 8 * h;
      rs[gi][h] = (gi * G < BN && m < p.M) ? __ldg(p.ln_rstd + ln_pixel(p, m, (n0 + gi * G) / G)) : 0.f;
      s1[gi][h] = 0.f;
      s2[gi][h] = 0.f;
    }
#pragma unroll
  for (int sc = 0; sc < BN / 64; ++sc) {
    const uint32_t box = smem_u32(ring + sc * kBoxBytes);
    float v[16], t1[2] = {0.f, 0.f}, t2[2] = {0.f, 0.f};  // v[2 jj + e]: dy xh of box column 8 jj + fcol + e
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      uint32_t rin[4];
      ldmatrix_x4(rin, box + box_off(mrow, 2 * q + mcb));
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int jj = 2 * q + (i >> 1), j = sc * 8 + jj, h = i & 1, c = j * 8 + fcol;
        const float2 d = unpack2(pack2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], VDK_DTYPE_BF16), VDK_DTYPE_BF16);
        acc[4 * j + 2 * h] = d.x;
        acc[4 * j + 2 * h + 1] = d.y;
        const float2 yv = unpack2(rin[i], VDK_DTYPE_BF16);
        const float2 w = *reinterpret_cast<const float2*>(par + c);
        const float2 iw = *reinterpret_cast<const float2*>(par + BN + c);
        const float2 b = *reinterpret_cast<const float2*>(par + 2 * BN + c);
        const float h0 = (yv.x - b.x) * iw.x, h1 = (yv.y - b.y) * iw.y;
        const float g0 = d.x * w.x, g1 = d.y * w.y;
        t1[h] += g0;
        t2[h] = fmaf(g0, h0, t2[h]);
        t1[h] += g1;
        t2[h] = fmaf(g1, h1, t2[h]);
        v[2 * jj] = h == 0 ? d.x * h0 : fmaf(d.x, h0, v[2 * jj]);
        v[2 * jj + 1] = h == 0 ? d.y * h1 : fmaf(d.y, h1, v[2 * jj + 1]);
      }
    }
    const int gi = sc * 64 / G;
#pragma unroll
    for (int gg = 0; gg < kGroups; ++gg)
      if (gg == gi)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          s1[gg][h] += t1[h];
          s2[gg][h] += t2[h];
        }
    halve_columns(v, lane);
    colp[sc][0] += v[0];
    colp[sc][1] += v[1];
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e) v[2 * jj + e] = acc[4 * (sc * 8 + jj) + e] + acc[4 * (sc * 8 + jj) + 2 + e];
    halve_columns(v, lane);
    colp[sc][2] += v[0];
    colp[sc][3] += v[1];
  }
  const float inv_g = 1.0f / static_cast<float>(G);
#pragma unroll
  for (int gi = 0; gi < kGroups; ++gi) {
    if (gi * G >= BN) break;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      s1[gi][h] += __shfl_xor_sync(0xffffffffu, s1[gi][h], 1);
      s1[gi][h] += __shfl_xor_sync(0xffffffffu, s1[gi][h], 2);
      s2[gi][h] += __shfl_xor_sync(0xffffffffu, s2[gi][h], 1);
      s2[gi][h] += __shfl_xor_sync(0xffffffffu, s2[gi][h], 2);
    }
  }
  if (p.ln_cluster > 1) {  // G > BN: one group per tile (gi = 0)
    const uint32_t rank = cluster_ctarank();
    if (leader) mbar_arrive_expect_tx(xbar, p.ln_cluster * 64 * 8);
    if ((lane & 3) == 0)
      for (int r = 0; r < p.ln_cluster; ++r)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          st_async_f2(smem_u32(xch + (rank * 64 + frow + 8 * h) * 8), smem_u32(xbar), r, s1[0][h], s2[0][h]);
    mbar_wait<true>(xbar, xphase);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float a = 0.f, b = 0.f;
      for (int r = 0; r < p.ln_cluster; ++r) {
        const float2 t = *reinterpret_cast<const float2*>(xch + (r * 64 + frow + 8 * h) * 8);
        a += t.x;
        b += t.y;
      }
      s1[0][h] = a;
      s2[0][h] = b;
    }
  }
#pragma unroll
  for (int gi = 0; gi < kGroups; ++gi)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      s1[gi][h] *= inv_g;
      s2[gi][h] *= inv_g;
    }
  __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(p.D);
#pragma unroll
  for (int sc = 0; sc < BN / 64; ++sc) {
    uint8_t* boxp = ring + sc * kBoxBytes;
    const uint32_t box = smem_u32(boxp);
    const int gi = sc * 64 / G;
    float m1[2], m2[2], r[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {  // the group's row statistics, selected without dynamic register indexing
      m1[h] = s1[0][h]; m2[h] = s2[0][h]; r[h] = rs[0][h];
#pragma unroll
      for (int gg = 1; gg < kGroups; ++gg)
        if (gg == gi) { m1[h] = s1[gg][h]; m2[h] = s2[gg][h]; r[h] = rs[gg][h]; }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t addr = box + box_off(mrow, 2 * q + mcb);
      uint32_t rin[4], rq[4];
      ldmatrix_x4(rin, addr);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int j = sc * 8 + 2 * q + (i >> 1), h = i & 1, c = j * 8 + fcol;
        const float2 yv = unpack2(rin[i], VDK_DTYPE_BF16);
        const float2 w = *reinterpret_cast<const float2*>(par + c);
        const float2 iw = *reinterpret_cast<const float2*>(par + BN + c);
        const float2 b = *reinterpret_cast<const float2*>(par + 2 * BN + c);
        const float h0 = (yv.x - b.x) * iw.x, h1 = (yv.y - b.y) * iw.y;
        const float o0 = r[h] * (acc[4 * j + 2 * h] * w.x - m1[h] - h0 * m2[h]);
        const float o1 = r[h] * (acc[4 * j + 2 * h + 1] * w.y - m1[h] - h1 * m2[h]);
        rq[i] = pack2(o0, o1, VDK_DTYPE_BF16);
      }
      stmatrix_x4(addr, rq);
    }
    __syncwarp();  // the warp reads back only its own 16 rows
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const int row = wl * 16 + it * 4 + (lane >> 3), chunk = lane & 7, m = wrow0 + row;
      if (m < p.M) {
        const int n = n0 + sc * 64 + chunk * 8, qg = n / G;
        const long long off = p.ln_wo == 0 ? static_cast<long long>(m) * p.ldd + n : ln_pixel(p, m, qg) * G + (n - qg * G);
        *reinterpret_cast<uint4*>(dst + off) = *reinterpret_cast<const uint4*>(boxp + box_off(row, chunk));
      }
    }
  }
}

// kTA / kTB: operand stored with the contraction index as the slow dimension ([K,M] / [K,N] row-major: MN-major)
// kMode: kGemmPlain, kConvDense, kConvIm2col or kConvGrouped (see above)
template <int BN, bool kBf16, int kTA, int kTB, int kMode>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tn_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
               const __grid_constant__ CUtensorMap map_d, const __grid_constant__ CUtensorMap map_aux,
               const __grid_constant__ CUtensorMap map_r, const GemmParams p) {
  using Cfg = GemmCfg<BN>;
  constexpr int kStages = Cfg::kStages;
  constexpr int kRing = Cfg::kRing;
  extern __shared__ uint8_t smem_raw[];
  // align inside the dynamic smem window without a pointer->integer->pointer round trip (which would demote every
  // later access to generic LD/ST)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* ring_all = smem + kStages * Cfg::kStageBytes;                   // [2][kRing] boxes, 1024-byte aligned
  float* par_all = reinterpret_cast<float*>(ring_all + Cfg::kRingBytes);  // [2][3][BN] bias, gamma, beta
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(par_all + 2 * Cfg::kParFloats);
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* res_bar = empty_bar + kStages;  // [2]: a consumer warpgroup's residual boxes have landed
  // A's column sums: two producer warps read every A stage as well and release it on the empty barrier
  constexpr bool kColSums = kTA && kMode == kGemmPlain;
  const bool col_sums = kColSums && p.partial_out && p.split_stride > 0 && p.col_sums != nullptr;
  constexpr bool kConvEx = kMode == kConvExDense || kMode == kConvExIm2col;


  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_a);
    prefetch_tensormap(&map_b);
    prefetch_tensormap(&map_d);
    if (p.aux != nullptr) prefetch_tensormap(&map_aux);
    if (kMode == kGemmLnBwd || p.epilogue == VDK_EPI_SCALE_RESIDUAL || p.epilogue == VDK_EPI_MUL_GELU_GRAD ||
        (kMode != kGemmPlain && p.epilogue == VDK_EPI_RESIDUAL_RELU) || (kConvEx && p.epilogue == VDK_EPI_SILU_RESIDUAL))
      prefetch_tensormap(&map_r);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], col_sums ? 10 : 8);  // one arrival per consumer warp (and per column-sum warp)
    }
    mbar_init(&res_bar[0], 1);
    mbar_init(&res_bar[1], 1);
    if constexpr (kMode == kGemmLnBwd)
      for (int i = 0; i < 4; ++i) mbar_init(reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(res_bar + 2) + kLnXchBytes) + i, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if constexpr (kMode == kGemmLnBwd) {
    if (p.ln_cluster > 1) cluster_sync_all();  // every rank's exchange barriers are initialised before the first st.async
  }

  if (threadIdx.x < 128) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    // the tile grid, computed in each role after its register hand-over (kept live across the hand-over, it spills)
    const int num_m = (p.M + kBM - 1) / kBM;
    const int num_n = (p.N + BN - 1) / BN;
    const int num_kb_total = (p.K + kBK - 1) / kBK;
    const int kb_per_split = (num_kb_total + p.split_k - 1) / p.split_k;
    const int num_tiles = num_m * num_n * p.split_k;  // work items; split index is the slowest dimension
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int mn = tile % (num_m * num_n), split = tile / (num_m * num_n);
        const int m0 = (mn / num_n) * kBM;
        const int n0 = (mn % num_n) * BN;
        const int kb0 = split * kb_per_split;
        const int kb1 = min(kb0 + kb_per_split, num_kb_total);
        // im2col: the tile's first output pixel, as the input position of its filter window's top-left tap.  The TMA unit
        // walks the next 127 pixels through the map's bounding box (across rows and images); rows past M read as zero.
        int cw = 0, ch = 0, cn = 0;
        if constexpr (kMode == kConvIm2col || kMode == kConvGrouped || kMode == kConvGroupedEx) {
          cn = m0 / p.cv_howo;
          const int r = m0 - cn * p.cv_howo, ho = r / p.cv_wo;
          ch = ho * p.cv_stride - p.cv_pad;
          cw = (r - ho * p.cv_wo) * p.cv_stride - p.cv_pad;
        } else if constexpr (kMode == kConvExIm2col) {
          cn = m0 / p.cv_howo;
          const int r = m0 - cn * p.cv_howo, ho = r / p.cv_wo;
          ch = ho * p.cv_stride - (p.cv_pad & 0xff);
          cw = (r - ho * p.cv_wo) * p.cv_stride - (p.cv_pad >> 8);
        }
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait_relaxed<true>(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * Cfg::kStageBytes;
          uint8_t* sb = sa + Cfg::kStageA;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          if constexpr (kMode == kConvIm2col || kMode == kConvExIm2col) {  // K block kb = (filter tap, 64-channel block)
            const int tap = kb / p.cv_cpb, c0 = (kb - tap * p.cv_cpb) * kBK, dy = tap / p.cv_kw;
            tma_load_im2col_4d(sa, &map_a, &full_bar[stage], c0, cw, ch, cn, static_cast<uint16_t>(tap - dy * p.cv_kw),
                               static_cast<uint16_t>(dy), kEvictNormal);
          } else if constexpr (kMode == kConvGrouped) {  // cv_cpb = 2: the tile's own 128 input channels at every tap
            const int tap = kb >> 1, c0 = n0 + (kb & 1) * kBK, dy = tap / p.cv_kw;
            tma_load_im2col_4d(sa, &map_a, &full_bar[stage], c0, cw, ch, cn, static_cast<uint16_t>(tap - dy * p.cv_kw),
                               static_cast<uint16_t>(dy), kEvictNormal);
          } else if constexpr (kMode == kConvGroupedEx) {  // K block kb = (tap, 64-channel block from the tile's c_lo)
            const int tap = kb / p.cv_cpb, dy = tap / p.cv_kw;
            const int c0 = ((n0 / p.cv_cg_out * p.cv_cg_in) & ~7) + (kb - tap * p.cv_cpb) * kBK;
            tma_load_im2col_4d(sa, &map_a, &full_bar[stage], c0, cw, ch, cn, static_cast<uint16_t>(tap - dy * p.cv_kw),
                               static_cast<uint16_t>(dy), kEvictNormal);
          } else if (kTA) {  // [K,M] storage: 64-wide M blocks x 64 contraction rows, 8 KB each
#pragma unroll
            for (int j = 0; j < kBM / 64; ++j) tma_load_2d(sa + j * 8192, &map_a, &full_bar[stage], m0 + j * 64, kb * kBK, kEvictNormal);
          } else {
            tma_load_2d(sa, &map_a, &full_bar[stage], kb * kBK, m0, kEvictNormal);
          }
          if (kTB) {
#pragma unroll
            for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * 8192, &map_b, &full_bar[stage], n0 + j * 64, kb * kBK, kEvictLast);
          } else {
            tma_load_2d(sb, &map_b, &full_bar[stage], kb * kBK, n0, kEvictLast);
          }
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    } else if (col_sums && threadIdx.x >= 32 && threadIdx.x < 96) {
      // column sums of A (bias gradient of the weight gradient): warps 1-2 walk the consumers' stage / phase sequence.
      // Warp 1 + j sums box j of each A stage (64 contraction rows x 64 M columns, 128-byte rows) in fp32, of the 16-bit
      // values as stored: lane = 8-byte piece lane % 16 (4 columns) of rows lane / 16 + 2 i.  8-byte pieces keep four
      // accumulators per thread, so that four loads fit in flight within the producer's 40 registers.  They read the
      // stages of the work items with n0 == 0 only (one per M tile and split), but release every stage, so empty_bar's
      // arrival count is fixed.
      const int j = (threadIdx.x >> 5) - 1, lane = threadIdx.x & 31;
      const int piece = lane & 15, r0 = lane >> 4;
      // row r0 + 2 i sits at (r0 + 2 i) * 128 bytes, its 16-byte chunk c at c ^ (r0 + 2 (i % 4)) = (c ^ r0) ^ 2 (i % 4)
      // (r0 <= 1): four base offsets, one per i % 4; the rest are immediates
      uint32_t off[4];
#pragma unroll
      for (int q = 0; q < 4; ++q)
        off[q] = j * 8192 + r0 * 128 + q * 256 + (((((piece >> 1) ^ r0) << 4)) ^ (q << 5)) + (piece & 1) * 8;
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int mn = tile % (num_m * num_n), split = tile / (num_m * num_n);
        const int m0 = (mn / num_n) * kBM;
        const bool mine = (mn % num_n) == 0;
        const int kb0 = split * kb_per_split;
        const int kb1 = min(kb0 + kb_per_split, num_kb_total);
        float s[4] = {0.f, 0.f, 0.f, 0.f};
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait<true>(&full_bar[stage], phase);
          if (mine) {
            const uint8_t* sa = smem + stage * Cfg::kStageBytes;
#pragma unroll
            for (int i0 = 0; i0 < 32; i0 += 4) {  // four loads in flight, then their 16 additions
              uint2 v[4];
#pragma unroll
              for (int q = 0; q < 4; ++q) v[q] = *reinterpret_cast<const uint2*>(sa + off[q] + i0 * 256);
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                const uint32_t w[2] = {v[q].x, v[q].y};
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  if constexpr (kBf16) {  // a bf16 is the top half of its fp32
                    s[2 * e] += __uint_as_float(w[e] << 16);
                    s[2 * e + 1] += __uint_as_float(w[e] & 0xffff0000u);
                  } else {
                    const float2 f = unpack2(w[e], VDK_DTYPE_FP16);
                    s[2 * e] += f.x;
                    s[2 * e + 1] += f.y;
                  }
                }
              }
            }
          }
          __syncwarp();  // the warp's reads of the stage are done before it is released
          if (lane == 0) mbar_arrive(&empty_bar[stage]);
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
        if (mine) {  // the two row groups of a piece meet
#pragma unroll
          for (int e = 0; e < 4; ++e) s[e] += __shfl_xor_sync(0xffffffffu, s[e], 16);
          const int m = m0 + j * 64 + piece * 4;
          if (lane < 16 && m < p.M)  // M % 8 == 0 (MN-major A): the 4 columns are all in or all out
            *reinterpret_cast<float4*>(p.col_sums + static_cast<size_t>(split) * p.M + m) = make_float4(s[0], s[1], s[2], s[3]);
        }
      }
    }
  } else {
    // ===================== consumers: mainloop + epilogue =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int num_m = (p.M + kBM - 1) / kBM;
    const int num_n = (p.N + BN - 1) / BN;
    const int num_kb_total = (p.K + kBK - 1) / kBK;
    const int kb_per_split = (num_kb_total + p.split_k - 1) / p.split_k;
    const int num_tiles = num_m * num_n * p.split_k;  // work items; split index is the slowest dimension
    const int ct = threadIdx.x - 128;  // 0..255
    const int cg = ct >> 7;            // consumer warpgroup: accumulator rows cg*64 .. cg*64+63 of the tile
    const int wl = (ct >> 5) & 3, lane = ct & 31;
    const int fcol = (lane & 3) * 2;
    // epilogue: this thread's first fragment row in the warpgroup's box (the other is + 8), and the row / chunk parity
    // whose address this lane gives to stmatrix / ldmatrix
    const int frow = wl * 16 + (lane >> 2);
    const int mrow = wl * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
    const int mcb = lane >> 4;
    const bool leader = (ct & 127) == 0;  // issues, and waits for, every TMA transfer of this warpgroup's epilogue
    const uint32_t bar_id = 2 + cg;       // named barrier of this warpgroup's 128 threads
    uint8_t* ring = ring_all + cg * kRing * kBoxBytes;
    float* par = par_all + cg * Cfg::kParFloats;
    const bool f32 = p.out_dtype == VDK_DTYPE_FP32;
    const int box_cols = f32 ? 32 : 64;
    const bool has_res = kMode == kGemmLnBwd || p.epilogue == VDK_EPI_SCALE_RESIDUAL || p.epilogue == VDK_EPI_MUL_GELU_GRAD ||
                         (kMode != kGemmPlain && p.epilogue == VDK_EPI_RESIDUAL_RELU) ||
                         (kConvEx && p.epilogue == VDK_EPI_SILU_RESIDUAL);
    const bool reduce = p.partial_out && p.split_stride == 0;  // atomic split-K: TMA reduce-add into D
    int slot = 0;  // ring slot of the next box
    uint32_t res_phase = 0;
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    float colp[BN / 64][4] = {};  // kGemmLnBwd: this thread's column sums of dy xh / dy over the CTA's tiles
    uint32_t ln_tiles = 0;        // kGemmLnBwd: tiles this warpgroup has finished (exchange slot parity and phase)
    if constexpr (kMode == kGemmLnBwd) {
      // the launch makes gridDim.x a multiple of num_n, so every tile of this CTA has the same columns: gamma, 1 / gamma
      // and beta are staged once, with ln_bwd_kernel's handling of gamma == 0 and |gamma| < 1e-12
      const int n0 = (blockIdx.x % num_n) * BN;
      for (int c = ct & 127; c < BN; c += 128) {
        const int ch = (n0 + c) % p.ln_group;  // a tile may hold several LayerNorm groups (the downsample's patch rows)
        float w = p.gamma[ch];
        float iw = 0.f;
        if (w != 0.f) {
          if (fabsf(w) < 1e-12f) w = w < 0.f ? -1e-12f : 1e-12f;
          iw = 1.0f / w;
        }
        par[c] = w;
        par[BN + c] = iw;
        par[2 * BN + c] = p.beta[ch];
      }
      named_bar_sync(bar_id, 128);
    }
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int mn = tile % (num_m * num_n), split = tile / (num_m * num_n);
      const int m0 = (mn / num_n) * kBM;
      const int n0 = (mn % num_n) * BN;
      const int kb0 = split * kb_per_split;
      const int kb1 = min(kb0 + kb_per_split, num_kb_total);
      const int wrow0 = m0 + cg * 64;
      const bool live = wrow0 < p.M;  // warpgroup-uniform: the half tile below a ragged M has nothing to write
      const int nbox = (min(BN, p.N - n0) + box_cols - 1) / box_cols;
      const int npre = has_res ? min(nbox, kRing) : 0;  // residual boxes loaded while the MMAs run
      // the tile's per-column parameters (bias, gamma, beta) go to this warpgroup's copy in shared memory by cp.async, which
      // holds no registers while the MMAs run; the previous tile's epilogue has read that copy (its last barrier is behind
      // every thread of the warpgroup)
      if (kMode != kGemmLnBwd && live && (ct & 127) < BN / 4) {
        const int c = (ct & 127) * 4;  // this thread's 4 columns of each array
        const bool in = n0 + c < p.N;  // N % 8 == 0: the 4 columns are all in or all out
        if (p.bias != nullptr) cp_async_16_zfill(par + c, p.bias + (in ? n0 + c : 0), in);
        if (p.epilogue == VDK_EPI_SCALE_RESIDUAL || p.epilogue == VDK_EPI_LAYERNORM)
          cp_async_16_zfill(par + BN + c, p.gamma + (in ? n0 + c : 0), in);
        if (p.epilogue == VDK_EPI_LAYERNORM) cp_async_16_zfill(par + 2 * BN + c, p.beta + (in ? n0 + c : 0), in);
      }
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait<true>(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * Cfg::kStageBytes) + cg * 8192;  // K-major: 64 rows x 128 B; MN-major: 64-wide block
        const uint32_t sb = smem_u32(smem + stage * Cfg::kStageBytes + Cfg::kStageA);
        const uint64_t da = kTA ? wgmma_desc_mn_sw128(sa, 8192) : wgmma_desc_k_sw128(sa);
        const uint64_t db = kTB ? wgmma_desc_mn_sw128(sb, 8192) : wgmma_desc_k_sw128(sb);
        // one k16 step: K-major = 32 bytes inside the swizzle row (+2 in 16-byte units); MN-major = two 8-row groups (+128)
        constexpr uint32_t step_a = kTA ? 128u : 2u, step_b = kTB ? 128u : 2u;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k) {
          if constexpr (BN == 256) wgmma_m64n256k16_ss<kBf16, kTA, kTB>(acc, da + step_a * k, db + step_b * k, (kb > kb0 || k > 0) ? 1u : 0u);
          else wgmma_m64n128k16_ss<kBf16, kTA, kTB>(acc, da + step_a * k, db + step_b * k, (kb > kb0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        if (kb == kb0 && leader && live && npre > 0) {
          // under the tile's first MMAs: once the previous tile's stores have read the ring, TMA-load the residual boxes
          // into the slots this tile's boxes will use
          tma_store_wait_read<0>();
          mbar_arrive_expect_tx(&res_bar[cg], npre * kBoxBytes);
          for (int i = 0; i < npre; ++i)
            tma_load_3d(ring + ((slot + i) % kRing) * kBoxBytes, &map_r, &res_bar[cg], n0 + i * box_cols, wrow0, 0);
        }
        // the previous stage's MMAs have retired once at most this one is pending: its slot may be refilled
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      if (!live) continue;
      if constexpr (kMode == kGemmLnBwd) {
        mbar_wait<true>(&res_bar[cg], res_phase);
        res_phase ^= 1;
        uint8_t* xch = reinterpret_cast<uint8_t*>(res_bar + 2) + (cg * 2 + (ln_tiles & 1)) * (4 * 64 * 8);
        uint64_t* xbar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(res_bar + 2) + kLnXchBytes) + cg * 2 + (ln_tiles & 1);
        ln_bwd_tile<BN>(p, acc, colp, par, ring, wrow0, n0, fcol, frow, mrow, mcb, wl, lane, xch, xbar, (ln_tiles >> 1) & 1, leader);
        ++ln_tiles;
        // every warp has read the ring before the leader loads the next tile's y into it
        fence_proxy_async_smem();
        named_bar_sync(bar_id, 128);
        continue;
      }

      cp_async_wait_all();
      named_bar_sync(bar_id, 128);  // the warpgroup's staged parameters are visible
      float ln_mean[2] = {0.f, 0.f}, ln_rstd[2] = {1.f, 1.f};
      if (p.epilogue == VDK_EPI_LAYERNORM) {
        // the tile spans the whole row (N <= BN): the four threads of a fragment quad hold every column of its two rows,
        // and the butterfly leaves the same sums in all four.  The bias is added in place first (epi_pair skips it here),
        // so that the statistics and the normalisation see the same acc + bias without holding the bias in registers.
        if (p.bias != nullptr) {
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const float2 b = *reinterpret_cast<const float2*>(par + j * 8 + fcol);
            acc[4 * j] += b.x;
            acc[4 * j + 1] += b.y;
            acc[4 * j + 2] += b.x;
            acc[4 * j + 3] += b.y;
          }
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float sum = 0.f;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            if (j * 8 >= p.N) break;  // N % 8 == 0: the columns below N are a prefix of whole 8-column blocks
            sum += acc[4 * j + 2 * r];
            sum += acc[4 * j + 2 * r + 1];
          }
          sum += __shfl_xor_sync(0xffffffffu, sum, 1);
          sum += __shfl_xor_sync(0xffffffffu, sum, 2);
          const float mean = sum / static_cast<float>(p.N);
          float sq = 0.f;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            if (j * 8 >= p.N) break;
            const float d0 = acc[4 * j + 2 * r] - mean;
            sq = fmaf(d0, d0, sq);
            const float d1 = acc[4 * j + 2 * r + 1] - mean;
            sq = fmaf(d1, d1, sq);
          }
          sq += __shfl_xor_sync(0xffffffffu, sq, 1);
          sq += __shfl_xor_sync(0xffffffffu, sq, 2);
          ln_mean[r] = mean;
          ln_rstd[r] = rsqrtf(sq / static_cast<float>(p.N) + p.ln_eps);
        }
      }
      if (npre > 0) {
        mbar_wait<true>(&res_bar[cg], res_phase);
        res_phase ^= 1;
      }
      const int dz = (p.partial_out && p.split_stride > 0) ? split : 0;  // slab of a deterministic split-K partial
      int box_i = 0;                                                     // boxes of this tile so far
#pragma unroll
      for (int sc = 0; sc < BN / 64; ++sc) {
        if (n0 + sc * 64 >= p.N) continue;  // block-uniform
        if (f32) {
          // two boxes of 32 columns; a thread writes its float2 pairs (two wavefronts per warp store, the minimum)
#pragma unroll
          for (int hb = 0; hb < 2; ++hb) {
            const int bcol = n0 + sc * 64 + hb * 32;
            if (bcol >= p.N) continue;
            uint8_t* box = ring + slot * kBoxBytes;
            if (has_res && box_i >= npre) {  // an fp32 residual wider than the ring: load this box now
              if (leader) {
                mbar_arrive_expect_tx(&res_bar[cg], kBoxBytes);
                tma_load_3d(box, &map_r, &res_bar[cg], bcol, wrow0, 0);
              }
              mbar_wait<true>(&res_bar[cg], res_phase);
              res_phase ^= 1;
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const int j = sc * 8 + hb * 4 + q;
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int r = frow + 8 * h;
                float2* dst = reinterpret_cast<float2*>(box + box_off(r, 2 * q + (fcol >> 2)) + (fcol & 2) * 4);
                float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
                if (!p.partial_out) epi_pair<BN, kMode>(p, x0, x1, par, j * 8 + fcol, ln_mean[h], ln_rstd[h], has_res ? *dst : make_float2(0.f, 0.f));
                *dst = make_float2(x0, x1);
              }
            }
            epi_publish<kRing>(&map_d, box, slot, leader, bar_id, bcol, wrow0, dz, reduce);
            ++box_i;
          }
        } else {
          const int bcol = n0 + sc * 64;
          uint8_t* box = ring + slot * kBoxBytes;
          if (p.aux != nullptr) {
            // GELU with a saved pre-activation: store acc + bias, then apply the activation to the ROUNDED
            // pre-activation (what the backward will see, and what autocast's 16-bit Linear output hands to nn.GELU)
            // (the rounded pre-activation stays in the accumulator registers between the two boxes)
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              uint32_t rq[4];
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const int j = sc * 8 + 2 * q + (i >> 1), h = i & 1;
                float& x0 = acc[4 * j + 2 * h];
                float& x1 = acc[4 * j + 2 * h + 1];
                if (p.bias != nullptr) {
                  const float2 b = *reinterpret_cast<const float2*>(par + j * 8 + fcol);
                  x0 += b.x;
                  x1 += b.y;
                }
                rq[i] = pack2(x0, x1, p.out_dtype);
                const float2 a = unpack2(rq[i], p.out_dtype);
                x0 = a.x;
                x1 = a.y;
              }
              stmatrix_x4(smem_u32(box) + box_off(mrow, 2 * q + mcb), rq);
            }
            epi_publish<kRing>(&map_aux, box, slot, leader, bar_id, bcol, wrow0, 0, false);
            box = ring + slot * kBoxBytes;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              uint32_t rq[4];
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const int j = sc * 8 + 2 * q + (i >> 1), h = i & 1;
                float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
                gelu_pair(x0, x1);
                rq[i] = pack2(x0, x1, p.out_dtype);
              }
              stmatrix_x4(smem_u32(box) + box_off(mrow, 2 * q + mcb), rq);
            }
          } else {
            // the residual box (if any) was loaded into this slot; each warp reads and overwrites only its own rows
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const uint32_t addr = smem_u32(box) + box_off(mrow, 2 * q + mcb);
              uint32_t rin[4] = {0u, 0u, 0u, 0u}, rq[4];
              if (has_res) ldmatrix_x4(rin, addr);
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const int j = sc * 8 + 2 * q + (i >> 1), h = i & 1;
                float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
                epi_pair<BN, kMode>(p, x0, x1, par, j * 8 + fcol, ln_mean[h], ln_rstd[h], unpack2(rin[i], p.out_dtype));
                rq[i] = pack2(x0, x1, p.out_dtype);
              }
              stmatrix_x4(addr, rq);
            }
          }
          epi_publish<kRing>(&map_d, box, slot, leader, bar_id, bcol, wrow0, 0, false);
          ++box_i;
        }
      }
    }
    if (leader) tma_store_wait<0>();  // the ring stays valid until the last stores have read it
    if constexpr (kMode == kGemmLnBwd) {
      // the column sums of the 8 consumer warps meet in the (now idle) pipeline stages and are added in warp order into
      // this CTA's slab row, laid out [N / ln_group][dgamma, dbeta][ln_group]
      named_bar_sync(4, 256);  // both warpgroups are past their last MMAs
      float* part = reinterpret_cast<float*>(smem);  // [8 warps][2][BN]
      const int warp = ct >> 5, jj = ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1);
#pragma unroll
      for (int sc = 0; sc < BN / 64; ++sc)
#pragma unroll
        for (int i = 0; i < 4; ++i) part[(warp * 2 + (i >> 1)) * BN + sc * 64 + jj * 8 + fcol + (i & 1)] = colp[sc][i];
      named_bar_sync(4, 256);
      const int n0 = (blockIdx.x % num_n) * BN;
      float* row = p.ln_slab + static_cast<size_t>(blockIdx.x / num_n) * 2 * p.N;
      for (int t = ct; t < 2 * BN; t += 256) {
        const int q = t / BN, c = t - q * BN;
        float sum = 0.f;
#pragma unroll
        for (int w8 = 0; w8 < 8; ++w8) sum += part[(w8 * 2 + q) * BN + c];
        const int n = n0 + c, grp = n / p.ln_group;
        row[(grp * 2 + q) * p.ln_group + n - grp * p.ln_group] = sum;
      }
    }
  }
  if constexpr (kMode == kGemmLnBwd) {
    if (p.ln_cluster > 1) cluster_sync_all();  // no CTA leaves while a peer's st.async may still target it
  }
}

template <int BN, bool kBf16, int kTA, int kTB, int kMode = kGemmPlain>
static int launch_gemm(const CUtensorMap* maps, const GemmParams& p, cudaStream_t stream) {
  constexpr int kSmem = GemmCfg<BN>::kSmemBytes;
  auto kern = gemm_tn_kernel<BN, kBf16, kTA, kTB, kMode>;
  static bool attr_set = false;  // per instantiation
  if (!attr_set) {
    VDK_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
    attr_set = true;
  }
  const int num_tiles = ((p.M + kBM - 1) / kBM) * ((p.N + BN - 1) / BN) * p.split_k;
  const int grid = num_tiles < sm_count() ? num_tiles : sm_count();
  kern<<<grid, kGemmThreads, kSmem, stream>>>(maps[0], maps[1], maps[2], maps[3], maps[4], p);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

template <int BN, bool kBf16>
static int launch_gemm_major(const CUtensorMap* maps, const GemmParams& p, bool ta, bool tb, cudaStream_t s) {
  if (ta) return tb ? launch_gemm<BN, kBf16, 1, 1>(maps, p, s) : launch_gemm<BN, kBf16, 1, 0>(maps, p, s);
  return tb ? launch_gemm<BN, kBf16, 0, 1>(maps, p, s) : launch_gemm<BN, kBf16, 0, 0>(maps, p, s);
}

}  // namespace vdk

namespace vdk {

// kGemmLnBwd launch: a persistent grid of a multiple of num_n CTAs (each keeps one column range); rows wider than the
// tile (cluster = G / BN > 1) run as clusters of `cluster` CTAs along N, as many as can be co-resident.  Returns the grid.
template <int BN>
static int launch_gemm_ln_bwd(const CUtensorMap* maps, const GemmParams& p, int cluster, cudaStream_t s, int* grid_out) {
  constexpr int kSmem = GemmCfg<BN>::kSmemBytes + kLnSmemBytes;
  static_assert(kSmem <= 227 * 1024, "LN-backward GEMM shared memory budget");
  auto kern = gemm_tn_kernel<BN, true, 0, 1, kGemmLnBwd>;
  static int fit[5] = {};  // per cluster size: co-resident CTAs (queried once)
  cudaLaunchConfig_t cfg{};
  cfg.blockDim = dim3(kGemmThreads);
  cfg.dynamicSmemBytes = kSmem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (fit[cluster] == 0) {
    VDK_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
    int n = sm_count() / cluster;
    if (cluster > 1) {
      cfg.gridDim = dim3(cluster * sm_count());
      VDK_CUDA_OK(cudaOccupancyMaxActiveClusters(&n, kern, &cfg));
    }
    VDK_REQUIRE(n > 0, "vdk_gemm: no cluster of %d LN-backward GEMM CTAs fits on the device", cluster);
    fit[cluster] = n * cluster;
  }
  const int num_n = p.N / BN, num_tiles = ((p.M + kBM - 1) / kBM) * num_n;
  const int grid = std::min(num_tiles, fit[cluster] - fit[cluster] % num_n);
  cfg.gridDim = dim3(grid);
  VDK_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, maps[0], maps[1], maps[2], maps[3], maps[4], p));
  *grid_out = grid;
  return VDK_OK;
}

// VDK_EPI_LN_BWD: dgrad D = LayerNorm_backward(bf16(A . B^T)) (B stored [K,N]), then the fixed-order reduction of the
// per-CTA dgamma / dbeta partials
static int gemm_ln_bwd_run(const vdk_gemm_desc& g, cudaStream_t s) {
  const int G = g.ln_group;
  VDK_REQUIRE(g.in_dtype == VDK_DTYPE_BF16 && g.out_dtype == VDK_DTYPE_BF16 && !g.trans_a && g.trans_b && g.split_k <= 1 &&
                  !g.bias && !g.aux_out && !g.a_col_sums,
              "vdk_gemm: LN_BWD needs bf16 in and out, trans_b only, no split-K, bias or auxiliary output");
  VDK_REQUIRE(g.gamma && g.beta && g.residual && g.ln_rstd && g.ln_dgamma && g.ln_dbeta && g.ln_slab,
              "vdk_gemm: LN_BWD needs gamma, beta, the saved output (residual), ln_rstd, ln_dgamma, ln_dbeta and ln_slab");
  const int BN = (g.N % 256 == 0) ? 256 : 128;
  // a group is a whole number of tiles (up to 4: one cluster), or a tile a whole number of groups
  VDK_REQUIRE(G > 0 && G % 128 == 0 && g.N % G == 0 && (BN % G == 0 || (G % BN == 0 && G / BN <= 4 && G / BN != 3)),
              "vdk_gemm: LN_BWD group %d must be 128, 256, 512 or 1024 and divide N=%d (tile width %d)", G, g.N, BN);
  VDK_REQUIRE(g.lda >= g.K && g.lda % 8 == 0 && g.ldb >= g.N && g.ldb % 8 == 0 && g.ldd >= g.N && g.ldd % 8 == 0 &&
                  (reinterpret_cast<uintptr_t>(g.D) & 15) == 0,
              "vdk_gemm: LN_BWD pitches must cover the rows and keep them 16-byte aligned");
  VDK_REQUIRE(g.ln_wo >= 0 && (g.ln_wo == 0 || (g.N == 4 * G && g.M % g.ln_wo == 0)),
              "vdk_gemm: LN_BWD patch rows need N = 4 ln_group and M a multiple of ln_wo");
  VDK_REQUIRE(g.ldr >= g.N && g.ldr % 8 == 0 && (reinterpret_cast<uintptr_t>(g.residual) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(g.ln_slab) & 15) == 0,
              "vdk_gemm: LN_BWD saved-output rows and ln_slab must be 16-byte aligned");
  CUtensorMap maps[5];  // A, B, D (unused: D is written from the ring), aux_out (unused), y
  int rc = make_tma_2d_16bit(&maps[0], g.A, (uint64_t)g.M, (uint64_t)g.K, (uint64_t)g.lda, kBM, kBK);
  if (rc != VDK_OK) return rc;
  rc = make_tma_2d_16bit(&maps[1], g.B, (uint64_t)g.K, (uint64_t)g.N, (uint64_t)g.ldb, kBK, 64);
  if (rc != VDK_OK) return rc;
  rc = make_tma_epilogue_map(&maps[4], g.residual, 2, (uint64_t)g.M, (uint64_t)g.N, (uint64_t)g.ldr, 1, 0);
  if (rc != VDK_OK) return rc;
  maps[2] = maps[4];
  maps[3] = maps[4];
  GemmParams p{};
  p.M = g.M; p.N = g.N; p.K = g.K; p.D = g.D; p.ldd = g.ldd;
  p.gamma = g.gamma; p.beta = g.beta; p.residual = g.residual; p.ldr = g.ldr;
  p.out_dtype = VDK_DTYPE_BF16; p.epilogue = VDK_EPI_LN_BWD; p.split_k = 1;
  p.ln_slab = g.ln_slab; p.ln_rstd = g.ln_rstd; p.ln_group = G; p.ln_wo = g.ln_wo;
  p.ln_cluster = G > BN ? G / BN : 1;
  int grid = 0;
  {
    // algorithmic bytes: both operands, the saved output and rstd once, the output once
    ProfScope prof(kProfGemm, 2.0 * g.M * g.N * g.K,
                   2.0 * (static_cast<double>(g.M) * g.K + static_cast<double>(g.N) * g.K) + 4.0 * g.M * g.N + 4.0 * g.M * (g.N / G), s);
    rc = BN == 256 ? launch_gemm_ln_bwd<256>(maps, p, p.ln_cluster, s, &grid) : launch_gemm_ln_bwd<128>(maps, p, p.ln_cluster, s, &grid);
    if (rc != VDK_OK) return rc;
  }
  // one slab row per num_n CTAs, [N / G][dgamma, dbeta][G]: grid / num_n x N / G partials of each, 2 G floats apart
  const int n_part = grid / (g.N / BN) * (g.N / G);
  rc = launch_slab_reduce(g.ln_slab, n_part, static_cast<size_t>(2) * G, G / 4, g.ln_dgamma, 1, s);
  if (rc != VDK_OK) return rc;
  return launch_slab_reduce(g.ln_slab + G, n_part, static_cast<size_t>(2) * G, G / 4, g.ln_dbeta, 1, s);
}

int gemm_run(const vdk_gemm_desc& g, cudaStream_t s) {
  VDK_REQUIRE(g.A && g.B && g.D, "vdk_gemm: null operand");
  VDK_REQUIRE(g.M > 0 && g.N > 0 && g.K > 0, "vdk_gemm: empty problem M=%d N=%d K=%d", g.M, g.N, g.K);
  VDK_REQUIRE(g.in_dtype == VDK_DTYPE_BF16 || g.in_dtype == VDK_DTYPE_FP16, "vdk_gemm: in_dtype must be bf16/fp16");
  VDK_REQUIRE(g.out_dtype >= VDK_DTYPE_BF16 && g.out_dtype <= VDK_DTYPE_FP32, "vdk_gemm: bad out_dtype");
  // K itself is free: TMA zero-fills the contraction tail; only pitches and the output width need 16-byte granularity
  VDK_REQUIRE(g.N % 8 == 0, "vdk_gemm: N must be a multiple of 8 (N=%d)", g.N);
  VDK_REQUIRE(g.lda >= (g.trans_a ? g.M : g.K) && g.ldb >= (g.trans_b ? g.N : g.K) && g.ldd >= g.N && g.lda % 8 == 0 &&
                  g.ldb % 8 == 0,
              "vdk_gemm: bad pitches");
  if (g.trans_a) VDK_REQUIRE(g.M % 8 == 0, "vdk_gemm: trans_a needs M to be a multiple of 8");
  const int dalign = g.out_dtype == VDK_DTYPE_FP32 ? 4 : 8;
  VDK_REQUIRE(g.ldd % dalign == 0, "vdk_gemm: ldd must keep rows 16-byte aligned");
  VDK_REQUIRE((reinterpret_cast<uintptr_t>(g.D) & 15) == 0, "vdk_gemm: D must be 16-byte aligned");
  if (g.epilogue == VDK_EPI_LN_BWD) return gemm_ln_bwd_run(g, s);
  VDK_REQUIRE(g.epilogue >= VDK_EPI_NONE && g.epilogue <= VDK_EPI_MUL_GELU_GRAD, "vdk_gemm: bad epilogue");
  if (g.epilogue == VDK_EPI_MUL_GELU_GRAD) {
    VDK_REQUIRE(g.residual && g.out_dtype != VDK_DTYPE_FP32 && g.split_k <= 1 && !g.bias,
                "vdk_gemm: MUL_GELU_GRAD needs the saved pre-activation in `residual`, a 16-bit output and no bias");
    VDK_REQUIRE(g.ldr >= g.N && g.ldr % 8 == 0 && (reinterpret_cast<uintptr_t>(g.residual) & 15) == 0,
                "vdk_gemm: pre-activation rows must be 16-byte aligned");
  }
  if (g.epilogue == VDK_EPI_SCALE_RESIDUAL) {
    VDK_REQUIRE(g.gamma && g.residual, "vdk_gemm: SCALE_RESIDUAL needs gamma and residual");
    VDK_REQUIRE(g.ldr >= g.N && g.ldr % dalign == 0 && (reinterpret_cast<uintptr_t>(g.residual) & 15) == 0,
                "vdk_gemm: residual must be 16-byte aligned rows");
  }
  if (g.epilogue == VDK_EPI_LAYERNORM) {
    VDK_REQUIRE(g.gamma && g.beta, "vdk_gemm: LAYERNORM needs gamma (weight) and beta (bias)");
    VDK_REQUIRE(g.N <= 256, "vdk_gemm: LAYERNORM epilogue needs the whole row in one tile (N <= 256, got %d)", g.N);
    VDK_REQUIRE((reinterpret_cast<uintptr_t>(g.beta) & 15) == 0, "vdk_gemm: beta must be 16-byte aligned");
  }
  if (g.bias) VDK_REQUIRE((reinterpret_cast<uintptr_t>(g.bias) & 15) == 0, "vdk_gemm: bias must be 16-byte aligned");
  if (g.gamma) VDK_REQUIRE((reinterpret_cast<uintptr_t>(g.gamma) & 15) == 0, "vdk_gemm: gamma must be 16-byte aligned");
  int split = g.split_k < 1 ? 1 : g.split_k;
  {
    // every split must own at least one 64-wide K block (an empty split would publish an unwritten accumulator)
    const int kbt = (g.K + kBK - 1) / kBK;
    if (split > kbt) split = kbt;
    const int per = (kbt + split - 1) / split;
    split = (kbt + per - 1) / per;
  }
  if (g.split_stride != 0)
    VDK_REQUIRE(g.split_stride >= (long long)g.M * g.ldd && g.split_stride % 4 == 0, "vdk_gemm: split_stride must cover one [M,ldd] slab");
  if (g.split_k > 1)
    VDK_REQUIRE(g.out_dtype == VDK_DTYPE_FP32 && g.epilogue == VDK_EPI_NONE && !g.bias,
                "vdk_gemm: split_k > 1 needs fp32 output, no bias and no epilogue (partials are atomically added)");
  if (g.a_col_sums)
    VDK_REQUIRE(g.trans_a && g.split_k > 1 && g.split_stride != 0 && (reinterpret_cast<uintptr_t>(g.a_col_sums) & 15) == 0,
                "vdk_gemm: a_col_sums needs trans_a, split_k > 1 with split_stride > 0, and 16-byte alignment");

  // LayerNorm needs the whole row in one tile; otherwise narrow outputs use 128-column tiles (more tiles to
  // balance over 132 SMs) and wide ones 256.
  bool wide = (g.N % 256 == 0) || g.N > 512;
  if (g.epilogue == VDK_EPI_LAYERNORM) wide = g.N > 128;
  const int BN = wide ? 256 : 128;
  CUtensorMap maps[5];  // A, B, D, aux_out, residual
  CUtensorMap &ma = maps[0], &mb = maps[1], &md = maps[2], &maux = maps[3], &mr = maps[4];
  // K-major operand: rows = M (or N), box = tile rows x 64 contraction elements; MN-major: rows = contraction index,
  // box = 64 contraction rows x 64 M (or N) elements
  int rc = g.trans_a ? make_tma_2d_16bit(&ma, g.A, (uint64_t)g.K, (uint64_t)g.M, (uint64_t)g.lda, kBK, 64)
                     : make_tma_2d_16bit(&ma, g.A, (uint64_t)g.M, (uint64_t)g.K, (uint64_t)g.lda, kBM, kBK);
  if (rc != VDK_OK) return rc;
  rc = g.trans_b ? make_tma_2d_16bit(&mb, g.B, (uint64_t)g.K, (uint64_t)g.N, (uint64_t)g.ldb, kBK, 64)
                 : make_tma_2d_16bit(&mb, g.B, (uint64_t)g.N, (uint64_t)g.K, (uint64_t)g.ldb, BN, kBK);
  if (rc != VDK_OK) return rc;
  if (g.aux_out != nullptr) {
    VDK_REQUIRE(g.out_dtype != VDK_DTYPE_FP32 && g.split_k <= 1 && g.epilogue == VDK_EPI_GELU,
                "vdk_gemm: aux_out needs the GELU epilogue and a 16-bit output");
    VDK_REQUIRE((reinterpret_cast<uintptr_t>(g.aux_out) & 15) == 0, "vdk_gemm: aux_out must be 16-byte aligned");
  }
  // the epilogue's TMA views: D (a 3-D [split][M][ldd] view for split-K slabs), aux_out and the residual, which has D's
  // element type; the maps clip ragged M and N.  Unused views repeat D's map.
  const int osize = g.out_dtype == VDK_DTYPE_FP32 ? 4 : 2;
  const bool slabs = g.split_k > 1 && g.split_stride != 0;
  rc = make_tma_epilogue_map(&md, g.D, osize, (uint64_t)g.M, (uint64_t)g.N, (uint64_t)g.ldd, slabs ? (uint64_t)split : 1,
                             slabs ? (uint64_t)g.split_stride : 0);
  if (rc != VDK_OK) return rc;
  maux = md;
  mr = md;
  if (g.aux_out != nullptr) {
    rc = make_tma_epilogue_map(&maux, g.aux_out, 2, (uint64_t)g.M, (uint64_t)g.N, (uint64_t)g.ldd, 1, 0);
    if (rc != VDK_OK) return rc;
  }
  if (g.epilogue == VDK_EPI_SCALE_RESIDUAL || g.epilogue == VDK_EPI_MUL_GELU_GRAD) {
    rc = make_tma_epilogue_map(&mr, g.residual, osize, (uint64_t)g.M, (uint64_t)g.N, (uint64_t)g.ldr, 1, 0);
    if (rc != VDK_OK) return rc;
  }
  GemmParams p{g.M, g.N, g.K, g.D, g.ldd, g.bias, g.gamma, g.beta, g.residual, g.ldr, g.out_dtype, g.epilogue,
               g.ln_eps, split, g.split_k > 1 ? (long long)g.split_stride : 0ll, g.aux_out, (g.split_k > 1) ? 1 : 0};
  if (g.a_col_sums) p.col_sums = g.a_col_sums;  // aux_out needs split_k <= 1: the union's other member is unused here
  const bool bf = g.in_dtype == VDK_DTYPE_BF16;
  // algorithmic bytes: both operands once, the output once (x2 for an auxiliary 16-bit output), a 16-bit residual / saved tile once
  const double osz = g.out_dtype == VDK_DTYPE_FP32 ? 4.0 : 2.0;
  ProfScope prof(kProfGemm, 2.0 * g.M * g.N * g.K,
                 2.0 * (static_cast<double>(g.M) * g.K + static_cast<double>(g.N) * g.K) + osz * g.M * g.N * (g.split_k > 1 ? split : 1) +
                     (g.aux_out ? 2.0 * g.M * g.N : 0.0) + (g.residual ? osz * g.M * g.N : 0.0),
                 s);
  const bool ta = g.trans_a != 0, tb = g.trans_b != 0;
  if (wide) return bf ? launch_gemm_major<256, true>(maps, p, ta, tb, s) : launch_gemm_major<256, false>(maps, p, ta, tb, s);
  return bf ? launch_gemm_major<128, true>(maps, p, ta, tb, s) : launch_gemm_major<128, false>(maps, p, ta, tb, s);
}

// The launcher behind vdk_conv2d and vdk_conv2d_ex, on arguments its entry point has validated.  pad: low / high padding
// of the h and w axes.  ex: the vdk_conv2d_ex instantiations (SiLU epilogues, Cin a multiple of 8 with the weight's
// channels padded to Cinp = a multiple of 64 for k x k / strided convolutions).
struct ConvArgs {
  const void* x;
  const void* w;
  const float* bias;
  const void* residual;
  void* y;
  int B, H, W, Cin, Cout, kernel, stride, epilogue;
  int pad_h[2], pad_w[2];
  bool ex;
};

static int conv_launch(const ConvArgs& c, cudaStream_t s) {
  const int Ho = (c.H + c.pad_h[0] + c.pad_h[1] - c.kernel) / c.stride + 1;
  const int Wo = (c.W + c.pad_w[0] + c.pad_w[1] - c.kernel) / c.stride + 1;
  const bool dense = c.kernel == 1 && c.stride == 1 && (c.pad_h[0] | c.pad_h[1] | c.pad_w[0] | c.pad_w[1]) == 0;
  const int Cinp = dense ? c.Cin : (c.Cin + kBK - 1) / kBK * kBK;
  const long long M = static_cast<long long>(c.B) * Ho * Wo;
  const long long K = static_cast<long long>(c.kernel) * c.kernel * Cinp;
  VDK_REQUIRE(M < (1ll << 31) && K < (1ll << 31), "vdk_conv2d: problem too large (M=%lld K=%lld)", M, K);
  const bool wide = (c.Cout % 256 == 0) || c.Cout > 512;
  CUtensorMap maps[5];  // A, B, D, aux_out (unused), residual
  int rc = dense ? make_tma_2d_16bit(&maps[0], c.x, (uint64_t)M, (uint64_t)c.Cin, (uint64_t)c.Cin, kBM, kBK)
         : c.ex  ? make_tma_im2col_16bit_pads(&maps[0], c.x, c.B, c.H, c.W, c.Cin, c.kernel, c.stride, c.pad_h, c.pad_w)
                 : make_tma_im2col_16bit(&maps[0], c.x, c.B, c.H, c.W, c.Cin, c.kernel, c.stride, c.pad_h[0]);
  if (rc != VDK_OK) return rc;
  rc = make_tma_2d_16bit(&maps[1], c.w, (uint64_t)c.Cout, (uint64_t)K, (uint64_t)K, wide ? 256 : 128, kBK);
  if (rc != VDK_OK) return rc;
  rc = make_tma_epilogue_map(&maps[2], c.y, 2, (uint64_t)M, (uint64_t)c.Cout, (uint64_t)c.Cout, 1, 0);
  if (rc != VDK_OK) return rc;
  maps[3] = maps[2];
  maps[4] = maps[2];
  if (c.residual != nullptr) {
    rc = make_tma_epilogue_map(&maps[4], c.residual, 2, (uint64_t)M, (uint64_t)c.Cout, (uint64_t)c.Cout, 1, 0);
    if (rc != VDK_OK) return rc;
  }
  GemmParams p{};
  p.M = static_cast<int>(M); p.N = c.Cout; p.K = static_cast<int>(K);
  p.D = c.y; p.ldd = c.Cout; p.bias = c.bias; p.residual = c.residual; p.ldr = c.Cout;
  p.out_dtype = VDK_DTYPE_BF16; p.epilogue = c.epilogue; p.split_k = 1;
  p.cv_cpb = Cinp / kBK; p.cv_kw = c.kernel; p.cv_stride = c.stride;
  p.cv_pad = c.ex ? (c.pad_h[0] | c.pad_w[0] << 8) : c.pad_h[0];
  p.cv_wo = Wo; p.cv_howo = Ho * Wo;
  // algorithmic bytes: the input once, the weights once, the output once, the residual once (FLOPs: the executed K)
  ProfScope prof(kProfGemm, 2.0 * M * c.Cout * K,
                 2.0 * (static_cast<double>(c.B) * c.H * c.W * c.Cin + static_cast<double>(c.Cout) * K + M * c.Cout) +
                     (c.residual ? 2.0 * M * c.Cout : 0.0),
                 s);
  if (c.ex) {
    if (dense) return wide ? launch_gemm<256, true, 0, 0, kConvExDense>(maps, p, s) : launch_gemm<128, true, 0, 0, kConvExDense>(maps, p, s);
    return wide ? launch_gemm<256, true, 0, 0, kConvExIm2col>(maps, p, s) : launch_gemm<128, true, 0, 0, kConvExIm2col>(maps, p, s);
  }
  if (dense) return wide ? launch_gemm<256, true, 0, 0, kConvDense>(maps, p, s) : launch_gemm<128, true, 0, 0, kConvDense>(maps, p, s);
  return wide ? launch_gemm<256, true, 0, 0, kConvIm2col>(maps, p, s) : launch_gemm<128, true, 0, 0, kConvIm2col>(maps, p, s);
}

int conv_run(const vdk_conv_desc& c, cudaStream_t s) {
  VDK_REQUIRE(c.x && c.w && c.y, "vdk_conv2d: null operand");
  VDK_REQUIRE(c.B > 0 && c.H > 0 && c.W > 0, "vdk_conv2d: empty input B=%d H=%d W=%d", c.B, c.H, c.W);
  VDK_REQUIRE(c.Cin > 0 && c.Cin % 64 == 0, "vdk_conv2d: Cin must be a positive multiple of 64 (Cin=%d)", c.Cin);
  VDK_REQUIRE(c.Cout > 0 && c.Cout % 8 == 0, "vdk_conv2d: Cout must be a positive multiple of 8 (Cout=%d)", c.Cout);
  // the im2col map holds the bounding-box corners in 8 signed bits and the tap offsets in 8 unsigned bits
  VDK_REQUIRE(c.kernel >= 1 && c.kernel <= 16 && c.stride >= 1 && c.stride <= 8 && c.pad >= 0 && c.pad < c.kernel,
              "vdk_conv2d: unsupported kernel=%d stride=%d pad=%d", c.kernel, c.stride, c.pad);
  VDK_REQUIRE(c.H + 2 * c.pad >= c.kernel && c.W + 2 * c.pad >= c.kernel, "vdk_conv2d: kernel larger than the padded input");
  VDK_REQUIRE(c.epilogue == VDK_EPI_NONE || c.epilogue == VDK_EPI_RELU || c.epilogue == VDK_EPI_RESIDUAL_RELU,
              "vdk_conv2d: epilogue must be NONE, RELU or RESIDUAL_RELU (got %d)", c.epilogue);
  VDK_REQUIRE((c.epilogue == VDK_EPI_RESIDUAL_RELU) == (c.residual != nullptr),
              "vdk_conv2d: a residual is given exactly with the RESIDUAL_RELU epilogue");
  VDK_REQUIRE((reinterpret_cast<uintptr_t>(c.x) & 15) == 0 && (reinterpret_cast<uintptr_t>(c.w) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(c.y) & 15) == 0 && (reinterpret_cast<uintptr_t>(c.residual) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(c.bias) & 15) == 0,
              "vdk_conv2d: operands must be 16-byte aligned");
  // pad < kernel: a 1x1 convolution has no padding
  return conv_launch(ConvArgs{c.x, c.w, c.bias, c.residual, c.y, c.B, c.H, c.W, c.Cin, c.Cout, c.kernel, c.stride, c.epilogue,
                              {c.pad, c.pad}, {c.pad, c.pad}, false},
                     s);
}

int conv_ex_run(const vdk_conv_ex_desc& c, cudaStream_t s, bool allow_relu) {
  VDK_REQUIRE(c.x && c.w && c.y, "vdk_conv2d_ex: null operand");
  VDK_REQUIRE(c.B > 0 && c.H > 0 && c.W > 0, "vdk_conv2d_ex: empty input B=%d H=%d W=%d", c.B, c.H, c.W);
  VDK_REQUIRE(c.Cin > 0 && c.Cin % 8 == 0, "vdk_conv2d_ex: Cin must be a positive multiple of 8 (Cin=%d)", c.Cin);
  VDK_REQUIRE(c.Cout > 0 && c.Cout % 8 == 0, "vdk_conv2d_ex: Cout must be a positive multiple of 8 (Cout=%d)", c.Cout);
  VDK_REQUIRE(c.kernel >= 1 && c.kernel <= 16 && c.stride >= 1 && c.stride <= 8, "vdk_conv2d_ex: unsupported kernel=%d stride=%d",
              c.kernel, c.stride);
  // the low pads go to 8 bits of cv_pad each; every pad stays below the kernel, as the im2col map's corners need
  VDK_REQUIRE(c.pad_h_lo >= 0 && c.pad_h_hi >= 0 && c.pad_w_lo >= 0 && c.pad_w_hi >= 0 && c.pad_h_lo < c.kernel &&
                  c.pad_h_hi < c.kernel && c.pad_w_lo < c.kernel && c.pad_w_hi < c.kernel,
              "vdk_conv2d_ex: pads (%d, %d, %d, %d) must lie in [0, kernel)", c.pad_h_lo, c.pad_h_hi, c.pad_w_lo, c.pad_w_hi);
  VDK_REQUIRE(c.H + c.pad_h_lo + c.pad_h_hi >= c.kernel && c.W + c.pad_w_lo + c.pad_w_hi >= c.kernel,
              "vdk_conv2d_ex: kernel larger than the padded input");
  VDK_REQUIRE(c.epilogue == VDK_EPI_NONE || c.epilogue == VDK_EPI_SILU || c.epilogue == VDK_EPI_SILU_RESIDUAL ||
                  c.epilogue == VDK_EPI_HARDSWISH || (allow_relu && c.epilogue == VDK_EPI_RELU),
              "vdk_conv2d_ex: epilogue must be NONE, SILU, SILU_RESIDUAL or HARDSWISH (got %d)", c.epilogue);
  VDK_REQUIRE((c.epilogue == VDK_EPI_SILU_RESIDUAL) == (c.residual != nullptr),
              "vdk_conv2d_ex: a residual is given exactly with the SILU_RESIDUAL epilogue");
  VDK_REQUIRE((reinterpret_cast<uintptr_t>(c.x) & 15) == 0 && (reinterpret_cast<uintptr_t>(c.w) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(c.y) & 15) == 0 && (reinterpret_cast<uintptr_t>(c.residual) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(c.bias) & 15) == 0,
              "vdk_conv2d_ex: operands must be 16-byte aligned");
  return conv_launch(ConvArgs{c.x, c.w, c.bias, c.residual, c.y, c.B, c.H, c.W, c.Cin, c.Cout, c.kernel, c.stride, c.epilogue,
                              {c.pad_h_lo, c.pad_h_hi}, {c.pad_w_lo, c.pad_w_hi}, true},
                     s);
}

int conv_grouped_run(const vdk_conv_desc& c, int groups, cudaStream_t s) {
  VDK_REQUIRE(c.x && c.w && c.y, "vdk_conv2d_grouped: null operand");
  VDK_REQUIRE(c.B > 0 && c.H > 0 && c.W > 0, "vdk_conv2d_grouped: empty input B=%d H=%d W=%d", c.B, c.H, c.W);
  VDK_REQUIRE(c.Cin == c.Cout && c.Cin > 0 && c.Cin % 128 == 0,
              "vdk_conv2d_grouped: Cin must equal Cout and be a positive multiple of 128 (Cin=%d Cout=%d)", c.Cin, c.Cout);
  VDK_REQUIRE(groups >= 2 && c.Cin % groups == 0 && 128 % (c.Cin / groups) == 0,
              "vdk_conv2d_grouped: groups=%d must be >= 2 with Cin / groups dividing 128 (Cin=%d)", groups, c.Cin);
  VDK_REQUIRE(c.kernel >= 1 && c.kernel <= 16 && c.stride >= 1 && c.stride <= 8 && c.pad >= 0 && c.pad < c.kernel,
              "vdk_conv2d_grouped: unsupported kernel=%d stride=%d pad=%d", c.kernel, c.stride, c.pad);
  VDK_REQUIRE(c.H + 2 * c.pad >= c.kernel && c.W + 2 * c.pad >= c.kernel,
              "vdk_conv2d_grouped: kernel larger than the padded input");
  VDK_REQUIRE(c.epilogue == VDK_EPI_RELU && c.residual == nullptr,
              "vdk_conv2d_grouped: epilogue must be RELU, without a residual (got %d)", c.epilogue);
  VDK_REQUIRE((reinterpret_cast<uintptr_t>(c.x) & 15) == 0 && (reinterpret_cast<uintptr_t>(c.w) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(c.y) & 15) == 0 && (reinterpret_cast<uintptr_t>(c.bias) & 15) == 0,
              "vdk_conv2d_grouped: operands must be 16-byte aligned");
  const int Ho = (c.H + 2 * c.pad - c.kernel) / c.stride + 1, Wo = (c.W + 2 * c.pad - c.kernel) / c.stride + 1;
  const long long M = static_cast<long long>(c.B) * Ho * Wo;
  const long long K = static_cast<long long>(c.kernel) * c.kernel * 128;  // executed: each tile's 128 input channels
  VDK_REQUIRE(M < (1ll << 31), "vdk_conv2d_grouped: problem too large (M=%lld)", M);
  CUtensorMap maps[5];  // A, B, D, aux_out and residual (unused)
  int rc = make_tma_im2col_16bit(&maps[0], c.x, c.B, c.H, c.W, c.Cin, c.kernel, c.stride, c.pad);
  if (rc != VDK_OK) return rc;
  rc = make_tma_2d_16bit(&maps[1], c.w, (uint64_t)c.Cout, (uint64_t)K, (uint64_t)K, 128, kBK);
  if (rc != VDK_OK) return rc;
  rc = make_tma_epilogue_map(&maps[2], c.y, 2, (uint64_t)M, (uint64_t)c.Cout, (uint64_t)c.Cout, 1, 0);
  if (rc != VDK_OK) return rc;
  maps[3] = maps[2];
  maps[4] = maps[2];
  GemmParams p{};
  p.M = static_cast<int>(M); p.N = c.Cout; p.K = static_cast<int>(K);
  p.D = c.y; p.ldd = c.Cout; p.bias = c.bias; p.residual = nullptr; p.ldr = c.Cout;
  p.out_dtype = VDK_DTYPE_BF16; p.epilogue = c.epilogue; p.split_k = 1;
  p.cv_cpb = 2; p.cv_kw = c.kernel; p.cv_stride = c.stride; p.cv_pad = c.pad;
  p.cv_wo = Wo; p.cv_howo = Ho * Wo;
  // executed FLOPs (the block-diagonal K); the useful ones are a factor 128 / (Cin / groups) fewer
  ProfScope prof(kProfGemm, 2.0 * M * c.Cout * K,
                 2.0 * (static_cast<double>(c.B) * c.H * c.W * c.Cin + static_cast<double>(c.Cout) * K + M * c.Cout), s);
  return launch_gemm<128, true, 0, 0, kConvGrouped>(maps, p, s);
}

int conv_grouped_ex_cpb(int Cin, int Cout, int groups) {
  const int cgi = Cin / groups, cgo = Cout / groups;
  int cpb = 1;
  for (int n0 = 0; n0 < Cout; n0 += 128) {
    const int n1 = std::min(n0 + 128, Cout) - 1;
    const int span = (n1 / cgo + 1) * cgi - ((n0 / cgo * cgi) & ~7);  // from the tile's 16-byte-aligned c_lo
    cpb = std::max(cpb, (span + kBK - 1) / kBK);
  }
  return cpb;
}

int conv_grouped_ex_run(const vdk_conv_desc& c, int groups, cudaStream_t s) {
  VDK_REQUIRE(c.x && c.w && c.y, "vdk_conv2d_grouped_ex: null operand");
  VDK_REQUIRE(c.B > 0 && c.H > 0 && c.W > 0, "vdk_conv2d_grouped_ex: empty input B=%d H=%d W=%d", c.B, c.H, c.W);
  VDK_REQUIRE(c.Cin > 0 && c.Cin % 8 == 0 && c.Cout > 0 && c.Cout % 8 == 0,
              "vdk_conv2d_grouped_ex: Cin and Cout must be positive multiples of 8 (Cin=%d Cout=%d)", c.Cin, c.Cout);
  VDK_REQUIRE(groups >= 1 && c.Cin % groups == 0 && c.Cout % groups == 0,
              "vdk_conv2d_grouped_ex: groups=%d must be >= 1 and divide Cin=%d and Cout=%d", groups, c.Cin, c.Cout);
  VDK_REQUIRE(c.kernel >= 1 && c.kernel <= 16 && c.stride >= 1 && c.stride <= 8 && c.pad >= 0 && c.pad < c.kernel,
              "vdk_conv2d_grouped_ex: unsupported kernel=%d stride=%d pad=%d", c.kernel, c.stride, c.pad);
  VDK_REQUIRE(c.H + 2 * c.pad >= c.kernel && c.W + 2 * c.pad >= c.kernel,
              "vdk_conv2d_grouped_ex: kernel larger than the padded input");
  VDK_REQUIRE(c.epilogue == VDK_EPI_NONE || c.epilogue == VDK_EPI_RELU || c.epilogue == VDK_EPI_RESIDUAL_RELU,
              "vdk_conv2d_grouped_ex: epilogue must be NONE, RELU or RESIDUAL_RELU (got %d)", c.epilogue);
  VDK_REQUIRE((c.epilogue == VDK_EPI_RESIDUAL_RELU) == (c.residual != nullptr),
              "vdk_conv2d_grouped_ex: a residual is given exactly with the RESIDUAL_RELU epilogue");
  VDK_REQUIRE((reinterpret_cast<uintptr_t>(c.x) & 15) == 0 && (reinterpret_cast<uintptr_t>(c.w) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(c.y) & 15) == 0 && (reinterpret_cast<uintptr_t>(c.residual) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(c.bias) & 15) == 0,
              "vdk_conv2d_grouped_ex: operands must be 16-byte aligned");
  if (groups == 1) {
    // a dense 1x1 / stride-1 convolution: the plain GEMM over [B*H*W, Cin], K = Cin (TMA zero-fills the last K block)
    VDK_REQUIRE(c.kernel == 1 && c.stride == 1,
                "vdk_conv2d_grouped_ex: groups=1 takes a 1x1 / stride-1 kernel only (kernel=%d stride=%d)", c.kernel, c.stride);
    return conv_launch(ConvArgs{c.x, c.w, c.bias, c.residual, c.y, c.B, c.H, c.W, c.Cin, c.Cout, 1, 1, c.epilogue, {0, 0}, {0, 0},
                                false},
                       s);
  }
  const int Ho = (c.H + 2 * c.pad - c.kernel) / c.stride + 1, Wo = (c.W + 2 * c.pad - c.kernel) / c.stride + 1;
  const int cpb = conv_grouped_ex_cpb(c.Cin, c.Cout, groups);
  const long long M = static_cast<long long>(c.B) * Ho * Wo;
  const long long K = static_cast<long long>(c.kernel) * c.kernel * cpb * kBK;  // executed per output channel
  VDK_REQUIRE(M < (1ll << 31), "vdk_conv2d_grouped_ex: problem too large (M=%lld)", M);
  CUtensorMap maps[5];  // A, B, D, aux_out (unused), residual
  const int pads[2] = {c.pad, c.pad};
  int rc = make_tma_im2col_16bit_pads(&maps[0], c.x, c.B, c.H, c.W, c.Cin, c.kernel, c.stride, pads, pads);
  if (rc != VDK_OK) return rc;
  rc = make_tma_2d_16bit(&maps[1], c.w, (uint64_t)c.Cout, (uint64_t)K, (uint64_t)K, 128, kBK);
  if (rc != VDK_OK) return rc;
  rc = make_tma_epilogue_map(&maps[2], c.y, 2, (uint64_t)M, (uint64_t)c.Cout, (uint64_t)c.Cout, 1, 0);
  if (rc != VDK_OK) return rc;
  maps[3] = maps[2];
  maps[4] = maps[2];
  if (c.residual != nullptr) {
    rc = make_tma_epilogue_map(&maps[4], c.residual, 2, (uint64_t)M, (uint64_t)c.Cout, (uint64_t)c.Cout, 1, 0);
    if (rc != VDK_OK) return rc;
  }
  GemmParams p{};
  p.M = static_cast<int>(M); p.N = c.Cout; p.K = static_cast<int>(K);
  p.D = c.y; p.ldd = c.Cout; p.bias = c.bias; p.residual = c.residual;
  p.out_dtype = VDK_DTYPE_BF16; p.epilogue = c.epilogue; p.split_k = 1;
  p.cv_cpb = cpb; p.cv_kw = c.kernel; p.cv_stride = c.stride; p.cv_pad = c.pad;
  p.cv_wo = Wo; p.cv_howo = Ho * Wo;
  p.cv_cg_in = c.Cin / groups; p.cv_cg_out = c.Cout / groups;
  // executed FLOPs; the useful ones are a factor cpb * 64 / (Cin / groups) fewer
  ProfScope prof(kProfGemm, 2.0 * M * c.Cout * K,
                 2.0 * (static_cast<double>(c.B) * c.H * c.W * c.Cin + static_cast<double>(c.Cout) * K + M * c.Cout) +
                     (c.residual ? 2.0 * M * c.Cout : 0.0),
                 s);
  return launch_gemm<128, true, 0, 0, kConvGroupedEx>(maps, p, s);
}

}  // namespace vdk

extern "C" int vdk_conv2d(const vdk_conv_desc* desc, void* stream) {
  VDK_REQUIRE(desc, "vdk_conv2d: null descriptor");
  return vdk::conv_run(*desc, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vdk_conv2d_ex(const vdk_conv_ex_desc* desc, void* stream) {
  VDK_REQUIRE(desc, "vdk_conv2d_ex: null descriptor");
  return vdk::conv_ex_run(*desc, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vdk_conv2d_grouped(const vdk_conv_desc* desc, int groups, void* stream) {
  VDK_REQUIRE(desc, "vdk_conv2d_grouped: null descriptor");
  return vdk::conv_grouped_run(*desc, groups, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vdk_conv2d_grouped_ex(const vdk_conv_desc* desc, int groups, void* stream) {
  VDK_REQUIRE(desc, "vdk_conv2d_grouped_ex: null descriptor");
  return vdk::conv_grouped_ex_run(*desc, groups, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vdk_gemm_effective_splits(int K, int split_k) {
  int split = split_k < 1 ? 1 : split_k;
  const int kbt = (K + vdk::kBK - 1) / vdk::kBK;
  if (split > kbt) split = kbt;
  const int per = (kbt + split - 1) / split;
  return (kbt + per - 1) / per;
}

extern "C" int vdk_gemm(const vdk_gemm_desc* desc, void* stream) {
  VDK_REQUIRE(desc, "vdk_gemm: null descriptor");
  return vdk::gemm_run(*desc, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vdk_gemm_tn(const void* A, const void* B, void* D, int M, int N, int K, int lda, int ldb, int ldd,
                           int in_dtype, int out_dtype, int epilogue, const float* bias, const float* gamma,
                           const void* residual, int ldr, void* stream) {
  vdk_gemm_desc g{};
  g.A = A; g.B = B; g.D = D;
  g.M = M; g.N = N; g.K = K; g.lda = lda; g.ldb = ldb; g.ldd = ldd;
  g.in_dtype = in_dtype; g.out_dtype = out_dtype; g.epilogue = epilogue;
  g.bias = bias; g.gamma = gamma; g.residual = residual; g.ldr = ldr;
  g.split_k = 1;
  return vdk::gemm_run(g, reinterpret_cast<cudaStream_t>(stream));
}
