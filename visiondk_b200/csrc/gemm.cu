// gemm.cu — D = epilogue(A . B^T) on sm_90a warpgroup tensor cores (wgmma), operands staged by TMA.
//
// Replaces the library GEMMs behind timm's ConvNeXt/ViT Linear layers and patchify convolutions that
// models/faceX/backbone/timm_wrapper.py:52 runs, and the neck Linear of timm_wrapper.py:36 (SURVEY K1-K5).
//
// One persistent CTA per SM, 384 threads:
//   warpgroup 0    : TMA producer (one thread; A tile 128x64, B tile BNx64 per stage, 128-byte swizzle), registers
//                    handed to the consumers with setmaxnreg
//   warpgroups 1-2 : consumers, 64 rows each: wgmma m64 x BN x 16 into registers (fp32), then the epilogue.  The
//                    accumulator leaves the registers 64 columns at a time through shared memory so that each thread
//                    finishes 32 consecutive columns of one row (bias / GELU / layer-scale+residual / LayerNorm /
//                    GELU' -> 16-byte global stores) while the producer already fills the stages of the next tile.
#include "vdk_host.h"
#include "vdk_ptx.cuh"

#include <cstdlib>

namespace vdk {

constexpr int kBM = 128;
constexpr int kBK = 64;  // 64 x 16-bit = one 128-byte swizzle row
constexpr int kGemmThreads = 384;  // producer warpgroup, two consumer warpgroups
constexpr int kAccLd = 64 + 4;     // fp32 row pitch of the staged 128 x 64 accumulator chunk (conflict-free row reads)

struct GemmParams {
  int M, N, K;
  void* D;
  int ldd;
  const float* bias;
  const float* gamma;  // layer-scale (SCALE_RESIDUAL) or LayerNorm weight (LAYERNORM)
  const float* beta;   // LayerNorm bias
  const void* residual;  // SCALE_RESIDUAL: added; MUL_GELU_GRAD: the saved 16-bit pre-activation whose GELU' scales the output
  int ldr;
  int out_dtype;
  int epilogue;
  float ln_eps;
  int split_k;  // > 1: each tile's K range is split over split_k work items, fp32 partials are atomically added
  long long split_stride;  // > 0: split s writes its partial tile to D + s*split_stride with plain stores (deterministic)
  void* aux;  // GELU only: also store the pre-activation (acc + bias) here, pitch ldd (saved for the backward)
  int partial_out;  // the caller asked for split-K: raw fp32 partials are added / slab-stored even if one split remains
};

template <int BN>
struct GemmCfg {
  static constexpr int kStageA = kBM * kBK * 2;
  static constexpr int kStageB = BN * kBK * 2;
  static constexpr int kStageBytes = kStageA + kStageB;
  static constexpr int kStages = (BN == 256) ? 3 : 5;
  static constexpr int kAccBytes = kBM * kAccLd * 4;
  // stages + staged accumulator chunk + bias [BN] + LayerNorm mean / rstd [2][128] + barriers + 1 KB align slack
  static constexpr int kSmemBytes = kStages * kStageBytes + kAccBytes + BN * 4 + 2 * kBM * 4 + 2 * kStages * 8 + 1024;
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

// Per-chunk epilogue arithmetic on this thread's 32 consecutive columns [col0, col0 + ncols) of row `row`.
// `bsm`: this tile's bias values for columns [col0, col0 + 32) in shared memory (zero beyond N): staged once per tile so
// that the epilogue's critical path holds no global loads.
__device__ __forceinline__ void add_bias32(float (&v)[32], const float* bsm) {
#pragma unroll
  for (int j = 0; j < 32; j += 4) {
    const float4 b = *reinterpret_cast<const float4*>(bsm + j);
    v[j] += b.x; v[j + 1] += b.y; v[j + 2] += b.z; v[j + 3] += b.w;
  }
}
__device__ __forceinline__ void epi_math(const GemmParams& p, float (&v)[32], int row, int col0, int ncols, float ln_mean,
                                         float ln_rstd, const float* bsm) {
  if (p.bias != nullptr) add_bias32(v, bsm);
  if (p.epilogue == VDK_EPI_MUL_GELU_GRAD) {
    if (row < p.M) {
      const uint16_t* pre = reinterpret_cast<const uint16_t*>(p.residual) + static_cast<size_t>(row) * p.ldr + col0;
#pragma unroll
      for (int j = 0; j < 32; j += 8) {
        if (j < ncols) {
          const uint4 t = *reinterpret_cast<const uint4*>(pre + j);
          const float2 a0 = unpack2(t.x, p.out_dtype), a1 = unpack2(t.y, p.out_dtype);
          const float2 a2 = unpack2(t.z, p.out_dtype), a3 = unpack2(t.w, p.out_dtype);
          const float2 g0 = gelu_grad_pair(a0.x, a0.y), g1 = gelu_grad_pair(a1.x, a1.y);
          const float2 g2 = gelu_grad_pair(a2.x, a2.y), g3 = gelu_grad_pair(a3.x, a3.y);
          v[j] *= g0.x; v[j + 1] *= g0.y; v[j + 2] *= g1.x; v[j + 3] *= g1.y;
          v[j + 4] *= g2.x; v[j + 5] *= g2.y; v[j + 6] *= g3.x; v[j + 7] *= g3.y;
        }
      }
    }
  } else if (p.epilogue == VDK_EPI_GELU) {
#pragma unroll
    for (int j = 0; j < 32; j += 2) gelu_pair(v[j], v[j + 1]);
  } else if (p.epilogue == VDK_EPI_LAYERNORM) {
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      if (j < ncols) {
        const float4 g = __ldg(reinterpret_cast<const float4*>(p.gamma + col0 + j));
        const float4 b = __ldg(reinterpret_cast<const float4*>(p.beta + col0 + j));
        v[j] = (v[j] - ln_mean) * ln_rstd * g.x + b.x;
        v[j + 1] = (v[j + 1] - ln_mean) * ln_rstd * g.y + b.y;
        v[j + 2] = (v[j + 2] - ln_mean) * ln_rstd * g.z + b.z;
        v[j + 3] = (v[j + 3] - ln_mean) * ln_rstd * g.w + b.w;
      }
    }
  } else if (p.epilogue == VDK_EPI_SCALE_RESIDUAL) {
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      if (j < ncols) {
        const float4 g = __ldg(reinterpret_cast<const float4*>(p.gamma + col0 + j));
        v[j] *= g.x; v[j + 1] *= g.y; v[j + 2] *= g.z; v[j + 3] *= g.w;
      }
    }
    if (row < p.M) {
      if (p.out_dtype == VDK_DTYPE_FP32) {
        const float* res = reinterpret_cast<const float*>(p.residual) + static_cast<size_t>(row) * p.ldr + col0;
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          if (j < ncols) {
            const float4 t = *reinterpret_cast<const float4*>(res + j);
            v[j] += t.x; v[j + 1] += t.y; v[j + 2] += t.z; v[j + 3] += t.w;
          }
        }
      } else {
        const uint16_t* res = reinterpret_cast<const uint16_t*>(p.residual) + static_cast<size_t>(row) * p.ldr + col0;
#pragma unroll
        for (int j = 0; j < 32; j += 8) {
          if (j < ncols) {
            const uint4 t = *reinterpret_cast<const uint4*>(res + j);
            const float2 a0 = unpack2(t.x, p.out_dtype), a1 = unpack2(t.y, p.out_dtype);
            const float2 a2 = unpack2(t.z, p.out_dtype), a3 = unpack2(t.w, p.out_dtype);
            v[j] += a0.x; v[j + 1] += a0.y; v[j + 2] += a1.x; v[j + 3] += a1.y;
            v[j + 4] += a2.x; v[j + 5] += a2.y; v[j + 6] += a3.x; v[j + 7] += a3.y;
          }
        }
      }
    }
  }
}
// kTA / kTB: operand stored with the contraction index as the slow dimension ([K,M] / [K,N] row-major: MN-major)
template <int BN, bool kBf16, int kTA, int kTB>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tn_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const GemmParams p) {
  using Cfg = GemmCfg<BN>;
  constexpr int kStages = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  // align inside the dynamic smem window without a pointer->integer->pointer round trip (which would demote every
  // later access to generic LD/ST)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  float* acc_sm = reinterpret_cast<float*>(smem + kStages * Cfg::kStageBytes);  // [128][kAccLd]
  float* bias_sm = acc_sm + kBM * kAccLd;                                      // [BN] bias of the tile being finished
  float* ln_sm = bias_sm + BN;                                                 // [2][128] LayerNorm mean, rstd per row
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ln_sm + 2 * kBM);
  uint64_t* empty_bar = full_bar + kStages;

  const int num_m = (p.M + kBM - 1) / kBM;
  const int num_n = (p.N + BN - 1) / BN;
  const int num_kb_total = (p.K + kBK - 1) / kBK;
  const int kb_per_split = (num_kb_total + p.split_k - 1) / p.split_k;
  const int num_tiles = num_m * num_n * p.split_k;  // work items; split index is the slowest dimension

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_a);
    prefetch_tensormap(&map_b);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (threadIdx.x < 128) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int mn = tile % (num_m * num_n), split = tile / (num_m * num_n);
        const int m0 = (mn / num_n) * kBM;
        const int n0 = (mn % num_n) * BN;
        const int kb0 = split * kb_per_split;
        const int kb1 = min(kb0 + kb_per_split, num_kb_total);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait_relaxed<true>(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * Cfg::kStageBytes;
          uint8_t* sb = sa + Cfg::kStageA;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          if (kTA) {  // [K,M] storage: 64-wide M blocks x 64 contraction rows, 8 KB each
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
    }
  } else {
    // ===================== consumers: mainloop + epilogue =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int ct = threadIdx.x - 128;  // 0..255
    const int cg = ct >> 7;            // consumer warpgroup: accumulator rows cg*64 .. cg*64+63 of the tile
    const int wl = (ct >> 5) & 3, lane = ct & 31;
    const int frow = cg * 64 + wl * 16 + (lane >> 2);  // first of this thread's two fragment rows (the other is + 8)
    const int fcol = (lane & 3) * 2;
    const int erow = ct & 127, half = ct >> 7;         // epilogue: row and 32-column half of a staged chunk
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int mn = tile % (num_m * num_n), split = tile / (num_m * num_n);
      const int m0 = (mn / num_n) * kBM;
      const int n0 = (mn % num_n) * BN;
      const int kb0 = split * kb_per_split;
      const int kb1 = min(kb0 + kb_per_split, num_kb_total);
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

      if (p.epilogue == VDK_EPI_LAYERNORM) {
        // the tile spans the whole row (N <= BN): the four threads of a fragment quad hold every column of its two rows
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float sum = 0.f;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = n0 + j * 8 + fcol + e;
              if (col < p.N) sum += acc[4 * j + 2 * r + e] + (p.bias ? __ldg(p.bias + col) : 0.f);
            }
          sum += __shfl_xor_sync(0xffffffffu, sum, 1);
          sum += __shfl_xor_sync(0xffffffffu, sum, 2);
          const float mean = sum / static_cast<float>(p.N);
          float sq = 0.f;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = n0 + j * 8 + fcol + e;
              if (col < p.N) {
                const float d = acc[4 * j + 2 * r + e] + (p.bias ? __ldg(p.bias + col) : 0.f) - mean;
                sq = fmaf(d, d, sq);
              }
            }
          sq += __shfl_xor_sync(0xffffffffu, sq, 1);
          sq += __shfl_xor_sync(0xffffffffu, sq, 2);
          if ((lane & 3) == 0) {
            ln_sm[frow + 8 * r] = mean;
            ln_sm[kBM + frow + 8 * r] = rsqrtf(sq / static_cast<float>(p.N) + p.ln_eps);
          }
        }
      }
      if (p.bias != nullptr && ct < BN) bias_sm[ct] = (n0 + ct < p.N) ? __ldg(p.bias + n0 + ct) : 0.f;
      const int row = m0 + erow;
#pragma unroll
      for (int sc = 0; sc < BN / 64; ++sc) {
        if (n0 + sc * 64 < p.N) {  // block-uniform
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = sc * 8 + jj;
            *reinterpret_cast<float2*>(acc_sm + frow * kAccLd + jj * 8 + fcol) = make_float2(acc[4 * j], acc[4 * j + 1]);
            *reinterpret_cast<float2*>(acc_sm + (frow + 8) * kAccLd + jj * 8 + fcol) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
          }
          named_bar_sync(1, 256);  // the chunk (and, before the first one, the bias and LayerNorm statistics) is in smem
          float v[32];
#pragma unroll
          for (int j = 0; j < 32; j += 4) {
            const float4 t = *reinterpret_cast<const float4*>(acc_sm + erow * kAccLd + half * 32 + j);
            v[j] = t.x; v[j + 1] = t.y; v[j + 2] = t.z; v[j + 3] = t.w;
          }
          named_bar_sync(1, 256);  // every thread holds its piece: the buffer may take the next chunk
          const float ln_mean = p.epilogue == VDK_EPI_LAYERNORM ? ln_sm[erow] : 0.f;
          const float ln_rstd = p.epilogue == VDK_EPI_LAYERNORM ? ln_sm[kBM + erow] : 1.f;
          const int col0 = n0 + sc * 64 + half * 32;
          const int ncols = min(32, p.N - col0);  // multiple of 8 (N % 8 == 0 is required)
          if (row < p.M && ncols > 0) {
            if (p.partial_out) {
              // split-K: raw fp32 partial sums.  With a slab stride every split owns its own copy of D (plain stores,
              // the consumer adds the slabs in a fixed order: deterministic); otherwise they are atomically added
              // into a D the caller zeroed.
              if (p.split_stride > 0) {
                float* out = reinterpret_cast<float*>(p.D) + static_cast<size_t>(split) * p.split_stride +
                             static_cast<size_t>(row) * p.ldd + col0;
#pragma unroll
                for (int j = 0; j < 32; j += 4)
                  if (j < ncols) *reinterpret_cast<float4*>(out + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
              } else {
                float* out = reinterpret_cast<float*>(p.D) + static_cast<size_t>(row) * p.ldd + col0;
#pragma unroll
                for (int j = 0; j < 32; ++j)
                  if (j < ncols) atomicAdd(out + j, v[j]);
              }
            } else {
              if (p.aux != nullptr) {
                // GELU with a saved pre-activation: store acc + bias, then apply the activation to the ROUNDED
                // pre-activation (what the backward will see, and what autocast's 16-bit Linear output hands to nn.GELU)
                if (p.bias != nullptr) add_bias32(v, bias_sm + (col0 - n0));
                uint16_t* aux = reinterpret_cast<uint16_t*>(p.aux) + static_cast<size_t>(row) * p.ldd + col0;
#pragma unroll
                for (int j = 0; j < 32; j += 8) {
                  if (j < ncols) {
                    uint4 t;
                    t.x = pack2(v[j], v[j + 1], p.out_dtype);
                    t.y = pack2(v[j + 2], v[j + 3], p.out_dtype);
                    t.z = pack2(v[j + 4], v[j + 5], p.out_dtype);
                    t.w = pack2(v[j + 6], v[j + 7], p.out_dtype);
                    *reinterpret_cast<uint4*>(aux + j) = t;
                  }
                }
#pragma unroll
                for (int j = 0; j < 32; j += 2) {
                  float2 a = unpack2(pack2(v[j], v[j + 1], p.out_dtype), p.out_dtype);
                  gelu_pair(a.x, a.y);
                  v[j] = a.x;
                  v[j + 1] = a.y;
                }
              } else {
                epi_math(p, v, row, col0, ncols, ln_mean, ln_rstd, bias_sm + (col0 - n0));
              }
              if (p.out_dtype == VDK_DTYPE_FP32) {
                float* out = reinterpret_cast<float*>(p.D) + static_cast<size_t>(row) * p.ldd + col0;
#pragma unroll
                for (int j = 0; j < 32; j += 4)
                  if (j < ncols) *reinterpret_cast<float4*>(out + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
              } else {
                uint16_t* out = reinterpret_cast<uint16_t*>(p.D) + static_cast<size_t>(row) * p.ldd + col0;
#pragma unroll
                for (int j = 0; j < 32; j += 8) {
                  if (j < ncols) {
                    uint4 t;
                    t.x = pack2(v[j], v[j + 1], p.out_dtype);
                    t.y = pack2(v[j + 2], v[j + 3], p.out_dtype);
                    t.z = pack2(v[j + 4], v[j + 5], p.out_dtype);
                    t.w = pack2(v[j + 6], v[j + 7], p.out_dtype);
                    *reinterpret_cast<uint4*>(out + j) = t;
                  }
                }
              }
            }
          }
        }
      }
      named_bar_sync(1, 256);  // bias and LayerNorm statistics of this tile are consumed
    }
  }
}

template <int BN, bool kBf16, int kTA, int kTB>
static int launch_gemm(const CUtensorMap& ma, const CUtensorMap& mb, const GemmParams& p, cudaStream_t stream) {
  constexpr int kSmem = GemmCfg<BN>::kSmemBytes;
  auto kern = gemm_tn_kernel<BN, kBf16, kTA, kTB>;
  static bool attr_set = false;  // per instantiation
  if (!attr_set) {
    VDK_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
    attr_set = true;
  }
  const int num_tiles = ((p.M + kBM - 1) / kBM) * ((p.N + BN - 1) / BN) * p.split_k;
  const int grid = num_tiles < sm_count() ? num_tiles : sm_count();
  kern<<<grid, kGemmThreads, kSmem, stream>>>(ma, mb, p);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

template <int BN, bool kBf16>
static int launch_gemm_major(const CUtensorMap& ma, const CUtensorMap& mb, const GemmParams& p, bool ta, bool tb,
                             cudaStream_t s) {
  if (ta) return tb ? launch_gemm<BN, kBf16, 1, 1>(ma, mb, p, s) : launch_gemm<BN, kBf16, 1, 0>(ma, mb, p, s);
  return tb ? launch_gemm<BN, kBf16, 0, 1>(ma, mb, p, s) : launch_gemm<BN, kBf16, 0, 0>(ma, mb, p, s);
}

}  // namespace vdk

namespace vdk {

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

  // LayerNorm needs the whole row in one tile; otherwise narrow outputs use 128-column tiles (more tiles to
  // balance over 132 SMs) and wide ones 256.
  bool wide = (g.N % 256 == 0) || g.N > 512;
  if (g.epilogue == VDK_EPI_LAYERNORM) wide = g.N > 128;
  const int BN = wide ? 256 : 128;
  CUtensorMap ma, mb;
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
  GemmParams p{g.M, g.N, g.K, g.D, g.ldd, g.bias, g.gamma, g.beta, g.residual, g.ldr, g.out_dtype, g.epilogue,
               g.ln_eps, split, g.split_k > 1 ? (long long)g.split_stride : 0ll, g.aux_out, (g.split_k > 1) ? 1 : 0};
  const bool bf = g.in_dtype == VDK_DTYPE_BF16;
  // algorithmic bytes: both operands once, the output once (x2 for an auxiliary 16-bit output), a 16-bit residual / saved tile once
  const double osz = g.out_dtype == VDK_DTYPE_FP32 ? 4.0 : 2.0;
  ProfScope prof(kProfGemm, 2.0 * g.M * g.N * g.K,
                 2.0 * (static_cast<double>(g.M) * g.K + static_cast<double>(g.N) * g.K) + osz * g.M * g.N * (g.split_k > 1 ? split : 1) +
                     (g.aux_out ? 2.0 * g.M * g.N : 0.0) + (g.residual ? osz * g.M * g.N : 0.0),
                 s);
  const bool ta = g.trans_a != 0, tb = g.trans_b != 0;
  if (wide) return bf ? launch_gemm_major<256, true>(ma, mb, p, ta, tb, s) : launch_gemm_major<256, false>(ma, mb, p, ta, tb, s);
  return bf ? launch_gemm_major<128, true>(ma, mb, p, ta, tb, s) : launch_gemm_major<128, false>(ma, mb, p, ta, tb, s);
}

}  // namespace vdk

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
