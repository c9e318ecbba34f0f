// swin.cu — timm 0.9.16 SwinTransformerV2 (swinv2_base_window8_256, swinv2_large_window12to16_192to256) embedding forward
// for the faceX / CBIR extract path, NHWC bf16.
//
// Replaces TimmWrapper.forward for Swin V2 backbones (models/faceX/backbone/timm_wrapper.py:16-21, 30-38, 51-54: timm
// SwinTransformerV2 with num_classes=0, global_pool='' -> its NHWC [B, 8, 8, C] map, which the wrapper's rank rule sends
// through BatchNorm2d(8) -> Flatten -> Linear -> BatchNorm1d) and F.normalize (face_model.py:139).
//
// Written here:
//   window_attention   shifted-window cosine attention of one (image, window, head) per CTA, read straight from the qkv
//                      GEMM's output in natural token order: the roll, the window partition, their inverses and the shift
//                      mask are index arithmetic, and no score leaves the chip (mma.sync m16n8k16 for Q K^T and P V)
//   postnorm_residual  x <- x + LayerNorm(y) * gamma + beta (timm's res-post-norm), one warp per row
// Every Linear is the wgmma GEMM (gemm.cu); the patch embedding is the ConvNeXt stem's patchify + GEMM with the LayerNorm
// epilogue, patch merging a 2x2/s2 vdk_conv2d + ln_patchify, and the neck the shared launch_neck.
#include "vdk_host.h"
#include "vdk_ptx.cuh"

#include <algorithm>
#include "convnext_internal.h"

namespace vdk {

constexpr int kWinD = 32;  // head dim of both Swin V2 towers

__device__ __forceinline__ void win_mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ float win_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// byte offset of 16-byte chunk `chunk` (0..3) of row `row` in a [rows][32] bf16 tile: 64-byte rows, chunk index XOR
// ((row >> 1) & 3), so that the 8 rows one ldmatrix matrix reads fall in 8 distinct 16-byte bank groups
__device__ __forceinline__ int win_tile_off(int row, int chunk) { return row * 64 + ((chunk ^ ((row >> 1) & 3)) << 4); }

// timm's shift regions on one axis of length L (rolled coordinate r): slices (0:-w), (-w:-s), (-s:)
__device__ __forceinline__ int win_region(int r, int L, int w, int s) { return r < L - w ? 0 : (r < L - s ? 1 : 2); }

// qkv: [B, H, W, 3, heads, 32] bf16 (the qkv Linear's output as stored, natural token order); out: [B, H, W, heads * 32].
// CTA = one (image, window, head): the window's q, k, v rows are gathered with 16-byte cp.async from their rolled positions,
// the per-head relative-position bias table [(2w-1)^2] is staged in shared memory.  Each warp owns 16-query-row blocks and
// keeps a whole score row (64 or 256 keys) in registers: the softmax is exact (max, then exp and sum), with no rescale.
template <int kW>
__global__ void __launch_bounds__(kW == 8 ? 128 : 256)
window_attention_kernel(const __nv_bfloat16* __restrict__ qkv, int H, int Wd, int heads, int shift,
                        const float* __restrict__ scale, const float* __restrict__ bias, __nv_bfloat16* __restrict__ out) {
  constexpr int kN = kW * kW;                    // tokens per window
  constexpr int kWarps = kW == 8 ? 4 : 8;
  constexpr int kRowBlocks = kN / 16 / kWarps;   // 16-row blocks per warp: 1 (w = 8) or 2 (w = 16)
  constexpr int kJ = kN / 8;                     // 8-key score tiles of a row block
  constexpr int kT = 2 * kW - 1;                 // side of the relative-position table
  extern __shared__ __align__(128) uint8_t win_smem[];
  uint8_t* sq = win_smem;  // q, k, v: [kN][32] bf16 each
  uint8_t* sk = sq + kN * 64;
  uint8_t* sv = sk + kN * 64;
  float* s_qs = reinterpret_cast<float*>(sv + kN * 64);  // [kN] scale / max(|q|, 1e-12)
  float* s_rk = s_qs + kN;                                // [kN] 1 / max(|k|, 1e-12)
  float* s_bias = s_rk + kN;                              // [kT * kT]

  const int C = heads * kWinD;
  const int nwx = Wd / kW, nwin = (H / kW) * nwx;
  int item = blockIdx.x;
  const int h = item % heads;
  item /= heads;
  const int win = item % nwin, b = item / nwin;
  const int wy = win / nwx, wx = win - wy * nwx;
  // token t = (ty, tx) of the window lies at rolled (wy w + ty, wx w + tx), i.e. at natural ((wy w + ty + shift) mod H, ...);
  // the output goes back to the same natural position (window_reverse, then the roll by +shift)
  auto token = [&](int t) -> int64_t {
    int y = wy * kW + t / kW + shift, x = wx * kW + t % kW + shift;
    if (y >= H) y -= H;
    if (x >= Wd) x -= Wd;
    return (static_cast<int64_t>(b) * H + y) * Wd + x;
  };

  const int64_t ld = 3 * static_cast<int64_t>(C);
  for (int idx = threadIdx.x; idx < kN * 12; idx += blockDim.x) {
    const int t = idx / 12, rem = idx - t * 12, m = rem >> 2, ch = rem & 3;  // m: 0 q, 1 k, 2 v
    const __nv_bfloat16* src = qkv + token(t) * ld + m * C + h * kWinD + ch * 8;
    cp_async_16_zfill(win_smem + m * (kN * 64) + win_tile_off(t, ch), src, true);
  }
  for (int i = threadIdx.x; i < kT * kT; i += blockDim.x) s_bias[i] = __ldg(bias + static_cast<int64_t>(h) * kT * kT + i);
  cp_async_wait_all();
  __syncthreads();
  // fp32 norms of the stored bf16 q and k rows, with F.normalize's max(|.|, 1e-12)
  const float sc = __ldg(scale + h);
  for (int r = threadIdx.x; r < 2 * kN; r += blockDim.x) {
    const int t = r % kN;
    const uint8_t* tile = r < kN ? sq : sk;
    float ss = 0.f;
#pragma unroll
    for (int ch = 0; ch < 4; ++ch) {
      const uint4 u = *reinterpret_cast<const uint4*>(tile + win_tile_off(t, ch));
      const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = __bfloat1622float2(p[i]);
        ss = fmaf(f.x, f.x, ss);
        ss = fmaf(f.y, f.y, ss);
      }
    }
    const float nrm = fmaxf(sqrtf(ss), 1e-12f);
    if (r < kN) s_qs[t] = sc / nrm;
    else s_rk[t] = 1.f / nrm;
  }
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, tq = lane & 3, li = lane >> 3, lr = lane & 7;
  const uint32_t sqb = smem_u32(sq), skb = smem_u32(sk), svb = smem_u32(sv);
  constexpr float kLog2e = 1.4426950408889634f;
#pragma unroll 1
  for (int rb = 0; rb < kRowBlocks; ++rb) {
    const int row0 = (rb * kWarps + warp) * 16;
    uint32_t qa[2][4];
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) ldmatrix_x4(qa[kk], sqb + win_tile_off(row0 + (li & 1) * 8 + lr, kk * 2 + (li >> 1)));
    float sacc[kJ][4];
#pragma unroll
    for (int j = 0; j < kJ; ++j)
#pragma unroll
      for (int c = 0; c < 4; ++c) sacc[j][c] = 0.f;
#pragma unroll
    for (int jp = 0; jp < kJ / 2; ++jp) {
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        uint32_t kb[4];
        ldmatrix_x4(kb, skb + win_tile_off(jp * 16 + (li >> 1) * 8 + lr, kk * 2 + (li & 1)));
        win_mma_16816(sacc[2 * jp], qa[kk], kb[0], kb[1]);
        win_mma_16816(sacc[2 * jp + 1], qa[kk], kb[2], kb[3]);
      }
    }
    // score = dot * scale / (|q| |k|) + bias[idx] (+ -100 across shift regions), rows i0 = row0 + g and i0 + 8
    const int i0 = row0 + g;
    const float qs[2] = {s_qs[i0], s_qs[i0 + 8]};
    int qy[2], qx[2], qreg[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int i = i0 + rr * 8;
      qy[rr] = i / kW;
      qx[rr] = i % kW;
      qreg[rr] = shift ? win_region(wy * kW + qy[rr], H, kW, shift) * 3 + win_region(wx * kW + qx[rr], Wd, kW, shift) : 0;
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < kJ; ++j) {
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int rr = c >> 1, col = j * 8 + 2 * tq + (c & 1);
        const int ky = col / kW, kx = col % kW;
        float v = sacc[j][c] * (qs[rr] * s_rk[col]) + s_bias[(qy[rr] - ky + kW - 1) * kT + (qx[rr] - kx + kW - 1)];
        if (shift) {
          const int kreg = win_region(wy * kW + ky, H, kW, shift) * 3 + win_region(wx * kW + kx, Wd, kW, shift);
          if (kreg != qreg[rr]) v += -100.f;
        }
        sacc[j][c] = v;
        mx[rr] = fmaxf(mx[rr], v);
      }
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 1));
      mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 2));
    }
    // P = exp(score - max) rounded to bf16 for P V; the row sum is of the unrounded fp32 values
    float o[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int c = 0; c < 4; ++c) o[j][c] = 0.f;
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int kk = 0; kk < kN / 16; ++kk) {
      uint32_t pa[4];
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        const int j = 2 * kk + jj;
        const float p0 = win_exp2((sacc[j][0] - mx[0]) * kLog2e), p1 = win_exp2((sacc[j][1] - mx[0]) * kLog2e);
        const float p2 = win_exp2((sacc[j][2] - mx[1]) * kLog2e), p3 = win_exp2((sacc[j][3] - mx[1]) * kLog2e);
        rs[0] += p0 + p1;
        rs[1] += p2 + p3;
        __nv_bfloat162 lo = __floats2bfloat162_rn(p0, p1), hi = __floats2bfloat162_rn(p2, p3);
        pa[jj * 2] = *reinterpret_cast<uint32_t*>(&lo);
        pa[jj * 2 + 1] = *reinterpret_cast<uint32_t*>(&hi);
      }
#pragma unroll
      for (int jp = 0; jp < 2; ++jp) {
        uint32_t vb[4];
        ldmatrix_x4_trans(vb, svb + win_tile_off(kk * 16 + (li & 1) * 8 + lr, jp * 2 + (li >> 1)));
        win_mma_16816(o[2 * jp], pa, vb[0], vb[1]);
        win_mma_16816(o[2 * jp + 1], pa, vb[2], vb[3]);
      }
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      rs[rr] += __shfl_xor_sync(0xffffffffu, rs[rr], 1);
      rs[rr] += __shfl_xor_sync(0xffffffffu, rs[rr], 2);
    }
    const float inv0 = 1.0f / rs[0], inv1 = 1.0f / rs[1];
    // stage the 16 x 32 output block in this warp's own q rows (no other warp reads them), then 16-byte stores
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      __nv_bfloat162 lo = __floats2bfloat162_rn(o[j][0] * inv0, o[j][1] * inv0);
      __nv_bfloat162 hi = __floats2bfloat162_rn(o[j][2] * inv1, o[j][3] * inv1);
      *reinterpret_cast<__nv_bfloat162*>(sq + win_tile_off(i0, j) + 4 * tq) = lo;
      *reinterpret_cast<__nv_bfloat162*>(sq + win_tile_off(i0 + 8, j) + 4 * tq) = hi;
    }
    __syncwarp();
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int idx = lane + 32 * k, r = row0 + (idx >> 2), ch = idx & 3;
      *reinterpret_cast<uint4*>(out + token(r) * C + h * kWinD + ch * 8) = *reinterpret_cast<const uint4*>(sq + win_tile_off(r, ch));
    }
  }
}

// x[m, :] <- bf16(x[m, :] + LayerNorm(y[m, :]) * gamma + beta) over C (a multiple of 8, <= 1536): one warp per row, each lane
// holding up to 6 16-byte vectors of y; fp32 statistics (the mean, then the mean squared deviation)
__global__ void __launch_bounds__(256) postnorm_residual_kernel(__nv_bfloat16* x, const __nv_bfloat16* __restrict__ y,
                                                                int64_t M, int C, const float* __restrict__ ln_w,
                                                                const float* __restrict__ ln_b, float eps) {
  constexpr int kMaxVec = 6;
  const int lane = threadIdx.x & 31;
  const int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (row >= M) return;  // uniform over the warp
  const int nv = C / 8;
  const __nv_bfloat16* yr = y + row * C;
  __nv_bfloat16* xr = x + row * C;
  float v[kMaxVec][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    const int c8 = lane + 32 * i;
    if (c8 < nv) {
      const uint4 u = *reinterpret_cast<const uint4*>(yr + c8 * 8);
      const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = __bfloat1622float2(p[k]);
        v[i][2 * k] = f.x;
        v[i][2 * k + 1] = f.y;
        s += f.x + f.y;
      }
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  const float mean = s / static_cast<float>(C);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    if (lane + 32 * i < nv) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float d = v[i][k] - mean;
        q = fmaf(d, d, q);
      }
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) q += __shfl_xor_sync(0xffffffffu, q, off);
  const float rstd = rsqrtf(q / static_cast<float>(C) + eps);
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    const int c8 = lane + 32 * i;
    if (c8 < nv) {
      const uint4 u = *reinterpret_cast<const uint4*>(xr + c8 * 8);
      const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&u);
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(ln_w + c8 * 8)), g1 = __ldg(reinterpret_cast<const float4*>(ln_w + c8 * 8 + 4));
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(ln_b + c8 * 8)), b1 = __ldg(reinterpret_cast<const float4*>(ln_b + c8 * 8 + 4));
      const float gv[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      uint4 o;
      uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 xf = __bfloat1622float2(p[k]);
        __nv_bfloat162 r = __floats2bfloat162_rn(xf.x + ((v[i][2 * k] - mean) * rstd * gv[2 * k] + bv[2 * k]),
                                                 xf.y + ((v[i][2 * k + 1] - mean) * rstd * gv[2 * k + 1] + bv[2 * k + 1]));
        ow[k] = *reinterpret_cast<uint32_t*>(&r);
      }
      *reinterpret_cast<uint4*>(xr + c8 * 8) = o;
    }
  }
}

static int check_window_shape(int batch, int H, int W, int heads, int window, int shift) {
  VDK_REQUIRE(batch > 0 && heads > 0, "window_attention: batch and heads must be positive");
  VDK_REQUIRE(window == 8 || window == 16, "window_attention: window must be 8 or 16 (got %d)", window);
  VDK_REQUIRE(H > 0 && W > 0 && H % window == 0 && W % window == 0, "window_attention: H=%d and W=%d must be multiples of the window %d",
              H, W, window);
  VDK_REQUIRE(shift == 0 || (shift == window / 2 && H > window && W > window),
              "window_attention: shift must be 0 or window/2, and 0 when the map is a single window (got %d)", shift);
  VDK_REQUIRE(static_cast<int64_t>(batch) * (H / window) * (W / window) * heads < (1ll << 31), "window_attention: too many windows");
  return VDK_OK;
}

template <int kW>
static int launch_window_attention_t(const __nv_bfloat16* qkv, int B, int H, int W, int heads, int shift, const float* scale,
                                     const float* bias, __nv_bfloat16* out, cudaStream_t s) {
  constexpr int kN = kW * kW, kT = 2 * kW - 1;
  constexpr size_t kSmem = 3 * kN * 64 + 2 * kN * sizeof(float) + kT * kT * sizeof(float);
  static const cudaError_t attr =
      cudaFuncSetAttribute(window_attention_kernel<kW>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSmem));
  VDK_CUDA_OK(attr);
  const int64_t items = static_cast<int64_t>(B) * (H / kW) * (W / kW) * heads;
  window_attention_kernel<kW><<<static_cast<unsigned>(items), kW == 8 ? 128 : 256, kSmem, s>>>(qkv, H, W, heads, shift, scale, bias, out);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

static int launch_window_attention(const __nv_bfloat16* qkv, int B, int H, int W, int heads, int window, int shift,
                                   const float* scale, const float* bias, __nv_bfloat16* out, cudaStream_t s) {
  const double tokens = static_cast<double>(B) * H * W, C = heads * kWinD;
  ProfScope prof(kProfAttention, 4.0 * tokens * window * window * C, 8.0 * tokens * C, s);
  return window == 8 ? launch_window_attention_t<8>(qkv, B, H, W, heads, shift, scale, bias, out, s)
                     : launch_window_attention_t<16>(qkv, B, H, W, heads, shift, scale, bias, out, s);
}

static int launch_postnorm_residual(__nv_bfloat16* x, const __nv_bfloat16* y, int64_t M, int C, const float* ln_w,
                                    const float* ln_b, float eps, cudaStream_t s) {
  VDK_REQUIRE(C >= 8 && C % 8 == 0 && C <= 1536, "postnorm_residual: C must be a multiple of 8 in [8, 1536] (got %d)", C);
  ProfScope prof(kProfOther, 0.0, 6.0 * static_cast<double>(M) * C, s);
  postnorm_residual_kernel<<<static_cast<unsigned>((M * 32 + 255) / 256), 256, 0, s>>>(x, y, M, C, ln_w, ln_b, eps);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

static int check_swinv2(const vdk_swinv2_net* n) {
  VDK_REQUIRE(n, "vdk_swinv2: null network");
  VDK_REQUIRE(n->image_size == 256, "vdk_swinv2: image_size must be 256, the towers' size (got %d)", n->image_size);
  VDK_REQUIRE(n->feat_dim > 0 && n->feat_dim % 8 == 0, "vdk_swinv2: feat_dim must be a multiple of 8");
  // the merge convs need C % 64 == 0, the patch embedding's LayerNorm epilogue C <= 256
  VDK_REQUIRE(n->embed_dim > 0 && n->embed_dim % 64 == 0 && n->embed_dim <= 256,
              "vdk_swinv2: embed_dim must be a multiple of 64, <= 256 (got %d)", n->embed_dim);
  VDK_REQUIRE(n->stem_w && n->stem_b && n->stem_ln_w && n->stem_ln_b, "vdk_swinv2: missing patch embedding");
  int nb = 0, map = n->image_size / 4;
  for (int s = 0; s < 4; ++s) {
    VDK_REQUIRE(n->depths[s] >= 1, "vdk_swinv2: every stage needs at least one block");
    const int w = n->window[s], sh = n->shift[s];
    VDK_REQUIRE((w == 8 || w == 16) && map % w == 0, "vdk_swinv2: stage %d window %d must be 8 or 16 and divide the %d map", s, w, map);
    VDK_REQUIRE(sh == 0 || (sh == w / 2 && map > w), "vdk_swinv2: stage %d shift %d must be 0 or window/2 (0 on a single window)", s, sh);
    if (s > 0) {
      VDK_REQUIRE(n->merge_w[s] && n->merge_ln_w[s] && n->merge_ln_b[s], "vdk_swinv2: stage %d misses its patch merging", s);
      map /= 2;
    }
    nb += n->depths[s];
  }
  VDK_REQUIRE(nb <= VDK_SWINV2_MAX_BLOCKS, "vdk_swinv2: too many blocks (%d)", nb);
  for (int i = 0; i < nb; ++i) {
    const vdk_swinv2_block& b = n->blocks[i];
    VDK_REQUIRE(b.qkv_w && b.qkv_b && b.attn_scale && b.attn_bias && b.proj_w && b.proj_b && b.norm1_w && b.norm1_b && b.fc1_w &&
                    b.fc1_b && b.fc2_w && b.fc2_b && b.norm2_w && b.norm2_b,
                "vdk_swinv2: block %d misses a weight", i);
  }
  VDK_REQUIRE(n->norm_w && n->norm_b && n->neck_w && n->neck_b, "vdk_swinv2: missing final norm or neck");
  return VDK_OK;
}

}  // namespace vdk

using namespace vdk;

extern "C" int vdk_window_attention_fwd(const void* qkv, int batch, int H, int W, int heads, int window, int shift,
                                        const float* scale, const float* bias, void* out, void* stream) {
  VDK_REQUIRE(qkv && out && scale && bias, "vdk_window_attention_fwd: null operand");
  VDK_REQUIRE(((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(out)) & 15) == 0,
              "vdk_window_attention_fwd: qkv and out must be 16-byte aligned");
  const int rc = check_window_shape(batch, H, W, heads, window, shift);
  if (rc != VDK_OK) return rc;
  return launch_window_attention(static_cast<const __nv_bfloat16*>(qkv), batch, H, W, heads, window, shift, scale, bias,
                                 static_cast<__nv_bfloat16*>(out), reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vdk_postnorm_residual(void* x, const void* y, int64_t rows, int C, const float* ln_w, const float* ln_b, float eps,
                                     void* stream) {
  VDK_REQUIRE(x && y && ln_w && ln_b && rows > 0, "vdk_postnorm_residual: null operand or no rows");
  VDK_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(ln_w) |
                reinterpret_cast<uintptr_t>(ln_b)) & 15) == 0,
              "vdk_postnorm_residual: operands must be 16-byte aligned");
  return launch_postnorm_residual(static_cast<__nv_bfloat16*>(x), static_cast<const __nv_bfloat16*>(y), rows, C, ln_w, ln_b, eps,
                                  reinterpret_cast<cudaStream_t>(stream));
}

// x (residual stream, B*4096*C0), y (attention out / fc2 out / final norm, same size), big (qkv 3x, MLP hidden 4x, stem
// patch rows, merged maps, neck slabs): stage 1 holds the largest maps (each merge quarters the tokens, doubles C)
extern "C" size_t vdk_swinv2_workspace_bytes(const vdk_swinv2_net* net, int batch) {
  if (!net || batch <= 0 || net->image_size <= 0 || net->embed_dim <= 0) return 0;
  const size_t m = static_cast<size_t>(batch) * (net->image_size / 4) * (net->image_size / 4);
  const size_t mc = m * net->embed_dim;
  return 2 * up256(mc * 2) + up256(std::max(4 * mc, m * 48) * 2) + 1024;
}

extern "C" int vdk_swinv2_forward(const vdk_swinv2_net* net, const float* images, int batch, int l2_normalize, float* embeddings,
                                  void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_swinv2(net);
  if (rc != VDK_OK) return rc;
  VDK_REQUIRE(images && embeddings && batch > 0, "vdk_swinv2_forward: null image/embedding buffer");
  VDK_REQUIRE(workspace && workspace_bytes >= vdk_swinv2_workspace_bytes(net, batch), "vdk_swinv2_forward: workspace too small");
  VDK_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0 && (reinterpret_cast<uintptr_t>(images) & 15) == 0,
              "vdk_swinv2_forward: workspace must be 256-byte and images 16-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int S = net->image_size;
  const size_t m0 = static_cast<size_t>(batch) * (S / 4) * (S / 4), mc = m0 * net->embed_dim;
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  __nv_bfloat16* x = reinterpret_cast<__nv_bfloat16*>(ws);
  __nv_bfloat16* y = reinterpret_cast<__nv_bfloat16*>(ws + up256(mc * 2));
  __nv_bfloat16* big = reinterpret_cast<__nv_bfloat16*>(ws + 2 * up256(mc * 2));
  const size_t big_bytes = workspace_bytes - 2 * up256(mc * 2);

  auto gemm = [&](const void* A, const void* Bw, void* D, int M, int N, int K, int epi, const float* bias, const float* gamma,
                  const float* beta) -> int {
    vdk_gemm_desc g{};
    g.A = A; g.B = Bw; g.D = D;
    g.M = M; g.N = N; g.K = K; g.lda = K; g.ldb = K; g.ldd = N;
    g.in_dtype = VDK_DTYPE_BF16; g.out_dtype = VDK_DTYPE_BF16; g.epilogue = epi;
    g.bias = bias; g.gamma = gamma; g.beta = beta; g.ln_eps = 1e-5f; g.split_k = 1;
    return gemm_run(g, s);
  };

  // ---- patch embedding: conv 4x4/s4 as a GEMM over (c, kh, kw) patch rows, + bias + LayerNorm in the epilogue ----
  int H = S / 4, C = net->embed_dim;
  if ((rc = launch_stem_patchify(images, batch, S, big, s)) != VDK_OK) return rc;
  if ((rc = gemm(big, net->stem_w, x, batch * H * H, C, 48, VDK_EPI_LAYERNORM, net->stem_b, net->stem_ln_w, net->stem_ln_b)) != VDK_OK)
    return rc;
  int blk = 0;
  for (int st = 0; st < 4; ++st) {
    if (st > 0) {
      // ---- patch merging: the 2x2 gather + reduction as a 2x2/s2 conv (weight in (kh, kw, c) order), then LayerNorm ----
      vdk_conv_desc d{};
      d.x = x; d.w = net->merge_w[st]; d.y = big;
      d.B = batch; d.H = H; d.W = H; d.Cin = C; d.Cout = 2 * C;
      d.kernel = 2; d.stride = 2; d.pad = 0; d.epilogue = VDK_EPI_NONE;
      if ((rc = conv_run(d, s)) != VDK_OK) return rc;
      H /= 2;
      C *= 2;
      if ((rc = launch_ln_patchify(big, batch, H, H, C, net->merge_ln_w[st], net->merge_ln_b[st], 1e-5f, 1, x, nullptr, s)) != VDK_OK)
        return rc;
    }
    const int M = batch * H * H, heads = C / kWinD;
    for (int j = 0; j < net->depths[st]; ++j, ++blk) {
      const vdk_swinv2_block& b = net->blocks[blk];
      const int shift = (j % 2) ? net->shift[st] : 0;
      // x = x + norm1(proj(window_attention(qkv(x))))
      if ((rc = gemm(x, b.qkv_w, big, M, 3 * C, C, VDK_EPI_NONE, b.qkv_b, nullptr, nullptr)) != VDK_OK) return rc;
      if ((rc = launch_window_attention(big, batch, H, H, heads, net->window[st], shift, b.attn_scale, b.attn_bias, y, s)) != VDK_OK)
        return rc;
      if ((rc = gemm(y, b.proj_w, big, M, C, C, VDK_EPI_NONE, b.proj_b, nullptr, nullptr)) != VDK_OK) return rc;
      if ((rc = launch_postnorm_residual(x, big, M, C, b.norm1_w, b.norm1_b, 1e-5f, s)) != VDK_OK) return rc;
      // x = x + norm2(fc2(GELU(fc1(x))))
      if ((rc = gemm(x, b.fc1_w, big, M, 4 * C, C, VDK_EPI_GELU, b.fc1_b, nullptr, nullptr)) != VDK_OK) return rc;
      if ((rc = gemm(big, b.fc2_w, y, M, C, 4 * C, VDK_EPI_NONE, b.fc2_b, nullptr, nullptr)) != VDK_OK) return rc;
      if ((rc = launch_postnorm_residual(x, y, M, C, b.norm2_w, b.norm2_b, 1e-5f, s)) != VDK_OK) return rc;
    }
  }
  // ---- final LayerNorm (model.norm), then the neck: BN2d over h -> Flatten (h, w, c) -> Linear -> BN1d, folded ----
  if ((rc = launch_ln_patchify(x, batch, H, H, C, net->norm_w, net->norm_b, 1e-5f, 1, y, nullptr, s)) != VDK_OK) return rc;
  return launch_neck(y, batch, H * H * C, net->feat_dim, net->neck_w, net->neck_b, l2_normalize, reinterpret_cast<float*>(big),
                     big_bytes, embeddings, s);
}
