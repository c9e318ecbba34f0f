// train_ops.cu — the HBM-bound kernels of the ConvNeXt training backward (everything that is not a GEMM):
// column sums (bias gradients), LayerNorm backward (with the 2x2 un-patchify of the downsample layers), depthwise-7x7
// backward (data and weight gradient), BatchNorm forward/backward with batch statistics (the neck in train mode),
// layer-scale gradient finalisation, weight packing (fp32 master -> bf16 kernel layouts) and the inverse permutation for gradients.
//
// Replaces the autograd backward of timm's ConvNeXtBlock / downsample / stem and of the reference neck
// (models/faceX/backbone/timm_wrapper.py:30-38 in train mode: BatchNorm with batch statistics), i.e. what
// `scaler.scale(loss).backward()` at engine/procedure/train.py:206 runs through ATen/cuDNN.
#include "vdk_host.h"
#include "vdk_ptx.cuh"
#include "convnext_internal.h"

namespace vdk {

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

__device__ __forceinline__ void unpack8(const uint4& t, float (&v)[8]) {
  const float2 a0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.x));
  const float2 a1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.y));
  const float2 a2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.z));
  const float2 a3 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.w));
  v[0] = a0.x; v[1] = a0.y; v[2] = a1.x; v[3] = a1.y; v[4] = a2.x; v[5] = a2.y; v[6] = a3.x; v[7] = a3.y;
}
__device__ __forceinline__ uint4 pack8(const float (&v)[8]) {
  __nv_bfloat162 o0 = __floats2bfloat162_rn(v[0], v[1]), o1 = __floats2bfloat162_rn(v[2], v[3]);
  __nv_bfloat162 o2 = __floats2bfloat162_rn(v[4], v[5]), o3 = __floats2bfloat162_rn(v[6], v[7]);
  uint4 t;
  t.x = *reinterpret_cast<uint32_t*>(&o0); t.y = *reinterpret_cast<uint32_t*>(&o1);
  t.z = *reinterpret_cast<uint32_t*>(&o2); t.w = *reinterpret_cast<uint32_t*>(&o3);
  return t;
}

// ------------------------------------------------------------------------------------------------
// LayerNorm backward over C (optionally through the 2x2/s2 patch regrouping of the downsample layers)
// ------------------------------------------------------------------------------------------------
// dy, y: [rows, patch*patch*C] (grad of / saved LayerNorm output, patch-row layout), rstd[pixel], dx: NHWC [B,H,W,C].
//   xh = (y - beta) / gamma;  g = dy * gamma;  dx = rstd * (g - mean_C(g) - xh * mean_C(g * xh)) (+ addend)
//   dgamma += sum_pixels dy * xh;  dbeta += sum_pixels dy
// A pixel is shared by LPP lanes (IT 16-byte vectors each); a warp handles U x (32 / LPP) pixels per trip with all
// of their loads issued before the first use (U * IT = 4 vectors of dy and of y in flight per lane), and the bf16
// inputs stay packed in registers between the statistics pass and the output pass, so the narrow instantiations stay
// within 128 registers and the kernel HBM-bound. gamma / beta / 1/gamma live in shared memory; dgamma / dbeta are
// combined per warp by shuffles, per block in shared memory, and leave as one global atomic per channel per block.
//
// Accuracy: xh comes from the saved bf16 y, so it carries y's rounding amplified by 1/|gamma|: an error of up to
// ulp_bf16(y) / (2 |gamma|) per element, which exceeds bf16 precision of xh itself once |beta / gamma| >> |xh|.  A
// channel with gamma == 0 has no xh in y at all: it is taken as 0, so that channel's dx lacks its -xh * mean(g * xh)
// term and its dgamma receives nothing (both finite).
//
// IT = 6 (C up to 1536, ConvNeXt-L stage 3) carries 96 dgamma / dbeta accumulators and runs at the 255-register cap
// with a 36-byte spill (ptxas, sm_90a); IT = 3 and IT = 2 spill 200-400 bytes under their 128-register bound.

template <int LPP, int IT, int U>
__global__ void __launch_bounds__(256, IT >= 4 ? 1 : 2)
ln_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ y, const float* __restrict__ rstd,
              int B, int H, int W, int C, const float* __restrict__ ln_w, const float* __restrict__ ln_b, int patch,
              __nv_bfloat16* __restrict__ dx, const __nv_bfloat16* __restrict__ addend, float* __restrict__ dgamma,
              float* __restrict__ dbeta) {
  constexpr int kPPW = 32 / LPP;
  extern __shared__ float ln_sm[];
  const int Cp = LPP * IT * 8;  // padded channel count (>= C)
  float* s_w = ln_sm;           // gamma
  float* s_iw = s_w + Cp;       // 1 / gamma
  float* s_b = s_iw + Cp;       // beta
  float* s_dg = s_b + Cp;       // block partial of dgamma
  float* s_db = s_dg + Cp;      // block partial of dbeta
  for (int c = threadIdx.x; c < Cp; c += 256) {
    float w = c < C ? ln_w[c] : 1.f;
    float iw = 0.f;  // gamma == 0: y holds no trace of xh, which is taken as 0 (that channel's dgamma stays unknown)
    if (w != 0.f) {
      if (fabsf(w) < 1e-12f) w = w < 0.f ? -1e-12f : 1e-12f;
      iw = 1.0f / w;
    }
    s_w[c] = w;
    s_iw[c] = iw;
    s_b[c] = c < C ? ln_b[c] : 0.f;
    s_dg[c] = 0.f;
    s_db[c] = 0.f;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, sub = lane % LPP;
  const int64_t npix = static_cast<int64_t>(B) * H * W;
  const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
  const int64_t warp_id = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const float inv_c = 1.0f / static_cast<float>(C);
  float gw[IT][8], gb[IT][8];
#pragma unroll
  for (int i = 0; i < IT; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) { gw[i][j] = 0.f; gb[i][j] = 0.f; }

  for (int64_t base = warp_id * (kPPW * U); base < npix; base += nwarps * (kPPW * U)) {
    uint4 rdy[U][IT], ry[U][IT];
    int64_t pix[U], roff[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      pix[u] = base + u * kPPW + lane / LPP;
      const bool ok = pix[u] < npix;
      int64_t orow = pix[u];
      int ocol0 = 0;
      if (patch == 2 && ok) {
        const int xw = static_cast<int>(pix[u] % W);
        const int yh = static_cast<int>((pix[u] / W) % H);
        const int b = static_cast<int>(pix[u] / (static_cast<int64_t>(W) * H));
        orow = (static_cast<int64_t>(b) * (H / 2) + (yh >> 1)) * (W / 2) + (xw >> 1);
        ocol0 = ((yh & 1) * 2 + (xw & 1)) * C;
      }
      roff[u] = orow * (static_cast<int64_t>(C) * patch * patch) + ocol0;
#pragma unroll
      for (int i = 0; i < IT; ++i) {
        const int c = (sub + i * LPP) * 8;
        rdy[u][i] = make_uint4(0, 0, 0, 0);
        ry[u][i] = make_uint4(0, 0, 0, 0);
        if (ok && c < C) {
          rdy[u][i] = __ldg(reinterpret_cast<const uint4*>(dy + roff[u] + c));
          ry[u][i] = __ldg(reinterpret_cast<const uint4*>(y + roff[u] + c));
        }
      }
    }
    float s1[U], s2[U];
#pragma unroll
    for (int u = 0; u < U; ++u) { s1[u] = 0.f; s2[u] = 0.f; }
#pragma unroll
    for (int i = 0; i < IT; ++i) {
      const int c = (sub + i * LPP) * 8;
      float w[8], iw[8], bb[8];
      *reinterpret_cast<float4*>(&w[0]) = *reinterpret_cast<const float4*>(s_w + c);
            *reinterpret_cast<float4*>(&w[4]) = *reinterpret_cast<const float4*>(s_w + c + 4);
      *reinterpret_cast<float4*>(&iw[0]) = *reinterpret_cast<const float4*>(s_iw + c);
            *reinterpret_cast<float4*>(&iw[4]) = *reinterpret_cast<const float4*>(s_iw + c + 4);
      *reinterpret_cast<float4*>(&bb[0]) = *reinterpret_cast<const float4*>(s_b + c);
            *reinterpret_cast<float4*>(&bb[4]) = *reinterpret_cast<const float4*>(s_b + c + 4);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const bool okc = pix[u] < npix && c < C;
        float vdy[8], vy[8];
        unpack8(rdy[u][i], vdy);
        unpack8(ry[u][i], vy);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float h = okc ? (vy[j] - bb[j]) * iw[j] : 0.f;
          const float g = vdy[j] * w[j];
          s1[u] += g;
          s2[u] = fmaf(g, h, s2[u]);
          gw[i][j] = fmaf(vdy[j], h, gw[i][j]);
          gb[i][j] += vdy[j];
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
#pragma unroll
      for (int off = LPP / 2; off > 0; off >>= 1) {
        s1[u] += __shfl_xor_sync(0xffffffffu, s1[u], off);
        s2[u] += __shfl_xor_sync(0xffffffffu, s2[u], off);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (pix[u] < npix) {
        const float rs = rstd[pix[u]];
        const float m1 = s1[u] * inv_c, m2 = s2[u] * inv_c;
#pragma unroll
        for (int i = 0; i < IT; ++i) {
          const int c = (sub + i * LPP) * 8;
          if (c < C) {
            float w[8], iw[8], bb[8];
            *reinterpret_cast<float4*>(&w[0]) = *reinterpret_cast<const float4*>(s_w + c);
            *reinterpret_cast<float4*>(&w[4]) = *reinterpret_cast<const float4*>(s_w + c + 4);
            *reinterpret_cast<float4*>(&iw[0]) = *reinterpret_cast<const float4*>(s_iw + c);
            *reinterpret_cast<float4*>(&iw[4]) = *reinterpret_cast<const float4*>(s_iw + c + 4);
            *reinterpret_cast<float4*>(&bb[0]) = *reinterpret_cast<const float4*>(s_b + c);
            *reinterpret_cast<float4*>(&bb[4]) = *reinterpret_cast<const float4*>(s_b + c + 4);
            float vdy[8], vy[8], o[8];
            if constexpr (IT > 4) {  // recompute g and xh from the packed inputs rather than keep 16 IT floats live
              asm volatile("" : "+r"(rdy[u][i].x), "+r"(rdy[u][i].y), "+r"(rdy[u][i].z), "+r"(rdy[u][i].w));
              asm volatile("" : "+r"(ry[u][i].x), "+r"(ry[u][i].y), "+r"(ry[u][i].z), "+r"(ry[u][i].w));
            }
            unpack8(rdy[u][i], vdy);
            unpack8(ry[u][i], vy);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float h = (vy[j] - bb[j]) * iw[j];
              o[j] = rs * (vdy[j] * w[j] - m1 - h * m2);
            }
            if (addend) {
              float a[8];
              unpack8(__ldg(reinterpret_cast<const uint4*>(addend + pix[u] * C + c)), a);
#pragma unroll
              for (int j = 0; j < 8; ++j) o[j] += a[j];
            }
            *reinterpret_cast<uint4*>(dx + pix[u] * C + c) = pack8(o);
          }
        }
      }
    }
  }
  // lanes that handled the same channels (kPPW pixel slots per warp) are combined, then warps meet in shared memory
#pragma unroll
  for (int i = 0; i < IT; ++i) {
    const int c = (sub + i * LPP) * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float a = gw[i][j], b2 = gb[i][j];
#pragma unroll
      for (int off = LPP; off < 32; off <<= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, off);
        b2 += __shfl_xor_sync(0xffffffffu, b2, off);
      }
      if (lane < LPP) {
        atomicAdd(s_dg + c + j, a);
        atomicAdd(s_db + c + j, b2);
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += 256) {
    atomicAdd(dgamma + c, s_dg[c]);
    atomicAdd(dbeta + c, s_db[c]);
  }
}

template <int LPP, int IT, int U>
static void ln_bwd_launch(const __nv_bfloat16* dy, const __nv_bfloat16* y, const float* rstd, int B, int H, int W, int C,
                          const float* ln_w, const float* ln_b, int patch, __nv_bfloat16* dx, const __nv_bfloat16* addend,
                          float* dgamma, float* dbeta, cudaStream_t s) {
  const int64_t npix = static_cast<int64_t>(B) * H * W;
  const int64_t pix_per_block_trip = 8 * (32 / LPP) * U;
  const int blocks = static_cast<int>(std::max<int64_t>(1, std::min<int64_t>((npix + pix_per_block_trip - 1) / pix_per_block_trip,
                                                                              sm_count() * (IT >= 4 ? 1 : 2))));
  const size_t smem = static_cast<size_t>(LPP) * IT * 8 * 5 * sizeof(float);
  ln_bwd_kernel<LPP, IT, U><<<blocks, 256, smem, s>>>(dy, y, rstd, B, H, W, C, ln_w, ln_b, patch, dx, addend, dgamma, dbeta);
}

int launch_ln_bwd(const __nv_bfloat16* dy, const __nv_bfloat16* y, const float* rstd, int B, int H, int W, int C,
                  const float* ln_w, const float* ln_b, int patch, __nv_bfloat16* dx, const __nv_bfloat16* addend,
                  float* dgamma, float* dbeta, cudaStream_t s) {
  VDK_REQUIRE(C % 8 == 0 && C <= 1536, "ln_bwd: C must be a multiple of 8, <= 1536 (got %d)", C);
  const int vecs = C / 8;
  if (vecs <= 8) ln_bwd_launch<8, 1, 4>(dy, y, rstd, B, H, W, C, ln_w, ln_b, patch, dx, addend, dgamma, dbeta, s);
  else if (vecs <= 16) ln_bwd_launch<16, 1, 4>(dy, y, rstd, B, H, W, C, ln_w, ln_b, patch, dx, addend, dgamma, dbeta, s);
  else if (vecs <= 32) ln_bwd_launch<32, 1, 4>(dy, y, rstd, B, H, W, C, ln_w, ln_b, patch, dx, addend, dgamma, dbeta, s);
  else if (vecs <= 64) ln_bwd_launch<32, 2, 2>(dy, y, rstd, B, H, W, C, ln_w, ln_b, patch, dx, addend, dgamma, dbeta, s);
  else if (vecs <= 96) ln_bwd_launch<32, 3, 1>(dy, y, rstd, B, H, W, C, ln_w, ln_b, patch, dx, addend, dgamma, dbeta, s);  // ViT-B: C = 768
  else if (vecs <= 128) ln_bwd_launch<32, 4, 1>(dy, y, rstd, B, H, W, C, ln_w, ln_b, patch, dx, addend, dgamma, dbeta, s);
  else ln_bwd_launch<32, 6, 1>(dy, y, rstd, B, H, W, C, ln_w, ln_b, patch, dx, addend, dgamma, dbeta, s);  // ConvNeXt-L: C = 1536
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

// ------------------------------------------------------------------------------------------------
// depthwise 7x7 backward of a block, from one staging of the output gradient g = dconv:
//   data gradient    dx[b,y,x,c] = bf16(sum_{dy,dx} w[dy*7+dx][c] g[b,y+dy-3,x+dx-3,c] + addend[b,y,x,c])  (w: reversed taps)
//   weight gradient  dw[tap][c] += sum_{b,y,x} g[b,y,x,c] x[b,y+dy-3,x+dx-3,c];  dbias[c] += sum g
// ------------------------------------------------------------------------------------------------
// CTA = (group of images, T x T pixel tile, 64-channel chunk).  A producer warp streams each image's x halo and g halo
// ((T+6)^2 x 64, zero-filled out of bounds by TMA, so no masks) through a two-stage mbarrier ring, so image i+1 loads
// while image i computes.  Fourteen consumer warps read the same stage at once:
//   warps 0-6 (weight gradient): a thread owns 4 channels, ONE filter row dy and one 7-pixel half of every tile row; per
//     strip it reads 7 gradient (the halo's interior) and 13 input vectors for 7 x 7 x 4 FMAs, the 28 accumulators of its
//     filter row staying in registers.  Every image starts a fresh chain that is then added to the thread's total, so
//     a CTA can take many images (one wave of CTAs, each pipelining its images) without lengthening any chain.
//   warps 7-13 (data gradient): a thread owns 4 channels of a 7-pixel strip of a tile row: 7 filter rows, each 13 g
//     vectors against 7 taps (fp32, staged once per CTA) for 7 x 7 x 4 FMAs, then the addend and one bf16 store.
// After the last image the weight-gradient halves meet in shared memory and each CTA issues one atomic per (tap, channel).
// Either half may be switched off (null taps / null dw49).  C need only be a multiple of 8: the last chunk reads channels
// past C as TMA zero fill and stores nothing for them.
//
// Roundings.  Data gradient: 49 FMAs from zero, then the addend: 50 per output.  Weight gradient: a term passes its image's
// chain (T x 7 FMAs), the adds of the per-image partials (ipc - 1), the nh strip partials and one atomic per CTA:
// T * 7 + ipc - 1 + nh + groups * tiles, with groups = ceil(B / ipc).
constexpr int kBwdT = 14;
constexpr int kBwdC = 64;
constexpr int kBwdR = 7;             // strip length (pixels) = taps per filter row
constexpr int kBwdHalfWarps = 7;     // consumer warps per half
constexpr int kBwdThreads = (2 * kBwdHalfWarps + 1) * 32;

__device__ __forceinline__ float2 bf16lo_hi(uint32_t t) {  // bf16 pair -> fp32 pair: a shift and a mask
  return make_float2(__uint_as_float(t << 16), __uint_as_float(t & 0xffff0000u));
}

// TT: compile-time tile edge (14 or 7: every shared-memory offset an immediate, no bounds predicates) or 0 = runtime
template <int TT>
__global__ void __launch_bounds__(kBwdThreads, 1)
dwconv7_bwd_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_g, int B, int H,
                   int W, int C, int T_rt, int ipc, const float* __restrict__ w49, const __nv_bfloat16* __restrict__ addend,
                   __nv_bfloat16* __restrict__ dx_out, float* __restrict__ dw49, float* __restrict__ dbias) {
  extern __shared__ uint8_t bw_raw[];
  uint8_t* smem = bw_raw + ((128u - (smem_u32(bw_raw) & 127u)) & 127u);
  const int T = TT > 0 ? TT : T_rt;
  const int halo = T + 6;
  const int nh = (T + kBwdR - 1) / kBwdR;  // strips per tile row
  const int planes = 7 * nh;               // (half, dy) pairs of the weight gradient
  const int h_bytes = (halo * halo * kBwdC * 2 + 127) & ~127;
  const int stage_bytes = 2 * h_bytes;     // x halo, then g halo
  float* wsm = reinterpret_cast<float*>(smem + 2 * stage_bytes);  // [49][64] taps of this chunk (data gradient)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(wsm + 49 * kBwdC);
  uint64_t* empty_bar = full_bar + 2;
  float* red = reinterpret_cast<float*>(smem);  // aliases stage 0 once every image is done
  const bool do_data = w49 != nullptr, do_wgrad = dw49 != nullptr;

  const int tiles_w = (W + T - 1) / T, tiles_h = (H + T - 1) / T;
  const int n_cc = (C + kBwdC - 1) / kBwdC;
  int bid = blockIdx.x;
  const int cc = bid % n_cc; bid /= n_cc;
  const int tw = bid % tiles_w; bid /= tiles_w;
  const int th = bid % tiles_h;
  const int b0 = (bid / tiles_h) * ipc;
  const int n_img = min(B, b0 + ipc) - b0;
  const int oy0 = th * T, ox0 = tw * T;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_g);
    if (do_wgrad) prefetch_tensormap(&map_x);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2 * kBwdHalfWarps);
    }
    fence_mbar_init();
  }
  if (do_data) {
    for (int i = threadIdx.x; i < 49 * (kBwdC / 4); i += blockDim.x) {
      const int t = i / (kBwdC / 4), q = i - t * (kBwdC / 4);
      const int c = cc * kBwdC + q * 4;
      *reinterpret_cast<float4*>(wsm + t * kBwdC + q * 4) =
          c < C ? __ldg(reinterpret_cast<const float4*>(w49 + static_cast<size_t>(t) * C + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  __syncthreads();

  const int quad = threadIdx.x & 15;
  const int cq = cc * kBwdC + quad * 4;  // first of this thread's 4 channels
  float2 tot[7][2];                      // weight gradient: this thread's filter row over all its images
  float btot[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int d = 0; d < 7; ++d) tot[d][0] = tot[d][1] = make_float2(0.f, 0.f);
  const int plane = (threadIdx.x >> 4) % (2 * kBwdHalfWarps);  // weight-gradient plane / data-gradient strip slot
  const int hh = plane / 7, dy = plane - hh * 7;                 // (weight gradient)

  if (warp == 2 * kBwdHalfWarps) {
    // ===================== producer: one image ahead of the consumers =====================
    if (lane == 0) {
      for (int i = 0; i < n_img; ++i) {
        const int buf = i & 1;
        mbar_wait_relaxed(&empty_bar[buf], ((i >> 1) & 1) ^ 1);  // both halves are done with image i - 2
        uint8_t* st = smem + buf * stage_bytes;
        mbar_arrive_expect_tx(&full_bar[buf], (do_wgrad ? 2 : 1) * halo * halo * kBwdC * 2);
        if (do_wgrad) tma_load_4d(st, &map_x, &full_bar[buf], cc * kBwdC, ox0 - 3, oy0 - 3, b0 + i);
        tma_load_4d(st + h_bytes, &map_g, &full_bar[buf], cc * kBwdC, ox0 - 3, oy0 - 3, b0 + i);
      }
    }
    __syncwarp();  // the warp reaches the final __syncthreads converged
  } else if (warp < kBwdHalfWarps) {
    // ===================== weight gradient =====================
    const bool active = do_wgrad && plane < planes;
    const int px0 = hh * kBwdR;
    for (int i = 0; i < n_img; ++i) {
      const int buf = i & 1;
      mbar_wait(&full_bar[buf], (i >> 1) & 1);
      if (active) {
        const uint8_t* sx = smem + buf * stage_bytes;
        const uint8_t* sg = sx + h_bytes;
        float2 acc[7][2];
#pragma unroll
        for (int d = 0; d < 7; ++d) acc[d][0] = acc[d][1] = make_float2(0.f, 0.f);
        float bsum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
        for (int py = 0; py < T; ++py) {
          float2 g[kBwdR][2];
          const uint8_t* gr = sg + (((py + 3) * halo + px0 + 3) * kBwdC + quad * 4) * 2;  // the halo's interior
#pragma unroll
          for (int r = 0; r < kBwdR; ++r) {
            uint2 t = make_uint2(0u, 0u);
            if (TT > 0 || px0 + r < T) t = *reinterpret_cast<const uint2*>(gr + r * kBwdC * 2);
            g[r][0] = bf16lo_hi(t.x);
            g[r][1] = bf16lo_hi(t.y);
          }
          if (dy == 0) {
#pragma unroll
            for (int r = 0; r < kBwdR; ++r) {
              bsum[0] += g[r][0].x; bsum[1] += g[r][0].y; bsum[2] += g[r][1].x; bsum[3] += g[r][1].y;
            }
          }
          const uint8_t* xr = sx + (((py + dy) * halo + px0) * kBwdC + quad * 4) * 2;
#pragma unroll
          for (int ix = 0; ix < kBwdR + 6; ++ix) {
            uint2 t = make_uint2(0u, 0u);
            if (TT > 0 || px0 + ix < halo) t = *reinterpret_cast<const uint2*>(xr + ix * kBwdC * 2);
            const float2 a = bf16lo_hi(t.x), c = bf16lo_hi(t.y);
#pragma unroll
            for (int r = 0; r < kBwdR; ++r) {  // input column ix meets strip pixel r through tap ix - r
              const int d = ix - r;
              if (d >= 0 && d < 7) {
                acc[d][0] = ffma2(g[r][0], a, acc[d][0]);
                acc[d][1] = ffma2(g[r][1], c, acc[d][1]);
              }
            }
          }
        }
#pragma unroll
        for (int d = 0; d < 7; ++d) {
          tot[d][0] = make_float2(tot[d][0].x + acc[d][0].x, tot[d][0].y + acc[d][0].y);
          tot[d][1] = make_float2(tot[d][1].x + acc[d][1].x, tot[d][1].y + acc[d][1].y);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) btot[k] += bsum[k];
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[buf]);
    }
  } else {
    // ===================== data gradient =====================
    const int strips = T * nh;
    const bool has_c = do_data && cq < C;
    for (int i = 0; i < n_img; ++i) {
      const int buf = i & 1;
      const int b = b0 + i;
      mbar_wait(&full_bar[buf], (i >> 1) & 1);
      const uint8_t* sg = smem + buf * stage_bytes + h_bytes;
      for (int s = plane; has_c && s < strips; s += 2 * kBwdHalfWarps) {
        const int py = s / nh, px0 = (s - py * nh) * kBwdR;
        const int oy = oy0 + py;
        // the strip's addend is requested before its taps run, so its global-memory latency hides under them
        bool out[kBwdR];
        uint2 ad[kBwdR];
#pragma unroll
        for (int p = 0; p < kBwdR; ++p) {
          const int ox = ox0 + px0 + p;
          out[p] = oy < H && ox < W && (TT > 0 || px0 + p < T);
          ad[p] = make_uint2(0u, 0u);
          if (addend && out[p])
            ad[p] = __ldg(reinterpret_cast<const uint2*>(addend + ((static_cast<int64_t>(b) * H + oy) * W + ox) * C + cq));
        }
        float2 acc[kBwdR][2];
#pragma unroll
        for (int p = 0; p < kBwdR; ++p) acc[p][0] = acc[p][1] = make_float2(0.f, 0.f);
#pragma unroll 1
        for (int fy = 0; fy < 7; ++fy) {
          float2 wlo[7], whi[7];
          const float* wrow = wsm + fy * (7 * kBwdC) + quad * 4;
#pragma unroll
          for (int d = 0; d < 7; ++d) {
            const float4 t = *reinterpret_cast<const float4*>(wrow + d * kBwdC);
            wlo[d] = make_float2(t.x, t.y);
            whi[d] = make_float2(t.z, t.w);
          }
          const uint8_t* gr = sg + (((py + fy) * halo + px0) * kBwdC + quad * 4) * 2;
#pragma unroll
          for (int ix = 0; ix < kBwdR + 6; ++ix) {
            uint2 t = make_uint2(0u, 0u);
            if (TT > 0 || px0 + ix < halo) t = *reinterpret_cast<const uint2*>(gr + ix * kBwdC * 2);
            const float2 a = bf16lo_hi(t.x), c = bf16lo_hi(t.y);
#pragma unroll
            for (int p = 0; p < kBwdR; ++p) {  // g column ix feeds output pixel p through tap ix - p
              const int d = ix - p;
              if (d >= 0 && d < 7) {
                acc[p][0] = ffma2(a, wlo[d], acc[p][0]);
                acc[p][1] = ffma2(c, whi[d], acc[p][1]);
              }
            }
          }
        }
#pragma unroll
        for (int p = 0; p < kBwdR; ++p) {
          if (!out[p]) continue;
          const int64_t off = ((static_cast<int64_t>(b) * H + oy) * W + ox0 + px0 + p) * C + cq;
          float o0 = acc[p][0].x, o1 = acc[p][0].y, o2 = acc[p][1].x, o3 = acc[p][1].y;
          if (addend) {
            const float2 a = bf16lo_hi(ad[p].x), c = bf16lo_hi(ad[p].y);
            o0 += a.x; o1 += a.y; o2 += c.x; o3 += c.y;
          }
          __nv_bfloat162 lo = __floats2bfloat162_rn(o0, o1), hi = __floats2bfloat162_rn(o2, o3);
          uint2 t;
          t.x = *reinterpret_cast<uint32_t*>(&lo);
          t.y = *reinterpret_cast<uint32_t*>(&hi);
          *reinterpret_cast<uint2*>(dx_out + off) = t;
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[buf]);
    }
  }
  if (!do_wgrad) return;  // uniform over the CTA

  __syncthreads();  // every stage read is done: red may overwrite stage 0
  if (warp < kBwdHalfWarps && plane < planes) {
#pragma unroll
    for (int d = 0; d < 7; ++d)
      *reinterpret_cast<float4*>(red + (plane * 7 + d) * kBwdC + quad * 4) =
          make_float4(tot[d][0].x, tot[d][0].y, tot[d][1].x, tot[d][1].y);
    if (dy == 0) {
#pragma unroll
      for (int k = 0; k < 4; ++k) red[(planes * 7 + hh) * kBwdC + quad * 4 + k] = btot[k];
    }
  }
  __syncthreads();
  for (int o = threadIdx.x; o < 50 * kBwdC; o += blockDim.x) {
    const int slot = o / kBwdC, ch = o - slot * kBwdC;  // slot = dy * 7 + dx, or 49 for the bias
    if (cc * kBwdC + ch >= C) continue;                 // zero-filled channels of a ragged last chunk
    float s = 0.f;
    if (slot < 49) {
      const int sdy = slot / 7, sdx = slot - sdy * 7;
      for (int h2 = 0; h2 < nh; ++h2) s += red[((h2 * 7 + sdy) * 7 + sdx) * kBwdC + ch];
      atomicAdd(dw49 + slot * C + cc * kBwdC + ch, s);
    } else {
      for (int h2 = 0; h2 < nh; ++h2) s += red[(planes * 7 + h2) * kBwdC + ch];
      atomicAdd(dbias + cc * kBwdC + ch, s);
    }
  }
}

// x / dw49 / dbias null: no weight gradient; w49 null: no data gradient
int launch_dwconv7_bwd(const __nv_bfloat16* x, const __nv_bfloat16* dconv, int B, int H, int W, int C, const float* w49,
                       const __nv_bfloat16* addend, __nv_bfloat16* dx, float* dw49, float* dbias, cudaStream_t s) {
  VDK_REQUIRE(C % 8 == 0, "dwconv7 backward: C must be a multiple of 8 (got %d)", C);
  VDK_REQUIRE((w49 == nullptr || dx != nullptr) && (dw49 == nullptr || (x != nullptr && dbias != nullptr)),
              "dwconv7 backward: missing operand");
  const double elems = static_cast<double>(B) * H * W * C;
  const int halves = (w49 ? 1 : 0) + (dw49 ? 1 : 0);
  // read g (+ x), write dx (+ read the addend)
  ProfScope prof(kProfDepthwise, 2.0 * 49.0 * elems * halves, 2.0 * elems * (1 + (dw49 ? 1 : 0) + (w49 ? (addend ? 2 : 1) : 0)), s);
  if (halves == 0) return VDK_OK;
  const int T = std::min(kBwdT, std::max(H, W));
  CUtensorMap mx, mg;
  int rc = make_tma_nhwc_16bit(&mg, dconv, B, H, W, C, T + 6, T + 6, kBwdC);
  if (rc != VDK_OK) return rc;
  mx = mg;
  if (dw49) {
    rc = make_tma_nhwc_16bit(&mx, x, B, H, W, C, T + 6, T + 6, kBwdC);
    if (rc != VDK_OK) return rc;
  }
  const int halo = T + 6, nh = (T + kBwdR - 1) / kBwdR;
  const int h_bytes = (halo * halo * kBwdC * 2 + 127) & ~127;
  VDK_REQUIRE((7 * 7 * nh + nh) * kBwdC * 4 <= 2 * h_bytes, "dwconv7 backward: reduction does not fit stage 0");
  const int smem = 4 * h_bytes + 49 * kBwdC * 4 + 4 * 8 + 128;
  VDK_CUDA_OK(cudaFuncSetAttribute(dwconv7_bwd_kernel<14>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  VDK_CUDA_OK(cudaFuncSetAttribute(dwconv7_bwd_kernel<7>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  VDK_CUDA_OK(cudaFuncSetAttribute(dwconv7_bwd_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  // images per CTA: one wave of CTAs (one per SM), each pipelining its images through the ring.  Never fewer than the
  // weight-gradient-only grouping of earlier releases (>= ~4 CTAs per SM, at most 16 images), so that the per-image
  // chains plus the fewer atomics never exceed that grouping's roundings (T*7*ipc + nh + groups*tiles).
  const int64_t per_image = static_cast<int64_t>((H + T - 1) / T) * ((W + T - 1) / T) * ((C + kBwdC - 1) / kBwdC);
  const int64_t ipc_min = std::max<int64_t>(1, std::min<int64_t>(16, (per_image * B) / (sm_count() * 4)));
  const int ipc = static_cast<int>(std::min<int64_t>(B, std::max<int64_t>(ipc_min, (per_image * B + sm_count() - 1) / sm_count())));
  const unsigned grid = static_cast<unsigned>(((B + ipc - 1) / ipc) * per_image);
  if (T == 14) dwconv7_bwd_kernel<14><<<grid, kBwdThreads, smem, s>>>(mx, mg, B, H, W, C, T, ipc, w49, addend, dx, dw49, dbias);
  else if (T == 7) dwconv7_bwd_kernel<7><<<grid, kBwdThreads, smem, s>>>(mx, mg, B, H, W, C, T, ipc, w49, addend, dx, dw49, dbias);
  else dwconv7_bwd_kernel<0><<<grid, kBwdThreads, smem, s>>>(mx, mg, B, H, W, C, T, ipc, w49, addend, dx, dw49, dbias);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

// ------------------------------------------------------------------------------------------------
// BatchNorm with batch statistics over the rows of an [R, C] matrix (channels last): forward and backward
// ------------------------------------------------------------------------------------------------
// one block per 32 channels, 8 warps stride the rows; two passes (mean, then centred variance) in fp32
template <typename TIn, typename TOut>
__global__ void __launch_bounds__(256)
bn_train_fwd_kernel(const TIn* __restrict__ x, int R, int C, const float* __restrict__ weight, const float* __restrict__ bias,
                    float eps, float momentum, TOut* __restrict__ y, float* __restrict__ save_mean,
                    float* __restrict__ save_rstd, float* __restrict__ running_mean, float* __restrict__ running_var) {
  __shared__ float red[8][33];
  __shared__ float s_mean[32], s_rstd[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  const bool ok = c < C;
  float s = 0.f;
  if (ok) for (int r = warp; r < R; r += 8) s += static_cast<float>(x[static_cast<int64_t>(r) * C + c]);
  red[warp][lane] = s;
  __syncthreads();
  if (warp == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w][lane];
    s_mean[lane] = t / static_cast<float>(R);
  }
  __syncthreads();
  const float mean = s_mean[lane];
  float q = 0.f;
  if (ok) for (int r = warp; r < R; r += 8) {
    const float d = static_cast<float>(x[static_cast<int64_t>(r) * C + c]) - mean;
    q = fmaf(d, d, q);
  }
  red[warp][lane] = q;
  __syncthreads();
  if (warp == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w][lane];
    const float var = t / static_cast<float>(R);  // biased: what normalises the batch
    s_rstd[lane] = rsqrtf(var + eps);
    if (ok) {
      save_mean[c] = mean;
      save_rstd[c] = s_rstd[lane];
      if (running_mean) {  // nn.BatchNorm: running_var uses the unbiased estimate
        running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
        const float unb = R > 1 ? t / static_cast<float>(R - 1) : var;
        running_var[c] = (1.f - momentum) * running_var[c] + momentum * unb;
      }
    }
  }
  __syncthreads();
  if (ok) {
    const float rs = s_rstd[lane], w = weight[c], b = bias[c];
    for (int r = warp; r < R; r += 8) {
      const float v = (static_cast<float>(x[static_cast<int64_t>(r) * C + c]) - mean) * rs * w + b;
      y[static_cast<int64_t>(r) * C + c] = static_cast<TOut>(v);
    }
  }
}

// dx = w * rstd * (dy - mean(dy) - xh * mean(dy * xh)), xh = (x - mean) * rstd; dweight = sum dy * xh; dbias = sum dy
template <typename TIn, typename TGrad>
__global__ void __launch_bounds__(256)
bn_train_bwd_kernel(const TGrad* __restrict__ dy, const TIn* __restrict__ x, int R, int C, const float* __restrict__ weight,
                    const float* __restrict__ save_mean, const float* __restrict__ save_rstd, TGrad* __restrict__ dx,
                    float* __restrict__ dweight, float* __restrict__ dbias) {
  __shared__ float red[2][8][33];
  __shared__ float s_a[32], s_b[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  const bool ok = c < C;
  const float mean = ok ? save_mean[c] : 0.f, rs = ok ? save_rstd[c] : 0.f;
  float s1 = 0.f, s2 = 0.f;
  if (ok) for (int r = warp; r < R; r += 8) {
    const float g = static_cast<float>(dy[static_cast<int64_t>(r) * C + c]);
    const float xh = (static_cast<float>(x[static_cast<int64_t>(r) * C + c]) - mean) * rs;
    s1 += g;
    s2 = fmaf(g, xh, s2);
  }
  red[0][warp][lane] = s1;
  red[1][warp][lane] = s2;
  __syncthreads();
  if (warp == 0) {
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
      a += red[0][w][lane];
      b += red[1][w][lane];
    }
    s_a[lane] = a;
    s_b[lane] = b;
    if (ok) {
      dbias[c] += a;
      dweight[c] += b;
    }
  }
  __syncthreads();
  if (ok) {
    const float w = weight[c], m1 = s_a[lane] / static_cast<float>(R), m2 = s_b[lane] / static_cast<float>(R);
    for (int r = warp; r < R; r += 8) {
      const float g = static_cast<float>(dy[static_cast<int64_t>(r) * C + c]);
      const float xh = (static_cast<float>(x[static_cast<int64_t>(r) * C + c]) - mean) * rs;
      dx[static_cast<int64_t>(r) * C + c] = static_cast<TGrad>(w * rs * (g - m1 - xh * m2));
    }
  }
}

// bf16 activations with C % 8 == 0 (the neck's BatchNorm2d: rows = batch * H * W): one block per 8-channel vector
// column, 256 threads stride the rows with 16-byte loads; the tensor is L2-resident between the passes.
__device__ __forceinline__ void block_sum8(float (&v)[8], float (*red)[8]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = wsum(v[j]);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();  // red may still be read from the previous call
  if (lane == 0) {
#pragma unroll
    for (int j = 0; j < 8; ++j) red[warp][j] = v[j];
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w][j];
    v[j] = t;
  }
}

__global__ void __launch_bounds__(256)
bn_train_fwd_vec_kernel(const __nv_bfloat16* __restrict__ x, int R, int C, const float* __restrict__ weight,
                        const float* __restrict__ bias, float eps, float momentum, __nv_bfloat16* __restrict__ y,
                        float* __restrict__ save_mean, float* __restrict__ save_rstd, float* __restrict__ running_mean,
                        float* __restrict__ running_var) {
  __shared__ float red[8][8];
  const int c0 = blockIdx.x * 8;
  const float inv_r = 1.0f / static_cast<float>(R);
  float mean[8], q[8], v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { mean[j] = 0.f; q[j] = 0.f; }
  for (int r = threadIdx.x; r < R; r += 256) {
    unpack8(__ldg(reinterpret_cast<const uint4*>(x + static_cast<int64_t>(r) * C + c0)), v);
#pragma unroll
    for (int j = 0; j < 8; ++j) mean[j] += v[j];
  }
  block_sum8(mean, red);
#pragma unroll
  for (int j = 0; j < 8; ++j) mean[j] *= inv_r;
  for (int r = threadIdx.x; r < R; r += 256) {
    unpack8(__ldg(reinterpret_cast<const uint4*>(x + static_cast<int64_t>(r) * C + c0)), v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float d = v[j] - mean[j];
      q[j] = fmaf(d, d, q[j]);
    }
  }
  block_sum8(q, red);
  float sc[8], sh[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float var = q[j] * inv_r;  // biased: what normalises the batch
    const float rs = rsqrtf(var + eps);
    sc[j] = rs * weight[c0 + j];
    sh[j] = bias[c0 + j] - mean[j] * sc[j];
    if (threadIdx.x == 0) {
      save_mean[c0 + j] = mean[j];
      save_rstd[c0 + j] = rs;
      if (running_mean) {  // nn.BatchNorm: running_var uses the unbiased estimate
        running_mean[c0 + j] = (1.f - momentum) * running_mean[c0 + j] + momentum * mean[j];
        const float unb = R > 1 ? q[j] / static_cast<float>(R - 1) : var;
        running_var[c0 + j] = (1.f - momentum) * running_var[c0 + j] + momentum * unb;
      }
    }
  }
  for (int r = threadIdx.x; r < R; r += 256) {
    unpack8(__ldg(reinterpret_cast<const uint4*>(x + static_cast<int64_t>(r) * C + c0)), v);
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = fmaf(v[j], sc[j], sh[j]);
    *reinterpret_cast<uint4*>(y + static_cast<int64_t>(r) * C + c0) = pack8(o);
  }
}

__global__ void __launch_bounds__(256)
bn_train_bwd_vec_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x, int R, int C,
                        const float* __restrict__ weight, const float* __restrict__ save_mean,
                        const float* __restrict__ save_rstd, __nv_bfloat16* __restrict__ dx, float* __restrict__ dweight,
                        float* __restrict__ dbias) {
  __shared__ float red[8][8];
  const int c0 = blockIdx.x * 8;
  float mean[8], rs[8], s1[8], s2[8], g[8], v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    mean[j] = save_mean[c0 + j];
    rs[j] = save_rstd[c0 + j];
    s1[j] = 0.f;
    s2[j] = 0.f;
  }
  for (int r = threadIdx.x; r < R; r += 256) {
    unpack8(__ldg(reinterpret_cast<const uint4*>(dy + static_cast<int64_t>(r) * C + c0)), g);
    unpack8(__ldg(reinterpret_cast<const uint4*>(x + static_cast<int64_t>(r) * C + c0)), v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s1[j] += g[j];
      s2[j] = fmaf(g[j], (v[j] - mean[j]) * rs[j], s2[j]);
    }
  }
  block_sum8(s1, red);
  block_sum8(s2, red);
  const float inv_r = 1.0f / static_cast<float>(R);
  float a[8], m1[8], m2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (threadIdx.x == 0) {
      dbias[c0 + j] += s1[j];
      dweight[c0 + j] += s2[j];
    }
    a[j] = weight[c0 + j] * rs[j];
    m1[j] = s1[j] * inv_r;
    m2[j] = s2[j] * inv_r;
  }
  for (int r = threadIdx.x; r < R; r += 256) {
    unpack8(__ldg(reinterpret_cast<const uint4*>(dy + static_cast<int64_t>(r) * C + c0)), g);
    unpack8(__ldg(reinterpret_cast<const uint4*>(x + static_cast<int64_t>(r) * C + c0)), v);
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = a[j] * (g[j] - m1[j] - (v[j] - mean[j]) * rs[j] * m2[j]);
    *reinterpret_cast<uint4*>(dx + static_cast<int64_t>(r) * C + c0) = pack8(o);
  }
}

// ------------------------------------------------------------------------------------------------
// weight packing: fp32 master -> bf16 kernel layout; permutation [a][b][c] -> [a][c][b]; gradient un-permutation
// ------------------------------------------------------------------------------------------------
// out_bf16[a][c][b] = in[a][b][c] * (row_scale ? row_scale[a] : 1)
__global__ void __launch_bounds__(256)
permute021_kernel(const float* __restrict__ in, int A, int Bd, int Cd, const float* __restrict__ row_scale,
                  __nv_bfloat16* __restrict__ out_bf16, float* __restrict__ out_f32, int accumulate) {
  const int64_t total = static_cast<int64_t>(A) * Bd * Cd;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    // i indexes the OUTPUT [a][c][b] so that writes are coalesced
    const int b = static_cast<int>(i % Bd);
    const int c = static_cast<int>((i / Bd) % Cd);
    const int a = static_cast<int>(i / (static_cast<int64_t>(Bd) * Cd));
    float v = in[(static_cast<int64_t>(a) * Bd + b) * Cd + c];
    if (row_scale) v *= row_scale[a];
    if (out_bf16) out_bf16[i] = __float2bfloat16_rn(v);
    if (out_f32) out_f32[i] = accumulate ? out_f32[i] + v : v;
  }
}

// the same permutation through a 32 x 32 shared-memory tile: reads coalesced along c, writes coalesced along b
__global__ void __launch_bounds__(256)
permute021_tiled_kernel(const float* __restrict__ in, int Bd, int Cd, const float* __restrict__ row_scale,
                        __nv_bfloat16* __restrict__ out_bf16, float* __restrict__ out_f32, int accumulate) {
  __shared__ float tile[32][33];
  const int a = blockIdx.z, b0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const float sc = row_scale ? row_scale[a] : 1.f;
  const int64_t base = static_cast<int64_t>(a) * Bd * Cd;
#pragma unroll
  for (int r = ty; r < 32; r += 8) {
    const int b = b0 + r, c = c0 + tx;
    if (b < Bd && c < Cd) tile[r][tx] = in[base + static_cast<int64_t>(b) * Cd + c] * sc;
  }
  __syncthreads();
#pragma unroll
  for (int r = ty; r < 32; r += 8) {
    const int c = c0 + r, b = b0 + tx;
    if (b < Bd && c < Cd) {
      const int64_t o = base + static_cast<int64_t>(c) * Bd + b;
      const float v = tile[tx][r];
      if (out_bf16) out_bf16[o] = __float2bfloat16_rn(v);
      if (out_f32) out_f32[o] = accumulate ? out_f32[o] + v : v;
    }
  }
}

// layer-scale gradient finalisation for fc2 (out = x + gamma * (h W2^T + b2)):
//   G[c,k] = sum_m dOut[m,c] h[m,k] (the wgrad GEMM without gamma), sdo[c] = sum_m dOut[m,c]
//   dW2[c,k] += gamma[c] G[c,k];  dgamma[c] += sum_k G[c,k] W2[c,k] + b2[c] sdo[c];  db2[c] += gamma[c] sdo[c]
__global__ void __launch_bounds__(256)
layerscale_finalize_kernel(const float* __restrict__ G, const float* __restrict__ W2, const float* __restrict__ b2,
                           const float* __restrict__ gamma, const float* __restrict__ sdo, int C, int K4,
                           float* __restrict__ dW2, float* __restrict__ dgamma, float* __restrict__ db2) {
  __shared__ float red[8];
  const int c = blockIdx.x;
  const float gm = gamma[c];
  float dot = 0.f;
  for (int k = threadIdx.x; k < K4; k += 256) {
    const float g = G[static_cast<int64_t>(c) * K4 + k];
    dot = fmaf(g, W2[static_cast<int64_t>(c) * K4 + k], dot);
    dW2[static_cast<int64_t>(c) * K4 + k] += gm * g;
  }
  dot = wsum(dot);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = dot;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w];
    dgamma[c] += t + b2[c] * sdo[c];
    db2[c] += gm * sdo[c];
  }
}

__global__ void cast_f32_bf16_kernel(const float* __restrict__ in, int64_t n, __nv_bfloat16* __restrict__ out) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    out[i] = __float2bfloat16_rn(in[i]);
}
__global__ void add_f32_kernel(float* __restrict__ dst, const float* __restrict__ src, int64_t n) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    dst[i] += src[i];
}

static int blocks_for(int64_t n) { return static_cast<int>(std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, 132 * 16))); }

int launch_permute021(const float* in, int A, int Bd, int Cd, const float* row_scale, __nv_bfloat16* out_bf16,
                      float* out_f32, int accumulate, cudaStream_t s) {
  if (Bd >= 16 && Cd >= 16 && A <= 65535 && (Bd + 31) / 32 <= 65535) {
    const dim3 grid((Cd + 31) / 32, (Bd + 31) / 32, A);
    permute021_tiled_kernel<<<grid, 256, 0, s>>>(in, Bd, Cd, row_scale, out_bf16, out_f32, accumulate);
  } else {
    permute021_kernel<<<blocks_for(static_cast<int64_t>(A) * Bd * Cd), 256, 0, s>>>(in, A, Bd, Cd, row_scale, out_bf16, out_f32,
                                                                                   accumulate);
  }
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}
int launch_cast_bf16(const float* in, int64_t n, __nv_bfloat16* out, cudaStream_t s) {
  cast_f32_bf16_kernel<<<blocks_for(n), 256, 0, s>>>(in, n, out);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}
int launch_layerscale_finalize(const float* G, const float* W2, const float* b2, const float* gamma, const float* sdo, int C,
                               int K4, float* dW2, float* dgamma, float* db2, cudaStream_t s) {
  layerscale_finalize_kernel<<<C, 256, 0, s>>>(G, W2, b2, gamma, sdo, C, K4, dW2, dgamma, db2);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}
int launch_bn_fwd_bf16(const __nv_bfloat16* x, int R, int C, const float* w, const float* b, float eps, float momentum,
                       __nv_bfloat16* y, float* save_mean, float* save_rstd, float* run_mean, float* run_var, cudaStream_t s) {
  if (C % 8 == 0)
    bn_train_fwd_vec_kernel<<<C / 8, 256, 0, s>>>(x, R, C, w, b, eps, momentum, y, save_mean, save_rstd, run_mean, run_var);
  else
    bn_train_fwd_kernel<__nv_bfloat16, __nv_bfloat16><<<(C + 31) / 32, 256, 0, s>>>(x, R, C, w, b, eps, momentum, y, save_mean,
                                                                                    save_rstd, run_mean, run_var);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}
int launch_bn_fwd_f32(const float* x, int R, int C, const float* w, const float* b, float eps, float momentum, float* y,
                      float* save_mean, float* save_rstd, float* run_mean, float* run_var, cudaStream_t s) {
  bn_train_fwd_kernel<float, float><<<(C + 31) / 32, 256, 0, s>>>(x, R, C, w, b, eps, momentum, y, save_mean, save_rstd, run_mean,
                                                                  run_var);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}
int launch_bn_bwd_bf16(const __nv_bfloat16* dy, const __nv_bfloat16* x, int R, int C, const float* w, const float* save_mean,
                       const float* save_rstd, __nv_bfloat16* dx, float* dweight, float* dbias, cudaStream_t s) {
  if (C % 8 == 0)
    bn_train_bwd_vec_kernel<<<C / 8, 256, 0, s>>>(dy, x, R, C, w, save_mean, save_rstd, dx, dweight, dbias);
  else
    bn_train_bwd_kernel<__nv_bfloat16, __nv_bfloat16><<<(C + 31) / 32, 256, 0, s>>>(dy, x, R, C, w, save_mean, save_rstd, dx,
                                                                                    dweight, dbias);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}
int launch_bn_bwd_f32(const float* dy, const float* x, int R, int C, const float* w, const float* save_mean,
                      const float* save_rstd, float* dx, float* dweight, float* dbias, cudaStream_t s) {
  bn_train_bwd_kernel<float, float><<<(C + 31) / 32, 256, 0, s>>>(dy, x, R, C, w, save_mean, save_rstd, dx, dweight, dbias);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}
int launch_add_f32(float* dst, const float* src, int64_t n, cudaStream_t s) {
  add_f32_kernel<<<blocks_for(n), 256, 0, s>>>(dst, src, n);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

}  // namespace vdk

// ---- C-ABI exports of the building blocks (unit parity tests; the product calls them through convnext_train.cu) ----
using namespace vdk;

extern "C" int vdk_layernorm_bwd(const void* dy, const void* y, const float* rstd, int batch, int H, int W, int C,
                                 const float* ln_w, const float* ln_b, int patch, void* dx, const void* addend, float* dgamma,
                                 float* dbeta, void* stream) {
  VDK_REQUIRE(dy && y && rstd && ln_w && ln_b && dx && dgamma && dbeta, "vdk_layernorm_bwd: null operand");
  VDK_REQUIRE(patch == 1 || (patch == 2 && H % 2 == 0 && W % 2 == 0), "vdk_layernorm_bwd: patch must be 1 or 2");
  return launch_ln_bwd(reinterpret_cast<const __nv_bfloat16*>(dy), reinterpret_cast<const __nv_bfloat16*>(y), rstd, batch, H, W, C,
                       ln_w, ln_b, patch, reinterpret_cast<__nv_bfloat16*>(dx), reinterpret_cast<const __nv_bfloat16*>(addend),
                       dgamma, dbeta, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vdk_dwconv7(int mode, const void* x, int batch, int H, int W, int C, const float* w49, const float* bias,
                           const float* ln_w, const float* ln_b, float eps, void* y, float* rstd_out, const void* addend,
                           void* stream) {
  VDK_REQUIRE(x && y && w49 && (mode == 1 || (bias && ln_w && ln_b)), "vdk_dwconv7: null operand");
  return launch_dwconv7(mode, reinterpret_cast<const __nv_bfloat16*>(x), batch, H, W, C, w49, bias, ln_w, ln_b, eps,
                        reinterpret_cast<__nv_bfloat16*>(y), rstd_out, reinterpret_cast<const __nv_bfloat16*>(addend),
                        reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vdk_dwconv7_wgrad(const void* x, const void* dconv, int batch, int H, int W, int C, float* dw49, float* dbias,
                                 void* stream) {
  VDK_REQUIRE(x && dconv && dw49 && dbias, "vdk_dwconv7_wgrad: null operand");
  return launch_dwconv7_bwd(reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<const __nv_bfloat16*>(dconv), batch, H, W, C,
                            nullptr, nullptr, nullptr, dw49, dbias, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vdk_dwconv7_bwd(const void* x, const void* dconv, int batch, int H, int W, int C, const float* w49,
                               const void* addend, void* dx, float* dw49, float* dbias, void* stream) {
  VDK_REQUIRE(x && dconv && w49 && dx && dw49 && dbias, "vdk_dwconv7_bwd: null operand");
  return launch_dwconv7_bwd(reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<const __nv_bfloat16*>(dconv), batch, H, W, C,
                            w49, reinterpret_cast<const __nv_bfloat16*>(addend), reinterpret_cast<__nv_bfloat16*>(dx), dw49, dbias,
                            reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vdk_batchnorm_train_fwd(const void* x, int rows, int C, int is_bf16, const float* weight, const float* bias,
                                       float eps, float momentum, void* y, float* save_mean, float* save_rstd,
                                       float* running_mean, float* running_var, void* stream) {
  VDK_REQUIRE(x && y && weight && bias && save_mean && save_rstd && rows > 1, "vdk_batchnorm_train_fwd: bad arguments");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (is_bf16)
    return launch_bn_fwd_bf16(reinterpret_cast<const __nv_bfloat16*>(x), rows, C, weight, bias, eps, momentum,
                              reinterpret_cast<__nv_bfloat16*>(y), save_mean, save_rstd, running_mean, running_var, s);
  return launch_bn_fwd_f32(reinterpret_cast<const float*>(x), rows, C, weight, bias, eps, momentum, reinterpret_cast<float*>(y),
                           save_mean, save_rstd, running_mean, running_var, s);
}

extern "C" int vdk_batchnorm_train_bwd(const void* dy, const void* x, int rows, int C, int is_bf16, const float* weight,
                                       const float* save_mean, const float* save_rstd, void* dx, float* dweight, float* dbias,
                                       void* stream) {
  VDK_REQUIRE(dy && x && weight && save_mean && save_rstd && dx && dweight && dbias, "vdk_batchnorm_train_bwd: null operand");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (is_bf16)
    return launch_bn_bwd_bf16(reinterpret_cast<const __nv_bfloat16*>(dy), reinterpret_cast<const __nv_bfloat16*>(x), rows, C, weight,
                              save_mean, save_rstd, reinterpret_cast<__nv_bfloat16*>(dx), dweight, dbias, s);
  return launch_bn_bwd_f32(reinterpret_cast<const float*>(dy), reinterpret_cast<const float*>(x), rows, C, weight, save_mean,
                           save_rstd, reinterpret_cast<float*>(dx), dweight, dbias, s);
}
