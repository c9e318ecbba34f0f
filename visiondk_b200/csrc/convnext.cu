// convnext.cu — ConvNeXt (timm 0.9.16 layout) embedding forward for the faceX/CBIR extract path, NHWC bf16.
//
// Replaces timm's ConvNeXt forward + the reference neck + F.normalize:
//   models/faceX/backbone/timm_wrapper.py:51-54 (TimmWrapper.forward), :30-38 (output_layer),
//   models/faceX/face_model.py:137-139 (extract_cbir: model(x) then F.normalize).
//
// Dense contractions run on the wgmma GEMM (gemm.cu) with fused epilogues; everything around them is an
// HBM-bound kernel written here:
//   stem_patchify     NCHW fp32 image -> 4x4 patch rows [B*H/4*W/4, 48] bf16          (then GEMM + bias + LayerNorm)
//   dwconv7_ln        depthwise 7x7 (pad 3) + bias + LayerNorm over C, NHWC bf16      (then GEMM+GELU, GEMM+gamma+res)
//   ln_patchify       LayerNorm over C [+ 2x2/s2 patch gather]                        (downsample conv / head norm)
//   neck_finalize     split-K partials + folded BN bias [+ L2 normalise] -> fp32 embeddings
#include "vdk_host.h"
#include "vdk_ptx.cuh"

#include <cstdlib>
#include "convnext_internal.h"

namespace vdk {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

// ------------------------------------------------------------------------------------------------
// stem: 4x4 stride-4 patches of an NCHW fp32 image -> rows of 48 (c, kh, kw) in bf16
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) stem_patchify_kernel(const float* __restrict__ x, int B, int H, int W,
                                                            __nv_bfloat16* __restrict__ out) {
  // one thread per (patch, c, kh): reads 4 contiguous pixels, writes 4 contiguous bf16
  const int PH = H / 4, PW = W / 4;
  const int64_t total = static_cast<int64_t>(B) * PH * PW * 12;
  for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int ck = static_cast<int>(t % 12);
    const int64_t patch = t / 12;
    const int c = ck >> 2, kh = ck & 3;
    const int pw = static_cast<int>(patch % PW);
    const int ph = static_cast<int>((patch / PW) % PH);
    const int b = static_cast<int>(patch / (static_cast<int64_t>(PW) * PH));
    const float4 v = *reinterpret_cast<const float4*>(x + ((static_cast<int64_t>(b) * 3 + c) * H + (ph * 4 + kh)) * W + pw * 4);
    __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
    uint2 o;
    o.x = *reinterpret_cast<uint32_t*>(&lo);
    o.y = *reinterpret_cast<uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(out + patch * 48 + ck * 4) = o;
  }
}

int launch_stem_patchify(const float* images, int B, int S, __nv_bfloat16* out, cudaStream_t s) {
  const int64_t total = static_cast<int64_t>(B) * (S / 4) * (S / 4) * 12;
  const int blocks = static_cast<int>(std::min<int64_t>((total + 255) / 256, 132 * 16));
  stem_patchify_kernel<<<blocks, 256, 0, s>>>(images, B, S, S, out);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

// ------------------------------------------------------------------------------------------------
// depthwise 7x7 + bias + LayerNorm(C)
// ------------------------------------------------------------------------------------------------
// One CTA = a TH x TW tile of output pixels x ALL channels (LayerNorm couples the channels of a pixel).  The
// (TH+6) x (TW+6) x C input halo is brought into shared memory by TMA as a 4-D NHWC box whose out-of-bounds part
// is zero-filled by the hardware — exactly the convolution's zero padding, so the arithmetic loop has no bounds
// checks.  A "group" of C/4 threads (4 contiguous channels each: conflict-free 8-byte LDS, coalesced 8-byte STG)
// owns one output row of the tile at a time; the 49 taps of a thread's 4 channels are read one filter row at a
// time (L1-resident), accumulators stay in registers, and LayerNorm over C is a reduction inside the group.
// FMA-bound: 49 FMAs per output against 2 + 2 bytes of HBM traffic.  y = LayerNorm_C(conv + bias), optionally saving
// 1/sigma per pixel for the backward (the backward-data pass is dwconv7_bwd_kernel, train_ops.cu).
template <int TW>
__global__ void __launch_bounds__(512)
dwconv7_ln_kernel(const __grid_constant__ CUtensorMap map_x, int B, int H, int W, int C, int TH, int box_c,
                  int tpg /*threads per group, whole warps*/,
                  const float* __restrict__ w49,  // [49][C]
                  const float* __restrict__ bias, const float* __restrict__ ln_w, const float* __restrict__ ln_b,
                  float eps, __nv_bfloat16* __restrict__ y, float* __restrict__ rstd_out) {
  extern __shared__ uint8_t dw_smem_raw[];
  // aligned without a pointer->integer->pointer round trip, so the tile reads below stay LDS (not generic LD)
  uint8_t* smem = dw_smem_raw + ((128u - (smem_u32(dw_smem_raw) & 127u)) & 127u);
  const int box_h = TH + 6, box_w = TW + 6;
  const int n_chunks = C / box_c;
  const int box_bytes = box_h * box_w * box_c * 2;
  const int chunk_bytes = (box_bytes + 127) & ~127;  // chunk stride: every TMA destination 128-byte aligned
  float* red = reinterpret_cast<float*>(smem + n_chunks * chunk_bytes);  // [group][TW][warps per group <= 16]
  uint64_t* bar = reinterpret_cast<uint64_t*>(red + 16 * TW * 16);

  const int groups = blockDim.x / tpg;
  const int grp = threadIdx.x / tpg;
  const int tig = threadIdx.x - grp * tpg;
  const int tiles_w = (W + TW - 1) / TW, tiles_h = (H + TH - 1) / TH;
  const int tw = blockIdx.x % tiles_w;
  const int th = (blockIdx.x / tiles_w) % tiles_h;
  const int b = blockIdx.x / (tiles_w * tiles_h);
  const int oy0 = th * TH, ox0 = tw * TW;
  const int c0 = tig * 4;
  const bool has_c = c0 < C;
  const int lane = threadIdx.x & 31;
  const int wig = tig >> 5, nwig = tpg >> 5;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_x);
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(bar, n_chunks * box_bytes);
    for (int ch = 0; ch < n_chunks; ++ch)
      tma_load_4d(smem + ch * chunk_bytes, &map_x, bar, ch * box_c, ox0 - 3, oy0 - 3, b);
  }
  // weights / affine parameters of this thread's channels while the tile is in flight
  float4 bc = make_float4(0.f, 0.f, 0.f, 0.f), g4 = bc, b4 = bc;
  if (has_c) {
    bc = __ldg(reinterpret_cast<const float4*>(bias + c0));
    g4 = __ldg(reinterpret_cast<const float4*>(ln_w + c0));
    b4 = __ldg(reinterpret_cast<const float4*>(ln_b + c0));
  }
  const int pix_stride = box_c * 2;  // bytes between neighbouring pixels of one chunk
  const uint8_t* tbase = smem + (has_c ? (c0 / box_c) * chunk_bytes + (c0 % box_c) * 2 : 0);
  mbar_wait(bar, 0);

  const float inv_c = 1.0f / static_cast<float>(C);
  const int rounds = (TH + groups - 1) / groups;
  for (int rd = 0; rd < rounds; ++rd) {
    const int oyl = rd * groups + grp;  // output row inside the tile
    const bool active = has_c && oyl < TH && oy0 + oyl < H;
    float acc[TW][4];
#pragma unroll
    for (int p = 0; p < TW; ++p) {
      acc[p][0] = bc.x; acc[p][1] = bc.y; acc[p][2] = bc.z; acc[p][3] = bc.w;
    }
    if (active) {
#pragma unroll 1
      for (int dy = 0; dy < 7; ++dy) {
        float4 wrow[7];
#pragma unroll
        for (int dx = 0; dx < 7; ++dx) wrow[dx] = __ldg(reinterpret_cast<const float4*>(w49 + (dy * 7 + dx) * C + c0));
        const uint8_t* rowp = tbase + static_cast<size_t>((oyl + dy) * box_w) * pix_stride;
#pragma unroll
        for (int ix = 0; ix < TW + 6; ++ix) {
          const uint2 t = *reinterpret_cast<const uint2*>(rowp + ix * pix_stride);
          const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.x));
          const float2 c = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.y));
#pragma unroll
          for (int p = 0; p < TW; ++p) {
            const int dx = ix - p;  // input column ix feeds output pixel p through tap dx
            if (dx >= 0 && dx < 7) {
              acc[p][0] = fmaf(a.x, wrow[dx].x, acc[p][0]);
              acc[p][1] = fmaf(a.y, wrow[dx].y, acc[p][1]);
              acc[p][2] = fmaf(c.x, wrow[dx].z, acc[p][2]);
              acc[p][3] = fmaf(c.y, wrow[dx].w, acc[p][3]);
            }
          }
        }
      }
    }
    // LayerNorm over C for the TW pixels of this row: mean, then centred second moment, reduced in the group
    float mean[TW], rstd[TW];
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
      float sred[TW];
#pragma unroll
      for (int p = 0; p < TW; ++p) {
        float v = 0.f;
        if (active) {
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const float d = pass == 0 ? acc[p][c] : acc[p][c] - mean[p];
            v += pass == 0 ? d : d * d;
          }
        }
        sred[p] = warp_sum(v);
      }
      if (nwig > 1) {  // uniform across the CTA
        if (lane == 0) {
#pragma unroll
          for (int p = 0; p < TW; ++p) red[(grp * TW + p) * 16 + wig] = sred[p];
        }
        __syncthreads();
#pragma unroll
        for (int p = 0; p < TW; ++p) sred[p] = 0.f;
#pragma unroll 1
        for (int w = 0; w < nwig; ++w) {  // not unrolled: a 16-way predicated unroll costs more than the conv itself
#pragma unroll
          for (int p = 0; p < TW; ++p) sred[p] += red[(grp * TW + p) * 16 + w];
        }
        __syncthreads();
      }
#pragma unroll
      for (int p = 0; p < TW; ++p) {
        if (pass == 0) mean[p] = sred[p] * inv_c;
        else rstd[p] = rsqrtf(sred[p] * inv_c + eps);
      }
    }
    if (active) {
#pragma unroll
      for (int p = 0; p < TW; ++p) {
        const int ox = ox0 + p;
        if (ox >= W) continue;
        const int64_t pix = (static_cast<int64_t>(b) * H + oy0 + oyl) * W + ox;
        if (rstd_out != nullptr && tig == 0) rstd_out[pix] = rstd[p];
        __nv_bfloat16* dst = y + pix * C + c0;
        __nv_bfloat162 lo = __floats2bfloat162_rn((acc[p][0] - mean[p]) * rstd[p] * g4.x + b4.x,
                                                  (acc[p][1] - mean[p]) * rstd[p] * g4.y + b4.y);
        __nv_bfloat162 hi = __floats2bfloat162_rn((acc[p][2] - mean[p]) * rstd[p] * g4.z + b4.z,
                                                  (acc[p][3] - mean[p]) * rstd[p] * g4.w + b4.w);
        uint2 t;
        t.x = *reinterpret_cast<uint32_t*>(&lo);
        t.y = *reinterpret_cast<uint32_t*>(&hi);
        *reinterpret_cast<uint2*>(dst) = t;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// the same operator, channel-chunked: CTA = (image, TH x 7 pixel tile, <=128-channel chunk), one warp per output row
// ------------------------------------------------------------------------------------------------
// The all-channel kernel above holds a (T+6)^2 x C halo per CTA (173 KB at C = 512): one CTA per SM, its TMA load
// fully exposed.  Here a CTA stages only its chunk (43 KB at 128 channels), three CTAs share an SM and hide each
// other's loads, and the tile count per SM is large enough that the tail wave no longer matters.  LayerNorm couples the
// chunks of a pixel: the C / chunk CTAs of a tile form a thread-block CLUSTER, each publishes (mean, centred sum of
// squares) of its channels per pixel in shared memory, and every CTA combines the partials of its peers through
// distributed shared memory (Chan's parallel-variance update: same two-pass numerics as the reference LayerNorm,
// one cluster barrier).
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ float2 ld_dsmem_f2(const void* local_smem, uint32_t rank) {
  uint32_t ra;
  float2 v;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(smem_u32(local_smem)), "r"(rank));
  asm volatile("ld.shared::cluster.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(ra) : "memory");
  return v;
}

constexpr int kDwTW = 7;

template <int CHUNK>
__global__ void __launch_bounds__(224, 3)
dwconv7_chunk_kernel(const __grid_constant__ CUtensorMap map_x, int B, int H, int W, int C, int TH, int nchunks,
                     const float* __restrict__ w49, const float* __restrict__ bias, const float* __restrict__ ln_w,
                     const float* __restrict__ ln_b, float eps, __nv_bfloat16* __restrict__ y, float* __restrict__ rstd_out) {
  extern __shared__ uint8_t dwc_smem_raw[];
  uint8_t* smem = dwc_smem_raw + ((128u - (smem_u32(dwc_smem_raw) & 127u)) & 127u);
  constexpr int box_w = kDwTW + 6;
  constexpr int chunk = CHUNK;  // compile-time: every shared-memory offset of the tap loop is an immediate
  const int tile_bytes = (TH + 6) * box_w * chunk * 2;
  float* wsm = reinterpret_cast<float*>(smem + ((tile_bytes + 127) & ~127));     // [49][chunk] taps of this chunk
  float2* part = reinterpret_cast<float2*>(wsm + 49 * chunk);                    // [7 rows][8]: (mean, M2) per pixel
  uint64_t* bar = reinterpret_cast<uint64_t*>(part + 7 * 8);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int bid = blockIdx.x;
  const int ck = bid % nchunks; bid /= nchunks;
  const int tiles_w = (W + kDwTW - 1) / kDwTW, tiles_h = (H + TH - 1) / TH;
  const int tw = bid % tiles_w; bid /= tiles_w;
  const int th = bid % tiles_h;
  const int b = bid / tiles_h;
  const int oy0 = th * TH, ox0 = tw * kDwTW;
  const int cl = lane * 4;
  const bool has_c = cl < chunk;
  const int c0 = ck * chunk + cl;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_x);
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(bar, tile_bytes);
    tma_load_4d(smem, &map_x, bar, ck * chunk, ox0 - 3, oy0 - 3, b);
  }
  float4 bc = make_float4(0.f, 0.f, 0.f, 0.f), g4 = bc, b4 = bc;
  if (has_c) {
    bc = __ldg(reinterpret_cast<const float4*>(bias + c0));
    g4 = __ldg(reinterpret_cast<const float4*>(ln_w + c0));
    b4 = __ldg(reinterpret_cast<const float4*>(ln_b + c0));
  }
  // the chunk's 49 x chunk taps: shared memory, while the tile is in flight
  for (int i = threadIdx.x; i < 49 * (chunk / 4); i += blockDim.x) {
    const int t = i / (chunk / 4), q = i - t * (chunk / 4);
    *reinterpret_cast<float4*>(wsm + t * chunk + q * 4) = __ldg(reinterpret_cast<const float4*>(w49 + t * C + ck * chunk + q * 4));
  }
  __syncthreads();
  constexpr int pix_stride = chunk * 2;
  const bool active = has_c && warp < TH && oy0 + warp < H;
  float2 acc[kDwTW][2];  // channel pairs (c0, c0+1), (c0+2, c0+3)
#pragma unroll
  for (int p = 0; p < kDwTW; ++p) {
    acc[p][0] = make_float2(bc.x, bc.y);
    acc[p][1] = make_float2(bc.z, bc.w);
  }
  mbar_wait(bar, 0);
  if (active) {
    const uint8_t* tbase = smem + cl * 2;
#pragma unroll 1
    for (int dy = 0; dy < 7; ++dy) {
      float2 wlo[7], whi[7];
      const float* wrow = wsm + dy * (7 * chunk) + cl;
#pragma unroll
      for (int dx = 0; dx < 7; ++dx) {
        const float4 t = *reinterpret_cast<const float4*>(wrow + dx * chunk);
        wlo[dx] = make_float2(t.x, t.y);
        whi[dx] = make_float2(t.z, t.w);
      }
      const uint8_t* rowp = tbase + (warp + dy) * (box_w * pix_stride);
#pragma unroll
      for (int ix = 0; ix < box_w; ++ix) {
        const uint2 t = *reinterpret_cast<const uint2*>(rowp + ix * pix_stride);
        // bf16 -> fp32 is a 16-bit shift: one ALU op per value
        const float2 a = make_float2(__uint_as_float(t.x << 16), __uint_as_float(t.x & 0xffff0000u));
        const float2 c = make_float2(__uint_as_float(t.y << 16), __uint_as_float(t.y & 0xffff0000u));
#pragma unroll
        for (int p = 0; p < kDwTW; ++p) {
          const int dx = ix - p;  // input column ix feeds output pixel p through tap dx
          if (dx >= 0 && dx < 7) {
            acc[p][0] = ffma2(a, wlo[dx], acc[p][0]);
            acc[p][1] = ffma2(c, whi[dx], acc[p][1]);
          }
        }
      }
    }
  }
  // ---- LayerNorm over C: local two-pass statistics of this chunk, then the cluster-wide combination ----
  float mean[kDwTW], rstd[kDwTW];
  const float inv_chunk = 1.0f / static_cast<float>(chunk), inv_c = 1.0f / static_cast<float>(C);
#pragma unroll
  for (int p = 0; p < kDwTW; ++p) {
    const float s = warp_sum(active ? (acc[p][0].x + acc[p][0].y) + (acc[p][1].x + acc[p][1].y) : 0.f);
    mean[p] = s * inv_chunk;
  }
#pragma unroll
  for (int p = 0; p < kDwTW; ++p) {
    float q = 0.f;
    if (active) {
      const float d0 = acc[p][0].x - mean[p], d1 = acc[p][0].y - mean[p];
      const float d2 = acc[p][1].x - mean[p], d3 = acc[p][1].y - mean[p];
      q = fmaf(d0, d0, fmaf(d1, d1, fmaf(d2, d2, d3 * d3)));
    }
    rstd[p] = warp_sum(q);  // centred sum of squares of this chunk, for now
  }
  if (nchunks == 1) {
#pragma unroll
    for (int p = 0; p < kDwTW; ++p) rstd[p] = rsqrtf(rstd[p] * inv_c + eps);
  } else {
    float2 mine = make_float2(0.f, 0.f);
#pragma unroll
    for (int p = 0; p < kDwTW; ++p)
      if (lane == p) mine = make_float2(mean[p], rstd[p]);
    if (lane < kDwTW && warp < 7) part[warp * 8 + lane] = mine;
    cluster_arrive();
    cluster_wait();
    const float inv_n = 1.0f / static_cast<float>(nchunks);
#pragma unroll
    for (int p = 0; p < kDwTW; ++p) {
      float2 r = make_float2(0.f, 0.f);
      if (lane < nchunks) r = ld_dsmem_f2(part + warp * 8 + p, static_cast<uint32_t>(lane));
      const float m = warp_sum(r.x) * inv_n;
      const float d = r.x - m;
      const float m2 = warp_sum(lane < nchunks ? fmaf(static_cast<float>(chunk) * d, d, r.y) : 0.f);
      mean[p] = m;
      rstd[p] = rsqrtf(m2 * inv_c + eps);
    }
    cluster_arrive();  // my reads of the peers' partials are done (matched by the wait before exit)
  }
  if (active) {
#pragma unroll
    for (int p = 0; p < kDwTW; ++p) {
      const int ox = ox0 + p;
      if (ox >= W) continue;
      const int64_t pix = (static_cast<int64_t>(b) * H + oy0 + warp) * W + ox;
      if (rstd_out != nullptr && lane == 0 && ck == 0) rstd_out[pix] = rstd[p];
      __nv_bfloat16* dst = y + pix * C + c0;
      __nv_bfloat162 lo = __floats2bfloat162_rn((acc[p][0].x - mean[p]) * rstd[p] * g4.x + b4.x,
                                                (acc[p][0].y - mean[p]) * rstd[p] * g4.y + b4.y);
      __nv_bfloat162 hi = __floats2bfloat162_rn((acc[p][1].x - mean[p]) * rstd[p] * g4.z + b4.z,
                                                (acc[p][1].y - mean[p]) * rstd[p] * g4.w + b4.w);
      uint2 t;
      t.x = *reinterpret_cast<uint32_t*>(&lo);
      t.y = *reinterpret_cast<uint32_t*>(&hi);
      *reinterpret_cast<uint2*>(dst) = t;
    }
  }
  if (nchunks > 1) cluster_wait();  // no CTA of the cluster leaves while a peer may still read its shared memory
}

// ------------------------------------------------------------------------------------------------
// the same operator, PERSISTENT and software-pipelined (the default): latency was the limiter of the kernel above
// ------------------------------------------------------------------------------------------------
// The one-tile-per-CTA kernel above is limited by latency, not by the FP32 pipe: every CTA pays tensormap prefetch + barrier init + a 43 KB TMA load + 25 KB of tap
// staging + a cluster barrier + remote partial reads, with nothing to overlap them but two sibling CTAs in the same phase.
// Here a CTA lives for the whole launch and keeps ONE channel chunk: the chunk's taps / bias / LayerNorm affine are staged
// once, a producer warp streams halo tiles (TH x 7 output pixels) through a two-deep TMA / mbarrier ring, TH compute warps
// (one output row each) run the tap loop of tile i+1 while the LayerNorm statistics of tile i cross the cluster
// (split-phase barrier.cluster: arrive after publishing the chunk's (mean, M2), wait only after the next tile's taps).
// LayerNorm numerics are unchanged: two-pass statistics per chunk, Chan's combination across the chunks of a pixel.
template <int CHUNK, int TH>
__global__ void __launch_bounds__((TH + 1) * 32, TH == 7 ? 2 : 1)
dwconv7_pipe_kernel(const __grid_constant__ CUtensorMap map_x, int B, int H, int W, int C, int nchunks, int n_tiles,
                    const float* __restrict__ w49, const float* __restrict__ bias, const float* __restrict__ ln_w,
                    const float* __restrict__ ln_b, float eps, __nv_bfloat16* __restrict__ y, float* __restrict__ rstd_out) {
  extern __shared__ uint8_t dwp_smem_raw[];
  uint8_t* smem = dwp_smem_raw + ((128u - (smem_u32(dwp_smem_raw) & 127u)) & 127u);
  constexpr int box_w = kDwTW + 6, box_h = TH + 6;
  constexpr int tile_bytes = box_h * box_w * CHUNK * 2;
  constexpr int tile_stride = (tile_bytes + 127) & ~127;
  float* wsm = reinterpret_cast<float*>(smem + 2 * tile_stride);   // [49][CHUNK] taps of this chunk
  float2* part = reinterpret_cast<float2*>(wsm + 49 * CHUNK);     // [2 tile parities][TH rows][8]: (mean, M2) per pixel
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(part + 2 * TH * 8);
  uint64_t* empty_bar = full_bar + 2;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ck = blockIdx.x % nchunks;  // == rank inside the cluster (nchunks > 1)
  const int group = blockIdx.x / nchunks, n_groups = gridDim.x / nchunks;
  const int tiles_w = (W + kDwTW - 1) / kDwTW, tiles_h = (H + TH - 1) / TH;
  const int n_my = group < n_tiles ? (n_tiles - group + n_groups - 1) / n_groups : 0;
  const bool clustered = nchunks > 1;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_x);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], TH);
    }
    fence_mbar_init();
  }
  for (int i = threadIdx.x; i < 49 * (CHUNK / 4); i += blockDim.x) {
    const int t = i / (CHUNK / 4), q = i - t * (CHUNK / 4);
    *reinterpret_cast<float4*>(wsm + t * CHUNK + q * 4) = __ldg(reinterpret_cast<const float4*>(w49 + t * C + ck * CHUNK + q * 4));
  }
  __syncthreads();

  auto tile_coords = [&](int it, int& b, int& oy0, int& ox0) {
    int t = group + it * n_groups;
    const int tw = t % tiles_w;
    t /= tiles_w;
    const int th = t % tiles_h;
    b = t / tiles_h;
    oy0 = th * TH;
    ox0 = tw * kDwTW;
  };

  if (warp == TH) {
    // ===================== producer: one tile ahead of the compute warps =====================
    if (lane == 0 && n_my > 0) {
      int b, oy0, ox0;
      tile_coords(0, b, oy0, ox0);
      mbar_arrive_expect_tx(&full_bar[0], tile_bytes);
      tma_load_4d(smem, &map_x, &full_bar[0], ck * CHUNK, ox0 - 3, oy0 - 3, b);
    }
    for (int it = 0; it < n_my; ++it) {
      if (lane == 0 && it + 1 < n_my) {
        const int j = it + 1, buf = j & 1;
        mbar_wait_relaxed(&empty_bar[buf], ((j >> 1) & 1) ^ 1);  // the tap loops of tile j - 2 are done with this buffer
        int b, oy0, ox0;
        tile_coords(j, b, oy0, ox0);
        mbar_arrive_expect_tx(&full_bar[buf], tile_bytes);
        tma_load_4d(smem + buf * tile_stride, &map_x, &full_bar[buf], ck * CHUNK, ox0 - 3, oy0 - 3, b);
      }
      if (clustered) {  // every thread of the cluster takes part in the per-tile barrier
        __syncwarp();
        cluster_arrive();
        cluster_wait();
      }
    }
    if (clustered) {
      __syncwarp();
      cluster_arrive();
      cluster_wait();
    }
    return;
  }

  // ===================== compute warps: warp w owns output row w of every tile =====================
  const int cl = lane * 4;
  const bool has_c = cl < CHUNK;
  const int c0 = ck * CHUNK + cl;
  float4 bc = make_float4(0.f, 0.f, 0.f, 0.f), g4 = bc, b4 = bc;
  if (has_c) {
    bc = __ldg(reinterpret_cast<const float4*>(bias + c0));
    g4 = __ldg(reinterpret_cast<const float4*>(ln_w + c0));
    b4 = __ldg(reinterpret_cast<const float4*>(ln_b + c0));
  }
  constexpr int pix_stride = CHUNK * 2;
  const float inv_chunk = 1.0f / static_cast<float>(CHUNK), inv_c = 1.0f / static_cast<float>(C);

  // tap loop of one tile row: acc[p] = bias + sum over the 7x7 window (FMAs over channel pairs)
  auto conv_row = [&](const uint8_t* tile, float2 (&acc)[kDwTW][2]) {
#pragma unroll
    for (int p = 0; p < kDwTW; ++p) {
      acc[p][0] = make_float2(bc.x, bc.y);
      acc[p][1] = make_float2(bc.z, bc.w);
    }
    const uint8_t* tbase = tile + cl * 2;
#pragma unroll 1
    for (int dy = 0; dy < 7; ++dy) {
      float2 wlo[7], whi[7];
      const float* wrow = wsm + dy * (7 * CHUNK) + cl;
#pragma unroll
      for (int dx = 0; dx < 7; ++dx) {
        const float4 t = *reinterpret_cast<const float4*>(wrow + dx * CHUNK);
        wlo[dx] = make_float2(t.x, t.y);
        whi[dx] = make_float2(t.z, t.w);
      }
      const uint8_t* rowp = tbase + (warp + dy) * (box_w * pix_stride);
#pragma unroll
      for (int ix = 0; ix < box_w; ++ix) {
        const uint2 t = *reinterpret_cast<const uint2*>(rowp + ix * pix_stride);
        const float2 a = make_float2(__uint_as_float(t.x << 16), __uint_as_float(t.x & 0xffff0000u));
        const float2 c = make_float2(__uint_as_float(t.y << 16), __uint_as_float(t.y & 0xffff0000u));
#pragma unroll
        for (int p = 0; p < kDwTW; ++p) {
          const int dx = ix - p;
          if (dx >= 0 && dx < 7) {
            acc[p][0] = ffma2(a, wlo[dx], acc[p][0]);
            acc[p][1] = ffma2(c, whi[dx], acc[p][1]);
          }
        }
      }
    }
  };

  // ---- conv + bias + LayerNorm over C, statistics exchanged across the cluster one tile behind the tap loop ----
  float2 acc[kDwTW][2];     // tile whose LayerNorm is pending
  float mean[kDwTW], m2[kDwTW];
  int pb = 0, poy0 = 0, pox0 = 0;
  bool pactive = false;

  auto local_stats = [&](bool active, int parity) {  // two-pass (mean, centred sum of squares) of this chunk, published for the peers
#pragma unroll
    for (int p = 0; p < kDwTW; ++p)
      mean[p] = warp_sum(active ? (acc[p][0].x + acc[p][0].y) + (acc[p][1].x + acc[p][1].y) : 0.f) * inv_chunk;
#pragma unroll
    for (int p = 0; p < kDwTW; ++p) {
      float q = 0.f;
      if (active) {
        const float d0 = acc[p][0].x - mean[p], d1 = acc[p][0].y - mean[p];
        const float d2 = acc[p][1].x - mean[p], d3 = acc[p][1].y - mean[p];
        q = fmaf(d0, d0, fmaf(d1, d1, fmaf(d2, d2, d3 * d3)));
      }
      m2[p] = warp_sum(q);
    }
    if (clustered) {
      float2 mine = make_float2(0.f, 0.f);
#pragma unroll
      for (int p = 0; p < kDwTW; ++p)
        if (lane == p) mine = make_float2(mean[p], m2[p]);
      if (lane < kDwTW) part[(parity * TH + warp) * 8 + lane] = mine;
    }
  };

  auto finish = [&](int parity) {  // combine the chunks' statistics (Chan), normalise, store the pending tile
    float rstd[kDwTW];
    if (clustered) {
      float2 r[kDwTW];
#pragma unroll
      for (int p = 0; p < kDwTW; ++p) {
        r[p] = make_float2(0.f, 0.f);
        if (lane < nchunks) r[p] = ld_dsmem_f2(part + (parity * TH + warp) * 8 + p, static_cast<uint32_t>(lane));
      }
      const float inv_n = 1.0f / static_cast<float>(nchunks);
#pragma unroll
      for (int p = 0; p < kDwTW; ++p) {
        const float m = warp_sum(r[p].x) * inv_n;
        const float d = r[p].x - m;
        const float q = warp_sum(lane < nchunks ? fmaf(static_cast<float>(CHUNK) * d, d, r[p].y) : 0.f);
        mean[p] = m;
        rstd[p] = rsqrtf(q * inv_c + eps);
      }
    } else {
#pragma unroll
      for (int p = 0; p < kDwTW; ++p) rstd[p] = rsqrtf(m2[p] * inv_c + eps);
    }
    if (pactive) {
#pragma unroll
      for (int p = 0; p < kDwTW; ++p) {
        const int ox = pox0 + p;
        if (ox >= W) continue;
        const int64_t pix = (static_cast<int64_t>(pb) * H + poy0 + warp) * W + ox;
        if (rstd_out != nullptr && lane == 0 && ck == 0) rstd_out[pix] = rstd[p];
        __nv_bfloat16* dst = y + pix * C + c0;
        __nv_bfloat162 lo = __floats2bfloat162_rn((acc[p][0].x - mean[p]) * rstd[p] * g4.x + b4.x,
                                                  (acc[p][0].y - mean[p]) * rstd[p] * g4.y + b4.y);
        __nv_bfloat162 hi = __floats2bfloat162_rn((acc[p][1].x - mean[p]) * rstd[p] * g4.z + b4.z,
                                                  (acc[p][1].y - mean[p]) * rstd[p] * g4.w + b4.w);
        uint2 t;
        t.x = *reinterpret_cast<uint32_t*>(&lo);
        t.y = *reinterpret_cast<uint32_t*>(&hi);
        *reinterpret_cast<uint2*>(dst) = t;
      }
    }
  };

  for (int it = 0; it < n_my; ++it) {
    const int buf = it & 1;
    int b, oy0, ox0;
    tile_coords(it, b, oy0, ox0);
    const bool active = has_c && oy0 + warp < H;
    float2 nxt[kDwTW][2];
    mbar_wait(&full_bar[buf], (it >> 1) & 1);
    if (active) conv_row(smem + buf * tile_stride, nxt);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[buf]);
    if (it > 0) {  // the previous tile: its statistics have had a whole tap loop to cross the cluster
      if (clustered) cluster_wait();
      finish((it - 1) & 1);
    }
#pragma unroll
    for (int p = 0; p < kDwTW; ++p) {
      acc[p][0] = nxt[p][0];
      acc[p][1] = nxt[p][1];
    }
    pb = b; poy0 = oy0; pox0 = ox0; pactive = active;
    local_stats(active, buf);
    if (clustered) cluster_arrive();
  }
  if (n_my > 0) {
    if (clustered) cluster_wait();
    finish((n_my - 1) & 1);
  }
  if (clustered) {  // no CTA of the cluster leaves while a peer may still read its partials
    cluster_arrive();
    cluster_wait();
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm over C of NHWC rows, optionally scattered into 2x2/stride-2 patch rows (kh, kw, c)
// ------------------------------------------------------------------------------------------------
template <int LPP>  // lanes per pixel (8, 16 or 32); each lane owns 8-channel (16-byte) vectors c = (sub + i*LPP)*8
__global__ void __launch_bounds__(256)
ln_patchify_kernel(const __nv_bfloat16* __restrict__ x, int B, int H, int W, int C, const float* __restrict__ ln_w,
                   const float* __restrict__ ln_b, float eps, int patch /*1 or 2*/, __nv_bfloat16* __restrict__ out,
                   float* __restrict__ rstd_out) {
  constexpr int kPPW = 32 / LPP;  // pixels per warp
  constexpr int kMaxIter = 8;     // C <= LPP * 8 * kMaxIter
  const int lane = threadIdx.x & 31;
  const int sub = lane % LPP;
  const int64_t warp_id = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int64_t pix = warp_id * kPPW + lane / LPP;
  const int64_t npix = static_cast<int64_t>(B) * H * W;
  const bool ok = pix < npix;
  const __nv_bfloat16* src = x + (ok ? pix : 0) * C;
  const int iters = (C + LPP * 8 - 1) / (LPP * 8);
  float v[kMaxIter][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxIter; ++i) {
    if (i < iters) {
      const int c = (sub + i * LPP) * 8;
      uint4 t = make_uint4(0, 0, 0, 0);
      if (ok && c < C) t = *reinterpret_cast<const uint4*>(src + c);
      const float2 a0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.x));
      const float2 a1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.y));
      const float2 a2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.z));
      const float2 a3 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.w));
      v[i][0] = a0.x; v[i][1] = a0.y; v[i][2] = a1.x; v[i][3] = a1.y;
      v[i][4] = a2.x; v[i][5] = a2.y; v[i][6] = a3.x; v[i][7] = a3.y;
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[i][j];
    }
  }
#pragma unroll
  for (int off = LPP / 2; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  const float mean = s / static_cast<float>(C);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxIter; ++i) {
    if (i < iters && (sub + i * LPP) * 8 < C) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[i][j] - mean;
        q = fmaf(d, d, q);
      }
    }
  }
#pragma unroll
  for (int off = LPP / 2; off > 0; off >>= 1) q += __shfl_xor_sync(0xffffffffu, q, off);
  const float rstd = rsqrtf(q / static_cast<float>(C) + eps);
  if (!ok) return;
  if (rstd_out != nullptr && sub == 0) rstd_out[pix] = rstd;
  int64_t orow;
  int ocol0;
  if (patch == 2) {
    const int xw = static_cast<int>(pix % W);
    const int yh = static_cast<int>((pix / W) % H);
    const int b = static_cast<int>(pix / (static_cast<int64_t>(W) * H));
    orow = (static_cast<int64_t>(b) * (H / 2) + (yh >> 1)) * (W / 2) + (xw >> 1);
    ocol0 = ((yh & 1) * 2 + (xw & 1)) * C;
  } else {
    orow = pix;
    ocol0 = 0;
  }
  __nv_bfloat16* dst = out + orow * (static_cast<int64_t>(C) * patch * patch) + ocol0;
#pragma unroll
  for (int i = 0; i < kMaxIter; ++i) {
    const int c = (sub + i * LPP) * 8;
    if (i < iters && c < C) {
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(ln_w + c)), g1 = __ldg(reinterpret_cast<const float4*>(ln_w + c + 4));
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(ln_b + c)), b1 = __ldg(reinterpret_cast<const float4*>(ln_b + c + 4));
      __nv_bfloat162 o0 = __floats2bfloat162_rn((v[i][0] - mean) * rstd * g0.x + b0.x, (v[i][1] - mean) * rstd * g0.y + b0.y);
      __nv_bfloat162 o1 = __floats2bfloat162_rn((v[i][2] - mean) * rstd * g0.z + b0.z, (v[i][3] - mean) * rstd * g0.w + b0.w);
      __nv_bfloat162 o2 = __floats2bfloat162_rn((v[i][4] - mean) * rstd * g1.x + b1.x, (v[i][5] - mean) * rstd * g1.y + b1.y);
      __nv_bfloat162 o3 = __floats2bfloat162_rn((v[i][6] - mean) * rstd * g1.z + b1.z, (v[i][7] - mean) * rstd * g1.w + b1.w);
      uint4 t;
      t.x = *reinterpret_cast<uint32_t*>(&o0); t.y = *reinterpret_cast<uint32_t*>(&o1);
      t.z = *reinterpret_cast<uint32_t*>(&o2); t.w = *reinterpret_cast<uint32_t*>(&o3);
      *reinterpret_cast<uint4*>(dst + c) = t;
    }
  }
}

int launch_ln_patchify(const __nv_bfloat16* x, int B, int H, int W, int C, const float* ln_w, const float* ln_b, float eps,
                       int patch, __nv_bfloat16* out, float* rstd_out, cudaStream_t s) {
  VDK_REQUIRE(C % 8 == 0 && C <= 2048, "layernorm_patchify: C must be a multiple of 8, <= 2048 (got %d)", C);
  const int64_t npix = static_cast<int64_t>(B) * H * W;
  const int vecs = C / 8;
  if (vecs <= 8) {
    const int64_t warps = (npix + 3) / 4;
    ln_patchify_kernel<8><<<static_cast<unsigned>((warps * 32 + 255) / 256), 256, 0, s>>>(x, B, H, W, C, ln_w, ln_b, eps, patch, out, rstd_out);
  } else if (vecs <= 16) {
    const int64_t warps = (npix + 1) / 2;
    ln_patchify_kernel<16><<<static_cast<unsigned>((warps * 32 + 255) / 256), 256, 0, s>>>(x, B, H, W, C, ln_w, ln_b, eps, patch, out, rstd_out);
  } else {
    ln_patchify_kernel<32><<<static_cast<unsigned>((npix * 32 + 255) / 256), 256, 0, s>>>(x, B, H, W, C, ln_w, ln_b, eps, patch, out, rstd_out);
  }
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

// ------------------------------------------------------------------------------------------------
// neck finalize: split-K partial sums + folded bias -> embedding rows (optionally L2-normalised)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
neck_finalize_kernel(const float* __restrict__ acc, int n_slabs, size_t slab_stride, int B, int F,
                     const float* __restrict__ bias, int l2norm, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= B) return;
  double ss = 0.0;
  // the canonical F.normalize of retrieval.cu: fixed-order fp64 sum of squares (lane-strided, xor butterfly)
  // split-K slabs are added in slab order: the embedding is bitwise reproducible run to run
  for (int i = lane; i < F; i += 32) {
    float v = bias[i];
    for (int sl = 0; sl < n_slabs; ++sl) v += acc[sl * slab_stride + static_cast<size_t>(row) * F + i];
    out[static_cast<size_t>(row) * F + i] = v;
    ss = fma(static_cast<double>(v), static_cast<double>(v), ss);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, off);
  const float denom = l2norm ? fmaxf(static_cast<float>(sqrt(ss)), 1e-12f) : 1.0f;
  if (l2norm)
    for (int i = lane; i < F; i += 32) out[static_cast<size_t>(row) * F + i] = __fdiv_rn(out[static_cast<size_t>(row) * F + i], denom);
}

int launch_neck_finalize(const float* slabs, int n_slabs, size_t slab_stride, int B, int F, const float* bias, int l2norm,
                         float* out, cudaStream_t s) {
  neck_finalize_kernel<<<(B * 32 + 255) / 256, 256, 0, s>>>(slabs, n_slabs, slab_stride, B, F, bias, l2norm, out);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

int launch_neck(const __nv_bfloat16* feats, int batch, int Kn, int F, const void* neck_w, const float* neck_b, int l2_normalize,
                float* scratch, size_t scratch_bytes, float* embeddings, cudaStream_t s) {
  const int tiles = ((batch + 127) / 128) * ((F + 255) / 256);
  // split-K over ~2 waves of CTAs; every split writes its own fp32 slab into the scratch buffer and neck_finalize adds the
  // slabs in order, so the embedding is bitwise reproducible
  const size_t slab = static_cast<size_t>(batch) * F;
  int split = std::max(1, (2 * sm_count()) / std::max(1, tiles));
  split = static_cast<int>(std::min<size_t>(split, scratch_bytes / (slab * sizeof(float))));
  split = vdk_gemm_effective_splits(Kn, std::max(1, split));
  {
    vdk_gemm_desc g{};
    g.A = feats; g.B = neck_w; g.D = scratch;
    g.M = batch; g.N = F; g.K = Kn; g.lda = Kn; g.ldb = Kn; g.ldd = F;
    g.in_dtype = VDK_DTYPE_BF16; g.out_dtype = VDK_DTYPE_FP32; g.epilogue = VDK_EPI_NONE;
    g.split_k = split;
    g.split_stride = split > 1 ? static_cast<long long>(slab) : 0;
    const int rc = gemm_run(g, s);
    if (rc != VDK_OK) return rc;
  }
  neck_finalize_kernel<<<(batch * 32 + 255) / 256, 256, 0, s>>>(scratch, split, slab, batch, F, neck_b, l2_normalize, embeddings);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

static int check_net(const vdk_convnext_net* n) {
  VDK_REQUIRE(n, "vdk_convnext: null network");
  VDK_REQUIRE(n->image_size > 0 && n->image_size % 32 == 0, "vdk_convnext: image_size must be a multiple of 32");
  VDK_REQUIRE(n->feat_dim > 0 && n->feat_dim % 8 == 0, "vdk_convnext: feat_dim must be a multiple of 8");
  int nb = 0;
  for (int s = 0; s < 4; ++s) {
    VDK_REQUIRE(n->dims[s] > 0 && n->dims[s] % 8 == 0 && n->dims[s] <= 2048, "vdk_convnext: dims must be multiples of 8, <= 2048");
    VDK_REQUIRE(n->depths[s] >= 0, "vdk_convnext: bad depth");
    nb += n->depths[s];
  }
  VDK_REQUIRE(nb <= VDK_CONVNEXT_MAX_BLOCKS, "vdk_convnext: too many blocks (%d)", nb);
  VDK_REQUIRE(n->dims[0] <= 256, "vdk_convnext: stem width must be <= 256 (LayerNorm epilogue tile)");
  return VDK_OK;
}

}  // namespace vdk

using namespace vdk;

template <int TW>
static int launch_dwconv_tw(const CUtensorMap& mx, int batch, int H, int W, int C, int TH, int box_c, const float* w49,
                            const float* bias, const float* ln_w, const float* ln_b, float eps, __nv_bfloat16* y,
                            float* rstd_out, cudaStream_t s) {
  const int tpg = ((C / 4) + 31) / 32 * 32;
  const int groups = std::max(1, std::min(512 / tpg, TH));
  const int n_chunks = C / box_c;
  const int smem = n_chunks * (((TH + 6) * (TW + 6) * box_c * 2 + 127) & ~127) + 16 * TW * 16 * 4 + 16 + 128;
  auto kern = dwconv7_ln_kernel<TW>;
  VDK_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  const unsigned grid = static_cast<unsigned>(batch) * ((H + TH - 1) / TH) * ((W + TW - 1) / TW);
  kern<<<grid, groups * tpg, smem, s>>>(mx, batch, H, W, C, TH, box_c, tpg, w49, bias, ln_w, ln_b, eps, y, rstd_out);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}


// Persistent launch: one CTA per SM (two for the 7-row tile), grid = co-resident clusters x chunks.
template <int CHUNK, int TH>
static int launch_dwconv7_pipe_t(const __nv_bfloat16* x, int batch, int H, int W, int C, const float* w49, const float* bias,
                                 const float* ln_w, const float* ln_b, float eps, __nv_bfloat16* y, float* rstd_out,
                                 cudaStream_t s) {
  const int nchunks = C / CHUNK;
  constexpr int tile_stride = ((TH + 6) * (kDwTW + 6) * CHUNK * 2 + 127) & ~127;
  constexpr int smem = 2 * tile_stride + 49 * CHUNK * 4 + 2 * TH * 8 * 8 + 4 * 8 + 128;
  static_assert(smem <= 227 * 1024, "dwconv7_pipe shared memory budget");
  CUtensorMap mx;
  int rc = make_tma_nhwc_16bit(&mx, x, batch, H, W, C, TH + 6, kDwTW + 6, CHUNK);
  if (rc != VDK_OK) return rc;
  auto kern = dwconv7_pipe_kernel<CHUNK, TH>;
  const int cluster = nchunks;
  struct Fit { int clusters; };
  static Fit fit[17] = {};  // per cluster size: co-resident clusters of this instantiation (queried once)
  cudaLaunchConfig_t cfg{};
  cfg.blockDim = dim3((TH + 1) * 32);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (fit[cluster].clusters == 0) {
    VDK_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    if (cluster > 8) VDK_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    cfg.gridDim = dim3(cluster * sm_count());
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess || n <= 0) {
      cudaGetLastError();
      fit[cluster].clusters = -1;
    } else {
      fit[cluster].clusters = n;
    }
  }
  if (fit[cluster].clusters < 0) return VDK_ERR_WORKSPACE;
  const int n_tiles = batch * ((H + TH - 1) / TH) * ((W + kDwTW - 1) / kDwTW);
  const int groups = std::min(n_tiles, fit[cluster].clusters);
  cfg.gridDim = dim3(static_cast<unsigned>(groups) * nchunks);
  VDK_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, mx, batch, H, W, C, nchunks, n_tiles, w49, bias, ln_w, ln_b, eps, y, rstd_out));
  return VDK_OK;
}

static int launch_dwconv7_pipe(const __nv_bfloat16* x, int batch, int H, int W, int C, int chunk, const float* w49,
                               const float* bias, const float* ln_w, const float* ln_b, float eps, __nv_bfloat16* y, float* rstd_out,
                               cudaStream_t s) {
  const bool tall = H > 7;  // 14-row tiles (15 warps, one CTA per SM) unless the map is 7 rows high
#define VDK_DWP(CHV)                                                                                                                  \
  return tall ? launch_dwconv7_pipe_t<CHV, 14>(x, batch, H, W, C, w49, bias, ln_w, ln_b, eps, y, rstd_out, s)                         \
              : launch_dwconv7_pipe_t<CHV, 7>(x, batch, H, W, C, w49, bias, ln_w, ln_b, eps, y, rstd_out, s)
  if (chunk == 128) { VDK_DWP(128); }
  if (chunk == 96) { VDK_DWP(96); }
  VDK_DWP(64);
#undef VDK_DWP
}

// mode 0: forward conv + bias + LayerNorm (rstd_out optional); mode 1: plain conv with `w49` (+ addend), the depthwise
// backward-data pass (dwconv7_bwd_kernel with its weight-gradient half off)
int vdk::launch_dwconv7(int mode, const __nv_bfloat16* x, int batch, int H, int W, int C, const float* w49, const float* bias,
                          const float* ln_w, const float* ln_b, float eps, __nv_bfloat16* y, float* rstd_out,
                          const __nv_bfloat16* addend, cudaStream_t s) {
  VDK_REQUIRE(C % 8 == 0 && C <= 2048, "dwconv7: C must be a multiple of 8, <= 2048 (got %d)", C);
  if (mode == 1) return launch_dwconv7_bwd(nullptr, x, batch, H, W, C, w49, addend, y, nullptr, nullptr, s);
  const double dw_elems = static_cast<double>(batch) * H * W * C;
  ProfScope prof(kProfDepthwise, 2.0 * 49.0 * dw_elems, 2.0 * dw_elems * 2.0, s);  // read x, write y
  {
    // channel-chunked kernel (clustered LayerNorm) whenever C splits into <= 16 chunks of <= 128 channels
    int chunk = 0;
    if (C % 128 == 0) chunk = 128;
    else if (C % 96 == 0) chunk = 96;
    else if (C % 64 == 0) chunk = 64;
    // VDK_DWCONV_PIPE=0 runs the one-tile-per-CTA chunk kernel below, which otherwise runs only where the persistent grid does
    // not fit the device: the switch lets the tests reach that fallback
    static const bool use_pipe = [] {
      const char* e = getenv("VDK_DWCONV_PIPE");
      return e ? atoi(e) != 0 : true;
    }();
    if (use_pipe && chunk > 0 && C / chunk <= 16) {
      const int rc = launch_dwconv7_pipe(x, batch, H, W, C, chunk, w49, bias, ln_w, ln_b, eps, y, rstd_out, s);
      if (rc != VDK_ERR_WORKSPACE) return rc;  // VDK_ERR_WORKSPACE: the persistent grid does not fit this device -> fall through
    }
    if (chunk > 0 && C / chunk <= 16) {
      const int nchunks = C / chunk;
      const int TH = std::min(7, H);
      CUtensorMap mx;
      int rc = make_tma_nhwc_16bit(&mx, x, batch, H, W, C, TH + 6, kDwTW + 6, chunk);
      if (rc != VDK_OK) return rc;
      const int smem = (((TH + 6) * (kDwTW + 6) * chunk * 2 + 127) & ~127) + 49 * chunk * 4 + 7 * 8 * 8 + 16 + 128;
      const unsigned grid = static_cast<unsigned>(batch) * ((H + TH - 1) / TH) * ((W + kDwTW - 1) / kDwTW) * nchunks;
      cudaLaunchConfig_t cfg{};
      cfg.gridDim = dim3(grid);
      cfg.blockDim = dim3(32 * TH);
      cfg.dynamicSmemBytes = smem;
      cfg.stream = s;
      cudaLaunchAttribute attr[1];
      attr[0].id = cudaLaunchAttributeClusterDimension;
      attr[0].val.clusterDim.x = nchunks;
      attr[0].val.clusterDim.y = 1;
      attr[0].val.clusterDim.z = 1;
      cfg.attrs = attr;
      cfg.numAttrs = 1;
#define VDK_DWC(CHV)                                                                                                     \
  do {                                                                                                                   \
    auto kern = dwconv7_chunk_kernel<CHV>;                                                                               \
    VDK_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024));                     \
    if (nchunks > 8) VDK_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));         \
    VDK_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, mx, batch, H, W, C, TH, nchunks, w49, bias, ln_w, ln_b, eps, y, rstd_out)); \
  } while (0)
      if (chunk == 128) VDK_DWC(128);
      else if (chunk == 96) VDK_DWC(96);
      else VDK_DWC(64);
#undef VDK_DWC
      return VDK_OK;
    }
  }
  // channel chunk of one TMA box: the largest divisor of C that is <= 256 and a multiple of 8
  int box_c = std::min(C, 256);
  while (C % box_c != 0 || box_c % 8 != 0) --box_c;
  // spatial tile: the largest of 7 / 4 / 2 whose halo (T+6)^2 x C x 2 B fits in ~200 KB of shared memory
  int T = 7;
  while (T > 2 && (T + 6) * (T + 6) * C * 2 > 200 * 1024) T = (T == 7) ? 4 : 2;
  VDK_REQUIRE((T + 6) * (T + 6) * C * 2 <= 200 * 1024, "dwconv7: C too large for the shared-memory halo (%d)", C);
  const int TH = std::min(T, H);
  CUtensorMap mx;
  int rc = make_tma_nhwc_16bit(&mx, x, batch, H, W, C, TH + 6, T + 6, box_c);
  if (rc != VDK_OK) return rc;
  if (T == 7) return launch_dwconv_tw<7>(mx, batch, H, W, C, TH, box_c, w49, bias, ln_w, ln_b, eps, y, rstd_out, s);
  if (T == 4) return launch_dwconv_tw<4>(mx, batch, H, W, C, TH, box_c, w49, bias, ln_w, ln_b, eps, y, rstd_out, s);
  return launch_dwconv_tw<2>(mx, batch, H, W, C, TH, box_c, w49, bias, ln_w, ln_b, eps, y, rstd_out, s);
}

static int launch_dwconv7_ln(const __nv_bfloat16* x, int batch, int H, int W, int C, const float* w49, const float* bias,
                             const float* ln_w, const float* ln_b, float eps, __nv_bfloat16* y, cudaStream_t s) {
  return launch_dwconv7(0, x, batch, H, W, C, w49, bias, ln_w, ln_b, eps, y, nullptr, nullptr, s);
}

extern "C" int vdk_dwconv7_ln(const void* x, int batch, int H, int W, int C, const float* w49, const float* bias,
                              const float* ln_w, const float* ln_b, float eps, void* y, void* stream) {
  VDK_REQUIRE(x && y && w49 && bias && ln_w && ln_b, "vdk_dwconv7_ln: null operand");
  VDK_REQUIRE(batch > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, "vdk_dwconv7_ln: bad shape (C must be a multiple of 8)");
  return launch_dwconv7_ln(reinterpret_cast<const __nv_bfloat16*>(x), batch, H, W, C, w49, bias, ln_w, ln_b, eps,
                           reinterpret_cast<__nv_bfloat16*>(y), reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vdk_layernorm_patchify(const void* x, int batch, int H, int W, int C, const float* ln_w,
                                      const float* ln_b, float eps, int patch, void* out, void* stream) {
  VDK_REQUIRE(x && out && ln_w && ln_b, "vdk_layernorm_patchify: null operand");
  VDK_REQUIRE(batch > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && C <= 2048, "vdk_layernorm_patchify: bad shape");
  VDK_REQUIRE(patch == 1 || (patch == 2 && H % 2 == 0 && W % 2 == 0), "vdk_layernorm_patchify: patch must be 1 or 2");
  return launch_ln_patchify(reinterpret_cast<const __nv_bfloat16*>(x), batch, H, W, C, ln_w, ln_b, eps, patch,
                            reinterpret_cast<__nv_bfloat16*>(out), nullptr, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" size_t vdk_convnext_workspace_bytes(const vdk_convnext_net* net, int batch) {
  if (!net || batch <= 0) return 0;
  const size_t hw0 = static_cast<size_t>(net->image_size / 4) * (net->image_size / 4);
  size_t max_mc = 0, max_m4c = 0;
  size_t hw = hw0;
  for (int s = 0; s < 4; ++s) {
    if (s > 0) hw /= 4;
    const size_t m = static_cast<size_t>(batch) * hw;
    max_mc = std::max(max_mc, m * net->dims[s]);
    max_m4c = std::max(max_m4c, m * net->dims[s] * 4);
  }
  const size_t patches = static_cast<size_t>(batch) * hw0 * 48;
  // x (residual stream), y (dwconv+LN / patch rows), h (hidden 4C or stem patches), neck accumulators
  return up256(max_mc * 2) * 2 + up256(std::max(max_m4c, patches) * 2) + up256(static_cast<size_t>(batch) * net->feat_dim * 4) + 1024;
}

extern "C" int vdk_convnext_forward(const vdk_convnext_net* net, const float* images, int batch, int l2_normalize,
                                    float* embeddings, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_net(net);
  if (rc != VDK_OK) return rc;
  VDK_REQUIRE(images && embeddings && batch > 0, "vdk_convnext_forward: null image/embedding buffer");
  VDK_REQUIRE(workspace && workspace_bytes >= vdk_convnext_workspace_bytes(net, batch),
              "vdk_convnext_forward: workspace too small");
  VDK_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0 && (reinterpret_cast<uintptr_t>(images) & 15) == 0,
              "vdk_convnext_forward: workspace must be 256-byte and images 16-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int S = net->image_size;
  const size_t hw0 = static_cast<size_t>(S / 4) * (S / 4);
  size_t max_mc = 0, max_m4c = 0, hwt = hw0;
  for (int st = 0; st < 4; ++st) {
    if (st > 0) hwt /= 4;
    max_mc = std::max(max_mc, static_cast<size_t>(batch) * hwt * net->dims[st]);
    max_m4c = std::max(max_m4c, static_cast<size_t>(batch) * hwt * net->dims[st] * 4);
  }
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  __nv_bfloat16* xbuf = reinterpret_cast<__nv_bfloat16*>(ws);
  ws += up256(max_mc * 2);
  __nv_bfloat16* ybuf = reinterpret_cast<__nv_bfloat16*>(ws);
  ws += up256(max_mc * 2);
  __nv_bfloat16* hbuf = reinterpret_cast<__nv_bfloat16*>(ws);
  ws += up256(std::max(max_m4c, static_cast<size_t>(batch) * hw0 * 48) * 2);
  (void)ws;

  auto gemm = [&](const void* A, const void* Bw, void* D, int M, int N, int K, int epi, const float* bias,
                  const float* gamma, const float* beta, const void* res, int out_dtype, int split) -> int {
    vdk_gemm_desc g{};
    g.A = A; g.B = Bw; g.D = D;
    g.M = M; g.N = N; g.K = K; g.lda = K; g.ldb = K; g.ldd = N;
    g.in_dtype = VDK_DTYPE_BF16; g.out_dtype = out_dtype; g.epilogue = epi;
    g.bias = bias; g.gamma = gamma; g.beta = beta; g.residual = res; g.ldr = N;
    g.ln_eps = 1e-6f; g.split_k = split;
    return gemm_run(g, s);
  };

  // ---- stem: conv4x4/s4 as a GEMM over patch rows, + bias + LayerNorm2d in the epilogue ----
  int H = S / 4, W = S / 4, C = net->dims[0];
  int M = batch * H * W;
  {
    if ((rc = launch_stem_patchify(images, batch, S, hbuf, s)) != VDK_OK) return rc;
    rc = gemm(hbuf, net->stem_w, xbuf, M, C, 48, VDK_EPI_LAYERNORM, net->stem_b, net->stem_ln_w, net->stem_ln_b, nullptr,
              VDK_DTYPE_BF16, 1);
    if (rc != VDK_OK) return rc;
  }
  int blk = 0;
  for (int st = 0; st < 4; ++st) {
    if (st > 0) {
      // ---- downsample: LayerNorm2d then conv2x2/s2 as a GEMM over (kh, kw, c) patch rows ----
      const vdk_convnext_down* d = &net->down[st];
      const int Cin = C;
      rc = launch_ln_patchify(xbuf, batch, H, W, Cin, d->ln_w, d->ln_b, 1e-6f, 2, ybuf, nullptr, s);
      if (rc != VDK_OK) return rc;
      H /= 2; W /= 2; C = net->dims[st];
      M = batch * H * W;
      rc = gemm(ybuf, d->conv_w, xbuf, M, C, 4 * Cin, VDK_EPI_NONE, d->conv_b, nullptr, nullptr, nullptr, VDK_DTYPE_BF16, 1);
      if (rc != VDK_OK) return rc;
    }
    for (int j = 0; j < net->depths[st]; ++j, ++blk) {
      const vdk_convnext_block* b = &net->blocks[blk];
      rc = launch_dwconv7_ln(xbuf, batch, H, W, C, b->dw_w, b->dw_b, b->ln_w, b->ln_b, 1e-6f, ybuf, s);
      if (rc != VDK_OK) return rc;
      rc = gemm(ybuf, b->fc1_w, hbuf, M, 4 * C, C, VDK_EPI_GELU, b->fc1_b, nullptr, nullptr, nullptr, VDK_DTYPE_BF16, 1);
      if (rc != VDK_OK) return rc;
      rc = gemm(hbuf, b->fc2_w, xbuf, M, C, 4 * C, VDK_EPI_SCALE_RESIDUAL, b->fc2_b, b->gamma, nullptr, xbuf, VDK_DTYPE_BF16, 1);
      if (rc != VDK_OK) return rc;
    }
  }
  // ---- head LayerNorm2d (applied by timm even with global_pool='') ----
  {
    rc = launch_ln_patchify(xbuf, batch, H, W, C, net->head_ln_w, net->head_ln_b, 1e-6f, 1, ybuf, nullptr, s);
    if (rc != VDK_OK) return rc;
  }
  // ---- neck: BN2d -> Flatten -> Linear -> BN1d, all folded into one skinny GEMM (eval statistics) ----
  return launch_neck(ybuf, batch, H * W * C, net->feat_dim, net->neck_w, net->neck_b, l2_normalize,
                     reinterpret_cast<float*>(hbuf), up256(std::max(max_m4c, static_cast<size_t>(batch) * hw0 * 48) * 2),
                     embeddings, s);
}
