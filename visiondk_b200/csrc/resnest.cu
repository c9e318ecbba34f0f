// resnest.cu — timm 0.9.16 ResNeSt (resnest14d/26d/50d, resnest50d_1s4x24d, resnest50d_4s2x40d) embedding forward for
// the faceX / CBIR extract path, NHWC bf16, every eval BatchNorm folded into its convolution.
//
// Replaces TimmWrapper.forward for ResNeSt backbones (models/faceX/backbone/timm_wrapper.py:16-21, 30-38, 51-54) and
// F.normalize (face_model.py:139).  The deep stem, its max pool, the avg_down shortcuts and the neck are the ResNet-D
// path's pieces (resnet.cu, launch_neck); conv1 and the shortcut are vdk_conv2d, the split conv is vdk_conv2d_grouped_ex
// (gemm.cu, kConvGroupedEx), conv3 its groups = 1 form (Cin = gw, a multiple of 8).  Written here, all deterministic
// (fixed summation orders, no atomics):
//   radix_mean     gap[b, c] = mean_hw sum_r u[b, hw, r C + c] in fp32
//   attn_excite    fc1 (grouped, bn1 folded) + ReLU, fc2 (grouped) + bias, radix softmax / sigmoid, several images per CTA
//   radix_combine  v = sum_r a_r u_r in fp32 -> bf16, with avd_last's AvgPool2d(3, 2, 1) fused (the full-resolution
//                  combined map is never stored)
//   avgpool3s2     avd_first's AvgPool2d(3, 2, 1, count_include_pad=True) over NHWC bf16
#include "vdk_host.h"

#include <algorithm>
#include "convnext_internal.h"

namespace vdk {

namespace {

constexpr int kExciteImgs = 8;        // images per attn_excite CTA: each weight is read once per 8 images
constexpr int kExciteChannels = 256;  // output channels c (all R radix rows of each) per attn_excite CTA
constexpr int kMaxRadix = 4;

__device__ __forceinline__ void load8(const __nv_bfloat16* p, float* f) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 v = __bfloat1622float2(h[i]);
    f[2 * i] = v.x;
    f[2 * i + 1] = v.y;
  }
}

__device__ __forceinline__ void store8(__nv_bfloat16* p, const float* f) {
  uint4 o;
  uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
    ow[i] = *reinterpret_cast<uint32_t*>(&h);
  }
  *reinterpret_cast<uint4*>(p) = o;
}

// gap[b, c] = sum_p sum_r u[b, p, r C + c] / HW: block (64 channels, image b) of 256 threads = 8 channel vectors x 32 pixel
// lanes; lane l adds pixels l, l + 32, ... in order (each pixel's radix terms r = 0 .. R-1 in order), then a fixed tree
// over the 32 lanes (se_mean_kernel's order).
__global__ void __launch_bounds__(256) radix_mean_kernel(const __nv_bfloat16* __restrict__ u, int HW, int C, int R,
                                                         float* __restrict__ gap) {
  __shared__ float part[32][64];
  const int b = blockIdx.y, cv = threadIdx.x & 7, lane = threadIdx.x >> 3, c0 = blockIdx.x * 64 + cv * 8;
  const bool live = c0 < C;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  if (live) {
    const __nv_bfloat16* src = u + static_cast<int64_t>(b) * HW * R * C + c0;
    for (int p = lane; p < HW; p += 32) {
      for (int r = 0; r < R; ++r) {
        float f[8];
        load8(src + (static_cast<int64_t>(p) * R + r) * C, f);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] += f[i];
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) part[lane][cv * 8 + i] = acc[i];
  __syncthreads();
  for (int half = 16; half > 0; half >>= 1) {
    if (lane < half) {
#pragma unroll
      for (int i = 0; i < 8; ++i) part[lane][cv * 8 + i] += part[lane + half][cv * 8 + i];
    }
    __syncthreads();
  }
  if (lane == 0 && live) {
#pragma unroll
    for (int i = 0; i < 8; ++i) gap[static_cast<int64_t>(b) * C + c0 + i] = part[0][cv * 8 + i] / static_cast<float>(HW);
  }
}

// attn[b, r C + c] for kExciteImgs images (blockIdx.x) and kExciteChannels channels c (blockIdx.y), fp32:
//   hid[j] = ReLU(b1[j] + sum_k w1[j, k] gap[g Cg + k])              j in group g = j / Ag  (fc1 + bn1, cardinality groups)
//   z[r] = b2[n_r] + sum_k w2[n_r, k] hid[g Ag + k], n_r = g R Cg + r Cg + i   for c = g Cg + i       (fc2)
//   attn[r C + c] = softmax_r z (R > 1) or sigmoid(z) (R = 1)
// fc1: one warp per hidden unit, lanes over k, every image's sum in registers, a fixed shuffle tree (each CTA recomputes
// the whole hidden layer: it is A x Cg MACs per image against fc2's R C x Ag); fc2: one thread per channel c, sequential
// over k, all R rows and all images at once.  Dynamic shared memory: kExciteImgs * (C + A) floats.
__global__ void __launch_bounds__(256) attn_excite_kernel(const float* __restrict__ gap, int B, int C, int R, int card, int A,
                                                          const float* __restrict__ w1, const float* __restrict__ b1,
                                                          const float* __restrict__ w2, const float* __restrict__ b2,
                                                          float* __restrict__ attn) {
  extern __shared__ float ex_smem[];
  float* g_s = ex_smem;                    // [kExciteImgs][C]
  float* hid = ex_smem + kExciteImgs * C;  // [kExciteImgs][A]
  const int b0 = blockIdx.x * kExciteImgs, nb = min(kExciteImgs, B - b0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int Cg = C / card, Ag = A / card;
  for (int t = threadIdx.x; t < kExciteImgs * C; t += blockDim.x) {
    const int i = t / C;
    g_s[t] = i < nb ? gap[static_cast<int64_t>(b0 + i) * C + (t - i * C)] : 0.f;
  }
  __syncthreads();
  for (int j = warp; j < A; j += blockDim.x / 32) {
    const float* wr = w1 + static_cast<int64_t>(j) * Cg;
    const float* gs = g_s + (j / Ag) * Cg;
    float a[kExciteImgs];
#pragma unroll
    for (int i = 0; i < kExciteImgs; ++i) a[i] = 0.f;
    for (int k = lane; k < Cg; k += 32) {
      const float w = wr[k];
#pragma unroll
      for (int i = 0; i < kExciteImgs; ++i) a[i] = fmaf(w, gs[i * C + k], a[i]);
    }
#pragma unroll
    for (int i = 0; i < kExciteImgs; ++i) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) a[i] += __shfl_xor_sync(0xffffffffu, a[i], o);
    }
    if (lane == 0) {
      const float bj = b1[j];
#pragma unroll
      for (int i = 0; i < kExciteImgs; ++i) hid[i * A + j] = fmaxf(a[i] + bj, 0.f);
    }
  }
  __syncthreads();
  const int c = blockIdx.y * kExciteChannels + threadIdx.x;
  if (c >= C) return;
  const int g = c / Cg, ii = c - g * Cg;
  const float* hs = hid + g * Ag;
  float z[kMaxRadix][kExciteImgs];
#pragma unroll
  for (int r = 0; r < kMaxRadix; ++r) {
#pragma unroll
    for (int i = 0; i < kExciteImgs; ++i) z[r][i] = 0.f;
  }
  const int64_t n0 = static_cast<int64_t>(g) * R * Cg + ii;  // fc2 row of radix r: n0 + r Cg
  for (int k = 0; k < Ag; ++k) {
    float h[kExciteImgs];
#pragma unroll
    for (int i = 0; i < kExciteImgs; ++i) h[i] = hs[i * A + k];
#pragma unroll
    for (int r = 0; r < kMaxRadix; ++r) {
      if (r < R) {
        const float w = w2[(n0 + r * Cg) * Ag + k];
#pragma unroll
        for (int i = 0; i < kExciteImgs; ++i) z[r][i] = fmaf(w, h[i], z[r][i]);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < kMaxRadix; ++r) {
    if (r < R) {
      const float bz = b2[n0 + r * Cg];
#pragma unroll
      for (int i = 0; i < kExciteImgs; ++i) z[r][i] += bz;
    }
  }
#pragma unroll
  for (int i = 0; i < kExciteImgs; ++i) {
    if (i >= nb) break;
    float* out = attn + static_cast<int64_t>(b0 + i) * R * C + c;
    if (R == 1) {
      out[0] = 1.f / (1.f + expf(-z[0][i]));
      continue;
    }
    float m = z[0][i];
#pragma unroll
    for (int r = 1; r < kMaxRadix; ++r)
      if (r < R) m = fmaxf(m, z[r][i]);
    float e[kMaxRadix], s = 0.f;
#pragma unroll
    for (int r = 0; r < kMaxRadix; ++r) {
      if (r < R) {
        e[r] = expf(z[r][i] - m);
        s += e[r];
      }
    }
#pragma unroll
    for (int r = 0; r < kMaxRadix; ++r)
      if (r < R) out[static_cast<int64_t>(r) * C] = e[r] / s;
  }
}

// v[b, ho, wo, c] = sum_r attn[b, r C + c] u[b, h, w, r C + c] (fp32: the r = 0 product, then one FMA per radix), stored as
// bf16.  kPool: avd_last's AvgPool2d(3, 2, 1) fused: the nine taps' combined values (zero outside the map) are added in
// (dy, dx) order in fp32 and divided by 9, then rounded once.  One thread = 8 channels of one output pixel.
template <bool kPool>
__global__ void __launch_bounds__(256) radix_combine_kernel(const __nv_bfloat16* __restrict__ u, const float* __restrict__ attn,
                                                            int B, int H, int W, int C, int R, int Ho, int Wo,
                                                            __nv_bfloat16* __restrict__ v) {
  const int cc = C / 8;
  const int64_t total = static_cast<int64_t>(B) * Ho * Wo * cc;
  for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c0 = static_cast<int>(t % cc) * 8;
    const int64_t m = t / cc;
    const int wo = static_cast<int>(m % Wo);
    const int ho = static_cast<int>((m / Wo) % Ho);
    const int b = static_cast<int>(m / (static_cast<int64_t>(Wo) * Ho));
    float a[kMaxRadix][8];
#pragma unroll
    for (int r = 0; r < kMaxRadix; ++r) {
      if (r < R) {
        const float* ap = attn + (static_cast<int64_t>(b) * R + r) * C + c0;
        const float4 a0 = *reinterpret_cast<const float4*>(ap), a1 = *reinterpret_cast<const float4*>(ap + 4);
        a[r][0] = a0.x; a[r][1] = a0.y; a[r][2] = a0.z; a[r][3] = a0.w;
        a[r][4] = a1.x; a[r][5] = a1.y; a[r][6] = a1.z; a[r][7] = a1.w;
      }
    }
    auto combine = [&](int h, int w, float* o) {
      const __nv_bfloat16* px = u + ((static_cast<int64_t>(b) * H + h) * W + w) * R * C + c0;
      float f[8];
      load8(px, f);
#pragma unroll
      for (int k = 0; k < 8; ++k) o[k] = a[0][k] * f[k];
#pragma unroll
      for (int r = 1; r < kMaxRadix; ++r) {
        if (r < R) {
          load8(px + static_cast<int64_t>(r) * C, f);
#pragma unroll
          for (int k = 0; k < 8; ++k) o[k] = fmaf(a[r][k], f[k], o[k]);
        }
      }
    };
    float out[8];
    if constexpr (kPool) {
#pragma unroll
      for (int k = 0; k < 8; ++k) out[k] = 0.f;
      for (int dy = 0; dy < 3; ++dy) {
        const int h = 2 * ho - 1 + dy;
        if (h < 0 || h >= H) continue;
        for (int dx = 0; dx < 3; ++dx) {
          const int w = 2 * wo - 1 + dx;
          if (w < 0 || w >= W) continue;
          float o[8];
          combine(h, w, o);
#pragma unroll
          for (int k = 0; k < 8; ++k) out[k] += o[k];
        }
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) out[k] /= 9.f;
    } else {
      combine(ho, wo, out);
    }
    store8(v + m * C + c0, out);
  }
}

// AvgPool2d(3, 2, padding 1, count_include_pad=True) over NHWC bf16: the in-map taps added in (dy, dx) order in fp32, / 9,
// one rounding.  One thread = 8 channels of one output pixel.
__global__ void __launch_bounds__(256) avgpool3s2_kernel(const __nv_bfloat16* __restrict__ x, int B, int H, int W, int C, int Ho,
                                                         int Wo, __nv_bfloat16* __restrict__ y) {
  const int cc = C / 8;
  const int64_t total = static_cast<int64_t>(B) * Ho * Wo * cc;
  for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c0 = static_cast<int>(t % cc) * 8;
    const int64_t m = t / cc;
    const int wo = static_cast<int>(m % Wo);
    const int ho = static_cast<int>((m / Wo) % Ho);
    const int b = static_cast<int>(m / (static_cast<int64_t>(Wo) * Ho));
    float s[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) s[k] = 0.f;
    for (int dy = 0; dy < 3; ++dy) {
      const int h = 2 * ho - 1 + dy;
      if (h < 0 || h >= H) continue;
      for (int dx = 0; dx < 3; ++dx) {
        const int w = 2 * wo - 1 + dx;
        if (w < 0 || w >= W) continue;
        float f[8];
        load8(x + ((static_cast<int64_t>(b) * H + h) * W + w) * C + c0, f);
#pragma unroll
        for (int k = 0; k < 8; ++k) s[k] += f[k];
      }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) s[k] /= 9.f;
    store8(y + m * C + c0, s);
  }
}

int avgpool3s2_run(const __nv_bfloat16* x, int B, int H, int W, int C, __nv_bfloat16* y, cudaStream_t s) {
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  avgpool3s2_kernel<<<grid_for(static_cast<int64_t>(B) * Ho * Wo * (C / 8)), 256, 0, s>>>(x, B, H, W, C, Ho, Wo, y);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

// the gate of a split-attention block: mean, excitation, combine (+ the fused stride-2 average pool)
int split_attn_gate(const __nv_bfloat16* u, int B, int H, int W, int C, int R, int card, int A, const float* w1, const float* b1,
                    const float* w2, const float* b2, float* gap, float* attn, int pool, __nv_bfloat16* v, cudaStream_t s) {
  radix_mean_kernel<<<dim3((C + 63) / 64, B), 256, 0, s>>>(u, H * W, C, R, gap);
  VDK_CUDA_OK(cudaGetLastError());
  attn_excite_kernel<<<dim3((B + kExciteImgs - 1) / kExciteImgs, (C + kExciteChannels - 1) / kExciteChannels), 256,
                       kExciteImgs * (C + A) * sizeof(float), s>>>(gap, B, C, R, card, A, w1, b1, w2, b2, attn);
  VDK_CUDA_OK(cudaGetLastError());
  const int Ho = pool ? (H - 1) / 2 + 1 : H, Wo = pool ? (W - 1) / 2 + 1 : W;
  const int grid = grid_for(static_cast<int64_t>(B) * Ho * Wo * (C / 8));
  if (pool) radix_combine_kernel<true><<<grid, 256, 0, s>>>(u, attn, B, H, W, C, R, Ho, Wo, v);
  else radix_combine_kernel<false><<<grid, 256, 0, s>>>(u, attn, B, H, W, C, R, Ho, Wo, v);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

// kExciteImgs * (C + A) floats must fit in the default 48 KB of dynamic shared memory
constexpr int kMaxGateFloats = 48 * 1024 / 4 / kExciteImgs;

int check_gate_shape(int C, int R, int card, int A) {
  VDK_REQUIRE(C > 0 && C % 8 == 0 && R >= 1 && R <= kMaxRadix && R * C <= 4096,
              "split attention: C=%d must be a positive multiple of 8 and 1 <= radix=%d <= %d with radix * C <= 4096", C, R,
              kMaxRadix);
  VDK_REQUIRE(card >= 1 && C % card == 0 && A > 0 && A % card == 0,
              "split attention: cardinality=%d must divide C=%d and the attention width A=%d", card, C, A);
  VDK_REQUIRE(C + A <= kMaxGateFloats, "split attention: C + A = %d exceeds %d", C + A, kMaxGateFloats);
  return VDK_OK;
}

int stage_width(const vdk_resnest_net* n, int s) { return ((64 << s) * n->base_width / 64) * n->cardinality; }

int check_resnest(const vdk_resnest_net* n) {
  VDK_REQUIRE(n, "vdk_resnest: null network");
  VDK_REQUIRE(n->image_size > 0 && n->image_size % 32 == 0, "vdk_resnest: image_size must be a multiple of 32 (got %d)",
              n->image_size);
  VDK_REQUIRE(n->feat_dim > 0 && n->feat_dim % 8 == 0, "vdk_resnest: feat_dim must be a multiple of 8");
  VDK_REQUIRE(n->radix >= 1 && n->cardinality >= 1 && n->base_width >= 1, "vdk_resnest: bad radix=%d cardinality=%d base_width=%d",
              n->radix, n->cardinality, n->base_width);
  int nb = 0;
  for (int s = 0; s < 4; ++s) {
    VDK_REQUIRE(n->depths[s] >= 1, "vdk_resnest: every stage needs at least one block");
    nb += n->depths[s];
    const int gw = stage_width(n, s);
    VDK_REQUIRE(gw % (n->cardinality * n->radix) == 0, "vdk_resnest: stage %d width %d is not a multiple of cardinality * radix", s,
                gw);
    const int rc = check_gate_shape(gw, n->radix, n->cardinality, n->attn[s]);
    if (rc != VDK_OK) return rc;
  }
  VDK_REQUIRE(nb <= VDK_RESNET_MAX_BLOCKS, "vdk_resnest: too many blocks (%d)", nb);
  for (int i = 0; i < 3; ++i) VDK_REQUIRE(n->stem[i].w && n->stem[i].b, "vdk_resnest: missing stem weights");
  int first = 0;
  for (int s = 0; s < 4; ++s) {
    for (int j = 0; j < n->depths[s]; ++j) {
      const vdk_resnest_block& b = n->blocks[first + j];
      VDK_REQUIRE(b.conv1.w && b.conv1.b && b.conv2.w && b.conv2.b && b.conv3.w && b.conv3.b && b.fc1_w && b.fc1_b && b.fc2_w &&
                      b.fc2_b,
                  "vdk_resnest: block %d misses a weight", first + j);
    }
    VDK_REQUIRE(n->blocks[first].down.w && n->blocks[first].down.b, "vdk_resnest: the first block of stage %d needs its shortcut conv", s);
    first += n->depths[s];
  }
  VDK_REQUIRE(n->neck_w && n->neck_b, "vdk_resnest: missing neck");
  return VDK_OK;
}

struct ResnestSizes {
  size_t act;   // elements of the largest map at most gw or 4 planes wide
  size_t big;   // elements of the largest split-conv output (R gw wide)
  size_t rows;  // elements of the stem's patch rows
  size_t gate;  // floats of the widest R gw row per image
};

ResnestSizes resnest_sizes(const vdk_resnest_net* n, int batch) {
  const size_t S = n->image_size, B = batch;
  ResnestSizes z{};
  z.act = B * (S / 2) * (S / 2) * 64;  // the stem's output (its 32-channel maps are smaller)
  size_t hin = S / 4;
  for (int s = 0; s < 4; ++s) {
    const size_t gw = stage_width(n, s), out = static_cast<size_t>(256) << s;
    const size_t ho = s == 0 ? hin : hin / 2;
    const size_t hs = n->avd_first ? ho : hin;  // the split conv of the stage's first block runs at hs
    z.act = std::max({z.act, B * hin * hin * gw, B * ho * ho * out});
    z.big = std::max(z.big, B * hs * hs * n->radix * gw);
    z.gate = std::max(z.gate, static_cast<size_t>(n->radix) * gw);
    hin = ho;
  }
  z.rows = B * (S / 2) * (S / 2) * 320;
  return z;
}

}  // namespace

}  // namespace vdk

using namespace vdk;

extern "C" size_t vdk_resnest_workspace_bytes(const vdk_resnest_net* net, int batch) {
  if (!net || batch <= 0 || net->image_size <= 0 || net->base_width <= 0 || net->cardinality <= 0 || net->radix <= 0) return 0;
  const ResnestSizes z = resnest_sizes(net, batch);
  // x (block input / output), shortcut, t1 (conv1 out, combined map, neck slabs), t2 (avd_first pool), the split conv's
  // output, stem patch rows, gap and attention
  return 4 * up256(z.act * 2) + up256(z.big * 2) + up256(z.rows * 2) + 2 * up256(batch * z.gate * 4) + 1024;
}

extern "C" int vdk_resnest_forward(const vdk_resnest_net* net, const float* images, int batch, int l2_normalize,
                                   float* embeddings, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_resnest(net);
  if (rc != VDK_OK) return rc;
  VDK_REQUIRE(images && embeddings && batch > 0, "vdk_resnest_forward: null image/embedding buffer");
  VDK_REQUIRE(workspace && workspace_bytes >= vdk_resnest_workspace_bytes(net, batch), "vdk_resnest_forward: workspace too small");
  VDK_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "vdk_resnest_forward: workspace must be 256-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const ResnestSizes z = resnest_sizes(net, batch);
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  auto take = [&](size_t bytes) {
    uint8_t* p = ws;
    ws += up256(bytes);
    return p;
  };
  __nv_bfloat16* x = reinterpret_cast<__nv_bfloat16*>(take(z.act * 2));
  __nv_bfloat16* sc = reinterpret_cast<__nv_bfloat16*>(take(z.act * 2));
  __nv_bfloat16* t1 = reinterpret_cast<__nv_bfloat16*>(take(z.act * 2));
  __nv_bfloat16* t2 = reinterpret_cast<__nv_bfloat16*>(take(z.act * 2));
  __nv_bfloat16* big = reinterpret_cast<__nv_bfloat16*>(take(z.big * 2));
  __nv_bfloat16* rows = reinterpret_cast<__nv_bfloat16*>(take(z.rows * 2));
  float* gap = reinterpret_cast<float*>(take(batch * z.gate * 4));
  float* attn = reinterpret_cast<float*>(take(batch * z.gate * 4));

  auto conv = [&](const void* in, int H, int Cin, const vdk_resnet_conv& c, int Cout, int k, int stride, int pad, int epi,
                  const void* res, void* out, int groups = 0) -> int {
    vdk_conv_desc d{};
    d.x = in; d.w = c.w; d.bias = c.b; d.residual = res; d.y = out;
    d.B = batch; d.H = H; d.W = H; d.Cin = Cin; d.Cout = Cout;
    d.kernel = k; d.stride = stride; d.pad = pad; d.epilogue = epi;
    return groups > 0 ? conv_grouped_ex_run(d, groups, s) : conv_run(d, s);
  };
  // the deep stem: three 3x3 convs (each + BN + ReLU) as GEMMs over zero-padded (kh, kw, c) patch rows
  const int S = net->image_size;
  int H = S / 2;
  if ((rc = launch_patch_rows_nchw(images, batch, S, S, 3, 3, 2, 1, H, H, 64, rows, s)) != VDK_OK) return rc;
  if ((rc = conv(rows, H, 64, net->stem[0], 32, 1, 1, 0, VDK_EPI_RELU, nullptr, t1)) != VDK_OK) return rc;
  if ((rc = launch_patch_rows_nhwc(t1, batch, H, H, 32, 3, 1, 1, H, H, 320, rows, s)) != VDK_OK) return rc;
  if ((rc = conv(rows, H, 320, net->stem[1], 32, 1, 1, 0, VDK_EPI_RELU, nullptr, t2)) != VDK_OK) return rc;
  if ((rc = launch_patch_rows_nhwc(t2, batch, H, H, 32, 3, 1, 1, H, H, 320, rows, s)) != VDK_OK) return rc;
  if ((rc = conv(rows, H, 320, net->stem[2], 64, 1, 1, 0, VDK_EPI_RELU, nullptr, sc)) != VDK_OK) return rc;
  if ((rc = launch_stem_maxpool(sc, batch, H, H, 64, x, s)) != VDK_OK) return rc;
  H /= 2;

  const int R = net->radix, card = net->cardinality;
  int C = 64, blk = 0;
  for (int st = 0; st < 4; ++st) {
    const int gw = stage_width(net, st), out = 256 << st, A = net->attn[st];
    for (int j = 0; j < net->depths[st]; ++j, ++blk) {
      const vdk_resnest_block& b = net->blocks[blk];
      const int stride = (st > 0 && j == 0) ? 2 : 1, Ho = H / stride;
      __nv_bfloat16* res = x;
      if (b.down.w) {  // avg_down: AvgPool2d(2, 2) + 1x1 conv folded into one 2x2/s2 conv on stride-2 blocks
        const int k = stride == 2 ? 2 : 1;
        if ((rc = conv(x, H, C, b.down, out, k, stride, 0, VDK_EPI_NONE, nullptr, sc)) != VDK_OK) return rc;
        res = sc;
      }
      if ((rc = conv(x, H, C, b.conv1, gw, 1, 1, 0, VDK_EPI_RELU, nullptr, t1)) != VDK_OK) return rc;
      const __nv_bfloat16* split_in = t1;
      int Hs = H;
      if (stride == 2 && net->avd_first) {
        if ((rc = avgpool3s2_run(t1, batch, H, H, gw, t2, s)) != VDK_OK) return rc;
        split_in = t2;
        Hs = Ho;
      }
      if ((rc = conv(split_in, Hs, gw, b.conv2, R * gw, 3, 1, 1, VDK_EPI_RELU, nullptr, big, card * R)) != VDK_OK) return rc;
      const int pool = stride == 2 && !net->avd_first;
      if ((rc = split_attn_gate(big, batch, Hs, Hs, gw, R, card, A, b.fc1_w, b.fc1_b, b.fc2_w, b.fc2_b, gap, attn, pool, t1, s)) !=
          VDK_OK)
        return rc;
      if ((rc = conv(t1, Ho, gw, b.conv3, out, 1, 1, 0, VDK_EPI_RESIDUAL_RELU, res, res, 1)) != VDK_OK) return rc;
      if (res == sc) std::swap(x, sc);
      H = Ho;
      C = out;
    }
  }
  return launch_neck(x, batch, H * H * C, net->feat_dim, net->neck_w, net->neck_b, l2_normalize, reinterpret_cast<float*>(t1),
                     up256(z.act * 2), embeddings, s);
}

extern "C" int vdk_resnest_struct_sizes(size_t* out, int n) {
  const size_t sizes[] = {sizeof(vdk_resnest_net)};
  const int k = static_cast<int>(sizeof(sizes) / sizeof(sizes[0]));
  for (int i = 0; i < n && i < k; ++i) out[i] = sizes[i];
  return k;
}

// Kernel-level entry points of the pieces above, for their tests.
extern "C" int vdk_split_attn_gate(const void* u, int B, int H, int W, int C, int radix, int cardinality, int A, const float* fc1_w,
                                   const float* fc1_b, const float* fc2_w, const float* fc2_b, float* gap, float* attn, int pool,
                                   void* v, void* stream) {
  VDK_REQUIRE(u && fc1_w && fc1_b && fc2_w && fc2_b && gap && attn && v, "vdk_split_attn_gate: null operand");
  VDK_REQUIRE(B > 0 && H > 0 && W > 0 && (pool == 0 || pool == 1), "vdk_split_attn_gate: bad shape B=%d H=%d W=%d pool=%d", B, H, W,
              pool);
  const int rc = check_gate_shape(C, radix, cardinality, A);
  if (rc != VDK_OK) return rc;
  VDK_REQUIRE(((reinterpret_cast<uintptr_t>(u) | reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(attn)) & 15) == 0,
              "vdk_split_attn_gate: 16-byte alignment");
  return split_attn_gate(static_cast<const __nv_bfloat16*>(u), B, H, W, C, radix, cardinality, A, fc1_w, fc1_b, fc2_w, fc2_b, gap,
                         attn, pool, static_cast<__nv_bfloat16*>(v), reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vdk_avgpool3s2(const void* x, int B, int H, int W, int C, void* y, void* stream) {
  VDK_REQUIRE(x && y && B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, "vdk_avgpool3s2: bad arguments");
  VDK_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0, "vdk_avgpool3s2: 16-byte alignment");
  return avgpool3s2_run(static_cast<const __nv_bfloat16*>(x), B, H, W, C, static_cast<__nv_bfloat16*>(y),
                        reinterpret_cast<cudaStream_t>(stream));
}
