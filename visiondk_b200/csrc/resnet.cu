// resnet.cu — timm 0.9.16 Bottleneck ResNet (resnet50/101/152, -D variants, wide_resnet*_2) embedding forward for the
// faceX / CBIR extract path, NHWC bf16, every eval BatchNorm folded into its convolution.
//
// Replaces TimmWrapper.forward for ResNet backbones (models/faceX/backbone/timm_wrapper.py:16-21, 30-38, 51-54: timm
// ResNet with num_classes=0, global_pool='' -> BatchNorm2d -> Flatten -> Linear -> BatchNorm1d) and F.normalize
// (face_model.py:139).
//
// Every convolution of the stages is vdk_conv2d (gemm.cu: 1x1 / stride 1 as a plain GEMM, 3x3 and stride-2 shortcuts as
// implicit GEMMs with TMA im2col A tiles) with the bias + ReLU / residual + ReLU epilogues.  Written here:
//   patch_rows   the stem's explicit im2col: fp32 NCHW image (or the deep stem's 32-channel bf16 maps) -> bf16 rows of
//                (kh, kw, c) zero padded to a multiple of 64, then a GEMM with the ReLU epilogue (Cin = 3 or 32 is too
//                narrow for the 64-channel im2col loads)
//   maxpool3s2   MaxPool2d(3, 2, padding 1) over NHWC, or the legacy SENet's unpadded ceil-mode form
//   se_*         the squeeze-excitation gate of the legacy SENets (mean, excitation, scale + residual + ReLU)
// and the neck is the ConvNeXt path's (launch_neck).  vdk_bottleneck_forward (end of file) runs the ResNeXts (grouped 3x3
// convs on vdk_conv2d_grouped) and the legacy SE-ResNets / SE-ResNeXts with the same pieces.
#include "vdk_host.h"

#include <algorithm>
#include "convnext_internal.h"

namespace vdk {

// out[m][e] for output pixel m = (b, ho, wo) and e = (dy * k + dx) * C + c < K: x[b, c, ho*stride - pad + dy, ...] (zero
// outside the image), 0 for K <= e < Kp.  One thread writes 8 consecutive entries (16 bytes) of a row.
template <typename T, bool kNCHW>
__global__ void __launch_bounds__(256) patch_rows_kernel(const T* __restrict__ x, int B, int H, int W, int C, int k,
                                                         int stride, int pad, int Ho, int Wo, int K, int Kp,
                                                         __nv_bfloat16* __restrict__ out) {
  const int chunks = Kp / 8;
  const int64_t total = static_cast<int64_t>(B) * Ho * Wo * chunks;
  for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int ch = static_cast<int>(t % chunks);
    const int64_t m = t / chunks;
    const int wo = static_cast<int>(m % Wo);
    const int ho = static_cast<int>((m / Wo) % Ho);
    const int b = static_cast<int>(m / (static_cast<int64_t>(Wo) * Ho));
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int e = ch * 8 + i;
      v[i] = 0.f;
      if (e < K) {
        const int tap = e / C, c = e - tap * C;
        const int dy = tap / k, dx = tap - dy * k;
        const int ih = ho * stride - pad + dy, iw = wo * stride - pad + dx;
        if (ih >= 0 && ih < H && iw >= 0 && iw < W) {
          const int64_t idx = kNCHW ? ((static_cast<int64_t>(b) * C + c) * H + ih) * W + iw
                                    : ((static_cast<int64_t>(b) * H + ih) * W + iw) * C + c;
          v[i] = static_cast<float>(x[idx]);
        }
      }
    }
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __nv_bfloat162 h = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
      ow[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    *reinterpret_cast<uint4*>(out + m * Kp + ch * 8) = o;
  }
}

// MaxPool2d(kernel 3, stride 2, padding kPad) over NHWC bf16 (padding never wins: it is -inf); one thread = 8 channels of
// one output pixel.  Exact (a max of bf16 values is one of them).  kPad = 1: timm's ResNet stem pool.  kPad = 0 with
// Ho = H / 2 on an even H: the legacy SENet's MaxPool2d(3, 2, ceil_mode=True), whose windows start one pixel later and
// whose last window is clipped at the border.
template <int kPad>
__global__ void __launch_bounds__(256) maxpool3s2_kernel(const __nv_bfloat16* __restrict__ x, int B, int H, int W, int C,
                                                         int Ho, int Wo, __nv_bfloat16* __restrict__ y) {
  const int cc = C / 8;
  const int64_t total = static_cast<int64_t>(B) * Ho * Wo * cc;
  for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c8 = static_cast<int>(t % cc);
    const int64_t m = t / cc;
    const int wo = static_cast<int>(m % Wo);
    const int ho = static_cast<int>((m / Wo) % Ho);
    const int b = static_cast<int>(m / (static_cast<int64_t>(Wo) * Ho));
    float mx[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) mx[i] = -INFINITY;
    for (int dy = 0; dy < 3; ++dy) {
      const int ih = ho * 2 - kPad + dy;
      if (ih < 0 || ih >= H) continue;
      for (int dx = 0; dx < 3; ++dx) {
        const int iw = wo * 2 - kPad + dx;
        if (iw < 0 || iw >= W) continue;
        const uint4 u = *reinterpret_cast<const uint4*>(x + ((static_cast<int64_t>(b) * H + ih) * W + iw) * C + c8 * 8);
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = __bfloat1622float2(h[i]);
          mx[2 * i] = fmaxf(mx[2 * i], f.x);
          mx[2 * i + 1] = fmaxf(mx[2 * i + 1], f.y);
        }
      }
    }
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __nv_bfloat162 h = __floats2bfloat162_rn(mx[2 * i], mx[2 * i + 1]);
      ow[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    *reinterpret_cast<uint4*>(y + m * C + c8 * 8) = o;
  }
}

// ---- squeeze-excitation (timm senet.py SEModule) after the BN-folded conv3 output y [B, HW, C] bf16 ----
// se_mean: mean[b, c] = sum_p y[b, p, c] / HW in fp32, deterministic: block (64 channels, image b) of 256 threads = 8
// channel vectors x 32 pixel lanes; lane l sums pixels l, l + 32, ... in order, then a fixed tree over the 32 lanes.
__global__ void __launch_bounds__(256) se_mean_kernel(const __nv_bfloat16* __restrict__ y, int HW, int C,
                                                      float* __restrict__ mean) {
  __shared__ float part[32][64];
  const int b = blockIdx.y, cv = threadIdx.x & 7, lane = threadIdx.x >> 3, c0 = blockIdx.x * 64 + cv * 8;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  const __nv_bfloat16* src = y + static_cast<int64_t>(b) * HW * C + c0;
  for (int p = lane; p < HW; p += 32) {
    const uint4 u = *reinterpret_cast<const uint4*>(src + static_cast<int64_t>(p) * C);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __bfloat1622float2(h[i]);
      acc[2 * i] += f.x;
      acc[2 * i + 1] += f.y;
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
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) mean[static_cast<int64_t>(b) * C + c0 + i] = part[0][cv * 8 + i] / static_cast<float>(HW);
  }
}

// se_excite: s[b, :] = gate(fc2(act(fc1(mean[b, :]) + b1)) + b2) in fp32, one block of 256 threads per image; act is
// ReLU (the legacy SENets, MobileNetV3) or SiLU (EfficientNetV2, silu_hidden); gate is sigmoid, or MobileNetV3's hard
// sigmoid relu6(v + 3) / 6 (hard_gate).  fc1: one warp per hidden unit, lanes over C, a fixed shuffle tree; fc2: one thread
// per channel, sequential over rd.
__global__ void __launch_bounds__(256) se_excite_kernel(const float* __restrict__ mean, int C, int rd,
                                                        const float* __restrict__ w1, const float* __restrict__ b1,
                                                        const float* __restrict__ w2, const float* __restrict__ b2,
                                                        float* __restrict__ s, int silu_hidden, int hard_gate) {
  extern __shared__ float se_smem[];
  float* m = se_smem;       // [C]
  float* hid = se_smem + C;  // [rd]
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int c = threadIdx.x; c < C; c += blockDim.x) m[c] = mean[static_cast<int64_t>(b) * C + c];
  __syncthreads();
  for (int j = warp; j < rd; j += blockDim.x / 32) {
    const float* wr = w1 + static_cast<int64_t>(j) * C;
    float a = 0.f;
    for (int c = lane; c < C; c += 32) a = fmaf(wr[c], m[c], a);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) {
      const float v = a + b1[j];
      hid[j] = silu_hidden ? v / (1.f + expf(-v)) : fmaxf(v, 0.f);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float* wr = w2 + static_cast<int64_t>(c) * rd;
    float a = 0.f;
    for (int j = 0; j < rd; ++j) a = fmaf(wr[j], hid[j], a);
    const float v = a + b2[c];
    s[static_cast<int64_t>(b) * C + c] = hard_gate ? fminf(fmaxf(v + 3.f, 0.f), 6.f) / 6.f : 1.f / (1.f + expf(-v));
  }
}

// se_scale: res[m, c] = ReLU(y[m, c] * s[b, c] + res[m, c]) (one fp32 FMA, then the bf16 rounding), in place into the
// shortcut like conv3's residual epilogue; one thread = 8 channels (16-byte vectors) of one pixel.
__global__ void __launch_bounds__(256) se_scale_kernel(const __nv_bfloat16* __restrict__ y, const float* __restrict__ s,
                                                       int64_t M, int HW, int C, __nv_bfloat16* res) {
  const int cc = C / 8;
  const int64_t total = M * cc;
  for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c8 = static_cast<int>(t % cc);
    const int64_t m = t / cc;
    const int64_t b = m / HW;
    const uint4 uy = *reinterpret_cast<const uint4*>(y + m * C + c8 * 8);
    const uint4 ur = *reinterpret_cast<const uint4*>(res + m * C + c8 * 8);
    const float4 s0 = *reinterpret_cast<const float4*>(s + b * C + c8 * 8);
    const float4 s1 = *reinterpret_cast<const float4*>(s + b * C + c8 * 8 + 4);
    const float sv[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    const __nv_bfloat162* hy = reinterpret_cast<const __nv_bfloat162*>(&uy);
    const __nv_bfloat162* hr = reinterpret_cast<const __nv_bfloat162*>(&ur);
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 fy = __bfloat1622float2(hy[i]), fr = __bfloat1622float2(hr[i]);
      __nv_bfloat162 h = __floats2bfloat162_rn(fmaxf(fmaf(fy.x, sv[2 * i], fr.x), 0.f), fmaxf(fmaf(fy.y, sv[2 * i + 1], fr.y), 0.f));
      ow[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    *reinterpret_cast<uint4*>(res + m * C + c8 * 8) = o;
  }
}

int launch_se_excite(const float* mean, int batch, int C, int rd, int silu_hidden, int hard_gate, const float* w1,
                     const float* b1, const float* w2, const float* b2, float* gate, cudaStream_t s) {
  se_excite_kernel<<<batch, 256, (C + rd) * sizeof(float), s>>>(mean, C, rd, w1, b1, w2, b2, gate, silu_hidden, hard_gate);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

int launch_patch_rows_nchw(const float* x, int B, int H, int W, int C, int k, int stride, int pad, int Ho, int Wo, int Kp,
                           __nv_bfloat16* out, cudaStream_t s) {
  const int64_t threads = static_cast<int64_t>(B) * Ho * Wo * (Kp / 8);
  patch_rows_kernel<float, true><<<grid_for(threads), 256, 0, s>>>(x, B, H, W, C, k, stride, pad, Ho, Wo, k * k * C, Kp, out);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

static int check_net(const vdk_resnet_net* n) {
  VDK_REQUIRE(n, "vdk_resnet: null network");
  // every map a stride-2 layer reads then has an even side: AvgPool2d(2, 2, ceil_mode=True) never sees a partial window
  VDK_REQUIRE(n->image_size > 0 && n->image_size % 32 == 0, "vdk_resnet: image_size must be a multiple of 32 (got %d)",
              n->image_size);
  VDK_REQUIRE(n->feat_dim > 0 && n->feat_dim % 8 == 0, "vdk_resnet: feat_dim must be a multiple of 8");
  VDK_REQUIRE(n->base_width == 64 || n->base_width == 128, "vdk_resnet: base_width must be 64 or 128 (got %d)", n->base_width);
  int nb = 0;
  for (int s = 0; s < 4; ++s) {
    VDK_REQUIRE(n->depths[s] >= 1, "vdk_resnet: every stage needs at least one block");
    nb += n->depths[s];
  }
  VDK_REQUIRE(nb <= VDK_RESNET_MAX_BLOCKS, "vdk_resnet: too many blocks (%d)", nb);
  for (int i = 0; i < (n->deep_stem ? 3 : 1); ++i) VDK_REQUIRE(n->stem[i].w && n->stem[i].b, "vdk_resnet: missing stem weights");
  for (int i = 0; i < nb; ++i) {
    const vdk_resnet_block& b = n->blocks[i];
    VDK_REQUIRE(b.conv1.w && b.conv1.b && b.conv2.w && b.conv2.b && b.conv3.w && b.conv3.b, "vdk_resnet: block %d misses a conv", i);
  }
  int first = 0;
  for (int s = 0; s < 4; ++s) {
    VDK_REQUIRE(n->blocks[first].down.w && n->blocks[first].down.b, "vdk_resnet: the first block of stage %d needs its shortcut conv", s);
    first += n->depths[s];
  }
  VDK_REQUIRE(n->neck_w && n->neck_b, "vdk_resnet: missing neck");
  return VDK_OK;
}

struct ResnetSizes {
  size_t act;   // elements of the largest activation map
  size_t rows;  // elements of the stem's patch rows
};

static ResnetSizes resnet_sizes(const vdk_resnet_net* n, int batch) {
  const size_t S = n->image_size, B = batch;
  ResnetSizes z;
  z.act = B * (S / 2) * (S / 2) * 64;  // stem output (the deep stem's 32-channel maps are smaller)
  size_t hin = S / 4;
  for (int s = 0; s < 4; ++s) {
    const size_t width = static_cast<size_t>(n->base_width) << s, out = static_cast<size_t>(256) << s;
    const size_t ho = s == 0 ? hin : hin / 2;
    z.act = std::max(z.act, B * hin * hin * width);  // conv1 of the first block runs at the input resolution
    z.act = std::max(z.act, B * ho * ho * out);
    hin = ho;
  }
  z.rows = B * (S / 2) * (S / 2) * (n->deep_stem ? 320 : 192);
  return z;
}

}  // namespace vdk

using namespace vdk;

extern "C" size_t vdk_resnet_workspace_bytes(const vdk_resnet_net* net, int batch) {
  if (!net || batch <= 0 || net->image_size <= 0 || net->base_width <= 0) return 0;
  const ResnetSizes z = resnet_sizes(net, batch);
  // x (block input / output), shortcut, t1 (conv1 out, neck slabs), t2 (conv2 out), stem patch rows
  return 4 * up256(z.act * 2) + up256(z.rows * 2) + 1024;
}

extern "C" int vdk_resnet_forward(const vdk_resnet_net* net, const float* images, int batch, int l2_normalize,
                                  float* embeddings, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_net(net);
  if (rc != VDK_OK) return rc;
  VDK_REQUIRE(images && embeddings && batch > 0, "vdk_resnet_forward: null image/embedding buffer");
  VDK_REQUIRE(workspace && workspace_bytes >= vdk_resnet_workspace_bytes(net, batch), "vdk_resnet_forward: workspace too small");
  VDK_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "vdk_resnet_forward: workspace must be 256-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const ResnetSizes z = resnet_sizes(net, batch);
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  __nv_bfloat16* buf[4];
  for (int i = 0; i < 4; ++i) {
    buf[i] = reinterpret_cast<__nv_bfloat16*>(ws);
    ws += up256(z.act * 2);
  }
  __nv_bfloat16* rows = reinterpret_cast<__nv_bfloat16*>(ws);
  __nv_bfloat16 *x = buf[0], *sc = buf[1], *t1 = buf[2], *t2 = buf[3];

  auto conv = [&](const void* in, int H, int W, int Cin, const vdk_resnet_conv& c, int Cout, int k, int stride, int pad,
                  int epi, const void* res, void* out) -> int {
    vdk_conv_desc d{};
    d.x = in; d.w = c.w; d.bias = c.b; d.residual = res; d.y = out;
    d.B = batch; d.H = H; d.W = W; d.Cin = Cin; d.Cout = Cout;
    d.kernel = k; d.stride = stride; d.pad = pad; d.epilogue = epi;
    return conv_run(d, s);
  };
  // stem convolution over explicit patch rows: a 1x1 conv (plain GEMM) over [B, Ho, Wo, Kp] + bias + ReLU
  auto stem_conv = [&](auto* in, bool nchw, int H, int C, int k, int stride, const vdk_resnet_conv& c, int Cout, void* out) -> int {
    const int pad = k / 2, Ho = (H + 2 * pad - k) / stride + 1;
    const int K = k * k * C, Kp = (K + 63) / 64 * 64;
    const int64_t threads = static_cast<int64_t>(batch) * Ho * Ho * (Kp / 8);
    using T = std::remove_cv_t<std::remove_pointer_t<decltype(in)>>;
    if (nchw) patch_rows_kernel<T, true><<<grid_for(threads), 256, 0, s>>>(in, batch, H, H, C, k, stride, pad, Ho, Ho, K, Kp, rows);
    else patch_rows_kernel<T, false><<<grid_for(threads), 256, 0, s>>>(in, batch, H, H, C, k, stride, pad, Ho, Ho, K, Kp, rows);
    VDK_CUDA_OK(cudaGetLastError());
    return conv(rows, Ho, Ho, Kp, c, Cout, 1, 1, 0, VDK_EPI_RELU, nullptr, out);
  };

  const int S = net->image_size;
  int H = S / 2;
  // ---- stem: conv 7x7/s2 + bn1 + ReLU, or the deep stem's three 3x3 convs (each + BN + ReLU) ----
  if (net->deep_stem) {
    if ((rc = stem_conv(images, true, S, 3, 3, 2, net->stem[0], 32, t1)) != VDK_OK) return rc;
    if ((rc = stem_conv(static_cast<const __nv_bfloat16*>(t1), false, H, 32, 3, 1, net->stem[1], 32, t2)) != VDK_OK) return rc;
    if ((rc = stem_conv(static_cast<const __nv_bfloat16*>(t2), false, H, 32, 3, 1, net->stem[2], 64, sc)) != VDK_OK) return rc;
  } else {
    if ((rc = stem_conv(images, true, S, 3, 7, 2, net->stem[0], 64, sc)) != VDK_OK) return rc;
  }
  // ---- max pool 3x3/s2 ----
  {
    const int Ho = H / 2;
    maxpool3s2_kernel<1><<<grid_for(static_cast<int64_t>(batch) * Ho * Ho * 8), 256, 0, s>>>(sc, batch, H, H, 64, Ho, Ho, x);
    VDK_CUDA_OK(cudaGetLastError());
    H = Ho;
  }
  // ---- stages of Bottleneck blocks: conv1 1x1 + ReLU, conv2 3x3/stride + ReLU, conv3 1x1 + shortcut + ReLU ----
  int C = 64, blk = 0;
  for (int st = 0; st < 4; ++st) {
    const int width = net->base_width << st, out = 256 << st;
    for (int j = 0; j < net->depths[st]; ++j, ++blk) {
      const vdk_resnet_block& b = net->blocks[blk];
      const int stride = (st > 0 && j == 0) ? 2 : 1, Ho = H / stride;
      if ((rc = conv(x, H, H, C, b.conv1, width, 1, 1, 0, VDK_EPI_RELU, nullptr, t1)) != VDK_OK) return rc;
      if ((rc = conv(t1, H, H, width, b.conv2, width, 3, stride, 1, VDK_EPI_RELU, nullptr, t2)) != VDK_OK) return rc;
      __nv_bfloat16* res = x;
      if (b.down.w) {
        // shortcut: 1x1/stride conv, or (avg_down, stride 2) AvgPool2d(2, 2) + 1x1 conv folded into one 2x2/s2 conv
        const int k = (net->avg_down && stride == 2) ? 2 : 1;
        if ((rc = conv(x, H, H, C, b.down, out, k, stride, 0, VDK_EPI_NONE, nullptr, sc)) != VDK_OK) return rc;
        res = sc;
      }
      if ((rc = conv(t2, Ho, Ho, width, b.conv3, out, 1, 1, 0, VDK_EPI_RESIDUAL_RELU, res, res)) != VDK_OK) return rc;
      if (res == sc) std::swap(x, sc);
      H = Ho;
      C = out;
    }
  }
  // ---- neck: BN2d -> Flatten -> Linear -> BN1d folded into one split-K GEMM over the (h, w, c) features ----
  return launch_neck(x, batch, H * H * C, net->feat_dim, net->neck_w, net->neck_b, l2_normalize, reinterpret_cast<float*>(t1),
                     up256(z.act * 2), embeddings, s);
}

// ---- general Bottleneck network: ResNeXt (grouped conv2), legacy SE-ResNet / SE-ResNeXt (SE gate, stride on conv1,
// ceil-mode stem pool).  vdk_resnet_forward above stays its own path. ----
namespace vdk {

static int se_gate(const __nv_bfloat16* y, int batch, int HW, int C, int rd, const float* w1, const float* b1, const float* w2,
                   const float* b2, float* mean, float* sc, __nv_bfloat16* res, cudaStream_t s) {
  int rc;
  se_mean_kernel<<<dim3(C / 64, batch), 256, 0, s>>>(y, HW, C, mean);
  VDK_CUDA_OK(cudaGetLastError());
  if ((rc = launch_se_excite(mean, batch, C, rd, 0, 0, w1, b1, w2, b2, sc, s)) != VDK_OK) return rc;
  const int64_t M = static_cast<int64_t>(batch) * HW;
  se_scale_kernel<<<grid_for(M * (C / 8)), 256, 0, s>>>(y, sc, M, HW, C, res);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

static int stem_pool_run(const __nv_bfloat16* x, int B, int H, int W, int C, int mode, __nv_bfloat16* y, cudaStream_t s) {
  const int pad = mode == VDK_STEM_POOL_CEIL ? 0 : 1;
  // floor mode with padding 1; ceil mode without padding (every window then starts inside the map, none is dropped)
  const int Ho = mode == VDK_STEM_POOL_CEIL ? (H - 2) / 2 + 1 : (H + 2 * pad - 3) / 2 + 1;
  const int Wo = mode == VDK_STEM_POOL_CEIL ? (W - 2) / 2 + 1 : (W + 2 * pad - 3) / 2 + 1;
  const int64_t threads = static_cast<int64_t>(B) * Ho * Wo * (C / 8);
  if (pad) maxpool3s2_kernel<1><<<grid_for(threads), 256, 0, s>>>(x, B, H, W, C, Ho, Wo, y);
  else maxpool3s2_kernel<0><<<grid_for(threads), 256, 0, s>>>(x, B, H, W, C, Ho, Wo, y);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

static int check_bottleneck(const vdk_bottleneck_net* n) {
  VDK_REQUIRE(n, "vdk_bottleneck: null network");
  VDK_REQUIRE(n->image_size > 0 && n->image_size % 32 == 0, "vdk_bottleneck: image_size must be a multiple of 32 (got %d)",
              n->image_size);
  VDK_REQUIRE(n->feat_dim > 0 && n->feat_dim % 8 == 0, "vdk_bottleneck: feat_dim must be a multiple of 8");
  VDK_REQUIRE(n->width >= 64 && n->width % 64 == 0 && n->width <= 512, "vdk_bottleneck: width must be 64..512 in steps of 64 (got %d)",
              n->width);
  VDK_REQUIRE(n->cardinality >= 1, "vdk_bottleneck: cardinality must be >= 1");
  if (n->cardinality > 1) {
    VDK_REQUIRE(n->width % 128 == 0 && n->width % n->cardinality == 0 && 128 % (n->width / n->cardinality) == 0,
                "vdk_bottleneck: grouped conv2 needs width a multiple of 128 and channels per group dividing 128 (width=%d, "
                "cardinality=%d)", n->width, n->cardinality);
  }
  VDK_REQUIRE(n->stem_pool == VDK_STEM_POOL_PAD1 || n->stem_pool == VDK_STEM_POOL_CEIL, "vdk_bottleneck: bad stem_pool %d",
              n->stem_pool);
  VDK_REQUIRE(!(n->stride_on_conv1 && n->avg_down), "vdk_bottleneck: stride_on_conv1 with avg_down is not a timm model");
  int nb = 0;
  for (int s = 0; s < 4; ++s) {
    VDK_REQUIRE(n->depths[s] >= 1, "vdk_bottleneck: every stage needs at least one block");
    nb += n->depths[s];
  }
  VDK_REQUIRE(nb <= VDK_RESNET_MAX_BLOCKS, "vdk_bottleneck: too many blocks (%d)", nb);
  for (int i = 0; i < (n->deep_stem ? 3 : 1); ++i) VDK_REQUIRE(n->stem[i].w && n->stem[i].b, "vdk_bottleneck: missing stem weights");
  int first = 0;
  for (int s = 0; s < 4; ++s) {
    for (int j = 0; j < n->depths[s]; ++j) {
      const vdk_bottleneck_block& b = n->blocks[first + j];
      VDK_REQUIRE(b.conv1.w && b.conv1.b && b.conv2.w && b.conv2.b && b.conv3.w && b.conv3.b, "vdk_bottleneck: block %d misses a conv",
                  first + j);
      if (b.se_fc1_w) {
        const int C = 256 << s;
        VDK_REQUIRE(b.se_fc1_b && b.se_fc2_w && b.se_fc2_b, "vdk_bottleneck: block %d has an incomplete SE module", first + j);
        VDK_REQUIRE(n->se_reduction > 0 && C % n->se_reduction == 0 && C / n->se_reduction >= 1,
                    "vdk_bottleneck: se_reduction %d must divide C=%d", n->se_reduction, C);
        VDK_REQUIRE((reinterpret_cast<uintptr_t>(b.se_fc1_w) & 3) == 0, "vdk_bottleneck: SE weights must be fp32-aligned");
      }
    }
    VDK_REQUIRE(n->blocks[first].down.w && n->blocks[first].down.b, "vdk_bottleneck: the first block of stage %d needs its shortcut conv", s);
    first += n->depths[s];
  }
  VDK_REQUIRE(n->neck_w && n->neck_b, "vdk_bottleneck: missing neck");
  return VDK_OK;
}

static ResnetSizes bottleneck_sizes(const vdk_bottleneck_net* n, int batch) {
  const size_t S = n->image_size, B = batch;
  ResnetSizes z;
  z.act = B * (S / 2) * (S / 2) * 64;
  size_t hin = S / 4;
  for (int s = 0; s < 4; ++s) {
    const size_t width = static_cast<size_t>(n->width) << s, out = static_cast<size_t>(256) << s;
    const size_t ho = s == 0 ? hin : hin / 2;
    z.act = std::max(z.act, B * hin * hin * width);  // conv1 of the first block at the input resolution (stride on conv2)
    z.act = std::max(z.act, B * ho * ho * out);
    hin = ho;
  }
  z.rows = B * (S / 2) * (S / 2) * (n->deep_stem ? 320 : 192);
  return z;
}

}  // namespace vdk

extern "C" size_t vdk_bottleneck_workspace_bytes(const vdk_bottleneck_net* net, int batch) {
  if (!net || batch <= 0 || net->image_size <= 0 || net->width <= 0) return 0;
  const ResnetSizes z = bottleneck_sizes(net, batch);
  // x, shortcut, t1 (conv1 out, conv3 out before the SE gate, neck slabs), t2 (conv2 out), stem patch rows, SE mean + gate
  return 4 * up256(z.act * 2) + up256(z.rows * 2) + 2 * up256(static_cast<size_t>(batch) * 2048 * 4) + 1024;
}

extern "C" int vdk_bottleneck_forward(const vdk_bottleneck_net* net, const float* images, int batch, int l2_normalize,
                                      float* embeddings, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_bottleneck(net);
  if (rc != VDK_OK) return rc;
  VDK_REQUIRE(images && embeddings && batch > 0, "vdk_bottleneck_forward: null image/embedding buffer");
  VDK_REQUIRE(workspace && workspace_bytes >= vdk_bottleneck_workspace_bytes(net, batch), "vdk_bottleneck_forward: workspace too small");
  VDK_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "vdk_bottleneck_forward: workspace must be 256-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const ResnetSizes z = bottleneck_sizes(net, batch);
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  __nv_bfloat16* buf[4];
  for (int i = 0; i < 4; ++i) {
    buf[i] = reinterpret_cast<__nv_bfloat16*>(ws);
    ws += up256(z.act * 2);
  }
  __nv_bfloat16* rows = reinterpret_cast<__nv_bfloat16*>(ws);
  ws += up256(z.rows * 2);
  float* se_mean = reinterpret_cast<float*>(ws);
  float* se_s = reinterpret_cast<float*>(ws + up256(static_cast<size_t>(batch) * 2048 * 4));
  __nv_bfloat16 *x = buf[0], *sc = buf[1], *t1 = buf[2], *t2 = buf[3];

  auto conv = [&](const void* in, int H, int Cin, const vdk_resnet_conv& c, int Cout, int k, int stride, int pad, int epi,
                  const void* res, void* out, int groups = 1) -> int {
    vdk_conv_desc d{};
    d.x = in; d.w = c.w; d.bias = c.b; d.residual = res; d.y = out;
    d.B = batch; d.H = H; d.W = H; d.Cin = Cin; d.Cout = Cout;
    d.kernel = k; d.stride = stride; d.pad = pad; d.epilogue = epi;
    return groups > 1 ? conv_grouped_run(d, groups, s) : conv_run(d, s);
  };
  auto stem_conv = [&](auto* in, bool nchw, int H, int C, int k, int stride, const vdk_resnet_conv& c, int Cout, void* out) -> int {
    const int pad = k / 2, Ho = (H + 2 * pad - k) / stride + 1;
    const int K = k * k * C, Kp = (K + 63) / 64 * 64;
    const int64_t threads = static_cast<int64_t>(batch) * Ho * Ho * (Kp / 8);
    using T = std::remove_cv_t<std::remove_pointer_t<decltype(in)>>;
    if (nchw) patch_rows_kernel<T, true><<<grid_for(threads), 256, 0, s>>>(in, batch, H, H, C, k, stride, pad, Ho, Ho, K, Kp, rows);
    else patch_rows_kernel<T, false><<<grid_for(threads), 256, 0, s>>>(in, batch, H, H, C, k, stride, pad, Ho, Ho, K, Kp, rows);
    VDK_CUDA_OK(cudaGetLastError());
    return conv(rows, Ho, Kp, c, Cout, 1, 1, 0, VDK_EPI_RELU, nullptr, out);
  };

  const int S = net->image_size;
  int H = S / 2;
  if (net->deep_stem) {
    if ((rc = stem_conv(images, true, S, 3, 3, 2, net->stem[0], 32, t1)) != VDK_OK) return rc;
    if ((rc = stem_conv(static_cast<const __nv_bfloat16*>(t1), false, H, 32, 3, 1, net->stem[1], 32, t2)) != VDK_OK) return rc;
    if ((rc = stem_conv(static_cast<const __nv_bfloat16*>(t2), false, H, 32, 3, 1, net->stem[2], 64, sc)) != VDK_OK) return rc;
  } else {
    if ((rc = stem_conv(images, true, S, 3, 7, 2, net->stem[0], 64, sc)) != VDK_OK) return rc;
  }
  // ---- max pool 3x3/s2: padding 1, or ceil mode without padding (the same H / 2 output on the even stem map) ----
  if ((rc = stem_pool_run(sc, batch, H, H, 64, net->stem_pool, x, s)) != VDK_OK) return rc;
  H /= 2;
  // ---- stages: conv1 1x1 + ReLU, conv2 3x3 (grouped when cardinality > 1) + ReLU, conv3 1x1 + shortcut + ReLU, or
  // with SE: conv3 + bias, then ReLU(conv3 * gate + shortcut) ----
  int C = 64, blk = 0;
  for (int st = 0; st < 4; ++st) {
    const int width = net->width << st, out = 256 << st;
    for (int j = 0; j < net->depths[st]; ++j, ++blk) {
      const vdk_bottleneck_block& b = net->blocks[blk];
      const int stride = (st > 0 && j == 0) ? 2 : 1, Ho = H / stride;
      const int s1 = net->stride_on_conv1 ? stride : 1, s2 = net->stride_on_conv1 ? 1 : stride;
      if ((rc = conv(x, H, C, b.conv1, width, 1, s1, 0, VDK_EPI_RELU, nullptr, t1)) != VDK_OK) return rc;
      if ((rc = conv(t1, H / s1, width, b.conv2, width, 3, s2, 1, VDK_EPI_RELU, nullptr, t2, net->cardinality)) != VDK_OK) return rc;
      __nv_bfloat16* res = x;
      if (b.down.w) {
        const int k = (net->avg_down && stride == 2) ? 2 : 1;
        if ((rc = conv(x, H, C, b.down, out, k, stride, 0, VDK_EPI_NONE, nullptr, sc)) != VDK_OK) return rc;
        res = sc;
      }
      if (b.se_fc1_w) {
        if ((rc = conv(t2, Ho, width, b.conv3, out, 1, 1, 0, VDK_EPI_NONE, nullptr, t1)) != VDK_OK) return rc;
        if ((rc = se_gate(t1, batch, Ho * Ho, out, out / net->se_reduction, b.se_fc1_w, b.se_fc1_b, b.se_fc2_w, b.se_fc2_b, se_mean,
                          se_s, res, s)) != VDK_OK)
          return rc;
      } else if ((rc = conv(t2, Ho, width, b.conv3, out, 1, 1, 0, VDK_EPI_RESIDUAL_RELU, res, res)) != VDK_OK) {
        return rc;
      }
      if (res == sc) std::swap(x, sc);
      H = Ho;
      C = out;
    }
  }
  return launch_neck(x, batch, H * H * C, net->feat_dim, net->neck_w, net->neck_b, l2_normalize, reinterpret_cast<float*>(t1),
                     up256(z.act * 2), embeddings, s);
}

namespace vdk {

int launch_patch_rows_nhwc(const __nv_bfloat16* x, int B, int H, int W, int C, int k, int stride, int pad, int Ho, int Wo, int Kp,
                           __nv_bfloat16* out, cudaStream_t s) {
  const int64_t threads = static_cast<int64_t>(B) * Ho * Wo * (Kp / 8);
  patch_rows_kernel<__nv_bfloat16, false><<<grid_for(threads), 256, 0, s>>>(x, B, H, W, C, k, stride, pad, Ho, Wo, k * k * C, Kp, out);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

int launch_stem_maxpool(const __nv_bfloat16* x, int B, int H, int W, int C, __nv_bfloat16* y, cudaStream_t s) {
  return stem_pool_run(x, B, H, W, C, VDK_STEM_POOL_PAD1, y, s);
}

}  // namespace vdk

// Kernel-level entry points of the pieces above, for their tests.
extern "C" int vdk_stem_maxpool(const void* x, int B, int H, int W, int C, int mode, void* y, void* stream) {
  VDK_REQUIRE(x && y && B > 0 && H >= 3 && W >= 3 && C > 0 && C % 8 == 0, "vdk_stem_maxpool: bad arguments");
  VDK_REQUIRE(mode == VDK_STEM_POOL_PAD1 || mode == VDK_STEM_POOL_CEIL, "vdk_stem_maxpool: bad mode %d", mode);
  VDK_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0, "vdk_stem_maxpool: 16-byte alignment");
  return stem_pool_run(static_cast<const __nv_bfloat16*>(x), B, H, W, C, mode, static_cast<__nv_bfloat16*>(y),
                       reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vdk_se_gate(const void* y, int B, int HW, int C, int rd, const float* fc1_w, const float* fc1_b,
                           const float* fc2_w, const float* fc2_b, float* mean, float* gate, void* residual, void* stream) {
  VDK_REQUIRE(y && fc1_w && fc1_b && fc2_w && fc2_b && mean && gate && residual, "vdk_se_gate: null operand");
  VDK_REQUIRE(B > 0 && HW > 0 && C > 0 && C % 64 == 0 && C <= 2048 && rd >= 1 && rd <= C, "vdk_se_gate: bad shape");
  VDK_REQUIRE(((reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(residual) | reinterpret_cast<uintptr_t>(gate)) & 15) == 0,
              "vdk_se_gate: 16-byte alignment");
  return se_gate(static_cast<const __nv_bfloat16*>(y), B, HW, C, rd, fc1_w, fc1_b, fc2_w, fc2_b, mean, gate,
                 static_cast<__nv_bfloat16*>(residual), reinterpret_cast<cudaStream_t>(stream));
}
