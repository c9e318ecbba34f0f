// effnet.cu — timm 0.9.16 tf_efficientnetv2_s / _m / _l embedding forward for the faceX / CBIR extract path, NHWC bf16,
// every eval BatchNorm folded into its convolution.
//
// Replaces TimmWrapper.forward for EfficientNetV2 backbones (models/faceX/backbone/timm_wrapper.py:16-21, 30-38, 51-54:
// timm EfficientNet with num_classes=0, global_pool='' -> BatchNorm2d -> Flatten -> Linear -> BatchNorm1d) and F.normalize
// (face_model.py:139).
//
// The dense convolutions are vdk_conv2d_ex (gemm.cu: TF-"same" padding, SiLU epilogues, Cin a multiple of 8); the conv_pwl
// projections are vdk_gemm with the SCALE_RESIDUAL epilogue at gamma = 1 (or no epilogue without a shortcut).  Written here:
//   dwconv3_silu  the InvertedResidual's depthwise 3x3 (stride 1 / 2, TF-"same") + bias + SiLU, which also emits the SE mean
//   se_apply      d *= gate before the projection GEMM reads d (one extra read + write of d; see DESIGN §7g)
// The SE excitation is resnet.cu's se_excite_kernel with the SiLU hidden activation, the stem is resnet.cu's patch rows +
// a GEMM, the neck is the ConvNeXt path's (launch_neck).
#include "vdk_host.h"

#include <algorithm>
#include "convnext_internal.h"

namespace vdk {

constexpr int kDwChannels = 32;  // channels per CTA of dwconv3_silu
constexpr int kDwPixelLanes = 64;

// y[b, ho, wo, c] = silu(bias[c] + sum_{dy, dx} w[dy*3 + dx][c] x[b, ho*S - pt + dy, wo*S - pl + dx, c]) (zero outside the
// image), rounded to bf16; mean[b, c] = the sum of the rounded y[b, :, :, c] over the map / (Ho Wo).  One CTA = one image x
// 32 channels, 256 threads = 4 channel vectors of 8 (16-byte loads) x 64 pixel lanes; lane l handles pixels l, l + 64, ...
// in order, then a fixed tree over the 64 lanes: the mean is bit-reproducible.  The taps are fp32 FMAs in (bias, dy, dx)
// order.  At the 7^2 / 14^2 maps of batch 256 the grid is (C / 32) x 256 >= 2048 CTAs.
template <int kStride>
__global__ void __launch_bounds__(256) dwconv3_silu_kernel(const __nv_bfloat16* __restrict__ x, int H, int W, int C, int Ho,
                                                           int Wo, int pt, int pl, const float* __restrict__ w,
                                                           const float* __restrict__ bias, __nv_bfloat16* __restrict__ y,
                                                           float* __restrict__ mean) {
  __shared__ float part[kDwPixelLanes][kDwChannels];
  const int b = blockIdx.y, cv = threadIdx.x & 3, lane = threadIdx.x >> 2;
  const int c0 = blockIdx.x * kDwChannels + cv * 8;
  float wt[9][8], bs[8], sum[8];
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const float4 a = *reinterpret_cast<const float4*>(w + static_cast<int64_t>(t) * C + c0);
    const float4 e = *reinterpret_cast<const float4*>(w + static_cast<int64_t>(t) * C + c0 + 4);
    wt[t][0] = a.x; wt[t][1] = a.y; wt[t][2] = a.z; wt[t][3] = a.w;
    wt[t][4] = e.x; wt[t][5] = e.y; wt[t][6] = e.z; wt[t][7] = e.w;
  }
  {
    const float4 a = *reinterpret_cast<const float4*>(bias + c0);
    const float4 e = *reinterpret_cast<const float4*>(bias + c0 + 4);
    bs[0] = a.x; bs[1] = a.y; bs[2] = a.z; bs[3] = a.w;
    bs[4] = e.x; bs[5] = e.y; bs[6] = e.z; bs[7] = e.w;
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) sum[i] = 0.f;
  const __nv_bfloat16* xb = x + static_cast<int64_t>(b) * H * W * C + c0;
  __nv_bfloat16* yb = y + static_cast<int64_t>(b) * Ho * Wo * C + c0;
  const int HWo = Ho * Wo;
  for (int p = lane; p < HWo; p += kDwPixelLanes) {
    const int ho = p / Wo, wo = p - ho * Wo;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = bs[i];
#pragma unroll
    for (int dy = 0; dy < 3; ++dy) {
      const int ih = ho * kStride - pt + dy;
      if (ih < 0 || ih >= H) continue;
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
        const int iw = wo * kStride - pl + dx;
        if (iw < 0 || iw >= W) continue;
        const uint4 u = *reinterpret_cast<const uint4*>(xb + (static_cast<int64_t>(ih) * W + iw) * C);
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = __bfloat1622float2(h[i]);
          acc[2 * i] = fmaf(wt[dy * 3 + dx][2 * i], f.x, acc[2 * i]);
          acc[2 * i + 1] = fmaf(wt[dy * 3 + dx][2 * i + 1], f.y, acc[2 * i + 1]);
        }
      }
    }
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float v0 = acc[2 * i] / (1.f + __expf(-acc[2 * i]));
      const float v1 = acc[2 * i + 1] / (1.f + __expf(-acc[2 * i + 1]));
      const __nv_bfloat162 hq = __floats2bfloat162_rn(v0, v1);
      ow[i] = *reinterpret_cast<const uint32_t*>(&hq);
      const float2 r = __bfloat1622float2(hq);
      sum[2 * i] += r.x;
      sum[2 * i + 1] += r.y;
    }
    *reinterpret_cast<uint4*>(yb + static_cast<int64_t>(p) * C) = o;
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) part[lane][cv * 8 + i] = sum[i];
  __syncthreads();
  for (int half = kDwPixelLanes / 2; half > 0; half >>= 1) {
    if (lane < half) {
#pragma unroll
      for (int i = 0; i < 8; ++i) part[lane][cv * 8 + i] += part[lane + half][cv * 8 + i];
    }
    __syncthreads();
  }
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) mean[static_cast<int64_t>(b) * C + c0 + i] = part[0][cv * 8 + i] / static_cast<float>(HWo);
  }
}

// d[m, c] = bf16(d[m, c] * gate[m / HW, c]) in place; one thread = 8 channels (16-byte vectors) of one pixel
__global__ void __launch_bounds__(256) se_apply_kernel(__nv_bfloat16* d, const float* __restrict__ gate, int64_t M, int HW, int C) {
  const int cc = C / 8;
  const int64_t total = M * cc;
  for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c8 = static_cast<int>(t % cc);
    const int64_t m = t / cc;
    const int64_t b = m / HW;
    uint4 u = *reinterpret_cast<const uint4*>(d + m * C + c8 * 8);
    const float4 g0 = *reinterpret_cast<const float4*>(gate + b * C + c8 * 8);
    const float4 g1 = *reinterpret_cast<const float4*>(gate + b * C + c8 * 8 + 4);
    const float gv[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __bfloat1622float2(h[i]);
      h[i] = __floats2bfloat162_rn(f.x * gv[2 * i], f.y * gv[2 * i + 1]);
    }
    *reinterpret_cast<uint4*>(d + m * C + c8 * 8) = u;
  }
}

__global__ void fill_kernel(float* p, int n, float v) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) p[i] = v;
}

int launch_se_apply(__nv_bfloat16* d, const float* gate, int64_t M, int HW, int C, cudaStream_t s) {
  se_apply_kernel<<<grid_for(M * (C / 8)), 256, 0, s>>>(d, gate, M, HW, C);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

int launch_fill(float* p, int n, float v, cudaStream_t s) {
  fill_kernel<<<1, 256, 0, s>>>(p, n, v);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

static int dw_run(const __nv_bfloat16* x, int B, int H, int W, int C, int stride, const float* w, const float* b,
                  __nv_bfloat16* y, float* mean, cudaStream_t s) {
  int pt, pb, pl, pr;
  same_pad(H, 3, stride, pt, pb);
  same_pad(W, 3, stride, pl, pr);
  const int Ho = (H + stride - 1) / stride, Wo = (W + stride - 1) / stride;
  ProfScope prof(kProfDepthwise, 2.0 * 9 * B * Ho * Wo * C, 2.0 * B * (static_cast<double>(H) * W + Ho * Wo) * C, s);
  const dim3 grid(C / kDwChannels, B);
  if (stride == 1) dwconv3_silu_kernel<1><<<grid, 256, 0, s>>>(x, H, W, C, Ho, Wo, pt, pl, w, b, y, mean);
  else dwconv3_silu_kernel<2><<<grid, 256, 0, s>>>(x, H, W, C, Ho, Wo, pt, pl, w, b, y, mean);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

static int se_run(__nv_bfloat16* d, const float* mean, int B, int HW, int C, int rd, const float* w1, const float* b1,
                  const float* w2, const float* b2, float* gate, cudaStream_t s) {
  ProfScope prof(kProfOther, 4.0 * B * C * rd + static_cast<double>(B) * HW * C, 4.0 * B * static_cast<double>(HW) * C, s);
  int rc = launch_se_excite(mean, B, C, rd, 1, 0, w1, b1, w2, b2, gate, s);
  if (rc != VDK_OK) return rc;
  return launch_se_apply(d, gate, static_cast<int64_t>(B) * HW, HW, C, s);
}

static int check_effnet(const vdk_effnetv2_net* n) {
  VDK_REQUIRE(n, "vdk_effnetv2: null network");
  VDK_REQUIRE(n->image_size > 0 && n->image_size % 32 == 0, "vdk_effnetv2: image_size must be a multiple of 32 (got %d)",
              n->image_size);
  VDK_REQUIRE(n->feat_dim > 0 && n->feat_dim % 8 == 0, "vdk_effnetv2: feat_dim must be a multiple of 8");
  VDK_REQUIRE(n->num_blocks >= 1 && n->num_blocks <= VDK_EFFNETV2_MAX_BLOCKS, "vdk_effnetv2: num_blocks must be 1..%d (got %d)",
              VDK_EFFNETV2_MAX_BLOCKS, n->num_blocks);
  VDK_REQUIRE(n->stem_ch > 0 && n->stem_ch % 8 == 0 && n->head_ch > 0 && n->head_ch % 8 == 0,
              "vdk_effnetv2: stem_ch and head_ch must be positive multiples of 8");
  VDK_REQUIRE(n->stem.w && n->stem.b && n->head.w && n->head.b && n->neck_w && n->neck_b, "vdk_effnetv2: missing stem, head or neck");
  int cin = n->stem_ch, strided = 0;
  for (int i = 0; i < n->num_blocks; ++i) {
    const vdk_effnetv2_block& b = n->blocks[i];
    VDK_REQUIRE(b.kind >= VDK_EFFNET_CN && b.kind <= VDK_EFFNET_IR, "vdk_effnetv2: block %d has bad kind %d", i, b.kind);
    VDK_REQUIRE(b.stride == 1 || b.stride == 2, "vdk_effnetv2: block %d stride must be 1 or 2", i);
    VDK_REQUIRE(b.cin == cin, "vdk_effnetv2: block %d takes %d channels, the previous block gives %d", i, b.cin, cin);
    VDK_REQUIRE(b.cout > 0 && b.cout % 8 == 0 && b.mid > 0 && b.mid % 8 == 0, "vdk_effnetv2: block %d widths must be multiples of 8", i);
    VDK_REQUIRE(b.conv.w && b.conv.b, "vdk_effnetv2: block %d misses its first conv", i);
    if (b.kind == VDK_EFFNET_CN) VDK_REQUIRE(b.mid == b.cout, "vdk_effnetv2: CN block %d needs mid == cout", i);
    if (b.kind != VDK_EFFNET_CN) VDK_REQUIRE(b.conv_pwl.w && b.conv_pwl.b, "vdk_effnetv2: block %d misses conv_pwl", i);
    if (b.kind == VDK_EFFNET_IR) {
      VDK_REQUIRE(b.mid % kDwChannels == 0 && b.mid <= 4096, "vdk_effnetv2: IR block %d mid must be a multiple of 32, <= 4096", i);
      VDK_REQUIRE(b.se_rd >= 1 && b.se_rd <= b.mid, "vdk_effnetv2: IR block %d has bad se_rd %d", i, b.se_rd);
      VDK_REQUIRE(b.dw_w && b.dw_b && b.se_w1 && b.se_b1 && b.se_w2 && b.se_b2, "vdk_effnetv2: IR block %d misses weights", i);
      VDK_REQUIRE(((reinterpret_cast<uintptr_t>(b.dw_w) | reinterpret_cast<uintptr_t>(b.dw_b)) & 15) == 0,
                  "vdk_effnetv2: depthwise weights must be 16-byte aligned");
    }
    strided += b.stride == 2;
    cin = b.cout;
  }
  // the stem halves the map, four stride-2 blocks make S / 32: the neck's K = (S / 32)^2 * head_ch
  VDK_REQUIRE(strided == 4, "vdk_effnetv2: the blocks must hold exactly four stride-2 blocks (got %d)", strided);
  return VDK_OK;
}

struct EffnetSizes {
  size_t act;      // elements of the largest activation map
  size_t rows;     // elements of the stem's patch rows
  int max_mid;     // widest SE gate
  int max_cout;    // widest shortcut projection (the gamma = 1 vector)
};

static EffnetSizes effnet_sizes(const vdk_effnetv2_net* n, int batch) {
  const size_t B = batch;
  size_t H = n->image_size / 2;
  EffnetSizes z{B * H * H * n->stem_ch, B * H * H * 64, 8, 8};
  for (int i = 0; i < n->num_blocks; ++i) {
    const vdk_effnetv2_block& b = n->blocks[i];
    const size_t Ho = (H + b.stride - 1) / b.stride;
    z.act = std::max(z.act, B * Ho * Ho * b.cout);
    if (b.kind == VDK_EFFNET_ER) z.act = std::max(z.act, B * Ho * Ho * b.mid);
    if (b.kind == VDK_EFFNET_IR) {
      z.act = std::max(z.act, B * H * H * b.mid);
      z.max_mid = std::max(z.max_mid, b.mid);
    }
    z.max_cout = std::max(z.max_cout, b.cout);
    H = Ho;
  }
  z.act = std::max(z.act, B * H * H * n->head_ch);
  return z;
}

}  // namespace vdk

using namespace vdk;

extern "C" size_t vdk_effnetv2_workspace_bytes(const vdk_effnetv2_net* net, int batch) {
  if (!net || batch <= 0 || net->image_size <= 0 || net->num_blocks < 1 || net->num_blocks > VDK_EFFNETV2_MAX_BLOCKS) return 0;
  const EffnetSizes z = effnet_sizes(net, batch);
  // x (block input), y (block output), e (expanded), d (depthwise output, neck slabs), stem patch rows, SE mean + gate, ones
  return 4 * up256(z.act * 2) + up256(z.rows * 2) + 2 * up256(static_cast<size_t>(batch) * z.max_mid * 4) +
         up256(static_cast<size_t>(z.max_cout) * 4) + 1024;
}

extern "C" int vdk_effnetv2_forward(const vdk_effnetv2_net* net, const float* images, int batch, int l2_normalize,
                                    float* embeddings, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_effnet(net);
  if (rc != VDK_OK) return rc;
  VDK_REQUIRE(images && embeddings && batch > 0, "vdk_effnetv2_forward: null image/embedding buffer");
  VDK_REQUIRE(workspace && workspace_bytes >= vdk_effnetv2_workspace_bytes(net, batch), "vdk_effnetv2_forward: workspace too small");
  VDK_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "vdk_effnetv2_forward: workspace must be 256-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const EffnetSizes z = effnet_sizes(net, batch);
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  __nv_bfloat16* buf[4];
  for (int i = 0; i < 4; ++i) {
    buf[i] = reinterpret_cast<__nv_bfloat16*>(ws);
    ws += up256(z.act * 2);
  }
  __nv_bfloat16* rows = reinterpret_cast<__nv_bfloat16*>(ws);
  ws += up256(z.rows * 2);
  float* se_mean = reinterpret_cast<float*>(ws);
  ws += up256(static_cast<size_t>(batch) * z.max_mid * 4);
  float* se_gate = reinterpret_cast<float*>(ws);
  ws += up256(static_cast<size_t>(batch) * z.max_mid * 4);
  float* ones = reinterpret_cast<float*>(ws);
  __nv_bfloat16 *x = buf[0], *y = buf[1], *e = buf[2], *d = buf[3];
  if ((rc = launch_fill(ones, z.max_cout, 1.f, s)) != VDK_OK) return rc;

  // TF-"same" k x k convolution on vdk_conv2d_ex
  auto conv = [&](const void* in, int H, int Cin, const vdk_resnet_conv& c, int Cout, int k, int stride, int epi, const void* res,
                  void* out) -> int {
    vdk_conv_ex_desc cd{};
    cd.x = in; cd.w = c.w; cd.bias = c.b; cd.residual = res; cd.y = out;
    cd.B = batch; cd.H = H; cd.W = H; cd.Cin = Cin; cd.Cout = Cout; cd.kernel = k; cd.stride = stride; cd.epilogue = epi;
    same_pad(H, k, stride, cd.pad_h_lo, cd.pad_h_hi);
    same_pad(H, k, stride, cd.pad_w_lo, cd.pad_w_hi);
    return conv_ex_run(cd, s);
  };
  // conv_pwl: [M, mid] x [cout, mid]^T + bias (+ the shortcut through SCALE_RESIDUAL at gamma = 1)
  auto project = [&](const __nv_bfloat16* a, int M, int mid, const vdk_resnet_conv& c, int cout, const __nv_bfloat16* res,
                     __nv_bfloat16* out) -> int {
    vdk_gemm_desc g{};
    g.A = a; g.B = c.w; g.D = out;
    g.M = M; g.N = cout; g.K = mid; g.lda = mid; g.ldb = mid; g.ldd = cout;
    g.in_dtype = VDK_DTYPE_BF16; g.out_dtype = VDK_DTYPE_BF16; g.bias = c.b; g.split_k = 1;
    g.epilogue = res ? VDK_EPI_SCALE_RESIDUAL : VDK_EPI_NONE;
    if (res) {
      g.gamma = ones; g.residual = res; g.ldr = cout;
    }
    return gemm_run(g, s);
  };

  const int S = net->image_size;
  int H = S / 2;
  // ---- stem: conv 3x3/s2 with TF-"same" (0, 1) padding on the even image = unpadded patch rows with Ho = S / 2 (the last
  // row / column of taps falls outside the image and reads zero), a GEMM with the SiLU epilogue ----
  if ((rc = launch_patch_rows_nchw(images, batch, S, S, 3, 3, 2, 0, H, H, 64, rows, s)) != VDK_OK) return rc;
  if ((rc = conv(rows, H, 64, net->stem, net->stem_ch, 1, 1, VDK_EPI_SILU, nullptr, x)) != VDK_OK) return rc;
  for (int i = 0; i < net->num_blocks; ++i) {
    const vdk_effnetv2_block& b = net->blocks[i];
    const int Ho = (H + b.stride - 1) / b.stride, M = batch * Ho * Ho;
    const bool skip = b.stride == 1 && b.cin == b.cout;
    if (b.kind == VDK_EFFNET_CN) {
      if ((rc = conv(x, H, b.cin, b.conv, b.cout, 3, b.stride, skip ? VDK_EPI_SILU_RESIDUAL : VDK_EPI_SILU, skip ? x : nullptr, y)) != VDK_OK)
        return rc;
    } else if (b.kind == VDK_EFFNET_ER) {
      if ((rc = conv(x, H, b.cin, b.conv, b.mid, 3, b.stride, VDK_EPI_SILU, nullptr, e)) != VDK_OK) return rc;
      if ((rc = project(e, M, b.mid, b.conv_pwl, b.cout, skip ? x : nullptr, y)) != VDK_OK) return rc;
    } else {
      if ((rc = conv(x, H, b.cin, b.conv, b.mid, 1, 1, VDK_EPI_SILU, nullptr, e)) != VDK_OK) return rc;
      if ((rc = dw_run(e, batch, H, H, b.mid, b.stride, b.dw_w, b.dw_b, d, se_mean, s)) != VDK_OK) return rc;
      if ((rc = se_run(d, se_mean, batch, Ho * Ho, b.mid, b.se_rd, b.se_w1, b.se_b1, b.se_w2, b.se_b2, se_gate, s)) != VDK_OK)
        return rc;
      if ((rc = project(d, M, b.mid, b.conv_pwl, b.cout, skip ? x : nullptr, y)) != VDK_OK) return rc;
    }
    std::swap(x, y);
    H = Ho;
  }
  const int c_last = net->blocks[net->num_blocks - 1].cout;
  if ((rc = conv(x, H, c_last, net->head, net->head_ch, 1, 1, VDK_EPI_SILU, nullptr, e)) != VDK_OK) return rc;
  // ---- neck: BN2d -> Flatten -> Linear -> BN1d folded into one split-K GEMM over the (h, w, c) features ----
  return launch_neck(e, batch, H * H * net->head_ch, net->feat_dim, net->neck_w, net->neck_b, l2_normalize,
                     reinterpret_cast<float*>(d), up256(z.act * 2), embeddings, s);
}

// Kernel-level entry points of the pieces above, for their tests.
extern "C" int vdk_dwconv3_silu(const void* x, int B, int H, int W, int C, int stride, const float* w, const float* b, void* y,
                                float* mean, void* stream) {
  VDK_REQUIRE(x && w && b && y && mean, "vdk_dwconv3_silu: null operand");
  VDK_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && C % kDwChannels == 0 && C <= 4096 && (stride == 1 || stride == 2),
              "vdk_dwconv3_silu: bad shape B=%d H=%d W=%d C=%d stride=%d", B, H, W, C, stride);
  VDK_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(w) |
                reinterpret_cast<uintptr_t>(b)) & 15) == 0,
              "vdk_dwconv3_silu: 16-byte alignment");
  return dw_run(static_cast<const __nv_bfloat16*>(x), B, H, W, C, stride, w, b, static_cast<__nv_bfloat16*>(y), mean,
                reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vdk_effnet_se(void* d, const float* mean, int B, int HW, int C, int rd, const float* w1, const float* b1,
                             const float* w2, const float* b2, float* gate, void* stream) {
  VDK_REQUIRE(d && mean && w1 && b1 && w2 && b2 && gate, "vdk_effnet_se: null operand");
  VDK_REQUIRE(B > 0 && HW > 0 && C > 0 && C % 8 == 0 && C <= 4096 && rd >= 1 && rd <= C, "vdk_effnet_se: bad shape");
  VDK_REQUIRE(((reinterpret_cast<uintptr_t>(d) | reinterpret_cast<uintptr_t>(gate)) & 15) == 0, "vdk_effnet_se: 16-byte alignment");
  return se_run(static_cast<__nv_bfloat16*>(d), mean, B, HW, C, rd, w1, b1, w2, b2, gate, reinterpret_cast<cudaStream_t>(stream));
}
