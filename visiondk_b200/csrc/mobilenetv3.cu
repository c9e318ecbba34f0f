// mobilenetv3.cu — timm 0.9.16 MobileNetV3 (large / small, full / minimal, TF-"same" or symmetric padding) embedding
// forward for the faceX / CBIR extract path, NHWC bf16, every eval BatchNorm folded into its convolution.
//
// Replaces TimmWrapper.forward for MobileNetV3 backbones (models/faceX/backbone/timm_wrapper.py:16-21, 30-38, 51-54: timm
// MobileNetV3 with num_classes=0, global_pool='' -> BatchNorm2d -> Flatten -> Linear -> BatchNorm1d) and F.normalize
// (face_model.py:139).
//
// The stem, the expansions, the CN 1x1 and conv_head are vdk_conv2d_ex (gemm.cu) with the ReLU or hard-swish epilogue;
// the projections are vdk_gemm with K = mid and, with a shortcut, SCALE_RESIDUAL at gamma = 1.  Written here:
//   dwconv_mnv3  the depthwise k x k (k 3 / 5, stride 1 / 2, separate low / high pads) + bias + ReLU / hard-swish for any
//                multiple-of-8 width, which also emits the SE mean
// The SE excitation is resnet.cu's se_excite_kernel with the ReLU hidden activation and the hard-sigmoid gate, applied by
// effnet.cu's se_apply; the neck is the ConvNeXt path's (launch_neck).
#include "vdk_host.h"

#include <algorithm>
#include <type_traits>
#include "convnext_internal.h"
#include "vdk_ptx.cuh"

namespace vdk {

constexpr int kMnv3Threads = 256;

// y[b, ho, wo, c] = act(bias[c] + sum_{dy, dx} w[dy*K + dx][c] x[b, ho*S - pt + dy, wo*S - pl + dx, c]) (zero outside the
// image), rounded to bf16.  One thread = CPT channels (one 16- or 4-byte vector) of a pixel: 8 for 3x3 (72 tap registers),
// 2 for 5x5, so that the 25 taps stay in registers (50 floats) under the 128-register cap of two 256-thread CTAs per SM
// (at 4 channels the 100 taps spill).  A CTA = one image x CV channel vectors (cv fastest, so a warp reads
// consecutive channels of consecutive pixels) x `lanes` pixel lanes, CV * lanes <= 256; CV = ceil(G / ceil(G / 32)) for G
// vectors per pixel (capping CV at 8 instead, for more pixel lanes per CTA, measured slower on every SE shape), and the
// 2-vector maps of width 16 get 128 lanes.  Grid (ceil(G / CV), B, P): blockIdx.z takes the z-th of P equal
// pixel ranges, which keeps the narrow, large maps' grids over two waves.  Lane l handles pixels p0 + l, p0 + l + lanes,
// ... in order; the taps are fp32 FMAs in (bias, dy, dx) order.
// mean (P == 1 only) [b, c] = the sum of the rounded y over the map / (Ho Wo): per-lane sums in pixel order, then the lanes
// folded in a fixed tree (lanes >= the largest power of two <= lanes first): bit-reproducible, no atomics.
template <int K, int S, int CPT, int ACT>
__global__ void __launch_bounds__(kMnv3Threads, 2) dwconv_mnv3_kernel(const __nv_bfloat16* __restrict__ x, int H, int W, int C,
                                                                   int Ho, int Wo, int pt, int pl, int CV, int lanes, int chunk,
                                                                   const float* __restrict__ w, const float* __restrict__ bias,
                                                                   __nv_bfloat16* __restrict__ y, float* __restrict__ mean) {
  __shared__ float part[kMnv3Threads * 8];  // [lanes][CV * CPT]
  const int b = blockIdx.y, cv = threadIdx.x % CV, lane = threadIdx.x / CV;
  const int c0 = (blockIdx.x * CV + cv) * CPT;
  const bool active = c0 < C;
  float sum[CPT];
#pragma unroll
  for (int i = 0; i < CPT; ++i) sum[i] = 0.f;
  if (active) {
    float wt[K * K][CPT], bs[CPT];
#pragma unroll
    for (int t = 0; t < K * K; ++t) {
#pragma unroll
      for (int q = 0; q < CPT; q += 2) {
        const float2 a = *reinterpret_cast<const float2*>(w + static_cast<int64_t>(t) * C + c0 + q);
        wt[t][q] = a.x; wt[t][q + 1] = a.y;
      }
    }
#pragma unroll
    for (int q = 0; q < CPT; q += 2) {
      const float2 a = *reinterpret_cast<const float2*>(bias + c0 + q);
      bs[q] = a.x; bs[q + 1] = a.y;
    }
    const __nv_bfloat16* xb = x + static_cast<int64_t>(b) * H * W * C + c0;
    __nv_bfloat16* yb = y + static_cast<int64_t>(b) * Ho * Wo * C + c0;
    const int p0 = blockIdx.z * chunk, p1 = min(p0 + chunk, Ho * Wo);
    using Vec = typename std::conditional<CPT == 8, uint4, typename std::conditional<CPT == 4, uint2, uint32_t>::type>::type;
    for (int p = p0 + lane; p < p1; p += lanes) {
      const int ho = p / Wo, wo = p - ho * Wo;
      float acc[CPT];
#pragma unroll
      for (int i = 0; i < CPT; ++i) acc[i] = bs[i];
#pragma unroll
      for (int dy = 0; dy < K; ++dy) {
        const int ih = ho * S - pt + dy;
        if (ih < 0 || ih >= H) continue;
#pragma unroll
        for (int dx = 0; dx < K; ++dx) {
          const int iw = wo * S - pl + dx;
          if (iw < 0 || iw >= W) continue;
          const Vec u = *reinterpret_cast<const Vec*>(xb + (static_cast<int64_t>(ih) * W + iw) * C);
          const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
          for (int i = 0; i < CPT / 2; ++i) {
            const float2 f = __bfloat1622float2(h[i]);
            acc[2 * i] = fmaf(wt[dy * K + dx][2 * i], f.x, acc[2 * i]);
            acc[2 * i + 1] = fmaf(wt[dy * K + dx][2 * i + 1], f.y, acc[2 * i + 1]);
          }
        }
      }
      Vec o;
      uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
      for (int i = 0; i < CPT / 2; ++i) {
        float v0 = acc[2 * i], v1 = acc[2 * i + 1];
        if (ACT == VDK_ACT_HARDSWISH) {
          v0 = hardswish(v0);
          v1 = hardswish(v1);
        } else {
          v0 = fmaxf(v0, 0.f);
          v1 = fmaxf(v1, 0.f);
        }
        const __nv_bfloat162 hq = __floats2bfloat162_rn(v0, v1);
        ow[i] = *reinterpret_cast<const uint32_t*>(&hq);
        const float2 r = __bfloat1622float2(hq);
        sum[2 * i] += r.x;
        sum[2 * i + 1] += r.y;
      }
      *reinterpret_cast<Vec*>(yb + static_cast<int64_t>(p) * C) = o;
    }
  }
  if (mean == nullptr) return;  // uniform over the grid
  const int row = CV * CPT;
#pragma unroll
  for (int i = 0; i < CPT; ++i) part[lane * row + cv * CPT + i] = sum[i];
  __syncthreads();
  int pow2 = 1;
  while (pow2 * 2 <= lanes) pow2 *= 2;
  if (lane < lanes - pow2) {
#pragma unroll
    for (int i = 0; i < CPT; ++i) part[lane * row + cv * CPT + i] += part[(lane + pow2) * row + cv * CPT + i];
  }
  __syncthreads();
  for (int half = pow2 / 2; half > 0; half >>= 1) {
    if (lane < half) {
#pragma unroll
      for (int i = 0; i < CPT; ++i) part[lane * row + cv * CPT + i] += part[(lane + half) * row + cv * CPT + i];
    }
    __syncthreads();
  }
  if (lane == 0 && active) {
#pragma unroll
    for (int i = 0; i < CPT; ++i) mean[static_cast<int64_t>(b) * C + c0 + i] = part[cv * CPT + i] / static_cast<float>(Ho * Wo);
  }
}

template <int K, int CPT, int ACT>
static void dw_launch(int stride, dim3 grid, int threads, const __nv_bfloat16* x, int H, int W, int C, int Ho, int Wo, int pt,
                      int pl, int CV, int lanes, int chunk, const float* w, const float* b, __nv_bfloat16* y, float* mean,
                      cudaStream_t s) {
  if (stride == 1)
    dwconv_mnv3_kernel<K, 1, CPT, ACT><<<grid, threads, 0, s>>>(x, H, W, C, Ho, Wo, pt, pl, CV, lanes, chunk, w, b, y, mean);
  else
    dwconv_mnv3_kernel<K, 2, CPT, ACT><<<grid, threads, 0, s>>>(x, H, W, C, Ho, Wo, pt, pl, CV, lanes, chunk, w, b, y, mean);
}

static void dw_pads(int H, int k, int stride, int pad, int& lo, int& hi) {
  if (pad == VDK_PAD_SAME) same_pad(H, k, stride, lo, hi);
  else lo = hi = k / 2;
}

static int dw_run(const __nv_bfloat16* x, int B, int H, int W, int C, int k, int stride, int pad, int act, const float* w,
                  const float* b, __nv_bfloat16* y, float* mean, cudaStream_t s) {
  int pt, pb, pl, pr;
  dw_pads(H, k, stride, pad, pt, pb);
  dw_pads(W, k, stride, pad, pl, pr);
  const int Ho = (H + pt + pb - k) / stride + 1, Wo = (W + pl + pr - k) / stride + 1;
  const int cpt = k == 3 ? 8 : 2, G = C / cpt;
  const int nx = (G + 31) / 32, CV = (G + nx - 1) / nx, lanes = kMnv3Threads / CV;
  // without a mean, split the map until the grid holds ~2 waves of 8 CTAs per SM, keeping >= 4 pixels per lane
  int P = 1;
  if (mean == nullptr) {
    const int64_t ctas = static_cast<int64_t>(nx) * B;
    const int want = static_cast<int>(std::min<int64_t>((2 * 132 * 8 + ctas - 1) / ctas, 1 << 16));
    P = std::max(1, std::min(want, Ho * Wo / (4 * lanes)));
  }
  const int chunk = (Ho * Wo + P - 1) / P;
  P = (Ho * Wo + chunk - 1) / chunk;
  ProfScope prof(kProfDepthwise, 2.0 * k * k * B * Ho * Wo * C, 2.0 * B * (static_cast<double>(H) * W + Ho * Wo) * C, s);
  const dim3 grid(nx, B, P);
  const int threads = CV * lanes;
  if (k == 3) {
    if (act == VDK_ACT_HARDSWISH) dw_launch<3, 8, VDK_ACT_HARDSWISH>(stride, grid, threads, x, H, W, C, Ho, Wo, pt, pl, CV, lanes, chunk, w, b, y, mean, s);
    else dw_launch<3, 8, VDK_ACT_RELU>(stride, grid, threads, x, H, W, C, Ho, Wo, pt, pl, CV, lanes, chunk, w, b, y, mean, s);
  } else {
    if (act == VDK_ACT_HARDSWISH) dw_launch<5, 2, VDK_ACT_HARDSWISH>(stride, grid, threads, x, H, W, C, Ho, Wo, pt, pl, CV, lanes, chunk, w, b, y, mean, s);
    else dw_launch<5, 2, VDK_ACT_RELU>(stride, grid, threads, x, H, W, C, Ho, Wo, pt, pl, CV, lanes, chunk, w, b, y, mean, s);
  }
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

static int se_run(__nv_bfloat16* d, const float* mean, int B, int HW, int C, int rd, const float* w1, const float* b1,
                  const float* w2, const float* b2, float* gate, cudaStream_t s) {
  ProfScope prof(kProfOther, 4.0 * B * C * rd + static_cast<double>(B) * HW * C, 4.0 * B * static_cast<double>(HW) * C, s);
  int rc = launch_se_excite(mean, B, C, rd, 0, 1, w1, b1, w2, b2, gate, s);
  if (rc != VDK_OK) return rc;
  return launch_se_apply(d, gate, static_cast<int64_t>(B) * HW, HW, C, s);
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static int check_mnv3(const vdk_mobilenetv3_net* n) {
  VDK_REQUIRE(n, "vdk_mobilenetv3: null network");
  VDK_REQUIRE(n->image_size > 0 && n->image_size % 32 == 0, "vdk_mobilenetv3: image_size must be a multiple of 32 (got %d)",
              n->image_size);
  VDK_REQUIRE(n->feat_dim > 0 && n->feat_dim % 8 == 0, "vdk_mobilenetv3: feat_dim must be a multiple of 8");
  VDK_REQUIRE(n->num_blocks >= 1 && n->num_blocks <= VDK_MOBILENETV3_MAX_BLOCKS,
              "vdk_mobilenetv3: num_blocks must be 1..%d (got %d)", VDK_MOBILENETV3_MAX_BLOCKS, n->num_blocks);
  VDK_REQUIRE(n->pad == VDK_PAD_SAME || n->pad == VDK_PAD_SYMMETRIC, "vdk_mobilenetv3: bad pad rule %d", n->pad);
  VDK_REQUIRE((n->stem_act == VDK_ACT_RELU || n->stem_act == VDK_ACT_HARDSWISH) &&
                  (n->head_act == VDK_ACT_RELU || n->head_act == VDK_ACT_HARDSWISH),
              "vdk_mobilenetv3: stem_act and head_act must be VDK_ACT_RELU or VDK_ACT_HARDSWISH");
  VDK_REQUIRE(n->stem_ch > 0 && n->stem_ch % 8 == 0 && n->head_ch > 0 && n->head_ch % 8 == 0,
              "vdk_mobilenetv3: stem_ch and head_ch must be positive multiples of 8");
  VDK_REQUIRE(n->stem.w && n->stem.b && n->head.w && n->head.b && n->neck_w && n->neck_b,
              "vdk_mobilenetv3: missing stem, head or neck");
  int cin = n->stem_ch, strided = 0;
  for (int i = 0; i < n->num_blocks; ++i) {
    const vdk_mobilenetv3_block& b = n->blocks[i];
    VDK_REQUIRE(b.kind >= VDK_MNV3_DS && b.kind <= VDK_MNV3_CN, "vdk_mobilenetv3: block %d has bad kind %d", i, b.kind);
    VDK_REQUIRE(b.act == VDK_ACT_RELU || b.act == VDK_ACT_HARDSWISH, "vdk_mobilenetv3: block %d has bad act %d", i, b.act);
    VDK_REQUIRE(b.cin == cin, "vdk_mobilenetv3: block %d takes %d channels, the previous block gives %d", i, b.cin, cin);
    VDK_REQUIRE(b.cout > 0 && b.cout % 8 == 0 && b.mid > 0 && b.mid % 8 == 0 && b.mid <= 4096,
                "vdk_mobilenetv3: block %d widths must be multiples of 8, mid <= 4096", i);
    if (b.kind == VDK_MNV3_CN) {
      VDK_REQUIRE(b.kernel == 1 && b.stride == 1 && b.mid == b.cout && b.se_rd == 0,
                  "vdk_mobilenetv3: CN block %d must be a 1x1 / stride-1 conv with mid == cout and no SE", i);
      VDK_REQUIRE(b.conv.w && b.conv.b, "vdk_mobilenetv3: CN block %d misses its conv", i);
    } else {
      VDK_REQUIRE(b.kernel == 3 || b.kernel == 5, "vdk_mobilenetv3: block %d kernel must be 3 or 5 (got %d)", i, b.kernel);
      VDK_REQUIRE(b.stride == 1 || b.stride == 2, "vdk_mobilenetv3: block %d stride must be 1 or 2", i);
      if (b.kind == VDK_MNV3_DS) VDK_REQUIRE(b.mid == b.cin, "vdk_mobilenetv3: DS block %d needs mid == cin", i);
      if (b.kind == VDK_MNV3_IR) VDK_REQUIRE(b.conv.w && b.conv.b, "vdk_mobilenetv3: IR block %d misses conv_pw", i);
      VDK_REQUIRE(b.dw_w && b.dw_b && b.conv_pwl.w && b.conv_pwl.b, "vdk_mobilenetv3: block %d misses weights", i);
      VDK_REQUIRE(aligned16(b.dw_w) && aligned16(b.dw_b), "vdk_mobilenetv3: depthwise weights must be 16-byte aligned");
      VDK_REQUIRE(b.se_rd >= 0 && b.se_rd <= b.mid, "vdk_mobilenetv3: block %d has bad se_rd %d", i, b.se_rd);
      if (b.se_rd > 0)
        VDK_REQUIRE(b.se_w1 && b.se_b1 && b.se_w2 && b.se_b2, "vdk_mobilenetv3: block %d misses its SE weights", i);
    }
    strided += b.stride == 2;
    cin = b.cout;
  }
  // the stem halves the map, four stride-2 blocks make S / 32: the neck's K = (S / 32)^2 * head_ch
  VDK_REQUIRE(strided == 4, "vdk_mobilenetv3: the blocks must hold exactly four stride-2 blocks (got %d)", strided);
  return VDK_OK;
}

struct Mnv3Sizes {
  size_t act;    // elements of the largest activation map
  size_t rows;   // elements of the stem's patch rows
  int max_mid;   // widest SE gate
  int max_cout;  // widest shortcut projection (the gamma = 1 vector)
};

static Mnv3Sizes mnv3_sizes(const vdk_mobilenetv3_net* n, int batch) {
  const size_t B = batch;
  size_t H = n->image_size / 2;
  Mnv3Sizes z{B * H * H * n->stem_ch, B * H * H * 64, 8, 8};
  for (int i = 0; i < n->num_blocks; ++i) {
    const vdk_mobilenetv3_block& b = n->blocks[i];
    const size_t Ho = (H + b.stride - 1) / b.stride;
    z.act = std::max({z.act, B * H * H * b.mid, B * Ho * Ho * b.cout});
    z.max_mid = std::max(z.max_mid, b.mid);
    z.max_cout = std::max(z.max_cout, b.cout);
    H = Ho;
  }
  z.act = std::max(z.act, B * H * H * n->head_ch);
  return z;
}

}  // namespace vdk

using namespace vdk;

extern "C" size_t vdk_mobilenetv3_workspace_bytes(const vdk_mobilenetv3_net* net, int batch) {
  if (!net || batch <= 0 || net->image_size <= 0 || net->num_blocks < 1 || net->num_blocks > VDK_MOBILENETV3_MAX_BLOCKS) return 0;
  const Mnv3Sizes z = mnv3_sizes(net, batch);
  // x (block input), y (block output), e (expanded), d (depthwise output, neck slabs), stem patch rows, SE mean + gate, ones
  return 4 * up256(z.act * 2) + up256(z.rows * 2) + 2 * up256(static_cast<size_t>(batch) * z.max_mid * 4) +
         up256(static_cast<size_t>(z.max_cout) * 4) + 1024;
}

extern "C" int vdk_mobilenetv3_forward(const vdk_mobilenetv3_net* net, const float* images, int batch, int l2_normalize,
                                       float* embeddings, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_mnv3(net);
  if (rc != VDK_OK) return rc;
  VDK_REQUIRE(images && embeddings && batch > 0, "vdk_mobilenetv3_forward: null image/embedding buffer");
  VDK_REQUIRE(workspace && workspace_bytes >= vdk_mobilenetv3_workspace_bytes(net, batch),
              "vdk_mobilenetv3_forward: workspace too small");
  VDK_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "vdk_mobilenetv3_forward: workspace must be 256-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const Mnv3Sizes z = mnv3_sizes(net, batch);
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

  // 1x1 convolution + folded BatchNorm (or conv_head's bias) + activation on vdk_conv2d_ex's plain-GEMM path
  auto conv1x1 = [&](const void* in, int H, int Cin, const vdk_resnet_conv& c, int Cout, int act, void* out) -> int {
    vdk_conv_ex_desc cd{};
    cd.x = in; cd.w = c.w; cd.bias = c.b; cd.y = out;
    cd.B = batch; cd.H = H; cd.W = H; cd.Cin = Cin; cd.Cout = Cout; cd.kernel = 1; cd.stride = 1;
    cd.epilogue = act == VDK_ACT_HARDSWISH ? VDK_EPI_HARDSWISH : VDK_EPI_RELU;
    return conv_ex_run(cd, s, true);
  };
  // the projection: [M, mid] x [cout, mid]^T + bias (+ the shortcut through SCALE_RESIDUAL at gamma = 1)
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
  // ---- stem: conv 3x3/s2 = patch rows with Ho = S / 2 (TF-"same" (0, 1) on the even image: no low pad, the last row /
  // column of taps falls outside and reads zero; symmetric: pad 1), a GEMM with the activation epilogue ----
  const int stem_pad = net->pad == VDK_PAD_SAME ? 0 : 1;
  if ((rc = launch_patch_rows_nchw(images, batch, S, S, 3, 3, 2, stem_pad, H, H, 64, rows, s)) != VDK_OK) return rc;
  if ((rc = conv1x1(rows, H, 64, net->stem, net->stem_ch, net->stem_act, x)) != VDK_OK) return rc;
  for (int i = 0; i < net->num_blocks; ++i) {
    const vdk_mobilenetv3_block& b = net->blocks[i];
    const int Ho = (H + b.stride - 1) / b.stride, M = batch * Ho * Ho;
    const bool skip = b.stride == 1 && b.cin == b.cout;
    if (b.kind == VDK_MNV3_CN) {
      if ((rc = conv1x1(x, H, b.cin, b.conv, b.cout, b.act, y)) != VDK_OK) return rc;
    } else {
      const __nv_bfloat16* dw_in = x;
      if (b.kind == VDK_MNV3_IR) {
        if ((rc = conv1x1(x, H, b.cin, b.conv, b.mid, b.act, e)) != VDK_OK) return rc;
        dw_in = e;
      }
      float* mean = b.se_rd > 0 ? se_mean : nullptr;
      if ((rc = dw_run(dw_in, batch, H, H, b.mid, b.kernel, b.stride, net->pad, b.act, b.dw_w, b.dw_b, d, mean, s)) != VDK_OK)
        return rc;
      if (b.se_rd > 0 &&
          (rc = se_run(d, se_mean, batch, Ho * Ho, b.mid, b.se_rd, b.se_w1, b.se_b1, b.se_w2, b.se_b2, se_gate, s)) != VDK_OK)
        return rc;
      if ((rc = project(d, M, b.mid, b.conv_pwl, b.cout, skip ? x : nullptr, y)) != VDK_OK) return rc;
    }
    std::swap(x, y);
    H = Ho;
  }
  const int c_last = net->blocks[net->num_blocks - 1].cout;
  if ((rc = conv1x1(x, H, c_last, net->head, net->head_ch, net->head_act, e)) != VDK_OK) return rc;
  // ---- neck: BN2d -> Flatten -> Linear -> BN1d folded into one split-K GEMM over the (h, w, c) features ----
  return launch_neck(e, batch, H * H * net->head_ch, net->feat_dim, net->neck_w, net->neck_b, l2_normalize,
                     reinterpret_cast<float*>(d), up256(z.act * 2), embeddings, s);
}

extern "C" int vdk_mobilenetv3_struct_sizes(size_t* out, int n) {
  const size_t sizes[] = {sizeof(vdk_mobilenetv3_net)};
  const int k = static_cast<int>(sizeof(sizes) / sizeof(sizes[0]));
  for (int i = 0; i < n && i < k; ++i) out[i] = sizes[i];
  return k;
}

// Kernel-level entry points of the pieces above, for their tests.
extern "C" int vdk_dwconv_mnv3(const void* x, int B, int H, int W, int C, int kernel, int stride, int pad, int act, const float* w,
                               const float* b, void* y, float* mean, void* stream) {
  VDK_REQUIRE(x && w && b && y, "vdk_dwconv_mnv3: null operand");
  VDK_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && C <= 4096 && (kernel == 3 || kernel == 5) &&
                  (stride == 1 || stride == 2),
              "vdk_dwconv_mnv3: bad shape B=%d H=%d W=%d C=%d kernel=%d stride=%d", B, H, W, C, kernel, stride);
  VDK_REQUIRE(pad == VDK_PAD_SAME || pad == VDK_PAD_SYMMETRIC, "vdk_dwconv_mnv3: bad pad rule %d", pad);
  VDK_REQUIRE(act == VDK_ACT_RELU || act == VDK_ACT_HARDSWISH, "vdk_dwconv_mnv3: bad act %d", act);
  VDK_REQUIRE(H + 2 * (kernel / 2) >= kernel && W + 2 * (kernel / 2) >= kernel, "vdk_dwconv_mnv3: map smaller than the kernel");
  VDK_REQUIRE(aligned16(x) && aligned16(y) && aligned16(w) && aligned16(b), "vdk_dwconv_mnv3: 16-byte alignment");
  return dw_run(static_cast<const __nv_bfloat16*>(x), B, H, W, C, kernel, stride, pad, act, w, b, static_cast<__nv_bfloat16*>(y),
                mean, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vdk_mnv3_se(void* d, const float* mean, int B, int HW, int C, int rd, const float* w1, const float* b1,
                           const float* w2, const float* b2, float* gate, void* stream) {
  VDK_REQUIRE(d && mean && w1 && b1 && w2 && b2 && gate, "vdk_mnv3_se: null operand");
  VDK_REQUIRE(B > 0 && HW > 0 && C > 0 && C % 8 == 0 && C <= 4096 && rd >= 1 && rd <= C, "vdk_mnv3_se: bad shape");
  VDK_REQUIRE(aligned16(d) && aligned16(gate), "vdk_mnv3_se: 16-byte alignment");
  return se_run(static_cast<__nv_bfloat16*>(d), mean, B, HW, C, rd, w1, b1, w2, b2, gate, reinterpret_cast<cudaStream_t>(stream));
}
