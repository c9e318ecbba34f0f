/* vdk_b200.h — C ABI of libvdk_b200.so, the sm_90a implementation of DORAEMON's (wuji3/visiondk)
 * embedding hot path.  The reference is pure Python and has no FFI of its own (SURVEY.md §8b); each
 * entry point below names the reference call site (file:line under /root/reference) whose arithmetic
 * it replaces.  A maintainer binds these with ctypes (INTEGRATION.md shows the stubs).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller unless the name says `host`;
 *   - `stream` is a cudaStream_t passed as void*; calls enqueue work and return without synchronising;
 *   - nothing is allocated behind the caller: scratch comes in as `workspace` (+ a *_workspace_bytes query);
 *   - return value: VDK_OK (0) or a negative VDK_ERR_*; vdk_last_error_string() explains the last failure
 *     on the calling thread.  There is no CPU fallback: without a CUDA device every compute call fails.
 */
#ifndef VDK_B200_H_
#define VDK_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VDK_OK 0
#define VDK_ERR_INVALID (-1)   /* bad argument / unsupported shape */
#define VDK_ERR_CUDA (-2)      /* a CUDA runtime or driver call failed */
#define VDK_ERR_WORKSPACE (-3) /* workspace too small */
#define VDK_ERR_OVERFLOW (-4)  /* a candidate buffer overflowed; caller must take the wide path */

/* ---- library ------------------------------------------------------------------------------- */
int vdk_version(void);                    /* major*10000 + minor*100 + patch */
const char* vdk_last_error_string(void);  /* thread-local, never NULL */
/* 0 when a device of compute capability 9.0 is present and usable, else VDK_ERR_CUDA. */
int vdk_device_check(void);

/* ---- dense contraction: D = epilogue(A . B^T) ---------------------------------------------- */
/* Replaces the cuBLAS/cuDNN GEMMs inside timm's ConvNeXt/ViT blocks that models/faceX/backbone/
 * timm_wrapper.py:52 runs (pointwise Linear layers, patchify convs as GEMMs) and the neck Linear
 * (timm_wrapper.py:36).  A is [M,K] row-major (pitch lda), B is [N,K] row-major (pitch ldb) — the
 * layout of nn.Linear.weight — both 16-bit (bf16 or fp16); accumulation is fp32 on wgmma (register accumulators). */
#define VDK_DTYPE_BF16 0
#define VDK_DTYPE_FP16 1
#define VDK_DTYPE_FP32 2

#define VDK_EPI_NONE 0           /* D = acc (+ bias[n]) */
#define VDK_EPI_GELU 1           /* D = gelu(acc + bias[n]): nn.GELU()'s erf form evaluated as 0.5 x (1 + tanh(x (c1 + c3 x^2))) with
                                    (c1, c3) fitted to it (max deviation 3.1e-4) in fp16x2; |err| <= 6e-4 |x| before the output
                                    rounding (tests/test_gemm_gpu.py sweeps every finite 16-bit x) */
#define VDK_EPI_SCALE_RESIDUAL 2 /* D = residual[m,n] + gamma[n] * (acc + bias[n])  (ConvNeXt layer-scale; gamma = 1: plain residual) */
#define VDK_EPI_LAYERNORM 3      /* D = LayerNorm_N(acc + bias) * gamma + beta; the tile must span the row (N <= 256) */
#define VDK_EPI_MUL_GELU_GRAD 4  /* D = acc * gelu'(residual[m,n]): dgrad through the MLP's GELU (residual = saved pre-activation);
                                    the derivative of the same fp16x2 form, |gelu'~ - gelu'| <= 8e-3 before the output rounding */
/* vdk_conv2d only (vdk_gemm rejects them): */
#define VDK_EPI_RELU 5           /* D = max(acc + bias[n], 0)  (conv + folded BatchNorm + ReLU) */
#define VDK_EPI_RESIDUAL_RELU 6  /* D = max(residual[m,n] + (acc + bias[n]), 0)  (last conv of a ResNet bottleneck) */
/* vdk_conv2d_ex only (vdk_gemm and vdk_conv2d reject them).  SiLU x / (1 + e^-x) with the approximate exp2 and reciprocal:
 * relative error <= 1e-6 for |x| <= 64 before the output rounding. */
#define VDK_EPI_SILU 7           /* D = silu(acc + bias[n])  (conv + folded BatchNorm + SiLU) */
#define VDK_EPI_SILU_RESIDUAL 8  /* D = residual[m,n] + silu(acc + bias[n])  (timm's ConvBnAct with skip: the activation first) */
#define VDK_EPI_HARDSWISH 9      /* D = v relu6(v + 3) / 6 with v = acc + bias[n]  (MobileNetV3's hard-swish, nn.Hardswish) */
/* vdk_gemm, trans_a = 0, trans_b = 1, bf16 in and out only: the LayerNorm backward of the layer whose output gradient the
 * GEMM computes.  dy = bf16(acc); per row and group of ln_group columns, with xh = (y - beta) / gamma from the saved
 * LayerNorm output y = residual and g = dy gamma:  D = rstd (g - mean(g) - xh mean(g xh));  ln_dgamma += sum_rows dy xh,
 * ln_dbeta += sum_rows dy (per-CTA partials reduced in a fixed order: deterministic).  The same arithmetic as
 * vdk_layernorm_bwd on bf16(dy), including its gamma == 0 / |gamma| < 1e-12 handling. */
#define VDK_EPI_LN_BWD 10

typedef struct vdk_gemm_desc {
  const void* A; /* [M,K] 16-bit, pitch lda */
  const void* B; /* [N,K] 16-bit, pitch ldb (nn.Linear.weight layout) */
  void* D;       /* [M,N] out_dtype, pitch ldd */
  int M, N, K, lda, ldb, ldd;
  int in_dtype, out_dtype, epilogue;
  const float* bias;    /* [N] or NULL */
  const float* gamma;   /* [N]: layer-scale (SCALE_RESIDUAL) or LayerNorm weight (LAYERNORM) */
  const float* beta;    /* [N]: LayerNorm bias */
  const void* residual; /* [M,ldr], dtype of D (SCALE_RESIDUAL) */
  int ldr;
  float ln_eps;
  int split_k; /* > 1: K is split over split_k CTAs per tile whose fp32 partials are atomically added into a
                  ZEROED fp32 D (skinny-M neck GEMM, timm_wrapper.py:36); epilogue NONE, no bias */
  long long split_stride; /* split_k > 1 only.  0: partials are atomically added into a zeroed D.  > 0 (elements):
                             split s stores its partial into the slab D + s*split_stride; the effective number of
                             splits is min(split_k, ceil(K/64)) rounded so that every split is non-empty — query it
                             with vdk_gemm_effective_splits.  Deterministic. */
  void* aux_out;  /* VDK_EPI_GELU only, may be NULL: also store the pre-activation acc + bias [M,ldd] (saved for backward) */
  int trans_a; /* 1: A is stored [K,M] row-major (pitch lda >= M): the contraction index is the slow dimension */
  int trans_b; /* 1: B is stored [K,N] row-major (pitch ldb >= N).  Backward GEMMs use these: dgrad
                  dX = dY . W (B = W stored [N_out,K_in] = [K,N] of this contraction) and wgrad dW = dY^T . X
                  (both operands stored with the token index slow) need no transposed copies. */
  float* a_col_sums; /* may be NULL; trans_a with split_k > 1 and split_stride > 0 only: split s also stores the column
                        sums of A over its K range, sum_k A[k,m] in fp32, to a_col_sums[s*M + m] (the bias gradient of
                        the wgrad above, from the A tiles the GEMM streams anyway).  16-byte aligned. */
  /* VDK_EPI_LN_BWD only (gamma, beta: the LayerNorm's weight and bias; residual: its saved bf16 output [M,ldr]): */
  const float* ln_rstd; /* 1/sigma per LayerNorm row (pixel) */
  float* ln_dgamma;     /* [ln_group] += */
  float* ln_dbeta;      /* [ln_group] += */
  float* ln_slab;       /* scratch of 2 * N * (number of SMs) floats, 16-byte aligned */
  int ln_group;         /* LayerNorm width: 128, 256, 512 or 1024, dividing N (128 unless N % 256 == 0); a width above
                           the 256-column tile runs as clusters of ln_group / 256 CTAs */
  int ln_wo;            /* 0: D is [M,ldd] like the GEMM output.  > 0: row m holds the 2x2 patch (b, ho, wo) of an NHWC
                           image of width 2 ln_wo, column q ln_group + c its pixel (2 ho + q / 2, 2 wo + q % 2), channel c
                           (N = 4 ln_group); D and ln_rstd are in that image's [B, 2 Ho, 2 ln_wo, ln_group] pixel order */
} vdk_gemm_desc;
int vdk_gemm(const vdk_gemm_desc* desc, void* stream);
/* Number of K splits vdk_gemm will actually use for (K, split_k). */
int vdk_gemm_effective_splits(int K, int split_k);

/* Positional convenience form of vdk_gemm (split_k = 1, no LayerNorm). */
int vdk_gemm_tn(const void* A, const void* B, void* D, int M, int N, int K, int lda, int ldb, int ldd,
                int in_dtype,          /* VDK_DTYPE_BF16 | VDK_DTYPE_FP16 */
                int out_dtype,         /* VDK_DTYPE_BF16 | VDK_DTYPE_FP16 | VDK_DTYPE_FP32 */
                int epilogue,          /* VDK_EPI_* */
                const float* bias,     /* [N] or NULL */
                const float* gamma,    /* [N], VDK_EPI_SCALE_RESIDUAL only */
                const void* residual,  /* [M,ldr] same dtype as D, VDK_EPI_SCALE_RESIDUAL only */
                int ldr, void* stream);

/* ---- dense 2-D convolution: implicit GEMM on the wgmma GEMM --------------------------------- */
/* y = epilogue(conv2d(x, w) + bias): NHWC bf16 activations, square kernel, equal stride and zero padding on both axes —
 * the Conv2d + eval BatchNorm (folded into w and bias) [+ residual] + ReLU of timm's ResNet Bottleneck
 * (timm/models/resnet.py).  The GEMM row is the output pixel (b, ho, wo), M = B*Ho*Wo; K = kernel*kernel*Cin in
 * (kh, kw, cin) order.  1x1 / stride-1 convolutions run as a plain GEMM over [B*H*W, Cin]; every other shape gathers its
 * A tiles straight from x with TMA im2col loads (no im2col buffer).  Ho = (H + 2 pad - kernel) / stride + 1. */
typedef struct vdk_conv_desc {
  const void* x;        /* [B, H, W, Cin] bf16 */
  const void* w;        /* [Cout, kernel, kernel, Cin] bf16 */
  const float* bias;    /* [Cout] or NULL */
  const void* residual; /* [B, Ho, Wo, Cout] bf16, VDK_EPI_RESIDUAL_RELU only; may be y itself (in place) */
  void* y;              /* [B, Ho, Wo, Cout] bf16 */
  int B, H, W, Cin, Cout;
  int kernel, stride, pad;
  int epilogue; /* VDK_EPI_NONE, VDK_EPI_RELU or VDK_EPI_RESIDUAL_RELU */
} vdk_conv_desc;
/* Cin a multiple of 64, Cout a multiple of 8, 1 <= kernel <= 16, 1 <= stride <= 8, 0 <= pad < kernel. */
int vdk_conv2d(const vdk_conv_desc* desc, void* stream);
/* Grouped form (`groups` groups of cg = Cin / groups channels): the 3x3 conv of timm's ResNeXt Bottleneck
 * (timm/models/resnet.py, cardinality > 1) and of the legacy SE-ResNeXt (timm/models/senet.py).  Each 128-channel output
 * tile contracts over the 128 input channels of its own groups, so desc->w is the block-diagonal weight [Cout, kernel,
 * kernel, 128]: output channel n of group g = n / cg in tile t = n / 128 holds timm's w[n, j - g cg + 128 t] at tile
 * channel j for j in group g, zero elsewhere.  K = kernel*kernel*128 are executed, 128 / cg times the useful MACs.
 * Cin == Cout a multiple of 128, groups >= 2 with cg dividing 128, epilogue VDK_EPI_RELU (no residual); kernel, stride and
 * pad as vdk_conv2d. */
int vdk_conv2d_grouped(const vdk_conv_desc* desc, int groups, void* stream);
/* Grouped form for any group widths: cgi = Cin / groups input and cgo = Cout / groups output channels per group (the
 * split-attention conv of timm's ResNeSt, timm/layers/split_attn.py, has Cout = radix * Cin and cgi as small as 10).  The
 * 128-channel output tile t (n0 = 128 t) contracts over the input channels of the groups its output channels belong to,
 * from c_lo(t) = (n0 / cgo) * cgi rounded down to a multiple of 8 on, as cpb 64-channel blocks per tap; cpb is the maximum
 * over the tiles of ceil(((min(n0 + 127, Cout - 1) / cgo + 1) * cgi - c_lo(t)) / 64).  desc->w is [Cout, kernel, kernel, cpb * 64] bf16:
 * output channel n of group g = n / cgo holds timm's w[n, j + c_lo(n / 128) - g cgi] at column j when that index lies in
 * [0, cgi), zero elsewhere.  Executed MACs: cpb * 64 / cgi times the useful ones.
 * Cin and Cout multiples of 8, groups >= 1 dividing both; epilogue VDK_EPI_NONE, VDK_EPI_RELU or VDK_EPI_RESIDUAL_RELU;
 * kernel, stride and pad as vdk_conv2d.  groups = 1 takes a 1x1 / stride-1 kernel only and runs as vdk_conv2d's plain GEMM
 * with K = Cin (w [Cout, Cin]), so that Cin need not be a multiple of 64 (ResNeSt's conv3). */
int vdk_conv2d_grouped_ex(const vdk_conv_desc* desc, int groups, void* stream);
/* Extended form for TensorFlow-"same" padded MBConv networks (timm's tf_efficientnetv2_* and *mobilenetv3_*,
 * timm/models/_efficientnet_blocks.py with Conv2dSame): separate low and high zero padding per axis, the SiLU and hard-swish
 * epilogues, and Cin any multiple of 8.
 * Ho = (H + pad_h_lo + pad_h_hi - kernel) / stride + 1, likewise Wo.  1x1 / stride-1 / unpadded convolutions run as a plain
 * GEMM over [B*H*W, Cin] with w [Cout, Cin]; every other shape is an implicit GEMM whose K blocks are 64 channels of one
 * tap, so w is [Cout, kernel, kernel, Cinp] with Cinp = Cin rounded up to a multiple of 64 and zero columns from Cin on
 * (executed MACs: Cinp / Cin times the useful ones; the input is read once, its padding channels are never stored). */
typedef struct vdk_conv_ex_desc {
  const void* x;        /* [B, H, W, Cin] bf16 */
  const void* w;        /* [Cout, Cin] (1x1 / stride 1 / unpadded) or [Cout, kernel, kernel, Cinp] bf16 */
  const float* bias;    /* [Cout] or NULL */
  const void* residual; /* [B, Ho, Wo, Cout] bf16, VDK_EPI_SILU_RESIDUAL only; may be y itself (in place) */
  void* y;              /* [B, Ho, Wo, Cout] bf16 */
  int B, H, W, Cin, Cout;
  int kernel, stride;
  int pad_h_lo, pad_h_hi, pad_w_lo, pad_w_hi; /* each in [0, kernel) */
  int epilogue; /* VDK_EPI_NONE, VDK_EPI_SILU, VDK_EPI_SILU_RESIDUAL or VDK_EPI_HARDSWISH */
} vdk_conv_ex_desc;
/* Cin and Cout multiples of 8, 1 <= kernel <= 16, 1 <= stride <= 8. */
int vdk_conv2d_ex(const vdk_conv_ex_desc* desc, void* stream);

/* ---- ResNet embedding forward (eval) --------------------------------------------------------- */
/* Replaces TimmWrapper.forward for timm's Bottleneck ResNets (resnet50/101/152, their -D variants, wide_resnet50_2/101_2;
 * models/faceX/backbone/timm_wrapper.py:16-21, 30-38, 51-54) followed by F.normalize (face_model.py:139): every eval
 * BatchNorm folded into its conv (bf16 weight [Cout, kh, kw, Cin], fp32 bias), NHWC bf16 activations in `workspace`. */
#define VDK_RESNET_MAX_BLOCKS 64
typedef struct vdk_resnet_conv {
  const void* w;  /* bf16 [Cout, kh, kw, Cin] (stem: [Cout, Kp] patch rows, see below) */
  const float* b; /* [Cout] */
} vdk_resnet_conv;
typedef struct vdk_resnet_block {
  vdk_resnet_conv conv1; /* 1x1, Cin -> width, + ReLU */
  vdk_resnet_conv conv2; /* 3x3 / stride (1, or 2 in the first block of stages 2-4), + ReLU */
  vdk_resnet_conv conv3; /* 1x1, width -> 4 * planes, + shortcut, + ReLU */
  vdk_resnet_conv down;  /* shortcut conv, w == NULL: identity.  1x1 / stride; with avg_down and stride 2 the
                            AvgPool2d(2, 2) is folded in: [Cout, 2, 2, Cin] with the 1x1 weight / 4 at every tap */
} vdk_resnet_block;
typedef struct vdk_resnet_net {
  int image_size; /* square input side, multiple of 32 */
  int feat_dim;   /* embedding width, multiple of 8 */
  int depths[4];
  int base_width; /* 64, or 128 for wide_resnet*_2: width of stage s's 3x3 conv = base_width * 2^s */
  int deep_stem;  /* 0: conv 7x7/s2 (stem[0], Kp = 192); 1: ResNet-D deep stem 3x3/s2 3->32 (Kp 64), 3x3 32->32, 3x3 32->64
                     (Kp 320 each) — all as GEMMs over zero-padded (kh, kw, c) patch rows */
  int avg_down;   /* 1: the shortcut of stride-2 blocks is AvgPool2d(2, 2) + 1x1 conv (ResNet-D) */
  vdk_resnet_conv stem[3]; /* the stem's BatchNorms folded in (bn1 into the last one) */
  vdk_resnet_block blocks[VDK_RESNET_MAX_BLOCKS]; /* stage-major */
  const void* neck_w;  /* [feat_dim, h*w*2048] bf16, K order (h, w, c), BN2d/BN1d eval statistics folded in */
  const float* neck_b; /* [feat_dim] */
} vdk_resnet_net;
size_t vdk_resnet_workspace_bytes(const vdk_resnet_net* net, int batch);
/* images: fp32 NCHW [batch,3,S,S]; embeddings: fp32 [batch, feat_dim], L2-normalised when l2_normalize != 0. */
int vdk_resnet_forward(const vdk_resnet_net* net, const float* images, int batch, int l2_normalize, float* embeddings,
                       void* workspace, size_t workspace_bytes, void* stream);
/* sizeof() of vdk_conv_desc and vdk_resnet_net, in that order (vdk_struct_sizes' contract for these two). */
int vdk_resnet_struct_sizes(size_t* out, int n);

/* ---- general Bottleneck network embedding forward (eval): ResNeXt, legacy SE-ResNet / SE-ResNeXt ---------------- */
/* Replaces TimmWrapper.forward for timm's ResNeXt (resnext50_32x4d, resnext101_32x8d / 64x4d, resnext50d_32x4d;
 * timm/models/resnet.py) and legacy SENet Bottleneck models (legacy_seresnet50/101/152, legacy_seresnext26/50/101_32x4d;
 * timm/models/senet.py) — models/faceX/backbone/timm_wrapper.py:16-21, 30-38, 51-54 — followed by F.normalize
 * (face_model.py:139).  Same layouts as vdk_resnet_net; a block's 3x3 conv is grouped when cardinality > 1, and a block
 * with SE weights runs out = ReLU(conv3 * sigmoid(fc2(ReLU(fc1(mean_hw(conv3))))) + shortcut) (timm senet.py SEModule). */
typedef struct vdk_bottleneck_block {
  vdk_resnet_conv conv1, conv2, conv3, down; /* as vdk_resnet_block; conv2 with cardinality > 1: vdk_conv2d_grouped's
                                                block-diagonal [width, 3, 3, 128] */
  const float* se_fc1_w; /* fp32 [rd, C], C = 4 * planes, rd = C / se_reduction; NULL: no SE module */
  const float* se_fc1_b; /* [rd] */
  const float* se_fc2_w; /* [C, rd] */
  const float* se_fc2_b; /* [C] */
} vdk_bottleneck_block;
#define VDK_STEM_POOL_PAD1 0 /* MaxPool2d(3, 2, padding=1) (timm ResNet) */
#define VDK_STEM_POOL_CEIL 1 /* MaxPool2d(3, 2, ceil_mode=True), no padding (legacy SENet) */
typedef struct vdk_bottleneck_net {
  int image_size;      /* square input side, multiple of 32 */
  int feat_dim;        /* embedding width, multiple of 8 */
  int depths[4];
  int width;           /* conv1 / conv2 width of stage 0, doubled per stage: 64 (ResNet, SE-ResNet), 128 (32x4d), 256 (32x8d,
                          64x4d) */
  int cardinality;     /* groups of the 3x3 conv: 1 dense, > 1 vdk_conv2d_grouped */
  int stride_on_conv1; /* 1: a stride-2 block strides its 1x1 conv1 (legacy SEResNetBottleneck); 0: its 3x3 conv2 */
  int stem_pool;       /* VDK_STEM_POOL_PAD1 or VDK_STEM_POOL_CEIL */
  int deep_stem;       /* as vdk_resnet_net */
  int avg_down;        /* as vdk_resnet_net */
  int se_reduction;    /* rd = C / se_reduction for the blocks with SE weights (16 in the legacy SENets) */
  vdk_resnet_conv stem[3];
  vdk_bottleneck_block blocks[VDK_RESNET_MAX_BLOCKS]; /* stage-major */
  const void* neck_w;  /* [feat_dim, h*w*2048] bf16, as vdk_resnet_net */
  const float* neck_b; /* [feat_dim] */
} vdk_bottleneck_net;
size_t vdk_bottleneck_workspace_bytes(const vdk_bottleneck_net* net, int batch);
/* images: fp32 NCHW [batch,3,S,S]; embeddings: fp32 [batch, feat_dim], L2-normalised when l2_normalize != 0. */
int vdk_bottleneck_forward(const vdk_bottleneck_net* net, const float* images, int batch, int l2_normalize, float* embeddings,
                           void* workspace, size_t workspace_bytes, void* stream);
/* sizeof() of vdk_bottleneck_net. */
int vdk_bottleneck_struct_sizes(size_t* out, int n);
/* The forward's stem pool alone: MaxPool2d(3, 2) over NHWC bf16 [B, H, W, C] (C a multiple of 8) with mode
 * VDK_STEM_POOL_PAD1 (padding 1) or VDK_STEM_POOL_CEIL (ceil_mode=True, no padding) into y [B, Ho, Wo, C]. */
int vdk_stem_maxpool(const void* x, int B, int H, int W, int C, int mode, void* y, void* stream);
/* The forward's SE gate alone, on y = the BN-folded conv3 output [B, HW, C] bf16 (C a multiple of 64, <= 2048):
 * mean [B, C] fp32 = the spatial mean, gate [B, C] fp32 = sigmoid(fc2_w ReLU(fc1_w mean + fc1_b) + fc2_b) (fc1_w [rd, C],
 * fc2_w [C, rd]), then residual [B, HW, C] bf16 = ReLU(y * gate + residual) in place. */
int vdk_se_gate(const void* y, int B, int HW, int C, int rd, const float* fc1_w, const float* fc1_b, const float* fc2_w,
                const float* fc2_b, float* mean, float* gate, void* residual, void* stream);

/* ---- EfficientNetV2 embedding forward (eval) ---------------------------------------------------- */
/* Replaces TimmWrapper.forward for timm's tf_efficientnetv2_s / _m / _l (timm/models/efficientnet.py,
 * _efficientnet_blocks.py; models/faceX/backbone/timm_wrapper.py:16-21, 30-38, 51-54) followed by F.normalize
 * (face_model.py:139).  Every eval BatchNorm (eps 1e-3) folded into its conv; NHWC bf16 activations in `workspace`; every
 * convolution TF-"same" padded: per axis total = max((ceil(H / s) - 1) s + k - H, 0), lo = total / 2, hi = total - lo.
 * Blocks (timm kinds), with a shortcut when stride == 1 and cin == cout:
 *   CN (ConvBnAct)      out = silu(conv3x3(x)) [+ x]
 *   ER (EdgeResidual)   out = conv_pwl(silu(conv3x3/s(x))) [+ x]
 *   IR (InvertedResid.) e = silu(conv_pw(x)); d = silu(dwconv3x3/s(e)); g = sigmoid(W2 silu(W1 mean_hw(d) + b1) + b2);
 *                       out = conv_pwl(d * g) [+ x]
 * then conv_head 1x1 + SiLU and the folded CNN neck over the (h, w, c) map. */
#define VDK_EFFNETV2_MAX_BLOCKS 80
#define VDK_EFFNET_CN 0
#define VDK_EFFNET_ER 1
#define VDK_EFFNET_IR 2
typedef struct vdk_effnetv2_block {
  int kind;   /* VDK_EFFNET_CN, _ER or _IR */
  int stride; /* 1 or 2 */
  int cin, cout;
  int mid;    /* ER, IR: the expanded width (IR: of the depthwise conv and the SE gate); CN: cout */
  int se_rd;  /* IR: the SE bottleneck width */
  vdk_resnet_conv conv;     /* CN conv / ER conv_exp: [out, 3, 3, Cinp] (vdk_conv2d_ex layout); IR conv_pw: [mid, cin] */
  const float* dw_w;        /* IR: fp32 [9, mid] taps in (dy, dx) order */
  const float* dw_b;        /* IR: [mid] */
  const float* se_w1;       /* IR: fp32 [se_rd, mid] conv_reduce */
  const float* se_b1;       /* [se_rd] */
  const float* se_w2;       /* [mid, se_rd] conv_expand */
  const float* se_b2;       /* [mid] */
  vdk_resnet_conv conv_pwl; /* ER, IR: [cout, mid] */
} vdk_effnetv2_block;
typedef struct vdk_effnetv2_net {
  int image_size; /* square input side, multiple of 32 */
  int feat_dim;   /* embedding width, multiple of 8 */
  int num_blocks;
  int stem_ch;    /* conv_stem 3x3/s2 3 -> stem_ch, as a GEMM over zero-padded (kh, kw, c) rows: stem.w [stem_ch, 64] */
  int head_ch;    /* conv_head 1x1 width (1280) */
  vdk_resnet_conv stem;
  vdk_effnetv2_block blocks[VDK_EFFNETV2_MAX_BLOCKS];
  vdk_resnet_conv head; /* [head_ch, cout of the last block] */
  const void* neck_w;   /* [feat_dim, h*w*head_ch] bf16, K order (h, w, c), BN2d/BN1d eval statistics folded in */
  const float* neck_b;  /* [feat_dim] */
} vdk_effnetv2_net;
size_t vdk_effnetv2_workspace_bytes(const vdk_effnetv2_net* net, int batch);
/* images: fp32 NCHW [batch,3,S,S]; embeddings: fp32 [batch, feat_dim], L2-normalised when l2_normalize != 0. */
int vdk_effnetv2_forward(const vdk_effnetv2_net* net, const float* images, int batch, int l2_normalize, float* embeddings,
                         void* workspace, size_t workspace_bytes, void* stream);
/* sizeof() of vdk_conv_ex_desc and vdk_effnetv2_net, in that order. */
int vdk_effnetv2_struct_sizes(size_t* out, int n);
/* The IR block's depthwise conv alone: y [B, Ho, Wo, C] bf16 = silu(dwconv3x3(x) + b) over x [B, H, W, C] bf16 (C a
 * multiple of 32, <= 4096), stride 1 or 2 with TF-"same" padding, w fp32 [9, C]; and mean [B, C] fp32 = the spatial mean of
 * the bf16 y, summed in a fixed order (bit-reproducible). */
int vdk_dwconv3_silu(const void* x, int B, int H, int W, int C, int stride, const float* w, const float* b, void* y, float* mean,
                     void* stream);
/* The IR block's SE gate alone, on the depthwise output d [B, HW, C] bf16 and its mean [B, C] fp32 (C a multiple of 8,
 * <= 4096): gate [B, C] fp32 = sigmoid(w2 silu(w1 mean + b1) + b2) (w1 [rd, C], w2 [C, rd]), then d = d * gate in place. */
int vdk_effnet_se(void* d, const float* mean, int B, int HW, int C, int rd, const float* w1, const float* b1, const float* w2,
                  const float* b2, float* gate, void* stream);

/* ---- MobileNetV3 embedding forward (eval) -------------------------------------------------------- */
/* Replaces TimmWrapper.forward for timm's MobileNetV3s at width 1.0 (tf_mobilenetv3_large_minimal_100, tf_mobilenetv3_large_100,
 * tf_mobilenetv3_small_100, tf_mobilenetv3_small_minimal_100, mobilenetv3_large_100, mobilenetv3_small_100;
 * timm/models/mobilenetv3.py, _efficientnet_blocks.py; models/faceX/backbone/timm_wrapper.py:16-21, 30-38, 51-54) followed
 * by F.normalize (face_model.py:139).  Every eval BatchNorm folded into its conv; NHWC bf16 activations in `workspace`.
 * act is ReLU or hard-swish per conv; padding is TF-"same" (tf_*) or symmetric k / 2.  Blocks, with a shortcut when
 * stride == 1 and cin == cout:
 *   DS (DepthwiseSeparable)  d = act(dwconv_k/s(x)); [d = d * hsig(W2 relu(W1 mean_hw(d) + b1) + b2)]; out = conv_pw(d) [+ x]
 *   IR (InvertedResidual)    e = act(conv_pw(x)); d = act(dwconv_k/s(e)); [SE as DS]; out = conv_pwl(d) [+ x]
 *   CN (ConvBnAct 1x1)       out = act(conv(x))
 * with hsig(v) = relu6(v + 3) / 6; then conv_head 1x1 (with bias) + act on the unpooled map and the folded CNN neck. */
#define VDK_MOBILENETV3_MAX_BLOCKS 24
#define VDK_MNV3_DS 0
#define VDK_MNV3_IR 1
#define VDK_MNV3_CN 2
#define VDK_ACT_RELU 0
#define VDK_ACT_HARDSWISH 1
#define VDK_PAD_SAME 0      /* TensorFlow "same": per axis total = max((ceil(H / s) - 1) s + k - H, 0), lo = total / 2 */
#define VDK_PAD_SYMMETRIC 1 /* k / 2 on every side */
typedef struct vdk_mobilenetv3_block {
  int kind;   /* VDK_MNV3_DS, _IR or _CN */
  int kernel; /* depthwise k: 3 or 5 (CN: 1) */
  int stride; /* 1 or 2 (CN: 1) */
  int cin, mid, cout; /* mid: the depthwise width (DS: cin; CN: cout), a multiple of 8 */
  int act;    /* VDK_ACT_RELU or VDK_ACT_HARDSWISH */
  int se_rd;  /* the SE bottleneck width; 0: no SE */
  vdk_resnet_conv conv;     /* IR conv_pw [mid, cin] / CN conv [cout, cin]; unused for DS */
  const float* dw_w;        /* DS, IR: fp32 [k*k, mid] taps in (dy, dx) order */
  const float* dw_b;        /* [mid] */
  const float* se_w1;       /* fp32 [se_rd, mid] conv_reduce */
  const float* se_b1;       /* [se_rd] */
  const float* se_w2;       /* [mid, se_rd] conv_expand */
  const float* se_b2;       /* [mid] */
  vdk_resnet_conv conv_pwl; /* DS conv_pw / IR conv_pwl: [cout, mid] */
} vdk_mobilenetv3_block;
typedef struct vdk_mobilenetv3_net {
  int image_size; /* square input side, multiple of 32 */
  int feat_dim;   /* embedding width, multiple of 8 */
  int num_blocks;
  int pad;        /* VDK_PAD_SAME or VDK_PAD_SYMMETRIC */
  int stem_ch;    /* conv_stem 3x3/s2 3 -> stem_ch, as a GEMM over zero-padded (kh, kw, c) rows: stem.w [stem_ch, 64] */
  int stem_act;   /* VDK_ACT_* */
  int head_ch;    /* conv_head 1x1 width (1280 large, 1024 small) */
  int head_act;   /* VDK_ACT_* */
  vdk_resnet_conv stem;
  vdk_mobilenetv3_block blocks[VDK_MOBILENETV3_MAX_BLOCKS];
  vdk_resnet_conv head; /* [head_ch, cout of the last block], conv_head's own bias */
  const void* neck_w;   /* [feat_dim, h*w*head_ch] bf16, K order (h, w, c), BN2d/BN1d eval statistics folded in */
  const float* neck_b;  /* [feat_dim] */
} vdk_mobilenetv3_net;
size_t vdk_mobilenetv3_workspace_bytes(const vdk_mobilenetv3_net* net, int batch);
/* images: fp32 NCHW [batch,3,S,S]; embeddings: fp32 [batch, feat_dim], L2-normalised when l2_normalize != 0. */
int vdk_mobilenetv3_forward(const vdk_mobilenetv3_net* net, const float* images, int batch, int l2_normalize, float* embeddings,
                            void* workspace, size_t workspace_bytes, void* stream);
/* sizeof() of vdk_mobilenetv3_net. */
int vdk_mobilenetv3_struct_sizes(size_t* out, int n);
/* The DS / IR block's depthwise conv alone: y [B, Ho, Wo, C] bf16 = act(dwconv_k(x) + b) over x [B, H, W, C] bf16 (C a multiple
 * of 8, <= 4096), k 3 or 5, stride 1 or 2, padding VDK_PAD_SAME or VDK_PAD_SYMMETRIC (Ho = ceil(H / stride) either way for
 * the even maps of the models; in general Ho = (H + lo + hi - k) / stride + 1), w fp32 [k*k, C], fp32 FMAs in (bias, dy, dx)
 * order.  mean [B, C] fp32 (may be NULL) = the spatial mean of the bf16 y, summed in a fixed order (bit-reproducible). */
int vdk_dwconv_mnv3(const void* x, int B, int H, int W, int C, int kernel, int stride, int pad, int act, const float* w,
                    const float* b, void* y, float* mean, void* stream);
/* The SE gate alone, on the depthwise output d [B, HW, C] bf16 and its mean [B, C] fp32 (C a multiple of 8, <= 4096):
 * gate [B, C] fp32 = relu6(w2 relu(w1 mean + b1) + b2 + 3) / 6 (w1 [rd, C], w2 [C, rd]), then d = d * gate in place. */
int vdk_mnv3_se(void* d, const float* mean, int B, int HW, int C, int rd, const float* w1, const float* b1, const float* w2,
                const float* b2, float* gate, void* stream);

/* ---- ResNeSt embedding forward (eval) ------------------------------------------------------------ */
/* Replaces TimmWrapper.forward for timm's ResNeSts with the width-32 deep stem (resnest14d, 26d, 50d, 50d_1s4x24d,
 * 50d_4s2x40d; timm/models/resnest.py, timm/layers/split_attn.py; models/faceX/backbone/timm_wrapper.py:16-21, 30-38,
 * 51-54) followed by F.normalize (face_model.py:139).  Stem, stem pool, avg_down shortcuts and neck as vdk_resnet_net with
 * deep_stem = avg_down = 1.  A block of stage s (planes = 64 << s, gw = floor(planes * base_width / 64) * cardinality,
 * C = gw, R = radix, A = attn[s]):
 *   t = ReLU(conv1(x));  on stride-2 blocks with avd_first: t = AvgPool2d(3, 2, 1)(t)   (count_include_pad: / 9)
 *   u = ReLU(conv(t)) 3x3 / s1 / p1, C -> R C, cardinality * R groups, output channel r C + c
 *   gap = mean_hw sum_r u_r;  z = fc2(ReLU(fc1(gap)))  (1x1, cardinality groups, with bias; bn1 folded into fc1)
 *   a[r, g C / card + i] = softmax_r z[g R C / card + r C / card + i]  (R > 1), sigmoid(z) (R = 1)
 *   v = sum_r a_r u_r;  on stride-2 blocks without avd_first: v = AvgPool2d(3, 2, 1)(v)
 *   out = ReLU(conv3(v) + shortcut(x)) */
typedef struct vdk_resnest_block {
  vdk_resnet_conv conv1; /* [gw, Cin] 1x1, bn1 folded */
  vdk_resnet_conv conv2; /* the split conv [R gw, 3, 3, cpb * 64] in vdk_conv2d_grouped_ex's layout, bn0 folded */
  const float* fc1_w;    /* fp32 [A, gw / cardinality], bn1 of the attention folded */
  const float* fc1_b;    /* [A] */
  const float* fc2_w;    /* fp32 [R gw, A / cardinality] */
  const float* fc2_b;    /* [R gw] */
  vdk_resnet_conv conv3; /* [4 planes, gw] 1x1, bn3 folded */
  vdk_resnet_conv down;  /* as vdk_resnet_block (avg_down) */
} vdk_resnest_block;
typedef struct vdk_resnest_net {
  int image_size;  /* square input side, multiple of 32 */
  int feat_dim;    /* embedding width, multiple of 8 */
  int depths[4];
  int radix;       /* 1 .. 4 */
  int cardinality; /* >= 1 */
  int base_width;  /* gw of stage s = floor((64 << s) * base_width / 64) * cardinality, a multiple of 8 */
  int avd_first;   /* 1: the stride-2 average pool before the split conv; 0: after the radix combine */
  int attn[4];     /* A per stage: make_divisible(gw R / 4, 8, min 32), a multiple of cardinality */
  vdk_resnet_conv stem[3]; /* the deep stem as vdk_resnet_net's */
  vdk_resnest_block blocks[VDK_RESNET_MAX_BLOCKS]; /* stage-major */
  const void* neck_w;  /* [feat_dim, h*w*2048] bf16, as vdk_resnet_net */
  const float* neck_b; /* [feat_dim] */
} vdk_resnest_net;
size_t vdk_resnest_workspace_bytes(const vdk_resnest_net* net, int batch);
/* images: fp32 NCHW [batch,3,S,S]; embeddings: fp32 [batch, feat_dim], L2-normalised when l2_normalize != 0. */
int vdk_resnest_forward(const vdk_resnest_net* net, const float* images, int batch, int l2_normalize, float* embeddings,
                        void* workspace, size_t workspace_bytes, void* stream);
/* sizeof() of vdk_resnest_net. */
int vdk_resnest_struct_sizes(size_t* out, int n);
/* The forward's split-attention gate alone, on u = the split conv's output [B, HW, R C] bf16 (C a multiple of 8, R C <= 4096,
 * 1 <= R <= 4; A a multiple of cardinality, cardinality dividing C): gap [B, C] fp32 = mean_hw sum_r u_r (fixed order),
 * attn [B, R C] fp32 = a[r, c] at r C + c as above, then v [B, Ho, Wo, C] bf16 = sum_r a_r u_r, over the H x W map
 * (HW = H W) when pool == 0, or AvgPool2d(3, 2, 1, count_include_pad) of it when pool == 1 (Ho = (H - 1) / 2 + 1). */
int vdk_split_attn_gate(const void* u, int B, int H, int W, int C, int radix, int cardinality, int A, const float* fc1_w,
                        const float* fc1_b, const float* fc2_w, const float* fc2_b, float* gap, float* attn, int pool, void* v,
                        void* stream);
/* AvgPool2d(3, 2, padding 1, count_include_pad=True) over NHWC bf16 x [B, H, W, C] (C a multiple of 8) into
 * y [B, (H - 1) / 2 + 1, (W - 1) / 2 + 1, C]: the fp32 sum of the nine taps (zeros outside) / 9, rounded once. */
int vdk_avgpool3s2(const void* x, int B, int H, int W, int C, void* y, void* stream);

/* ---- Swin Transformer V2 embedding forward (eval) ---------------------------------------------- */
/* Replaces TimmWrapper.forward for timm's SwinTransformerV2 towers (swinv2_base_window8_256,
 * swinv2_large_window12to16_192to256; models/faceX/backbone/timm_wrapper.py:16-21, 30-38, 51-54: timm 0.9.16 forward_features
 * returns an NHWC [B, 8, 8, C] map, so the wrapper's rank rule builds BatchNorm2d(8) over the h axis -> Flatten in (h, w, c)
 * order -> Linear -> BatchNorm1d) followed by F.normalize (face_model.py:139).  Head dim 32; every LayerNorm has eps 1e-5.
 * Blocks are res-post-norm: x = x + norm1(proj(attn(qkv(x)))); x = x + norm2(fc2(GELU(fc1(x)))). */
#define VDK_SWINV2_MAX_BLOCKS 24
typedef struct vdk_swinv2_block {
  const void* qkv_w;        /* [3C, C] bf16 (attn.qkv.weight) */
  const float* qkv_b;       /* [3C] = cat(q_bias, 0, v_bias) */
  const float* attn_scale;  /* [heads] exp(min(logit_scale, ln 100)) */
  const float* attn_bias;   /* [heads, (2w-1)^2] 16 sigmoid(cpb_mlp(relative_coords_table)), idx = (dy+w-1)(2w-1) + dx+w-1 */
  const void* proj_w;  const float* proj_b;   /* [C, C], [C] */
  const float* norm1_w; const float* norm1_b; /* [C] */
  const void* fc1_w;   const float* fc1_b;    /* [4C, C], [4C] (then exact GELU) */
  const void* fc2_w;   const float* fc2_b;    /* [C, 4C], [C] */
  const float* norm2_w; const float* norm2_b; /* [C] */
} vdk_swinv2_block;
typedef struct vdk_swinv2_net {
  int image_size;  /* 256 (the towers' size; the map is 64 -> 32 -> 16 -> 8) */
  int feat_dim;    /* embedding width, multiple of 8 */
  int embed_dim;   /* C of stage 0 (multiple of 64, <= 256), doubled by every patch merging */
  int depths[4];
  int window[4];   /* w = min(window, map) per stage: 8 or 16, dividing the map */
  int shift[4];    /* shift of the odd blocks of each stage: w/2, or 0 when the map is one window */
  const void* stem_w;      /* [C, 48] bf16, K order (c, kh, kw) = patch_embed.proj.weight flattened */
  const float* stem_b;     /* [C] */
  const float* stem_ln_w;  /* [C] patch_embed.norm */
  const float* stem_ln_b;
  const void* merge_w[4];      /* stage s > 0: [2Cin, 2, 2, Cin] bf16, downsample.reduction.weight permuted from timm's K order
                                  (w-offset, h-offset, c) to (kh, kw, c); index 0 unused */
  const float* merge_ln_w[4];  /* [2Cin] downsample.norm */
  const float* merge_ln_b[4];
  vdk_swinv2_block blocks[VDK_SWINV2_MAX_BLOCKS]; /* stage-major */
  const float* norm_w; const float* norm_b;  /* model.norm */
  const void* neck_w;   /* [feat_dim, 8*8*C] bf16, K order (h, w, c), BatchNorm2d (on h) and BatchNorm1d eval statistics folded */
  const float* neck_b;  /* [feat_dim] */
} vdk_swinv2_net;
size_t vdk_swinv2_workspace_bytes(const vdk_swinv2_net* net, int batch);
/* images: fp32 NCHW [batch,3,256,256]; embeddings: fp32 [batch, feat_dim], L2-normalised when l2_normalize != 0. */
int vdk_swinv2_forward(const vdk_swinv2_net* net, const float* images, int batch, int l2_normalize, float* embeddings,
                       void* workspace, size_t workspace_bytes, void* stream);
/* sizeof() of vdk_swinv2_net. */
int vdk_swinv2_struct_sizes(size_t* out, int n);
/* Shifted-window cosine attention of timm's WindowAttention (swin_transformer_v2.py, with SwinTransformerV2Block._attn's roll,
 * window_partition, window_reverse and attn_mask) on the qkv Linear's output as stored: qkv bf16 [batch, H, W, 3, heads, 32]
 * in natural token order -> out bf16 [batch, H, W, heads*32] in natural order.  Per (window, head):
 * softmax(normalize(q) normalize(k)^T * scale[h] + bias[h, idx] + mask) v, mask = -100 between timm's shift regions.
 * window 8 or 16 dividing H and W; shift 0 or window/2, and 0 when H == window or W == window. */
int vdk_window_attention_fwd(const void* qkv, int batch, int H, int W, int heads, int window, int shift, const float* scale,
                             const float* bias, void* out, void* stream);
/* The Swin V2 block's res-post-norm in place: x [rows, C] bf16 <- x + LayerNorm(y) * ln_w + ln_b (fp32 statistics; C a multiple
 * of 8 in [8, 1536]) — timm SwinTransformerV2Block.forward's x + norm1(...) and x + norm2(...). */
int vdk_postnorm_residual(void* x, const void* y, int64_t rows, int C, const float* ln_w, const float* ln_b, float eps, void* stream);

/* ---- ConvNeXt embedding forward (eval) ------------------------------------------------------ */
/* Replaces TimmWrapper.forward (models/faceX/backbone/timm_wrapper.py:51-54: timm ConvNeXt features with
 * num_classes=0, global_pool='' -> BatchNorm2d -> Flatten -> Linear -> BatchNorm1d, :30-38) followed by
 * F.normalize (models/faceX/face_model.py:139).  All pointers are device pointers to weights the caller packed
 * (visiondk_b200/backbone.py: layouts below); activations are NHWC bf16 in `workspace`. */
#define VDK_CONVNEXT_MAX_BLOCKS 64

typedef struct vdk_convnext_block {
  const float* dw_w;  /* depthwise 7x7 taps, [49][C] fp32 (tap-major, channel contiguous) */
  const float* dw_b;  /* [C] */
  const float* ln_w;  /* [C] LayerNorm(eps 1e-6) */
  const float* ln_b;  /* [C] */
  const void* fc1_w;  /* [4C, C] bf16 (nn.Linear.weight) */
  const float* fc1_b; /* [4C] */
  const void* fc2_w;  /* [C, 4C] bf16 */
  const float* fc2_b; /* [C] */
  const float* gamma; /* [C] layer scale */
  /* training only (may be NULL for inference): */
  const float* dw_w_flip; /* [49][C] taps in reverse order (backward-data of the depthwise conv) */
  const void* fc2_wg;     /* [C, 4C] bf16: gamma[c] * fc2.weight[c, :] (dgrad through layer scale) */
} vdk_convnext_block;

typedef struct vdk_convnext_down {
  const float* ln_w;   /* [Cin] LayerNorm2d(eps 1e-6) */
  const float* ln_b;   /* [Cin] */
  const void* conv_w;  /* [Cout, 4*Cin] bf16, K order (kh, kw, cin) */
  const float* conv_b; /* [Cout] */
} vdk_convnext_down;

typedef struct vdk_convnext_net {
  int image_size; /* square input side, multiple of 32 */
  int feat_dim;   /* embedding width (neck Linear out_features) */
  int depths[4];
  int dims[4];
  const void* stem_w;     /* [dims[0], 48] bf16, K order (c, kh, kw) = Conv2d(3,C0,4,4).weight flattened */
  const float* stem_b;    /* [dims[0]] */
  const float* stem_ln_w; /* [dims[0]] */
  const float* stem_ln_b;
  vdk_convnext_down down[4]; /* down[0] unused */
  vdk_convnext_block blocks[VDK_CONVNEXT_MAX_BLOCKS]; /* stage-major */
  const float* head_ln_w; /* [dims[3]] model.head.norm */
  const float* head_ln_b;
  const void* neck_w;  /* [feat_dim, h*w*dims[3]] bf16, K order (h, w, c), BN2d/BN1d eval statistics folded in */
  const float* neck_b; /* [feat_dim] folded bias */
} vdk_convnext_net;

/* Building blocks of the forward, exported for unit parity tests (NHWC bf16 activations):
 *   vdk_dwconv7_ln        y = LayerNorm_C(depthwise7x7(x, pad 3) + bias)         timm ConvNeXtBlock.conv_dw + .norm
 *   vdk_layernorm_patchify out = LayerNorm_C(x), patch == 2: regrouped as 2x2/stride-2 patch rows [B*H/2*W/2, 4C]
 *                          in (kh, kw, c) order (timm downsample LayerNorm2d + the im2col of its Conv2d(k2,s2)) */
int vdk_dwconv7_ln(const void* x, int batch, int H, int W, int C, const float* w49, const float* bias,
                   const float* ln_w, const float* ln_b, float eps, void* y, void* stream);
int vdk_layernorm_patchify(const void* x, int batch, int H, int W, int C, const float* ln_w, const float* ln_b,
                           float eps, int patch, void* out, void* stream);

/* ---- ConvNeXt training forward / backward -------------------------------------------------- */
/* fp32 tensors in timm's own layouts (device pointers): the master parameters, or — same struct — their gradients.
 * Replaces the train-mode forward of TimmWrapper (timm_wrapper.py:51-54, BatchNorm batch statistics at :34,37) and
 * its autograd backward, i.e. `scaler.scale(loss).backward()` at engine/procedure/train.py:206. */
typedef struct vdk_convnext_block_tensors {
  float* dw_w;  /* conv_dw.weight [C,1,7,7] */
  float* dw_b;
  float* ln_w;  /* norm.weight */
  float* ln_b;
  float* fc1_w; /* mlp.fc1.weight [4C,C] */
  float* fc1_b;
  float* fc2_w; /* mlp.fc2.weight [C,4C] */
  float* fc2_b;
  float* gamma;
} vdk_convnext_block_tensors;
typedef struct vdk_convnext_down_tensors {
  float* ln_w;
  float* ln_b;
  float* conv_w; /* downsample.1.weight [Cout,Cin,2,2] */
  float* conv_b;
} vdk_convnext_down_tensors;
typedef struct vdk_convnext_tensors {
  float* stem_w; /* stem.0.weight [C0,3,4,4] */
  float* stem_b;
  float* stem_ln_w;
  float* stem_ln_b;
  vdk_convnext_down_tensors down[4];
  vdk_convnext_block_tensors blocks[VDK_CONVNEXT_MAX_BLOCKS];
  float* head_ln_w;
  float* head_ln_b;
  float* bn2_w; /* output_layer.0 (BatchNorm2d) */
  float* bn2_b;
  float* bn2_running_mean;
  float* bn2_running_var;
  float* lin_w; /* output_layer.2.weight [F, C3*h*w] in timm's (c,h,w) flatten order */
  float* lin_b;
  float* bn1_w; /* output_layer.3 (BatchNorm1d) */
  float* bn1_b;
  float* bn1_running_mean;
  float* bn1_running_var;
} vdk_convnext_tensors;

/* Refreshes the bf16 / permuted kernel-layout weights of `net` (whose pointer fields address caller-allocated
 * buffers) from the fp32 masters: stem_w, down[].conv_w, blocks[].{dw_w, fc1_w, fc2_w, fc2_wg}, neck_w (un-folded,
 * (h,w,c) order), and blocks[].dw_w_flip (the reversed taps) where net carries that buffer.  fp32 vectors (biases,
 * norms, gamma) are used in place: point net's fields at the masters. */
int vdk_convnext_pack(const vdk_convnext_tensors* params, vdk_convnext_net* net, void* stream);
size_t vdk_convnext_train_workspace_bytes(const vdk_convnext_net* net, int batch);
/* images fp32 NCHW -> out_feats fp32 [batch, feat_dim] (NOT normalised: the head normalises).  Saves activations in
 * `workspace` for the backward; updates the BatchNorm running statistics in `params` with `bn_momentum`. */
int vdk_convnext_train_forward(const vdk_convnext_net* net, const vdk_convnext_tensors* params, const float* images,
                               int batch, float bn_momentum, float* out_feats, void* workspace, size_t workspace_bytes,
                               void* stream);
/* d_feats fp32 [batch, feat_dim] -> gradients ACCUMULATED (+=) into `grads` (same struct, timm layouts). */
int vdk_convnext_train_backward(const vdk_convnext_net* net, const vdk_convnext_tensors* params,
                                const vdk_convnext_tensors* grads, const float* d_feats, int batch, void* workspace,
                                size_t workspace_bytes, void* stream);
/* The same backward in consecutive UNIT ranges (unit 0 = neck + head LayerNorm, then per stage 3..0 one unit per block,
 * last block first, and one for the stage's downsample layer / the stem): lets the caller start the DDP all-reduce
 * (engine/vision_engine.py:509-510 wraps the model in DistributedDataParallel, whose buckets overlap the backward) of the
 * gradients a range completed while the next range computes.  Ranges must be issued in order and cover [0, units). */
int vdk_convnext_train_backward_units(const vdk_convnext_net* net);
int vdk_convnext_train_backward_range(const vdk_convnext_net* net, const vdk_convnext_tensors* params,
                                      const vdk_convnext_tensors* grads, const float* d_feats, int batch, void* workspace,
                                      size_t workspace_bytes, void* stream, int unit_begin, int unit_end);
/* Where the train workspace keeps one buffer: the saved activations of vdk_convnext_train_forward and the backward's scratch,
 * as a byte offset into the workspace and a size (both from the layout the train entry points use).  `index` selects the
 * block (Y, RSTD, HPRE, HPOST: 0 .. sum(depths) - 1, stage-major), the stage (PATCH, PRSTD: 1 .. 3) or, for XS, the
 * residual-stream node stage * (VDK_CONVNEXT_MAX_BLOCKS + 1) + j, j = 0 .. depths[stage]; it is ignored for the others.
 * An unknown id or an index out of range is refused with VDK_ERR_INVALID. */
enum {
  VDK_CONVNEXT_TRAIN_P0, VDK_CONVNEXT_TRAIN_Z0, VDK_CONVNEXT_TRAIN_RSTD0, VDK_CONVNEXT_TRAIN_XS, VDK_CONVNEXT_TRAIN_Y,
  VDK_CONVNEXT_TRAIN_RSTD, VDK_CONVNEXT_TRAIN_HPRE, VDK_CONVNEXT_TRAIN_HPOST, VDK_CONVNEXT_TRAIN_PATCH, VDK_CONVNEXT_TRAIN_PRSTD,
  VDK_CONVNEXT_TRAIN_F, VDK_CONVNEXT_TRAIN_FRSTD, VDK_CONVNEXT_TRAIN_FN, VDK_CONVNEXT_TRAIN_BN2_MEAN, VDK_CONVNEXT_TRAIN_BN2_RSTD,
  VDK_CONVNEXT_TRAIN_Z, VDK_CONVNEXT_TRAIN_ZSLAB, VDK_CONVNEXT_TRAIN_BN1_MEAN, VDK_CONVNEXT_TRAIN_BN1_RSTD, VDK_CONVNEXT_TRAIN_DXA,
  VDK_CONVNEXT_TRAIN_DXB, VDK_CONVNEXT_TRAIN_DY, VDK_CONVNEXT_TRAIN_DCONV, VDK_CONVNEXT_TRAIN_G, VDK_CONVNEXT_TRAIN_SDO,
  VDK_CONVNEXT_TRAIN_DW49, VDK_CONVNEXT_TRAIN_GWC, VDK_CONVNEXT_TRAIN_GWNECK, VDK_CONVNEXT_TRAIN_DZ, VDK_CONVNEXT_TRAIN_DZB,
  VDK_CONVNEXT_TRAIN_DFN, VDK_CONVNEXT_TRAIN_WSLAB, VDK_CONVNEXT_TRAIN_NUM_BUFFERS
};
int vdk_convnext_train_buffer(const vdk_convnext_net* net, int batch, int id, int index, size_t* offset, size_t* bytes);

/* Building blocks of the backward, exported for unit parity tests (NHWC bf16 activations, fp32 parameter grads +=):
 *   vdk_dwconv7             mode 0: LayerNorm_C(dwconv7(x)+bias) (rstd_out optional); mode 1: dwconv7(x) with `w49` (+addend)
 *                           — with reversed taps this is the depthwise backward-data pass
 *   vdk_dwconv7_wgrad       dw49[tap][c] += sum dconv * shifted x; dbias[c] += sum dconv (C a multiple of 8)
 *   vdk_dwconv7_bwd         both from one pass over dconv: dx = bf16(dwconv7(dconv) with `w49` (+addend)), and the
 *                           vdk_dwconv7_wgrad accumulation into dw49 / dbias (the training step's depthwise backward)
 *   vdk_layernorm_bwd       LayerNorm backward from the saved OUTPUT y and 1/sigma (patch = 2: through the 2x2 regrouping;
 *                           C a multiple of 8, <= 1536).  xhat = (y - beta) / gamma carries ulp(y) / (2 |gamma|) of error,
 *                           |beta / gamma| / |xhat| times bf16 precision; gamma = 0 takes xhat = 0 (that dgamma gets nothing)
 *   vdk_batchnorm_train_*   BatchNorm over the rows of [rows, C] with batch statistics (running stats updated) */
int vdk_dwconv7(int mode, const void* x, int batch, int H, int W, int C, const float* w49, const float* bias,
                const float* ln_w, const float* ln_b, float eps, void* y, float* rstd_out, const void* addend, void* stream);
int vdk_dwconv7_wgrad(const void* x, const void* dconv, int batch, int H, int W, int C, float* dw49, float* dbias,
                      void* stream);
int vdk_dwconv7_bwd(const void* x, const void* dconv, int batch, int H, int W, int C, const float* w49, const void* addend,
                    void* dx, float* dw49, float* dbias, void* stream);
int vdk_layernorm_bwd(const void* dy, const void* y, const float* rstd, int batch, int H, int W, int C, const float* ln_w,
                      const float* ln_b, int patch, void* dx, const void* addend, float* dgamma, float* dbeta, void* stream);
int vdk_batchnorm_train_fwd(const void* x, int rows, int C, int is_bf16, const float* weight, const float* bias, float eps,
                            float momentum, void* y, float* save_mean, float* save_rstd, float* running_mean,
                            float* running_var, void* stream);
int vdk_batchnorm_train_bwd(const void* dy, const void* x, int rows, int C, int is_bf16, const float* weight,
                            const float* save_mean, const float* save_rstd, void* dx, float* dweight, float* dbias,
                            void* stream);

size_t vdk_convnext_workspace_bytes(const vdk_convnext_net* net, int batch);
/* images: fp32 NCHW [batch,3,S,S] (what the reference's DataLoader yields); embeddings: fp32 [batch, feat_dim],
 * L2-normalised when l2_normalize != 0 (extract_cbir semantics). */
int vdk_convnext_forward(const vdk_convnext_net* net, const float* images, int batch, int l2_normalize,
                         float* embeddings, void* workspace, size_t workspace_bytes, void* stream);

/* ---- ViT inference forward (Transformer backbones of the CBIR extract path) ------------------- */
/* Replaces the eval forward of TimmWrapper for `timm-vit_*` backbones (models/faceX/backbone/timm_wrapper.py:16-21,
 * 39-47, 51-54: timm VisionTransformer with num_classes=0, global_pool='' -> every token after the final LayerNorm,
 * then LayerNorm -> Flatten -> Linear -> BatchNorm1d) as run by FeatureExtractor.extract_cbir (face_model.py:120-144).
 * All 16-bit weights are bf16 in nn.Linear layout [out, in]; vectors fp32; everything device memory. */
#define VDK_VIT_MAX_BLOCKS 48
typedef struct vdk_vit_block {
  const float* ln1_w; const float* ln1_b;
  const void* qkv_w;  const float* qkv_b;   /* [3*dim, dim], [3*dim]: rows ordered (q | k | v) x head x head_dim as in timm */
  const void* proj_w; const float* proj_b;  /* [dim, dim] */
  const float* ln2_w; const float* ln2_b;
  const void* fc1_w;  const float* fc1_b;   /* [mlp_dim, dim] */
  const void* fc2_w;  const float* fc2_b;   /* [dim, mlp_dim] */
  /* timm's LayerScale (DINOv2: blocks.{i}.ls1.gamma, ls2.gamma), [dim] each: x + ls1 * attn(...), x + ls2 * mlp(...).
   * NULL = no LayerScale.  Inference only. */
  const float* ls1; const float* ls2;
} vdk_vit_block;
typedef struct vdk_vit_net {
  int image_size, patch, dim, depth, heads, feat_dim;  /* head_dim = dim / heads: 64, 72 or 80 (training: 64) */
  const void* patch_w;      /* [dim, Kp] bf16, Kp = 3*patch*patch rounded up to 8, (c, kh, kw) order, zero padded */
  const float* patch_b;     /* [dim] */
  const float* cls_token;   /* [dim]; NULL = no class token (SigLIP, inference only): tokens = (image_size/patch)^2 */
  const float* pos_embed;   /* [tokens, dim]: [1 + (image_size/patch)^2, dim] with a class token */
  const float* ones;        /* [dim] of 1.0f (layer-scale slot of the residual epilogue: timm's default ViT has none) */
  vdk_vit_block blocks[VDK_VIT_MAX_BLOCKS];
  const float* norm_w; const float* norm_b;        /* model.norm, eps 1e-6 */
  const float* neck_ln_w; const float* neck_ln_b;  /* output_layer.0, eps 1e-5 */
  const void* neck_w;       /* [feat_dim, tokens*dim] bf16 with BatchNorm1d (eval) folded in */
  const float* neck_b;      /* [feat_dim] folded */
  /* timm's `pre_norm=True` variants (vit_*_clip_*: CLIP towers): a LayerNorm right after cls / position (model.norm_pre),
   * a bias-free patch embedding (patch_b == NULL) and LayerNorm eps 1e-5.  NULL / 0 = the plain ViT above (eps 1e-6).
   * Inference only: vdk_vit_train_* refuse a net with norm_pre_w set. */
  const float* norm_pre_w; const float* norm_pre_b;
  float ln_eps;             /* eps of norm_pre, the block norms and model.norm; 0 selects 1e-6 */
  int mlp_dim;              /* MLP hidden width (multiple of 8); 0 = 4 * dim.  Another width is inference only (SigLIP: 4304) */
} vdk_vit_net;
size_t vdk_vit_workspace_bytes(const vdk_vit_net* net, int batch);
/* images: fp32 NCHW [batch,3,S,S]; embeddings: fp32 [batch, feat_dim], L2-normalised when l2_normalize != 0. */
int vdk_vit_forward(const vdk_vit_net* net, const float* images, int batch, int l2_normalize, float* embeddings,
                    void* workspace, size_t workspace_bytes, void* stream);
/* softmax(Q K^T / sqrt(d)) V on the qkv Linear's output as stored: qkv bf16 [batch, tokens, 3, heads, head_dim] ->
 * out bf16 [batch, tokens, heads*head_dim]  (timm Attention.forward, scores never written to memory).  head_dim 64, 72 or 80
 * (other values: VDK_ERR_INVALID). */
int vdk_attention_fwd(const void* qkv, int batch, int tokens, int heads, int head_dim, void* out, void* stream);

/* ---- ViT training forward / backward (BASELINE config 3: ViT-B/16 + CircleLoss) ----------------------------------- */
/* fp32 tensors in timm layouts (parameters, or their gradients): what TimmWrapper('vit_*').train() holds. */
typedef struct vdk_vit_block_tensors {
  float* ln1_w; float* ln1_b; float* qkv_w; float* qkv_b; float* proj_w; float* proj_b;
  float* ln2_w; float* ln2_b; float* fc1_w; float* fc1_b; float* fc2_w; float* fc2_b;
} vdk_vit_block_tensors;
typedef struct vdk_vit_tensors {
  float* patch_w;   /* [dim, 3, P, P] */
  float* patch_b; float* cls_token; float* pos_embed;
  vdk_vit_block_tensors blocks[VDK_VIT_MAX_BLOCKS];
  float* norm_w; float* norm_b; float* neck_ln_w; float* neck_ln_b;
  float* lin_w;     /* output_layer.2.weight [feat_dim, tokens*dim] */
  float* lin_b;
  float* bn1_w; float* bn1_b; float* bn1_running_mean; float* bn1_running_var;  /* output_layer.3 */
} vdk_vit_tensors;
/* fp32 masters -> the bf16 GEMM weights of `net` (patch_w, qkv/proj/fc1/fc2, neck_w UNfolded: BatchNorm1d runs on batch
 * statistics in train mode).  Vector pointers of `net` are set by the caller (they may alias the masters). */
int vdk_vit_pack(const vdk_vit_tensors* params, vdk_vit_net* net, void* stream);
size_t vdk_vit_train_workspace_bytes(const vdk_vit_net* net, int batch);
/* Train-mode forward of TimmWrapper('vit_*') (timm_wrapper.py:51-54; neck :42-47 with BatchNorm1d batch statistics,
 * running stats updated): images fp32 NCHW -> out_feats fp32 [batch, feat_dim]; activations saved in `workspace`.
 * Needs 3*patch*patch % 8 == 0 and at most 208 tokens (the attention backward keeps one head's P in shared memory). */
int vdk_vit_train_forward(const vdk_vit_net* net, const vdk_vit_tensors* params, const float* images, int batch, float bn_momentum,
                          float* out_feats, void* workspace, size_t workspace_bytes, void* stream);
/* d_feats fp32 [batch, feat_dim] -> gradients ACCUMULATED (+=) into `grads`. */
int vdk_vit_train_backward(const vdk_vit_net* net, const vdk_vit_tensors* params, const vdk_vit_tensors* grads, const float* d_feats,
                           int batch, void* workspace, size_t workspace_bytes, void* stream);
/* The same backward in consecutive unit ranges (0 = neck + final LayerNorm, 1..depth = blocks depth-1..0, depth+1 = cls / position /
 * patch embedding): the DDP overlap of vdk_convnext_train_backward_range for Transformer backbones. */
int vdk_vit_train_backward_units(const vdk_vit_net* net);
int vdk_vit_train_backward_range(const vdk_vit_net* net, const vdk_vit_tensors* params, const vdk_vit_tensors* grads,
                                 const float* d_feats, int batch, void* workspace, size_t workspace_bytes, void* stream, int unit_begin,
                                 int unit_end);
/* The vdk_convnext_train_buffer of the ViT train workspace.  `index` selects the block (Y1 .. XO: 0 .. depth - 1); it is
 * ignored for the others. */
enum {
  VDK_VIT_TRAIN_ROWS, VDK_VIT_TRAIN_TOK, VDK_VIT_TRAIN_X0, VDK_VIT_TRAIN_Y1, VDK_VIT_TRAIN_R1, VDK_VIT_TRAIN_QKV, VDK_VIT_TRAIN_ATT,
  VDK_VIT_TRAIN_LSE, VDK_VIT_TRAIN_XM, VDK_VIT_TRAIN_Y2, VDK_VIT_TRAIN_R2, VDK_VIT_TRAIN_HPRE, VDK_VIT_TRAIN_HPOST, VDK_VIT_TRAIN_XO,
  VDK_VIT_TRAIN_F1, VDK_VIT_TRAIN_RF1, VDK_VIT_TRAIN_F2, VDK_VIT_TRAIN_RF2, VDK_VIT_TRAIN_Z, VDK_VIT_TRAIN_ZSLAB,
  VDK_VIT_TRAIN_BN_MEAN, VDK_VIT_TRAIN_BN_RSTD, VDK_VIT_TRAIN_DXA, VDK_VIT_TRAIN_DXB, VDK_VIT_TRAIN_DY, VDK_VIT_TRAIN_DBIG,
  VDK_VIT_TRAIN_DZ, VDK_VIT_TRAIN_DZB, VDK_VIT_TRAIN_GW, VDK_VIT_TRAIN_WSLAB, VDK_VIT_TRAIN_DTOK, VDK_VIT_TRAIN_NUM_BUFFERS
};
int vdk_vit_train_buffer(const vdk_vit_net* net, int batch, int id, int index, size_t* offset, size_t* bytes);
/* unit-test surface of the attention pair: forward that also saves the log2-domain log-sum-exp [batch, heads, tokens] (head_dim
 * 64, 72 or 80), and the backward dqkv = d(attention)/d(qkv) for d_out (both [batch, tokens, heads*64] bf16; head_dim 64 only). */
int vdk_attention_fwd_lse(const void* qkv, int batch, int tokens, int heads, int head_dim, void* out, float* lse2, void* stream);
int vdk_attention_bwd(const void* qkv, const void* out, const void* d_out, const float* lse2, int batch, int tokens, int heads,
                      int head_dim, void* dqkv, void* stream);

/* ---- margin-softmax heads + cross-entropy --------------------------------------------------- */
/* Replaces ArcFace.forward (models/faceX/head/arcface.py:20-36), CircleLoss.forward (models/faceX/head/
 * circleloss.py:21-43), nn.CrossEntropyLoss(label_smoothing) (models/losses/loss.py:71-73) and their autograd
 * backward, as called at engine/procedure/train.py:196.  fp32 in / fp32 out like the reference (no autocast on the
 * face path); the three contractions run on wgmma with a 3-way bf16 operand split (fp32-grade accuracy). */
#define VDK_HEAD_ARCFACE 0
#define VDK_HEAD_CIRCLELOSS 1
#define VDK_HEAD_MV_SOFTMAX 2 /* MV_Softmax.forward, models/faceX/head/mv_softmax.py:25-44 */

typedef struct vdk_head_desc {
  int kind;                 /* VDK_HEAD_* */
  int batch, feat_dim, num_class;
  float margin_arc, margin_am, scale; /* ArcFace(margin_arc, margin_am, scale); scale also MV_Softmax */
  float margin, gamma;                /* CircleLoss(margin, gamma); margin also MV_Softmax */
  float label_smooth;                 /* CrossEntropyLoss(label_smoothing) */
  float mv_weight;                    /* MV_Softmax(is_am, margin, mv_weight, scale) */
  int is_am;
} vdk_head_desc;

size_t vdk_head_workspace_bytes(const vdk_head_desc* d);
/* feats fp32 [B,D]; weight fp32 [D,C] (the head Parameter); labels int64 [B].
 * logits: fp32 [B,C] or NULL; loss: device scalar (mean CE); row_lse: fp32 [B] saved for the backward;
 * cos_saved: fp32 [B,C] clamped cos(theta) or NULL. */
int vdk_head_forward(const vdk_head_desc* d, const float* feats, const float* weight, const int64_t* labels,
                     float* logits, float* loss, float* row_lse, float* cos_saved, void* workspace,
                     size_t workspace_bytes, void* stream);
/* Fused backward of mean-CE(head(feats)) (dlogits == NULL; grad_loss: device scalar or NULL for 1), or the head-only
 * backward for a caller-supplied dlogits fp32 [B,C] (row_lse / grad_loss ignored).  dfeats [B,D], dweight [D,C]. */
int vdk_head_backward(const vdk_head_desc* d, const float* feats, const float* weight, const int64_t* labels,
                      const float* row_lse, const float* grad_loss, const float* dlogits, float* dfeats,
                      float* dweight, void* workspace, size_t workspace_bytes, void* stream);

/* Class-sharded head: rank `rank` of `world` holds the columns [class_offset, class_offset + d->num_class) of a head with
 * num_class_total classes, and every rank sees the same N = d->batch gathered rows (world equal batches of N / world, in rank
 * order) with GLOBAL labels.  The per-element arithmetic is the unsharded head's; with world = 1 and the whole head the five
 * calls below give vdk_head_forward / vdk_head_backward's results bit for bit.  Workspace: vdk_head_workspace_bytes(d), the
 * same buffer through one step (shard_forward reads the cosines shard_cos left in it, shard_finalize the normalised
 * features shard_backward left in it).  Label smoothing divides by num_class_total. */
typedef struct vdk_head_shard {
  int class_offset;     /* first class of this shard */
  int num_class_total;  /* C of the whole head (> 1); d->num_class is the shard's width (>= 1) */
  int world, rank;      /* d->batch is a multiple of world; this rank's own rows are [rank, rank + 1) * d->batch / world */
} vdk_head_shard;
/* sizeof(vdk_head_shard) (vdk_struct_sizes' contract for it). */
int vdk_head_shard_struct_sizes(size_t* out, int n);
/* 1. cos of the shard's columns into the workspace; label_cos fp32 [N]: the label column's cos where this shard owns the
 *    label, else 0 (summed over the ranks it is every row's label cos, which MV-Softmax needs before any logit). */
int vdk_head_shard_cos(const vdk_head_desc* d, const vdk_head_shard* s, const float* feats, const float* weight,
                       const int64_t* labels, float* label_cos, void* workspace, size_t workspace_bytes, void* stream);
/* 2. logits of the shard and per-row partials fp32 [N, 4]: (max z, sum exp(z - max), sum z, label z or 0).  label_cos: the
 *    rank-summed label cosines (MV-Softmax only; may be NULL otherwise).  logits / cos_saved: fp32 [N, d->num_class] or NULL. */
int vdk_head_shard_forward(const vdk_head_desc* d, const vdk_head_shard* s, const int64_t* labels, const float* label_cos,
                           float* logits, float* cos_saved, float* partials, void* workspace, size_t workspace_bytes,
                           void* stream);
/* 3. partials of every rank fp32 [world, N, 4] -> row_lse [N], row_loss [N] (CE with smoothing over num_class_total) and
 *    loss (device scalar): the mean of row_loss over this rank's own rows. */
int vdk_head_shard_combine(const vdk_head_desc* d, const vdk_head_shard* s, const float* partials, float* row_lse,
                           float* row_loss, float* loss, void* stream);
/* 4. dweight fp32 [D, d->num_class]: the gradient of the mean CE over all N rows (the rank-average of the per-rank losses'
 *    gradients); dfn fp32 [N, D]: this shard's part of d(loss_r)/d(normalised features) for every row, with each rank's
 *    loss the mean over its own rows (to be summed over the ranks).  grad_loss: device scalar or NULL for 1. */
int vdk_head_shard_backward(const vdk_head_desc* d, const vdk_head_shard* s, const float* feats, const float* weight,
                            const int64_t* labels, const float* label_cos, const float* row_lse, const float* grad_loss,
                            float* dfn, float* dweight, void* workspace, size_t workspace_bytes, void* stream);
/* 5. dfn summed over the ranks fp32 [N, D] -> dfeats fp32 [N / world, D] of this rank's own rows (normalisation backward). */
int vdk_head_shard_finalize(const vdk_head_desc* d, const vdk_head_shard* s, const float* dfn, float* dfeats,
                            void* workspace, size_t workspace_bytes, void* stream);

/* ---- optimizer step -------------------------------------------------------------------------- */
/* Replaces Trainer.update's clip_grad_norm_(max_norm=10) -> SGD step -> zero_grad -> ModelEMA.update
 * (engine/procedure/train.py:203-215, engine/optimizer.py:119-121, models/ema.py:28-37) on FLAT fp32 buffers
 * (parameters, gradients, momentum and EMA of one param group laid out contiguously by the caller). */
size_t vdk_grad_sumsq_workspace_bytes(void);
/* total_sumsq (device double) = [accumulate ? previous : 0] + sum(grads^2); deterministic summation order. */
int vdk_grad_sumsq(const float* grads, int64_t n, double* total_sumsq, int accumulate, void* workspace,
                   size_t workspace_bytes, void* stream);
/* One param group: g *= min(1, max_norm / (sqrt(total_sumsq) + 1e-6)); g += wd * p; buf = first_step ? g : mom*buf + g;
 * p -= lr * buf; ema = ema*d + (1-d)*p (ema may be NULL); g = 0 if zero_grad. */
int vdk_sgd_clip_ema_step(float* params, float* grads, float* momentum_buf, float* ema, int64_t n,
                          const double* total_sumsq, float max_norm, float lr, float momentum, float weight_decay,
                          int first_step, float ema_decay, float ema_one_minus_decay, int zero_grad, void* stream);
/* EMA of non-parameter float state (BatchNorm running statistics): ema = ema*d + (1-d)*src. */
int vdk_ema_update(float* ema, const float* src, int64_t n, float decay, float one_minus_decay, void* stream);

/* ---- retrieval: L2-normalise -> inner product -> top-k -------------------------------------- */
/* Replaces F.normalize at models/faceX/face_model.py:139, faiss index.add at
 * engine/cbir/evaluation.py:166-168 and faiss index.search at engine/cbir/evaluation.py:193
 * (cbir_eval.py:95,116).  Semantics: exact inner-product top-k; scores are the canonical fp32 scores
 * defined in oracle/retrieval.py (fixed-order fp64 accumulation), order = (score desc, id asc),
 * ids are int64, missing entries are id -1 / score -inf like faiss. */

/* Row preparation.  x: fp32 [n, dim] (pitch dim).  If `normalize`: xn = x / max(||x||, 1e-12) (F.normalize),
 * else xn = x.  Writes xn (fp32), xh = fp16(xn), row_norm[n] = ||xn||, row_err[n] >= ||xn - xh||.
 * Any of xn / row_norm may alias NULL to skip that output; xn may alias x (in place). */
int vdk_rows_prepare(const float* x, int64_t n, int dim, int normalize, float* xn, void* xh, float* row_norm,
                     float* row_err, void* stream);

typedef struct vdk_topk_plan {
  int64_t n_query;       /* rows of the query block */
  int64_t n_gallery;     /* rows of the (local shard of the) gallery */
  int dim;               /* embedding width, multiple of 64, <= 512 */
  int k;                 /* neighbours wanted, 1..1024 */
  int cand_capacity;     /* per-query slots for one range's admitted candidates (multiple of 32, >= 2k) */
  int carry_capacity;    /* per-query slots for survivors carried between ranges (in [2k, 4096]) */
  int n_stages;          /* gallery is scanned in n_stages ranges; thresholds tighten between them */
  int dense_mask;        /* bit s set: range s is scored densely (no admission threshold; must fit cand_capacity);
                            bit 0 is implied.  An all-dense plan cannot overflow a segment (the wide path). */
  int64_t stage_end[8];  /* exclusive end row of each stage (last == n_gallery) */
} vdk_topk_plan;

/* Fills stage boundaries / capacity for the given problem; returns VDK_OK. */
int vdk_topk_plan_default(vdk_topk_plan* plan, int64_t n_query, int64_t n_gallery, int dim, int k);
/* Scratch bytes vdk_ip_topk needs for this plan. */
size_t vdk_topk_workspace_bytes(const vdk_topk_plan* plan);

/* Exact inner-product top-k of q against g.
 *   q32/g32  : fp32 rows (what the scores are defined on), qh/gh: their fp16 copies from vdk_rows_prepare
 *   q_norm/q_err : per-query ||q|| and fp16 rounding-error norm; g_norm_max/g_err_max: device scalars, the
 *                  maxima over the gallery (vdk_reduce_max) — they bound the tensor-core score error.
 *   id_offset : added to every returned id (shard offset under multi-GPU sharding).
 *   out_scores: fp32 [n_query,k], out_ids: int64 [n_query,k].
 *   status    : device int32[4]: {overflow_rows, max_candidates_seen, rerank_rows_max, reserved}. */
int vdk_ip_topk(const vdk_topk_plan* plan, const float* q32, const void* qh, const float* q_norm,
                const float* q_err, const float* g32, const void* gh, const float* g_norm_max,
                const float* g_err_max, int64_t id_offset, float* out_scores, int64_t* out_ids, int32_t* status,
                void* workspace, size_t workspace_bytes, void* stream);

/* The two halves of vdk_ip_topk, for the SHARDED search (gallery rows split over GPUs, BASELINE config 4):
 *   vdk_ip_topk_filter  scans this shard (thresholds, ranges, selects), leaves every query's candidates in `workspace` and
 *                       writes kth_lb_out[n_query]: a lower bound of the shard's k-th largest canonical score (-inf if the
 *                       shard holds fewer than k rows);
 *   -- the ranks turn what they publish into a lower bound T of the GLOBAL k-th canonical score: the element-wise max of
 *      kth_lb, or better vdk_ip_topk_rank_sketch + vdk_topk_bound_from_sketches below --
 *   vdk_ip_topk_rerank  re-scores canonically only the candidates that can still reach the global top-k
 *                       (approx >= kth_lb_global - eps) and emits this shard's list, padded with (-FLT_MAX, -1).
 * The merged result (vdk_topk_merge*) is bit-identical to the unsharded search.  kth_lb_global == NULL re-ranks everything
 * (what vdk_ip_topk does).  Same plan, workspace and stream for both calls. */
int vdk_ip_topk_filter(const vdk_topk_plan* plan, const void* qh, const float* q_norm, const float* q_err, const void* gh,
                       const float* g_norm_max, const float* g_err_max, float* kth_lb_out, int32_t* status, void* workspace,
                       size_t workspace_bytes, void* stream);
/* The scan stage by stage, for shards that exchange their bounds BETWEEN gallery ranges: runs stages [stage_begin, stage_end) of
 * the plan (stage_begin == 0 initialises the workspace).  ext_lb (device fp32 [n_query], nullable): a lower bound of the GLOBAL
 * k-th canonical score derived from what all shards published after the previous stage (vdk_topk_bound_from_sketches) — it
 * tightens this shard's admission threshold and carry list (a candidate below ext_lb - eps cannot reach the global top-k), so
 * that after every exchange each shard filters as if it had scanned the union of all shards' prefixes.  kth_lb_out as in
 * vdk_ip_topk_filter, never below ext_lb. */
int vdk_ip_topk_filter_stages(const vdk_topk_plan* plan, const void* qh, const float* q_norm, const float* q_err, const void* gh,
                              const float* g_norm_max, const float* g_err_max, int stage_begin, int stage_end, const float* ext_lb,
                              float* kth_lb_out, int32_t* status, void* workspace, size_t workspace_bytes, void* stream);
int vdk_ip_topk_rerank(const vdk_topk_plan* plan, const float* q32, const float* g32, int64_t id_offset,
                       const float* kth_lb_global, float* out_scores, int64_t* out_ids, void* workspace, size_t workspace_bytes,
                       void* stream);

/* What shards exchange between gallery ranges (sharded search; no counterpart in the reference, which replicates the index:
 * engine/cbir/evaluation.py:159-162).  After `stages_done` stages of the plan ran (vdk_ip_topk_filter_stages), writes
 * sketch_out[n_query][n_ranks]: for every query and every ranks[i] (host array, 1 <= ranks[i] <= k, at most 8) a lower bound of
 * the canonical score of this shard's ranks[i]-th best row so far (-inf if it holds fewer candidates).  ranks[i] == k reports the
 * select's own k-th bound. */
int vdk_ip_topk_rank_sketch(const vdk_topk_plan* plan, int stages_done, const int32_t* ranks, int n_ranks, float* sketch_out,
                            void* workspace, size_t workspace_bytes, void* stream);
/* sketches: device fp32 [n_shards][n_query][n_ranks] (the all-gathered sketch_out of every shard, disjoint rows).
 * bound_inout[q] = max(bound_inout[q], largest reported score t with sum over shards of max{ranks[i] : sketch[i] >= t} >= k):
 * a lower bound of the GLOBAL k-th canonical score — the `ext_lb` of the next vdk_ip_topk_filter_stages call and the
 * kth_lb_global of vdk_ip_topk_rerank. */
int vdk_topk_bound_from_sketches(const float* sketches, int n_shards, int64_t n_query, const int32_t* ranks, int n_ranks, int k,
                                 float* bound_inout, void* stream);

/* Device pointer (inside `workspace`) to int32[n_query] flags the last vdk_ip_topk set for rows whose candidate lists
 * overflowed; status[0] counts them.  Their results are incomplete and must be recomputed with an all-dense plan. */
int vdk_topk_row_flags(const vdk_topk_plan* plan, const void* workspace, size_t workspace_bytes,
                       const int32_t** row_flags);

/* Exhaustive exact top-k for a FEW queries: canonical scores against every gallery row, exact selection on
 * (score desc, id asc) keys.  No candidate capacity, so it cannot overflow: the last resort for queries flagged by
 * vdk_ip_topk even under an all-dense plan (thousands of exact duplicates of a top-k member) — faiss' flat search
 * (engine/cbir/evaluation.py:193) answers such queries, so this path must too.  q32: fp32 [n_query, dim] (already
 * normalised if the index is a cosine index).  workspace >= vdk_ip_topk_exhaustive_workspace_bytes(n_gallery). */
size_t vdk_ip_topk_exhaustive_workspace_bytes(int64_t n_gallery);
int vdk_ip_topk_exhaustive(const float* q32, int64_t n_query, const float* g32, int64_t n_gallery, int dim, int k,
                           int64_t id_offset, float* out_scores, int64_t* out_ids, void* workspace, size_t workspace_bytes,
                           void* stream);

/* Measurement hook: launches ONLY the score/filter kernel of vdk_ip_topk for gallery rows [lo, hi), reusing the
 * thresholds a previous vdk_ip_topk left in `workspace` (dense != 0: the threshold-free first-range variant).
 * bench.py brackets this call with CUDA events to time the dominant kernel in isolation. */
int vdk_score_range(const vdk_topk_plan* plan, const void* qh, const void* gh, int64_t lo, int64_t hi, int dense,
                    void* workspace, size_t workspace_bytes, void* stream);

/* Max over a float vector into a device scalar (gallery-wide error/norm bounds). */
int vdk_reduce_max(const float* x, int64_t n, float* out, void* stream);

/* Merge `n_lists` per-shard top-k lists (each [n_query,k], already ordered) into the global top-k with
 * the same (score desc, id asc) rule.  Replaces faiss' IndexShards merge (the reference uses replicas,
 * engine/cbir/evaluation.py:159-162; sharding is BASELINE config 4). */
int vdk_topk_merge(const float* scores, const int64_t* ids, int n_lists, int64_t n_query, int k, float* out_scores,
                   int64_t* out_ids, void* stream);

/* The exchange format of the sharded search: one 64-bit word per list entry, (fp32 score bits << 32) | uint32 id
 * (id -1, the padding, becomes 0xffffffff; global ids must therefore stay below 2^32 - 1), so that the ranks' lists travel in
 * ONE all-gather.  vdk_topk_pack: (scores, ids)[n] -> packed[n].  vdk_topk_merge_packed: packed [n_lists, n_query, k] ->
 * global top-k, same rule as vdk_topk_merge. */
int vdk_topk_pack(const float* scores, const int64_t* ids, int64_t n, void* packed, void* stream);
int vdk_topk_merge_packed(const void* packed, int n_lists, int64_t n_query, int k, float* out_scores, int64_t* out_ids,
                          void* stream);

/* Brute-force canonical scores for verification at full size: out[i] = canonical_score(q[qi[i]], g[gi[i]]). */
int vdk_ip_exact_pairs(const float* q32, const float* g32, int dim, const int64_t* qi, const int64_t* gi, int64_t n,
                       float* out, void* stream);

/* ---- eval-time image preprocessing (SURVEY.md §8f-3: the GPU input pipeline) ------------------------------------------ */
/* Replaces, for a BATCH of decoded RGB images of different sizes, the `val.augment` list of configs/faceX/{face,cbir}.yaml:
 * ResizeAndPadding2Square(size, training=False) (dataset/transforms.py:325-365: PIL Image.resize(BILINEAR) of the longer side
 * to `size`, centred on a black square), T.ToTensor (:466-468) and T.Normalize(mean, std) (:474-477).  Bit-exact with
 * Pillow's 8-bit resampling + torch's fp32 arithmetic (oracle/preprocess.py, pinned against the installed Pillow / torchvision).
 *   packed : DEVICE uint8, every image as [height][width][3] (RGB) at images[i].offset
 *   images : HOST array of n descriptors
 *   out    : DEVICE fp32 [n, 3, size, size]
 * The call computes the resampling coefficients on the host (double precision, like Pillow), uploads them and synchronises
 * the stream once before launching (JPEG decoding itself stays on the host: out of scope). */
typedef struct vdk_image_desc {
  int64_t offset;   /* bytes from `packed` to the image's first pixel */
  int width, height;
} vdk_image_desc;
size_t vdk_preprocess_workspace_bytes(const vdk_image_desc* images, int n, int size);
int vdk_preprocess_resize_pad_normalize(const uint8_t* packed, const vdk_image_desc* images, int n, int size, const float* mean,
                                        const float* std_, float* out, void* workspace, size_t workspace_bytes, void* stream);

/* ---- training-time image augmentation (the `data.train.augment` list of configs/faceX/{face,cbir}.yaml) ---------------- */
/* Replaces, for a BATCH of decoded RGB images of different sizes at source resolution, the reference's training Compose
 * (dataset/transforms.py:403-555 as built by create_AugTransforms): per image an ordered list of byte-exact PIL stages, then
 * one resize stage into the size x size square, then ToTensor + Normalize.  The random draws are made on the host
 * (visiondk_b200/augment.py, in the reference's order and streams); a plan holds their outcome.
 *   BRIGHTNESS / SATURATION / CONTRAST : PIL.ImageEnhance.{Brightness,Color,Contrast}.enhance(alpha) (torchvision ColorJitter,
 *                                        transforms.py:170-179); the contrast mean is reduced on the device
 *   HUE        : torchvision adjust_hue on PIL (RGB->HSV, uint8 wrap-add of hue_shift, HSV->RGB)
 *   CUTOUT     : Image.paste of n solid boxes (transforms.py:63-109): box = x1, y1, mask_w, mask_h; color = r, g, b
 *   BLUR       : torchvision gaussian_blur on PIL (transforms.py:510-512): n-tap fp32 kernel, reflect padding, torch.round
 *   ROTATE     : Image.rotate(angle, BILINEAR), no expand, fill 0 (transforms.py:463-465): matrix = Pillow's affine matrix
 *   SHARPNESS  : ImageEnhance.Sharpness.enhance(alpha) (transforms.py:427-429)
 *   HFLIP      : T.RandomHorizontalFlip (transforms.py:451-453)
 * and the resize stage: ResizeAndPadding2Square(size, training=True) with BILINEAR or NEAREST (transforms.py:325-362), or
 * RandomResizedCrop's crop box resized to size x size with BILINEAR (transforms.py:390-400).
 *   packed : DEVICE uint8, every image as [height][width][3] (RGB) at images[i].offset
 *   images, plans : HOST arrays of n entries
 *   out    : DEVICE fp32 [n, 3, size, size]
 * The call uploads the plans and resampling tables and synchronises the stream once before launching. */
#define VDK_AUG_MAX_OPS 8
#define VDK_AUG_MAX_HOLES 8
#define VDK_AUG_MAX_KERNEL 9
enum { VDK_AUG_BRIGHTNESS = 1, VDK_AUG_CONTRAST = 2, VDK_AUG_SATURATION = 3, VDK_AUG_HUE = 4, VDK_AUG_CUTOUT = 5,
       VDK_AUG_BLUR = 6, VDK_AUG_ROTATE = 7, VDK_AUG_SHARPNESS = 8, VDK_AUG_HFLIP = 9 };
enum { VDK_AUG_RESIZE_PAD_BILINEAR = 0, VDK_AUG_RESIZE_PAD_NEAREST = 1, VDK_AUG_CROP_RESIZE = 2 };
typedef struct vdk_aug_op {
  double matrix[6];                  /* ROTATE: output pixel centre -> input position, as Pillow's Image.rotate builds it */
  float alpha;                       /* BRIGHTNESS, SATURATION, CONTRAST, SHARPNESS: the blend factor */
  int kind;                          /* VDK_AUG_* */
  int hue_shift;                     /* HUE: np.int32(hue_factor * 255).astype(np.uint8) */
  int n;                             /* CUTOUT: hole count; BLUR: kernel size (odd, <= VDK_AUG_MAX_KERNEL) */
  float kernel[VDK_AUG_MAX_KERNEL];  /* BLUR: torchvision's fp32 1-D gaussian kernel (the 2-D one is its fp32 outer product) */
  int box[VDK_AUG_MAX_HOLES][4];     /* CUTOUT: x1, y1, mask_w, mask_h of each hole, pasted in order */
  int color[VDK_AUG_MAX_HOLES][3];   /* CUTOUT: r, g, b of each hole */
} vdk_aug_op;
typedef struct vdk_aug_plan {
  vdk_aug_op ops[VDK_AUG_MAX_OPS];   /* applied in order at source resolution */
  int n_ops;
  int resize;                        /* VDK_AUG_RESIZE_PAD_BILINEAR / _NEAREST / VDK_AUG_CROP_RESIZE */
  int crop[4];                       /* CROP_RESIZE: left, top, width, height of the box (torchvision's j, i, w, h) */
} vdk_aug_plan;
size_t vdk_augment_workspace_bytes(const vdk_image_desc* images, const vdk_aug_plan* plans, int n, int size);
int vdk_augment_batch(const uint8_t* packed, const vdk_image_desc* images, const vdk_aug_plan* plans, int n, int size,
                      const float* mean, const float* std_, float* out, void* workspace, size_t workspace_bytes, void* stream);
/* sizeof() of vdk_aug_op and vdk_aug_plan, in that order (vdk_struct_sizes' contract for these two). */
int vdk_augment_struct_sizes(size_t* out, int n);

/* ---- baseline JPEG decoding (the image-folder input path: `Image.open(path).convert("RGB")`, dataset/basedataset.py:234-241) */
/* Decodes, for a BATCH of compressed files, the baseline JPEGs that libjpeg-turbo (as Pillow calls it: JDCT_ISLOW, fancy
 * upsampling, no draft mode) decodes, bit for bit: one SOF0/SOF1 frame of 8-bit samples, one interleaved Huffman scan over
 * all components, 1 component (Y replicated into R, G, B) or 3 components in YCbCr (JFIF, Adobe transform 1, or neither
 * marker and component ids other than 'R','G','B'), sampling 4:4:4, 4:2:2 (h2v1), 4:2:0 (h2v2) or 4:4:0 (h1v2), any restart
 * interval.  Everything else gets a fallback reason and is left to the host decoder (oracle/jpeg.py restates the arithmetic).
 *
 * 1. vdk_jpeg_parse (host only, no GPU): reads the headers of n files at packed + descs[i].data_offset (descs[i].data_bytes
 *    long) and fills the rest of each descriptor; descs[i].reason is VDK_JPEG_DEVICE or the fallback reason.  It also writes
 *    where each restart interval of the VDK_JPEG_DEVICE images starts (bytes from the file's start) into segs: image i's
 *    n_segments entries from segs[descs[i].seg_first], images one after the other.  Entries past seg_capacity are not
 *    written: when the last device image's seg_first + n_segments exceeds it, call again with a larger array.  Returns
 *    VDK_OK (a file the device does not take is not an error).
 * 2. the caller sets descs[i].out_offset (256-byte aligned) for every VDK_JPEG_DEVICE image: where its packed
 *    [height][width][3] RGB goes in `out` (the vdk_image_desc layout).
 * 3. vdk_jpeg_workspace_bytes (host only): lays the device images out in the workspace — writes their ws_* and *_cta_base
 *    fields and returns the bytes needed (2 bytes per coefficient + 1 per decoded sample), 0 on bad input.
 * 4. the caller copies the descriptors and the restart-interval table to the device (`descs_dev`, `segs_dev`, same bytes) and
 *    calls vdk_jpeg_decode with the same host descriptors: three kernels on `stream` (Huffman decode into int16
 *    coefficients, dequantise + islow IDCT into component planes, upsampling + YCbCr->RGB into `out`).  status[i] (DEVICE
 *    int32, n entries) is 0 when image i was decoded, or an OR of VDK_JPEG_BAD_* when its stream is not well formed (then
 *    `out` holds no valid pixels for it and the host decodes it); images that are not VDK_JPEG_DEVICE get
 *    VDK_JPEG_BAD_SKIPPED.  No allocation, no synchronisation.  `data` is the DEVICE copy of the packed files (same offsets
 *    as at parse time). */
enum { VDK_JPEG_DEVICE = 0, VDK_JPEG_NOT_JPEG = 1, VDK_JPEG_PROCESS = 2, VDK_JPEG_PRECISION = 3, VDK_JPEG_COLOR = 4,
       VDK_JPEG_SAMPLING = 5, VDK_JPEG_SCAN = 6, VDK_JPEG_MALFORMED = 7, VDK_JPEG_MPO = 8, VDK_JPEG_RESTART = 9,
       VDK_JPEG_TOO_LARGE = 10 /* a side above libjpeg's 65500, or more pixels than PIL.Image.MAX_IMAGE_PIXELS */ };
enum { VDK_JPEG_BAD_CODE = 1,      /* no Huffman code matches the next 16 bits */
       VDK_JPEG_BAD_AC_RUN = 2,    /* an AC run past coefficient 63 */
       VDK_JPEG_BAD_SHORT = 4,     /* a marker or the end of the scan before the last MCU of a restart interval */
       VDK_JPEG_BAD_EXTRA = 8,     /* whole bytes left over before a marker */
       VDK_JPEG_BAD_SKIPPED = 16 };
typedef struct vdk_jpeg_huff {
  uint16_t lut[512];      /* next 9 bits -> (code length << 8) | symbol; 0 when the code is longer than 9 bits */
  int32_t maxcode[18];    /* largest code of each length (-1: none); maxcode[17] is a sentinel above every 16-bit code */
  int32_t valoffset[17];  /* symbol of a code of length l = huffval[code + valoffset[l]] */
  uint8_t huffval[256];
} vdk_jpeg_huff;
typedef struct vdk_jpeg_desc {
  int64_t data_offset, data_bytes;  /* in: the file within the packed buffer */
  int64_t out_offset;               /* in (after parse): the RGB image within `out` */
  int64_t scan_begin, scan_end;     /* entropy-coded bytes [begin, end) from data_offset; scan_end is the EOI marker */
  int64_t seg_first;                /* set by vdk_jpeg_parse: the image's first entry in the restart-interval table */
  int64_t ws_coef, ws_plane;        /* set by vdk_jpeg_workspace_bytes: workspace byte offsets */
  int64_t idct_cta_base, color_cta_base;      /* set by vdk_jpeg_workspace_bytes: first CTA of the image in the grids */
  int width, height, ncomp, reason;
  int restart_interval;             /* MCUs per restart interval, 0 = none */
  int n_segments;                   /* restart intervals in the scan (1 without DRI) */
  int mcus_x, mcus_y, hmax, vmax;
  int h[3], v[3];                   /* sampling factors (1 x 1 for a single component) */
  int16_t quant[3][64];             /* natural order, cast to 16 bits like libjpeg's ISLOW_MULT_TYPE */
  vdk_jpeg_huff dc[3], ac[3];       /* per component */
  int64_t scan_first;               /* set by vdk_jpeg_parse_progressive: the image's first entry in the scan table */
  int n_scans, n_levels;            /* set by vdk_jpeg_parse_progressive: its scans, and 1 + their largest level */
} vdk_jpeg_desc;
int vdk_jpeg_parse(const uint8_t* packed, vdk_jpeg_desc* descs, int n, int64_t* segs, int64_t seg_capacity);
size_t vdk_jpeg_workspace_bytes(vdk_jpeg_desc* descs, int n);
int vdk_jpeg_decode(const uint8_t* data, const vdk_jpeg_desc* descs, const vdk_jpeg_desc* descs_dev, const int64_t* segs_dev,
                    int n, uint8_t* out, int32_t* status, void* workspace, size_t workspace_bytes, void* stream);
/* sizeof() of vdk_jpeg_huff and vdk_jpeg_desc, in that order. */
int vdk_jpeg_struct_sizes(size_t* out, int n);

/* ---- progressive JPEG decoding (the same input path; the same descriptors, workspace and status words) */
/* Decodes, bit for bit with the same libjpeg-turbo call, the progressive JPEGs whose frame the baseline decoder would take:
 * one SOF2 frame of 8-bit samples, 1 component or 3 in YCbCr, sampling 4:4:4 / 4:2:2 / 4:2:0 / 4:4:0, any restart interval,
 * and any scan script that libjpeg (jdphuff.c) accepts without a warning and that brings every coefficient of every
 * component to full precision (so libjpeg's block smoothing of incomplete scripts never applies).  Each scan uses the DHT and
 * DRI in force at its SOS; quantisation tables are latched at the first scan that contains the component (jdinput.c).
 * oracle/jpeg_progressive.py restates the arithmetic.
 *
 * 1. vdk_jpeg_parse as for baseline files; it gives progressive files VDK_JPEG_PROCESS.
 * 2. vdk_jpeg_parse_progressive (host only, no GPU): re-reads only the descriptors whose reason is VDK_JPEG_PROCESS and
 *    fills them like a baseline descriptor (size, components, sampling, MCU grid, latched quantisation tables; dc / ac are
 *    not used).  Their reason becomes VDK_JPEG_DEVICE_PROGRESSIVE or a fallback reason (VDK_JPEG_PROCESS for arithmetic,
 *    lossless and hierarchical frames; VDK_JPEG_SCAN for scripts that leave a coefficient unsent or not fully refined, or
 *    that libjpeg warns about (JWRN_BOGUS_PROGRESSION); VDK_JPEG_MALFORMED for scan parameters libjpeg refuses
 *    (JERR_BAD_PROGRESSION) and the header faults vdk_jpeg_parse refuses).  Every scan of a progressive image goes into
 *    `scans` (n_scans entries from scans[descs[i].scan_first]), and the restart-interval starts of each scan go into `segs`
 *    after those vdk_jpeg_parse wrote (scan j's n_segments entries from segs[scan.seg_first]; the image's descriptor spans
 *    them all with seg_first / n_segments).  Entries past scan_capacity / seg_capacity are not written: call both parsers
 *    again with larger arrays.  Returns VDK_OK.
 * 3. out_offset as in step 2 above, for the VDK_JPEG_DEVICE and VDK_JPEG_DEVICE_PROGRESSIVE images; vdk_jpeg_workspace_bytes
 *    lays out both kinds.
 * 4. vdk_jpeg_decode_ex: vdk_jpeg_decode plus the scan table (host `scans`, device copy `scans_dev`): the baseline Huffman
 *    kernel, then one progressive Huffman launch per dependency level across the batch (one thread per image, scan of that
 *    level and restart interval: jdphuff.c's DC first / DC refine / AC first / AC refine into the same zero-initialised int16
 *    store), then the IDCT and colour kernels once over both kinds.  Status words as for vdk_jpeg_decode (0 for a decoded
 *    image of either kind).  vdk_jpeg_decode itself skips VDK_JPEG_DEVICE_PROGRESSIVE images (VDK_JPEG_BAD_SKIPPED). */
enum { VDK_JPEG_DEVICE_PROGRESSIVE = 11 };
typedef struct vdk_jpeg_scan {
  int64_t scan_begin, scan_end;     /* entropy-coded bytes [begin, end) from the file's start; scan_end is the next marker */
  int64_t seg_first;                /* the scan's first entry in the restart-interval table */
  int n_segments;                   /* restart intervals in the scan (1 without DRI) */
  int restart_interval;             /* DRI in force at the SOS: MCUs (blocks in a one-component scan) per interval, 0 = none */
  int level;                        /* 1 + the largest level of the earlier scans that share a component and a coefficient
                                       with this one (0 if none): scans of one level write disjoint coefficients */
  int ncomp;                        /* components in the scan; more than one only in a DC scan (interleaved over MCUs) */
  int comp[3];                      /* their frame indexes, in frame order */
  int ss, se, ah, al;               /* spectral selection and successive approximation */
  int units_x, units_y;             /* MCU grid of an interleaved scan; the component's own blocks in a one-component scan */
  vdk_jpeg_huff tbl[3];             /* DC first: the DC table of each scan component; AC: tbl[0] is the AC table */
} vdk_jpeg_scan;
int vdk_jpeg_parse_progressive(const uint8_t* packed, vdk_jpeg_desc* descs, int n, vdk_jpeg_scan* scans, int64_t scan_capacity,
                               int64_t* segs, int64_t seg_capacity);
int vdk_jpeg_decode_ex(const uint8_t* data, const vdk_jpeg_desc* descs, const vdk_jpeg_desc* descs_dev, const int64_t* segs_dev,
                       const vdk_jpeg_scan* scans, const vdk_jpeg_scan* scans_dev, int n, uint8_t* out, int32_t* status,
                       void* workspace, size_t workspace_bytes, void* stream);
/* sizeof() of vdk_jpeg_scan. */
int vdk_jpeg_progressive_struct_sizes(size_t* out, int n);

/* Live kernel timing inside a real step (bench.py's roofline legs; not part of the reference's surface).  Between
 * vdk_prof_begin() and vdk_prof_end() every launch of the categories below is bracketed by two CUDA events on the stream it
 * is launched on; vdk_prof_end synchronises on them and returns, per category, the launch count, the summed event time and
 * the summed ALGORITHMIC flops / bytes of those launches.  Categories: 0 wgmma GEMM (vdk_gemm and every internal GEMM),
 * 1 depthwise 7x7 (forward+LN, data gradient, weight gradient), 2 attention (forward, backward), 3 retrieval score/filter,
 * 4 other.  Profiling perturbs the step (two event records per launch): never time a step with a profile open. */
typedef struct vdk_prof_total {
  long long launches;
  double ms;
  double flops;
  double bytes;
} vdk_prof_total;
#define VDK_PROF_CATEGORIES 5
int vdk_prof_begin(void);
int vdk_prof_end(vdk_prof_total* totals, int n_categories);

/* sizeof() of the by-pointer structs, in this order: vdk_gemm_desc, vdk_topk_plan, vdk_head_desc, vdk_convnext_net,
 * vdk_convnext_tensors, vdk_vit_net, vdk_vit_tensors.  Writes min(n, count) entries, returns the count: a binding checks its mirrors. */
int vdk_struct_sizes(size_t* out, int n);

#ifdef __cplusplus
}
#endif
#endif /* VDK_B200_H_ */
