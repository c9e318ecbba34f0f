// convnext_internal.h — launchers shared between the inference forward (convnext.cu) and the training
// forward/backward (convnext_train.cu).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

namespace vdk {

// mode 0: y = LayerNorm_C(dwconv7(x) + bias) (rstd_out optional: 1/sigma per pixel for the backward)
// mode 1: y = dwconv7(x) with the taps `w49` as given (+ addend): the backward-data pass uses reversed taps
int launch_dwconv7(int mode, const __nv_bfloat16* x, int batch, int H, int W, int C, const float* w49, const float* bias,
                   const float* ln_w, const float* ln_b, float eps, __nv_bfloat16* y, float* rstd_out,
                   const __nv_bfloat16* addend, cudaStream_t s);

// 4x4/stride-4 patches of the fp32 NCHW images [B, 3, S, S] -> bf16 rows [B*(S/4)^2, 48] in (c, kh, kw) order
int launch_stem_patchify(const float* images, int B, int S, __nv_bfloat16* out, cudaStream_t s);

// out = LayerNorm_C(x) per pixel, patch == 2: regrouped into 2x2/s2 patch rows (kh, kw, c); rstd_out optional
int launch_ln_patchify(const __nv_bfloat16* x, int B, int H, int W, int C, const float* ln_w, const float* ln_b, float eps,
                       int patch, __nv_bfloat16* out, float* rstd_out, cudaStream_t s);

// embeddings[row] = bias + sum of split-K slabs (fixed order) [, canonically L2-normalised]
// The CNN neck (BN2d -> Flatten -> Linear -> BN1d folded into neck_w / neck_b): feats [batch, Kn] bf16 (the final map in
// (h, w, c) order) -> embeddings [batch, F] fp32 [, L2-normalised], as a deterministic split-K GEMM whose fp32 slabs go
// to `scratch` (as many splits as fit in scratch_bytes, up to ~2 waves) + neck_finalize.
int launch_neck(const __nv_bfloat16* feats, int batch, int Kn, int F, const void* neck_w, const float* neck_b, int l2_normalize,
                float* scratch, size_t scratch_bytes, float* embeddings, cudaStream_t s);

int launch_neck_finalize(const float* slabs, int n_slabs, size_t slab_stride, int B, int F, const float* bias, int l2norm,
                         float* out, cudaStream_t s);

// ---- CNN pieces of resnet.cu shared with effnet.cu and mobilenetv3.cu ----
// gate[b, :] = g(w2 act(w1 mean[b, :] + b1) + b2) in fp32, act = ReLU (silu_hidden 0) or SiLU (1), g = sigmoid (hard_gate 0)
// or relu6(v + 3) / 6 (1); C + rd floats of shared memory
int launch_se_excite(const float* mean, int batch, int C, int rd, int silu_hidden, int hard_gate, const float* w1,
                     const float* b1, const float* w2, const float* b2, float* gate, cudaStream_t s);
// explicit im2col rows of fp32 NCHW images: out[m][(dy k + dx) C + c] bf16, zero outside the image and from k*k*C to Kp
int launch_patch_rows_nchw(const float* x, int B, int H, int W, int C, int k, int stride, int pad, int Ho, int Wo, int Kp,
                           __nv_bfloat16* out, cudaStream_t s);
// the same rows of NHWC bf16 maps (the deep stem's second and third convs)
int launch_patch_rows_nhwc(const __nv_bfloat16* x, int B, int H, int W, int C, int k, int stride, int pad, int Ho, int Wo, int Kp,
                           __nv_bfloat16* out, cudaStream_t s);
// timm's ResNet stem pool MaxPool2d(3, 2, padding 1) over NHWC bf16 (C a multiple of 8)
int launch_stem_maxpool(const __nv_bfloat16* x, int B, int H, int W, int C, __nv_bfloat16* y, cudaStream_t s);

// ---- MBConv pieces of effnet.cu shared with mobilenetv3.cu ----
// d[m, c] = bf16(d[m, c] * gate[m / HW, c]) in place over d [M, C] bf16 (C a multiple of 8)
int launch_se_apply(__nv_bfloat16* d, const float* gate, int64_t M, int HW, int C, cudaStream_t s);
// p[0 .. n) = v
int launch_fill(float* p, int n, float v, cudaStream_t s);

inline size_t up256(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }
// a grid-stride launch over `threads` threads: at most 16 CTAs of 256 per SM of the H100's 132
inline int grid_for(int64_t threads) { return static_cast<int>((threads + 255) / 256 < 132 * 16 ? (threads + 255) / 256 : 132 * 16); }
// TensorFlow "same" padding of one axis: the output has ceil(H / s) positions
inline void same_pad(int H, int k, int s, int& lo, int& hi) {
  const int out = (H + s - 1) / s;
  const int total = (out - 1) * s + k - H > 0 ? (out - 1) * s + k - H : 0;
  lo = total / 2;
  hi = total - lo;
}

}  // namespace vdk

namespace vdk {
// ---- training-side launchers (train_ops.cu) ----
int launch_ln_bwd(const __nv_bfloat16* dy, const __nv_bfloat16* y, const float* rstd, int B, int H, int W, int C,
                  const float* ln_w, const float* ln_b, int patch, __nv_bfloat16* dx, const __nv_bfloat16* addend,
                  float* dgamma, float* dbeta, cudaStream_t s);
// depthwise 7x7 backward from one staging of dconv: dx = bf16(correlation of dconv with w49 + addend) unless w49 is null,
// dw49 += / dbias += the weight gradient against x unless dw49 is null
int launch_dwconv7_bwd(const __nv_bfloat16* x, const __nv_bfloat16* dconv, int B, int H, int W, int C, const float* w49,
                       const __nv_bfloat16* addend, __nv_bfloat16* dx, float* dw49, float* dbias, cudaStream_t s);
int launch_permute021(const float* in, int A, int Bd, int Cd, const float* row_scale, __nv_bfloat16* out_bf16,
                      float* out_f32, int accumulate, cudaStream_t s);
int launch_cast_bf16(const float* in, int64_t n, __nv_bfloat16* out, cudaStream_t s);
int launch_layerscale_finalize(const float* G, const float* W2, const float* b2, const float* gamma, const float* sdo, int C,
                               int K4, float* dW2, float* dgamma, float* db2, cudaStream_t s);
int launch_bn_fwd_bf16(const __nv_bfloat16* x, int R, int C, const float* w, const float* b, float eps, float momentum,
                       __nv_bfloat16* y, float* save_mean, float* save_rstd, float* run_mean, float* run_var, cudaStream_t s);
int launch_bn_fwd_f32(const float* x, int R, int C, const float* w, const float* b, float eps, float momentum, float* y,
                      float* save_mean, float* save_rstd, float* run_mean, float* run_var, cudaStream_t s);
int launch_bn_bwd_bf16(const __nv_bfloat16* dy, const __nv_bfloat16* x, int R, int C, const float* w, const float* save_mean,
                       const float* save_rstd, __nv_bfloat16* dx, float* dweight, float* dbias, cudaStream_t s);
int launch_bn_bwd_f32(const float* dy, const float* x, int R, int C, const float* w, const float* save_mean,
                      const float* save_rstd, float* dx, float* dweight, float* dbias, cudaStream_t s);
int launch_add_f32(float* dst, const float* src, int64_t n, cudaStream_t s);
}  // namespace vdk
