// heads.cu — margin-softmax heads (ArcFace, CircleLoss) fused with cross-entropy, forward and backward.
//
// Replaces, for the faceX train step (engine/procedure/train.py:196: criterion(model(images, labels), labels)):
//   ArcFace.forward     models/faceX/head/arcface.py:20-36
//   CircleLoss.forward  models/faceX/head/circleloss.py:21-43
//   ce                  models/losses/loss.py:71-73 (nn.CrossEntropyLoss(label_smoothing))
// and their autograd backward.
//
// The reference runs this path in fp32 (no autocast, train.py:227).  The class-logit contraction cos = f~ . W~ and the
// two gradient contractions run on the wgmma GEMM with a 3-way bf16 split of every fp32 operand
// (x = p0 + p1 + p2, 8 mantissa bits each; the six products with i + j <= 2 are laid side by side along K).  Verified
// against fp64 (tests/test_heads_fp64_gpu.py): every output within its fp32 rounding bound; the cos RMS error, in units of
// 2^-24 sum|f~_k w~_k|, is 1.0 at D = 16, 3.0 at D = 128 and 6.2 at D = 512 on an H100 SXM, growing like sqrt(D) because
// the wgmma fp32 accumulator does not round to nearest (torch's fp32 matmul: 0.3-0.4; a 2-part split: 4-8 at D = 128).
// The same drift over dF~'s K = 6 Cp (3.5e5 at C = 58 671) gave an RMS of 31; dF~ therefore runs as fixed-order split-K
// slabs (dfn_splits), which measure 0.09.  Everything else (row/column normalisation, margins, online softmax, the normalisation backward) is fused into a few
// HBM-bound kernels.
#include "train_gemm.h"
#include "vdk_host.h"
#include "vdk_ptx.cuh"

#include <cfloat>

namespace vdk {

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}
__device__ __forceinline__ float warp_max_f(float v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, off));
  return v;
}

// part i of the 3-way bf16 split of x
__device__ __forceinline__ void split3(float x, __nv_bfloat16 (&p)[3]) {
  p[0] = __float2bfloat16_rn(x);
  const float r1 = x - __bfloat162float(p[0]);
  p[1] = __float2bfloat16_rn(r1);
  const float r2 = r1 - __bfloat162float(p[1]);
  p[2] = __float2bfloat16_rn(r2);
}
// term t of the side-by-side product layout: A-side uses parts (0,0,1,1,0,2), B-side (0,1,0,1,2,0)
__device__ __forceinline__ int split_part(int t, int b_side) {
  const int a_pat[6] = {0, 0, 1, 1, 0, 2};
  const int b_pat[6] = {0, 1, 0, 1, 2, 0};
  return b_side ? b_pat[t] : a_pat[t];
}

// dst[r, t*Kp + k] = part_t(src[r*ld + k] * scale_r * scale_k), r < R, k < K (zero for K <= k < Kp)
__global__ void __launch_bounds__(256)
split3_rows_kernel(const float* __restrict__ src, int R, int K, int ld, int Kp, const float* __restrict__ row_scale,
                   const float* __restrict__ col_scale, int b_side, __nv_bfloat16* __restrict__ dst,
                   float* __restrict__ scaled_copy /* [R,K] or null */) {
  const int64_t total = static_cast<int64_t>(R) * Kp;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / Kp), k = static_cast<int>(i % Kp);
    float v = 0.f;
    if (k < K) {
      v = src[static_cast<int64_t>(r) * ld + k];
      if (row_scale) v *= row_scale[r];
      if (col_scale) v *= col_scale[k];
      if (scaled_copy) scaled_copy[static_cast<int64_t>(r) * K + k] = v;
    }
    __nv_bfloat16 p[3];
    split3(v, p);
    __nv_bfloat16* d = dst + static_cast<int64_t>(r) * 6 * Kp + k;
#pragma unroll
    for (int t = 0; t < 6; ++t) d[static_cast<int64_t>(t) * Kp] = p[split_part(t, b_side)];
  }
}

// transposing variant: src is [K, R] (element (k, r) at src[k*ld + r]); dst[r, t*Kp + k] = part_t(src * scale_r)
__global__ void __launch_bounds__(256)
split3_cols_kernel(const float* __restrict__ src, int R, int K, int ld, int Rp, int Kp, const float* __restrict__ out_row_scale,
                   int b_side, __nv_bfloat16* __restrict__ dst) {
  __shared__ float tile[32][33];
  const int r0 = blockIdx.x * 32, k0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int j = ty; j < 32; j += 8) {
    const int k = k0 + j, r = r0 + tx;
    tile[j][tx] = (k < K && r < R) ? src[static_cast<int64_t>(k) * ld + r] : 0.f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int r = r0 + j, k = k0 + tx;
    if (r < Rp && k < Kp) {
      float v = tile[tx][j];
      if (out_row_scale && r < R) v *= out_row_scale[r];
      __nv_bfloat16 p[3];
      split3(v, p);
      __nv_bfloat16* d = dst + static_cast<int64_t>(r) * 6 * Kp + k;
#pragma unroll
      for (int t = 0; t < 6; ++t) d[static_cast<int64_t>(t) * Kp] = p[split_part(t, b_side)];
    }
  }
}

// inv[r] = 1 / max(||x_r||, 1e-12)  (F.normalize), one warp per row
__global__ void __launch_bounds__(256) row_inv_norm_kernel(const float* __restrict__ x, int R, int K, float* __restrict__ inv) {
  const int lane = threadIdx.x & 31;
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= R) return;
  float s = 0.f;
  for (int k = lane; k < K; k += 32) {
    const float v = x[static_cast<int64_t>(r) * K + k];
    s = fmaf(v, v, s);
  }
  s = warp_sum_f(s);
  if (lane == 0) inv[r] = 1.0f / fmaxf(sqrtf(s), 1e-12f);
}
// inv[c] = 1 / max(||W[:,c]||, 1e-12), thread per column (coalesced across columns)
__global__ void __launch_bounds__(256) col_inv_norm_kernel(const float* __restrict__ w, int D, int Cn, float* __restrict__ inv) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= Cn) return;
  float s = 0.f;
  for (int d = 0; d < D; ++d) {
    const float v = w[static_cast<int64_t>(d) * Cn + c];
    s = fmaf(v, v, s);
  }
  inv[c] = 1.0f / fmaxf(sqrtf(s), 1e-12f);
}

struct HeadCfg {
  int kind;  // VDK_HEAD_ARCFACE / VDK_HEAD_CIRCLELOSS / VDK_HEAD_MV_SOFTMAX
  float cos_m, sin_m, min_cos, margin_am, scale;  // arcface (cos_m, sin_m, scale also mv-softmax)
  float margin, gamma;                            // circleloss (margin also mv-softmax)
  float mv_weight;                                // mv-softmax
  int is_am;
  float label_smooth;
};

// MV-Softmax (mv_softmax.py:25-44) needs the label column's cosine `gt` of the row for every element: elements scoring
// above the margin-shifted target are "hard" (re-weighted; the comparison carries no gradient).  No clamp on cos there.
struct MvRow {
  float thr;       // hard-example threshold: cos(theta_y + m) (arc) or gt - m (am)
  float final_gt;  // the label column's logit / scale
  float dfinal;    // d final_gt / d gt
};
__device__ __forceinline__ MvRow mv_row(const HeadCfg& h, float gt) {
  MvRow r;
  if (h.is_am) {
    r.thr = gt - h.margin;
    r.final_gt = gt > h.margin ? gt - h.margin : gt;
    r.dfinal = 1.f;
  } else {
    const float s = sqrtf(1.0f - gt * gt);  // NaN for |gt| > 1, exactly like the reference
    const float ctm = gt * h.cos_m - s * h.sin_m;
    r.thr = ctm;
    r.final_gt = gt > 0.f ? ctm : gt;
    r.dfinal = gt > 0.f ? h.cos_m + (gt / s) * h.sin_m : 1.f;
  }
  return r;
}

// logit and d(logit)/d(cos) of one element (the reference's expressions, arcface.py:24-35 / circleloss.py:33-42)
__device__ __forceinline__ void head_logit(const HeadCfg& h, const MvRow& mv, float cos_raw, bool is_label, float& z,
                                           float& dz_dcos) {
  if (h.kind == VDK_HEAD_MV_SOFTMAX) {
    if (is_label) {
      z = mv.final_gt * h.scale;
      dz_dcos = mv.dfinal * h.scale;
    } else if (cos_raw > mv.thr) {
      z = (h.mv_weight * cos_raw + h.mv_weight - 1.0f) * h.scale;
      dz_dcos = h.mv_weight * h.scale;
    } else {
      z = cos_raw * h.scale;
      dz_dcos = h.scale;
    }
    return;
  }
  const float c = fminf(fmaxf(cos_raw, -1.f), 1.f);
  // torch.clamp's backward is a select, not a product: past the clamp the derivative is 0 even where the unclamped
  // expression is not finite (the label's c / s at c = 1, s = 0)
  const bool clamp_pass = cos_raw >= -1.f && cos_raw <= 1.f;
  float d;
  if (h.kind == VDK_HEAD_ARCFACE) {
    if (is_label) {
      if (c > h.min_cos) {
        const float s = sqrtf(1.0f - c * c);
        z = (c * h.cos_m - s * h.sin_m) * h.scale;
        d = (h.cos_m + (c / s) * h.sin_m) * h.scale;
      } else {
        z = (c - h.margin_am) * h.scale;
        d = h.scale;
      }
    } else {
      z = c * h.scale;
      d = h.scale;
    }
  } else {
    if (is_label) {
      const float ap = fmaxf((1.f + h.margin) - c, 0.f);  // detached
      z = ap * (c - (1.f - h.margin)) * h.gamma;
      d = ap * h.gamma;
    } else {
      const float an = fmaxf(c + h.margin, 0.f);  // detached
      z = an * (c - h.margin) * h.gamma;
      d = an * h.gamma;
    }
  }
  dz_dcos = clamp_pass ? d : 0.f;
}

// forward: one CTA per row; online softmax over the classes; optional logits output
__global__ void __launch_bounds__(256)
margin_ce_fwd_kernel(const float* __restrict__ cosm, int ldc, int B, int Cn, const int64_t* __restrict__ labels, HeadCfg h,
                     float* __restrict__ logits /*[B,Cn] or null*/, float* __restrict__ row_lse, float* __restrict__ row_loss) {
  __shared__ float red[3][8];
  const int row = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t y = labels[row];
  MvRow mv{0.f, 0.f, 0.f};
  if (h.kind == VDK_HEAD_MV_SOFTMAX) mv = mv_row(h, cosm[static_cast<int64_t>(row) * ldc + y]);
  float mx = -FLT_MAX, se = 0.f, sz = 0.f, zy = 0.f;
  for (int c = tid; c < Cn; c += 256) {
    float z, dz;
    head_logit(h, mv, cosm[static_cast<int64_t>(row) * ldc + c], c == y, z, dz);
    if (logits) logits[static_cast<int64_t>(row) * Cn + c] = z;
    if (c == y) zy = z;
    sz += z;
    if (z > mx) {
      se = se * __expf(mx - z) + 1.f;
      mx = z;
    } else {
      se += __expf(z - mx);
    }
  }
  // combine (max, sumexp) pairs, sums of z and the label logit across the block
  const float wm = warp_max_f(mx);
  se *= __expf(mx - wm);
  se = warp_sum_f(se);
  sz = warp_sum_f(sz);
  zy = warp_sum_f(zy);
  if (lane == 0) {
    red[0][warp] = wm;
    red[1][warp] = se;
    red[2][warp] = sz;
  }
  __shared__ float s_zy[8];
  if (lane == 0) s_zy[warp] = zy;
  __syncthreads();
  if (tid == 0) {
    float M = -FLT_MAX;
    for (int w = 0; w < 8; ++w) M = fmaxf(M, red[0][w]);
    float S = 0.f, Z = 0.f, ZY = 0.f;
    for (int w = 0; w < 8; ++w) {
      S += red[1][w] * __expf(red[0][w] - M);
      Z += red[2][w];
      ZY += s_zy[w];
    }
    const float lse = M + logf(S);
    row_lse[row] = lse;
    // CE with label smoothing: (1-e) * (lse - z_y) + e * (lse - mean_c z)
    row_loss[row] = (1.f - h.label_smooth) * (lse - ZY) + h.label_smooth * (lse - Z / static_cast<float>(Cn));
  }
}

__global__ void mean_kernel(const float* __restrict__ x, int n, float* out) {
  // single warp, fixed order: deterministic batch mean
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += 32) s += x[i];
  s = warp_sum_f(s);
  if (threadIdx.x == 0) *out = s / static_cast<float>(n);
}

// backward: dcos[b,c] = gout/B * (softmax - target) * dz/dcos * inv_wnorm[c]   (column norm folded in for dF~ = dcos' . W^T)
// and dcos_plain (without the column norm) for dW~ = f~^T . dcos
__global__ void __launch_bounds__(256)
margin_ce_bwd_kernel(const float* __restrict__ cosm, int ldc, int B, int Cn, const int64_t* __restrict__ labels, HeadCfg h,
                     const float* __restrict__ row_lse, const float* __restrict__ grad_out, const float* __restrict__ dlogits,
                     const float* __restrict__ inv_wnorm, float* __restrict__ dcos_plain, float* __restrict__ dcos_scaled,
                     int ldd) {
  const int row = blockIdx.x;
  const int64_t y = labels[row];
  const float g = (grad_out ? *grad_out : 1.f) / static_cast<float>(B);
  const float lse = row_lse ? row_lse[row] : 0.f;
  const float t_off = h.label_smooth / static_cast<float>(Cn);
  MvRow mv{0.f, 0.f, 0.f};
  if (h.kind == VDK_HEAD_MV_SOFTMAX) mv = mv_row(h, cosm[static_cast<int64_t>(row) * ldc + y]);
  for (int c = threadIdx.x; c < ldd; c += 256) {
    float v = 0.f;
    if (c < Cn) {
      float z, dz;
      head_logit(h, mv, cosm[static_cast<int64_t>(row) * ldc + c], c == y, z, dz);
      if (dlogits) {  // un-fused path: the caller's criterion produced d(loss)/d(logits)
        v = dlogits[static_cast<int64_t>(row) * Cn + c] * dz;
      } else {
        const float p = __expf(z - lse);
        const float target = (c == y ? (1.f - h.label_smooth) : 0.f) + t_off;
        v = g * (p - target) * dz;
      }
    }
    dcos_plain[static_cast<int64_t>(row) * ldd + c] = v;
    dcos_scaled[static_cast<int64_t>(row) * ldd + c] = c < Cn ? v * inv_wnorm[c] : 0.f;
  }
}

// df = (dF~ - f~ (f~ . dF~)) * inv_norm   (backward of F.normalize for ||f|| > eps), one warp per row
__global__ void __launch_bounds__(256)
fgrad_finalize_kernel(const float* __restrict__ dfn, const float* __restrict__ fn, const float* __restrict__ inv, int B, int D,
                      float* __restrict__ df) {
  const int lane = threadIdx.x & 31;
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= B) return;
  float dot = 0.f;
  for (int k = lane; k < D; k += 32) dot = fmaf(fn[static_cast<int64_t>(r) * D + k], dfn[static_cast<int64_t>(r) * D + k], dot);
  dot = warp_sum_f(dot);
  for (int k = lane; k < D; k += 32)
    df[static_cast<int64_t>(r) * D + k] = (dfn[static_cast<int64_t>(r) * D + k] - fn[static_cast<int64_t>(r) * D + k] * dot) * inv[r];
}
// dW[:,c] = (dW~[:,c] - W~[:,c] (W~[:,c] . dW~[:,c])) * inv_wnorm[c]; a block owns 32 columns, its 8 warps stride the
// D rows (coalesced 128-byte row segments) and meet in shared memory for the per-column dot product
__global__ void __launch_bounds__(256)
wgrad_finalize_kernel(const float* __restrict__ dwn, int ldw, const float* __restrict__ w, const float* __restrict__ inv, int D,
                      int Cn, float* __restrict__ dw) {
  __shared__ float red[8][32];
  const int lane = threadIdx.x & 31, grp = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  const bool ok = c < Cn;
  const float iv = ok ? inv[c] : 0.f;
  float dot = 0.f;
  if (ok)
    for (int d = grp; d < D; d += 8) dot = fmaf(w[static_cast<int64_t>(d) * Cn + c] * iv, dwn[static_cast<int64_t>(d) * ldw + c], dot);
  red[grp][lane] = dot;
  __syncthreads();
  dot = 0.f;
#pragma unroll
  for (int g = 0; g < 8; ++g) dot += red[g][lane];
  if (ok)
    for (int d = grp; d < D; d += 8)
      dw[static_cast<int64_t>(d) * Cn + c] = (dwn[static_cast<int64_t>(d) * ldw + c] - w[static_cast<int64_t>(d) * Cn + c] * iv * dot) * iv;
}

static size_t a256(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }
static int pad8(int v) { return (v + 7) & ~7; }

static int make_cfg(const vdk_head_desc* d, HeadCfg* h) {
  VDK_REQUIRE(d, "null head descriptor");
  VDK_REQUIRE(d->kind == VDK_HEAD_ARCFACE || d->kind == VDK_HEAD_CIRCLELOSS || d->kind == VDK_HEAD_MV_SOFTMAX,
              "head kind must be arcface, circleloss or mv-softmax");
  VDK_REQUIRE(d->batch > 0 && d->feat_dim > 0 && d->num_class > 1, "bad head shape");
  VDK_REQUIRE(d->label_smooth >= 0.f && d->label_smooth < 1.f, "label_smooth must be in [0,1)");
  h->kind = d->kind;
  h->cos_m = cosf(d->margin_arc);
  h->sin_m = sinf(d->margin_arc);
  h->min_cos = cosf(3.14159265358979323846f - d->margin_arc);
  h->margin_am = d->margin_am;
  h->scale = d->scale;
  h->margin = d->margin;
  h->gamma = d->gamma;
  h->mv_weight = d->mv_weight;
  h->is_am = d->is_am;
  if (d->kind == VDK_HEAD_MV_SOFTMAX) {  // MV_Softmax(is_am, margin, mv_weight, scale): cos/sin of ITS margin
    h->cos_m = cosf(d->margin);
    h->sin_m = sinf(d->margin);
  }
  h->label_smooth = d->label_smooth;
  return VDK_OK;
}

struct HeadWs {
  float *inv_f, *inv_w, *fn, *cosm, *row_loss, *dcos_plain, *dcos_scaled, *dfn, *dwn, *dfn_slabs;
  __nv_bfloat16 *a_split, *b_split;
  int Cp, Bp, Dp, dfn_splits;
};

// dF~ = dcos' . W^T contracts over K = 6 Cp (3.5e5 at C = 58 671).  The wgmma fp32 accumulator does not round to nearest, so
// one chain over K drifts with the number of k16 steps; the contraction is cut into split-K slabs of at most ~16 K-blocks
// (64 k16 steps, at most 256 slabs), each stored to its own fp32 slab and summed in a fixed order (deterministic).
static int dfn_splits(int Cp) {
  const int kbt = (6 * Cp + 63) / 64;
  return vdk_gemm_effective_splits(6 * Cp, std::min(256, (kbt + 15) / 16));
}
static size_t head_ws_layout(const vdk_head_desc* d, void* base, HeadWs* w) {
  const size_t B = d->batch, D = d->feat_dim, Cn = d->num_class;
  const size_t Cp = pad8(d->num_class), Bp = pad8(d->batch), Dp = pad8(d->feat_dim);
  uint8_t* p = reinterpret_cast<uint8_t*>(base);
  size_t off = 0;
  auto take = [&](size_t bytes) { uint8_t* r = p ? p + off : nullptr; off += a256(bytes); return r; };
  float* inv_f = reinterpret_cast<float*>(take(B * 4));
  float* inv_w = reinterpret_cast<float*>(take(Cn * 4));
  float* fn = reinterpret_cast<float*>(take(B * D * 4));
  float* cosm = reinterpret_cast<float*>(take(B * Cp * 4));
  float* row_loss = reinterpret_cast<float*>(take(B * 4));
  float* dcos_plain = reinterpret_cast<float*>(take(B * Cp * 4));
  float* dcos_scaled = reinterpret_cast<float*>(take(B * Cp * 4));
  float* dfn = reinterpret_cast<float*>(take(B * D * 4));
  float* dwn = reinterpret_cast<float*>(take(D * Cp * 4));
  const int splits = dfn_splits(static_cast<int>(Cp));
  float* dfn_slabs = splits > 1 ? reinterpret_cast<float*>(take(static_cast<size_t>(splits) * B * D * 4)) : nullptr;
  // split operands: the largest A side is max(B*6Dp, B*6Cp, D*6Bp), the largest B side max(Cp*6Dp, D*6Cp, Cp*6Bp)
  const size_t a_elems = std::max(std::max(B * 6 * Dp, B * 6 * Cp), D * 6 * Bp);
  const size_t b_elems = std::max(std::max(Cp * 6 * Dp, D * 6 * Cp), Cp * 6 * Bp);
  __nv_bfloat16* a_split = reinterpret_cast<__nv_bfloat16*>(take(a_elems * 2));
  __nv_bfloat16* b_split = reinterpret_cast<__nv_bfloat16*>(take(b_elems * 2));
  if (w) *w = HeadWs{inv_f, inv_w, fn, cosm, row_loss, dcos_plain, dcos_scaled, dfn, dwn, dfn_slabs, a_split, b_split,
                     static_cast<int>(Cp), static_cast<int>(Bp), static_cast<int>(Dp), splits};
  return off + 256;
}

static int split_gemm(const __nv_bfloat16* a, const __nv_bfloat16* b, float* d, int M, int N, int K6, int ldd, cudaStream_t s) {
  vdk_gemm_desc g{};
  g.A = a; g.B = b; g.D = d;
  g.M = M; g.N = N; g.K = K6; g.lda = K6; g.ldb = K6; g.ldd = ldd;
  g.in_dtype = VDK_DTYPE_BF16; g.out_dtype = VDK_DTYPE_FP32; g.epilogue = VDK_EPI_NONE;
  g.split_k = 1;
  return gemm_run(g, s);
}

static int blocks_for(int64_t n, int per_block) { return static_cast<int>(std::min<int64_t>((n + per_block - 1) / per_block, 132 * 32)); }

// cos = normalize(f) . normalize(W, dim 0) into ws.cosm (pitch Cp); also fills inv_f, inv_w, fn
static int head_cos(const vdk_head_desc* d, const float* feats, const float* weight, const HeadWs& w, cudaStream_t s) {
  const int B = d->batch, D = d->feat_dim, Cn = d->num_class;
  row_inv_norm_kernel<<<(B * 32 + 255) / 256, 256, 0, s>>>(feats, B, D, w.inv_f);
  col_inv_norm_kernel<<<(Cn + 255) / 256, 256, 0, s>>>(weight, D, Cn, w.inv_w);
  // A' = split(f * inv_f) [B, 6Dp]; also keeps f~ for the backward
  split3_rows_kernel<<<blocks_for(static_cast<int64_t>(B) * w.Dp, 256), 256, 0, s>>>(feats, B, D, D, w.Dp, w.inv_f, nullptr, 0,
                                                                                    w.a_split, w.fn);
  // B' = split(W^T * inv_w) [Cp, 6Dp]
  dim3 grid((w.Cp + 31) / 32, (w.Dp + 31) / 32);
  split3_cols_kernel<<<grid, 256, 0, s>>>(weight, Cn, D, Cn, w.Cp, w.Dp, w.inv_w, 1, w.b_split);
  VDK_CUDA_OK(cudaGetLastError());
  return split_gemm(w.a_split, w.b_split, w.cosm, B, w.Cp, 6 * w.Dp, w.Cp, s);
}

}  // namespace vdk

using namespace vdk;

extern "C" size_t vdk_head_workspace_bytes(const vdk_head_desc* d) {
  if (!d || d->batch <= 0 || d->feat_dim <= 0 || d->num_class <= 0) return 0;
  return head_ws_layout(d, nullptr, nullptr);
}

extern "C" int vdk_head_forward(const vdk_head_desc* d, const float* feats, const float* weight, const int64_t* labels,
                                float* logits, float* loss, float* row_lse, float* cos_saved, void* workspace,
                                size_t workspace_bytes, void* stream) {
  HeadCfg h;
  int rc = make_cfg(d, &h);
  if (rc != VDK_OK) return rc;
  VDK_REQUIRE(feats && weight && labels && loss && row_lse, "vdk_head_forward: null operand");
  VDK_REQUIRE(workspace && workspace_bytes >= vdk_head_workspace_bytes(d) && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0,
              "vdk_head_forward: workspace too small or misaligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  HeadWs w;
  head_ws_layout(d, workspace, &w);
  rc = head_cos(d, feats, weight, w, s);
  if (rc != VDK_OK) return rc;
  const int B = d->batch, Cn = d->num_class;
  margin_ce_fwd_kernel<<<B, 256, 0, s>>>(w.cosm, w.Cp, B, Cn, labels, h, logits, row_lse, w.row_loss);
  mean_kernel<<<1, 32, 0, s>>>(w.row_loss, B, loss);
  if (cos_saved)
    VDK_CUDA_OK(cudaMemcpy2DAsync(cos_saved, static_cast<size_t>(Cn) * 4, w.cosm, static_cast<size_t>(w.Cp) * 4,
                                  static_cast<size_t>(Cn) * 4, B, cudaMemcpyDeviceToDevice, s));
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_head_backward(const vdk_head_desc* d, const float* feats, const float* weight, const int64_t* labels,
                                 const float* row_lse, const float* grad_loss, const float* dlogits, float* dfeats,
                                 float* dweight,
                                 void* workspace, size_t workspace_bytes, void* stream) {
  HeadCfg h;
  int rc = make_cfg(d, &h);
  if (rc != VDK_OK) return rc;
  VDK_REQUIRE(feats && weight && labels && (row_lse || dlogits) && dfeats && dweight, "vdk_head_backward: null operand");
  VDK_REQUIRE(workspace && workspace_bytes >= vdk_head_workspace_bytes(d) && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0,
              "vdk_head_backward: workspace too small or misaligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  HeadWs w;
  head_ws_layout(d, workspace, &w);
  const int B = d->batch, D = d->feat_dim, Cn = d->num_class;
  VDK_REQUIRE(D % 8 == 0, "vdk_head_backward: feat_dim must be a multiple of 8 (it is the N of the dF~ GEMM)");
  // recompute cos (cheaper than keeping [B,C] alive between forward and backward at face-scale C)
  rc = head_cos(d, feats, weight, w, s);
  if (rc != VDK_OK) return rc;
  margin_ce_bwd_kernel<<<B, 256, 0, s>>>(w.cosm, w.Cp, B, Cn, labels, h, row_lse, grad_loss, dlogits, w.inv_w, w.dcos_plain,
                                         w.dcos_scaled, w.Cp);
  VDK_CUDA_OK(cudaGetLastError());
  // dF~ [B,D] = dcos' [B,C] . W^T   (A = dcos' rows over K=C, B = W rows [D, C])
  split3_rows_kernel<<<blocks_for(static_cast<int64_t>(B) * w.Cp, 256), 256, 0, s>>>(w.dcos_scaled, B, w.Cp, w.Cp, w.Cp, nullptr,
                                                                                    nullptr, 0, w.a_split, nullptr);
  split3_rows_kernel<<<blocks_for(static_cast<int64_t>(D) * w.Cp, 256), 256, 0, s>>>(weight, D, Cn, Cn, w.Cp, nullptr, nullptr, 1,
                                                                                    w.b_split, nullptr);
  VDK_CUDA_OK(cudaGetLastError());
  if (w.dfn_splits > 1) {
    vdk_gemm_desc g{};
    g.A = w.a_split; g.B = w.b_split; g.D = w.dfn_slabs;
    g.M = B; g.N = D; g.K = 6 * w.Cp; g.lda = 6 * w.Cp; g.ldb = 6 * w.Cp; g.ldd = D;
    g.in_dtype = VDK_DTYPE_BF16; g.out_dtype = VDK_DTYPE_FP32; g.epilogue = VDK_EPI_NONE;
    g.split_k = w.dfn_splits; g.split_stride = static_cast<long long>(B) * D;
    rc = gemm_run(g, s);
    if (rc != VDK_OK) return rc;
    rc = launch_slab_reduce(w.dfn_slabs, w.dfn_splits, static_cast<size_t>(B) * D, static_cast<int64_t>(B) * D / 4, w.dfn, 0, s);
  } else {
    rc = split_gemm(w.a_split, w.b_split, w.dfn, B, D, 6 * w.Cp, D, s);
  }
  if (rc != VDK_OK) return rc;
  fgrad_finalize_kernel<<<(B * 32 + 255) / 256, 256, 0, s>>>(w.dfn, w.fn, w.inv_f, B, D, dfeats);
  // dW~ [D,C] = f~^T [D,B] . dcos [B,C]   (A = f~^T over K=B, B = dcos^T [C, B])
  {
    dim3 ga((D + 31) / 32, (w.Bp + 31) / 32);
    split3_cols_kernel<<<ga, 256, 0, s>>>(w.fn, D, B, D, D, w.Bp, nullptr, 0, w.a_split);
    dim3 gb((w.Cp + 31) / 32, (w.Bp + 31) / 32);
    split3_cols_kernel<<<gb, 256, 0, s>>>(w.dcos_plain, w.Cp, B, w.Cp, w.Cp, w.Bp, nullptr, 1, w.b_split);
    VDK_CUDA_OK(cudaGetLastError());
  }
  rc = split_gemm(w.a_split, w.b_split, w.dwn, D, w.Cp, 6 * w.Bp, w.Cp, s);
  if (rc != VDK_OK) return rc;
  wgrad_finalize_kernel<<<(Cn + 31) / 32, 256, 0, s>>>(w.dwn, w.Cp, weight, w.inv_w, D, Cn, dweight);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}
