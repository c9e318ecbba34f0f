// convnext_train.cu — ConvNeXt + neck training forward (activations saved) and backward, orchestrated in C++ over the
// wgmma GEMM (gemm.cu: K-major and MN-major operands, so dgrad / wgrad need no transposed copies) and the HBM-bound
// kernels of convnext.cu / train_ops.cu.
//
// Replaces, for the faceX train step (engine/procedure/train.py:196,206): the forward of TimmWrapper in train mode
// (models/faceX/backbone/timm_wrapper.py:51-54; BatchNorm with batch statistics in the neck, :34,37) and the autograd
// backward of the whole backbone.  Gradients are ACCUMULATED (+=) into fp32 buffers in timm's parameter layouts.
#include "vdk_host.h"
#include "vdk_ptx.cuh"
#include "convnext_internal.h"
#include "train_gemm.h"

#include <vector>

namespace vdk {

static size_t al(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }

struct StageDims {
  int H, W, C;
  size_t M;
};

// Offsets (bytes) of everything the forward saves for the backward, plus scratch, inside the caller's workspace.
struct TrainLayout {
  StageDims st[4];
  int depth[4];
  int n_blocks;
  size_t p0, z0, rstd0;                                        // stem: patch rows [M0,48], pre-LN output, 1/sigma
  size_t xs[4][VDK_CONVNEXT_MAX_BLOCKS + 1];                   // residual stream at every node of a stage
  size_t y[VDK_CONVNEXT_MAX_BLOCKS], rstd[VDK_CONVNEXT_MAX_BLOCKS];
  size_t hpre[VDK_CONVNEXT_MAX_BLOCKS], hpost[VDK_CONVNEXT_MAX_BLOCKS];
  size_t patch[4], prstd[4];                                   // downsample: LayerNorm'ed 2x2 patch rows, 1/sigma
  size_t f, frstd, fn, bn2_mean, bn2_rstd, z, zslab, bn1_mean, bn1_rstd;
  size_t dxa, dxb, dy, dconv, G, sdo, dw49, gwc, gwneck, dz, dzb, dfn, wslab;
  size_t total;
};

static void make_layout(const vdk_convnext_net* net, int batch, TrainLayout* L) {
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += al(bytes); return o; };
  int H = net->image_size / 4, W = H;
  L->n_blocks = 0;
  for (int s = 0; s < 4; ++s) {
    if (s > 0) { H /= 2; W /= 2; }
    L->st[s] = {H, W, net->dims[s], static_cast<size_t>(batch) * H * W};
    L->depth[s] = net->depths[s];
    L->n_blocks += net->depths[s];
  }
  const size_t M0 = L->st[0].M;
  L->p0 = take(M0 * 48 * 2);
  L->z0 = take(M0 * net->dims[0] * 2);
  L->rstd0 = take(M0 * 4);
  int k = 0;
  size_t max_mc = 0, max_cc4 = 0;
  for (int s = 0; s < 4; ++s) {
    const size_t M = L->st[s].M, C = L->st[s].C;
    max_mc = std::max(max_mc, M * C);
    max_cc4 = std::max(max_cc4, C * 4 * C);
    if (s > 0) {
      L->patch[s] = take(M * 4 * L->st[s - 1].C * 2);
      L->prstd[s] = take(L->st[s - 1].M * 4);
      max_cc4 = std::max(max_cc4, C * 4 * static_cast<size_t>(L->st[s - 1].C));
    }
    for (int j = 0; j <= L->depth[s]; ++j) L->xs[s][j] = take(M * C * 2);
    for (int j = 0; j < L->depth[s]; ++j, ++k) {
      L->y[k] = take(M * C * 2);
      L->rstd[k] = take(M * 4);
      L->hpre[k] = take(M * 4 * C * 2);
      L->hpost[k] = take(M * 4 * C * 2);
    }
  }
  const size_t M3 = L->st[3].M, C3 = L->st[3].C, F = net->feat_dim, Kn = (M3 / batch) * C3;
  L->f = take(M3 * C3 * 2);
  L->frstd = take(M3 * 4);
  L->fn = take(M3 * C3 * 2);
  L->bn2_mean = take(C3 * 4);
  L->bn2_rstd = take(C3 * 4);
  L->z = take(static_cast<size_t>(batch) * F * 4);
  L->zslab = take(static_cast<size_t>(batch) * F * 4 * 160);
  L->bn1_mean = take(F * 4);
  L->bn1_rstd = take(F * 4);
  // backward scratch
  L->dxa = take(max_mc * 2);
  L->dxb = take(max_mc * 2);
  L->dy = take(max_mc * 2);
  L->dconv = take(max_mc * 2);
  L->G = take(max_cc4 * 4);
  // per-block scratch (zeroed once per backward): column sums of dOut, tap gradients in [49][C] layout
  L->sdo = take(static_cast<size_t>(L->n_blocks) * 2048 * 4);
  L->dw49 = take(static_cast<size_t>(L->n_blocks) * 49 * 2048 * 4);
  L->gwc = take(max_cc4 * 4);
  L->gwneck = take(F * Kn * 4);
  L->dz = take(static_cast<size_t>(batch) * F * 4);
  L->dzb = take(static_cast<size_t>(batch) * F * 2);
  L->dfn = take(M3 * C3 * 2);
  size_t slab = wgrad_slab_bytes(net->dims[0], 48, M0);
  for (int s = 0; s < 4; ++s) {
    const int C = L->st[s].C;
    slab = std::max(slab, wgrad_slab_bytes(C, 4 * C, L->st[s].M));
    slab = std::max(slab, wgrad_slab_bytes(4 * C, C, L->st[s].M));
    if (s > 0) slab = std::max(slab, wgrad_slab_bytes(C, 4 * L->st[s - 1].C, L->st[s].M));
  }
  L->wslab = take(slab);
  L->total = off + 256;
}

__global__ void slab_reduce_bias_kernel(const float* __restrict__ slabs, int n_slabs, size_t stride, const float* __restrict__ bias,
                                        int rows, int cols, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  float v = bias ? bias[i % cols] : 0.f;
  for (int s = 0; s < n_slabs; ++s) v += slabs[s * stride + i];
  out[i] = v;
}
// dst[i] (+)= sum_s slabs[s * stride + i]: 32 float4 columns x 8 slab groups per block; the groups meet in shared
// memory and are added in a fixed order
__global__ void __launch_bounds__(256)
slab_reduce_kernel(const float* __restrict__ slabs, int n_slabs, size_t stride, int64_t n4, float* __restrict__ dst,
                   int accumulate) {
  __shared__ float4 part[8][32];
  const int col = threadIdx.x & 31, grp = threadIdx.x >> 5;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * 32 + col;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (i < n4) {
#pragma unroll 4
    for (int s = grp; s < n_slabs; s += 8) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(slabs + static_cast<size_t>(s) * stride) + i);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  }
  part[grp][col] = acc;
  __syncthreads();
  if (grp == 0 && i < n4) {
    float4 t = part[0][col];
#pragma unroll
    for (int g = 1; g < 8; ++g) {
      const float4 v = part[g][col];
      t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
    }
    float4* o = reinterpret_cast<float4*>(dst) + i;
    if (accumulate) {
      const float4 d = *o;
      t.x += d.x; t.y += d.y; t.z += d.z; t.w += d.w;
    }
    *o = t;
  }
}
int launch_slab_reduce(const float* slabs, int n_slabs, size_t stride, int64_t n4, float* dst, int accumulate, cudaStream_t s) {
  slab_reduce_kernel<<<static_cast<unsigned>((n4 + 31) / 32), 256, 0, s>>>(slabs, n_slabs, stride, n4, dst, accumulate);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}
__global__ void col_sum_f32_small_kernel(const float* __restrict__ x, int rows, int cols, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  float s = 0.f;
  for (int r = 0; r < rows; ++r) s += x[static_cast<size_t>(r) * cols + c];
  out[c] += s;
}
__global__ void stem_patchify_train_kernel(const float* __restrict__ x, int B, int H, int W, __nv_bfloat16* __restrict__ out) {
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

}  // namespace vdk

using namespace vdk;

extern "C" size_t vdk_convnext_train_workspace_bytes(const vdk_convnext_net* net, int batch) {
  if (!net || batch <= 0) return 0;
  TrainLayout L;
  make_layout(net, batch, &L);
  return L.total;
}

// ---- weight packing, batched: the blocks of a stage have identical shapes, so ONE launch per (stage, kind) walks a table
// of per-block pointers passed by value (instead of ~190 small per-tensor launches per step) ----
constexpr int kPackTab = 32;
struct PackTab {
  const float* src[kPackTab];
  void* dst[kPackTab];
  void* dst2[kPackTab];
  const float* scale[kPackTab];
};

// dst[i] = bf16(src[i] * (scale ? scale[i / cols] : 1)) for tensor blockIdx.y;  dst2 (optional): the same without the scale
__global__ void __launch_bounds__(256)
pack_cast_kernel(PackTab t, int64_t n, int cols) {
  const float* __restrict__ src = t.src[blockIdx.y];
  __nv_bfloat16* __restrict__ dst = reinterpret_cast<__nv_bfloat16*>(t.dst[blockIdx.y]);
  __nv_bfloat16* __restrict__ dst2 = reinterpret_cast<__nv_bfloat16*>(t.dst2[blockIdx.y]);
  const float* __restrict__ sc = t.scale[blockIdx.y];
  for (int64_t i = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 4; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x * 4) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(src + i));  // n and cols are multiples of 4
    if (dst2 != nullptr) {
      __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
      uint2 o;
      o.x = *reinterpret_cast<uint32_t*>(&lo);
      o.y = *reinterpret_cast<uint32_t*>(&hi);
      *reinterpret_cast<uint2*>(dst2 + i) = o;
    }
    const float m = sc ? sc[i / cols] : 1.f;
    __nv_bfloat162 lo = __floats2bfloat162_rn(v.x * m, v.y * m), hi = __floats2bfloat162_rn(v.z * m, v.w * m);
    uint2 o;
    o.x = *reinterpret_cast<uint32_t*>(&lo);
    o.y = *reinterpret_cast<uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(dst + i) = o;
  }
}
// conv_dw.weight [C][49] -> taps [49][C] (dst) and the reversed taps [48 - t][C] for the backward-data pass (dst2, optional)
__global__ void __launch_bounds__(256)
pack_taps_kernel(PackTab t, int C) {
  const float* __restrict__ src = t.src[blockIdx.y];
  float* __restrict__ dst = reinterpret_cast<float*>(t.dst[blockIdx.y]);
  float* __restrict__ dst2 = reinterpret_cast<float*>(t.dst2[blockIdx.y]);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // output index [tap][c]
  if (i >= 49 * C) return;
  const int tap = i / C, c = i - tap * C;
  const float v = src[c * 49 + tap];
  if (dst != nullptr) dst[i] = v;
  if (dst2 != nullptr) dst2[(48 - tap) * C + c] = v;
}

// gradient of the taps back to timm's layout: dst[c][t] += src[t][c] for tensor blockIdx.y
__global__ void __launch_bounds__(256)
unpack_taps_grad_kernel(PackTab t, int C) {
  const float* __restrict__ src = t.src[blockIdx.y];
  float* __restrict__ dst = reinterpret_cast<float*>(t.dst[blockIdx.y]);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // input index [tap][c]
  if (i >= 49 * C) return;
  const int tap = i / C, c = i - tap * C;
  dst[c * 49 + tap] += src[i];
}

static int pack_impl(const vdk_convnext_tensors* p, const vdk_convnext_net* net, bool taps_and_weights, bool flip, cudaStream_t s) {
  auto bf = [](const void* q) { return const_cast<void*>(q); };
  int k0 = 0;
  for (int st = 0; st < 4; ++st) {
    const int C = net->dims[st], depth = net->depths[st];
    for (int j0 = 0; j0 < depth; j0 += kPackTab) {
      const int nb = std::min(kPackTab, depth - j0);
      PackTab fc1{}, fc2{}, taps{};
      bool any_flip = false;
      for (int j = 0; j < nb; ++j) {
        const vdk_convnext_block_tensors* b = &p->blocks[k0 + j0 + j];
        const vdk_convnext_block* o = &net->blocks[k0 + j0 + j];
        fc1.src[j] = b->fc1_w; fc1.dst[j] = bf(o->fc1_w);
        // fc2: plain cast (dst2) + gamma[c] * W2[c,:] (dst) in one pass when the layer-scaled copy is wanted
        fc2.src[j] = b->fc2_w;
        if (o->fc2_wg) { fc2.dst[j] = bf(o->fc2_wg); fc2.dst2[j] = bf(o->fc2_w); fc2.scale[j] = b->gamma; }
        else { fc2.dst[j] = bf(o->fc2_w); }
        taps.src[j] = b->dw_w;
        taps.dst[j] = taps_and_weights ? bf(o->dw_w) : nullptr;
        taps.dst2[j] = (flip && o->dw_w_flip) ? bf(o->dw_w_flip) : nullptr;
        any_flip = any_flip || taps.dst2[j] != nullptr;
      }
      const int64_t n = static_cast<int64_t>(4) * C * C;
      const unsigned gx = static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>((n / 4 + 255) / 256, 256)));
      if (taps_and_weights) {
        pack_cast_kernel<<<dim3(gx, nb), 256, 0, s>>>(fc1, n, 4 * C);  // no scale
        pack_cast_kernel<<<dim3(gx, nb), 256, 0, s>>>(fc2, n, 4 * C);
      }
      if (taps_and_weights || any_flip) pack_taps_kernel<<<dim3((49 * C + 255) / 256, nb), 256, 0, s>>>(taps, C);
    }
    k0 += depth;
  }
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_convnext_pack(const vdk_convnext_tensors* p, vdk_convnext_net* net, void* stream) {
  VDK_REQUIRE(p && net, "vdk_convnext_pack: null argument");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int C0 = net->dims[0];
  auto bf = [](const void* q) { return reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(q)); };
  for (int st = 0; st < 4; ++st)
    VDK_REQUIRE(net->dims[st] % 4 == 0, "vdk_convnext_pack: channel counts must be multiples of 4");
  RC(launch_cast_bf16(p->stem_w, static_cast<int64_t>(C0) * 48, bf(net->stem_w), s));
  for (int st = 1; st < 4; ++st) {
    // Conv2d(Cin,C,2,2).weight [C][Cin][4] -> [C][4][Cin]
    RC(launch_permute021(p->down[st].conv_w, net->dims[st], net->dims[st - 1], 4, nullptr, bf(net->down[st].conv_w), nullptr, 0, s));
  }
  // per block: conv_dw.weight [C][49] -> taps [49][C] (fp32, + the reversed taps when the net carries them), fc1 / fc2
  // casts, gamma[c] * W2[c,:]
  RC(pack_impl(p, net, true, true, s));
  const int C3 = net->dims[3], hw = (net->image_size / 32) * (net->image_size / 32);
  // Linear weight [F][C3][hw] -> [F][hw][C3]
  RC(launch_permute021(p->lin_w, net->feat_dim, C3, hw, nullptr, bf(net->neck_w), nullptr, 0, s));
  return VDK_OK;
}

__global__ void flip_taps_kernel(const float* __restrict__ w49, int C, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 49 * C) return;
  const int t = i / C, c = i - t * C;
  out[(48 - t) * C + c] = w49[i];
}

// Reversed taps from the PACKED taps of `net` (kept for callers that pack by other means; vdk_convnext_pack already
// writes them when the net carries dw_w_flip buffers).
extern "C" int vdk_convnext_pack_flip(const vdk_convnext_net* net, void* stream) {
  VDK_REQUIRE(net, "vdk_convnext_pack_flip: null net");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  int k = 0;
  for (int st = 0; st < 4; ++st)
    for (int j = 0; j < net->depths[st]; ++j, ++k) {
      const vdk_convnext_block* o = &net->blocks[k];
      if (!o->dw_w_flip) continue;
      flip_taps_kernel<<<(49 * net->dims[st] + 255) / 256, 256, 0, s>>>(o->dw_w, net->dims[st], const_cast<float*>(o->dw_w_flip));
    }
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_convnext_train_forward(const vdk_convnext_net* net, const vdk_convnext_tensors* p, const float* images,
                                          int batch, float bn_momentum, float* out_feats, void* workspace,
                                          size_t workspace_bytes, void* stream) {
  VDK_REQUIRE(net && p && images && out_feats && batch > 1, "vdk_convnext_train_forward: bad arguments (batch must be > 1)");
  TrainLayout L;
  make_layout(net, batch, &L);
  VDK_REQUIRE(workspace && workspace_bytes >= L.total && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0,
              "vdk_convnext_train_forward: workspace too small or misaligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  auto B16 = [&](size_t off) { return reinterpret_cast<__nv_bfloat16*>(ws + off); };
  auto F32 = [&](size_t off) { return reinterpret_cast<float*>(ws + off); };
  const Gemm G{s};
  const int S = net->image_size;

  // ---- stem: patch rows (saved) -> GEMM + bias -> LayerNorm2d (1/sigma saved) ----
  {
    const int M0 = static_cast<int>(L.st[0].M), C0 = L.st[0].C;
    const int64_t total = static_cast<int64_t>(M0) * 12;
    stem_patchify_train_kernel<<<static_cast<int>(std::min<int64_t>((total + 255) / 256, 132 * 16)), 256, 0, s>>>(images, batch, S, S,
                                                                                                             B16(L.p0));
    VDK_CUDA_OK(cudaGetLastError());
    RC(G.run(B16(L.p0), net->stem_w, B16(L.z0), M0, C0, 48, 48, 48, C0, VDK_EPI_NONE, net->stem_b, nullptr, nullptr, 0,
             VDK_DTYPE_BF16, 1, 0, 0, 0));
    RC(launch_ln_patchify(B16(L.z0), batch, L.st[0].H, L.st[0].W, C0, net->stem_ln_w, net->stem_ln_b, 1e-6f, 1, B16(L.xs[0][0]),
                          F32(L.rstd0), s));
  }
  int k = 0;
  for (int st = 0; st < 4; ++st) {
    const int H = L.st[st].H, W = L.st[st].W, C = L.st[st].C, M = static_cast<int>(L.st[st].M);
    if (st > 0) {
      const vdk_convnext_down* d = &net->down[st];
      const int Cin = L.st[st - 1].C;
      RC(launch_ln_patchify(B16(L.xs[st - 1][L.depth[st - 1]]), batch, L.st[st - 1].H, L.st[st - 1].W, Cin, d->ln_w, d->ln_b, 1e-6f,
                            2, B16(L.patch[st]), F32(L.prstd[st]), s));
      RC(G.run(B16(L.patch[st]), d->conv_w, B16(L.xs[st][0]), M, C, 4 * Cin, 4 * Cin, 4 * Cin, C, VDK_EPI_NONE, d->conv_b, nullptr,
               nullptr, 0, VDK_DTYPE_BF16, 1, 0, 0, 0));
    }
    for (int j = 0; j < L.depth[st]; ++j, ++k) {
      const vdk_convnext_block* b = &net->blocks[k];
      RC(launch_dwconv7(0, B16(L.xs[st][j]), batch, H, W, C, b->dw_w, b->dw_b, b->ln_w, b->ln_b, 1e-6f, B16(L.y[k]), F32(L.rstd[k]),
                        nullptr, s));
      RC(G.run(B16(L.y[k]), b->fc1_w, B16(L.hpost[k]), M, 4 * C, C, C, C, 4 * C, VDK_EPI_GELU, b->fc1_b, nullptr, nullptr, 0,
               VDK_DTYPE_BF16, 1, 0, 0, 0, B16(L.hpre[k])));
      RC(G.run(B16(L.hpost[k]), b->fc2_w, B16(L.xs[st][j + 1]), M, C, 4 * C, 4 * C, 4 * C, C, VDK_EPI_SCALE_RESIDUAL, b->fc2_b,
               b->gamma, B16(L.xs[st][j]), C, VDK_DTYPE_BF16, 1, 0, 0, 0));
    }
  }
  // ---- head LayerNorm2d -> neck: BatchNorm2d (batch stats) -> Flatten -> Linear -> BatchNorm1d (batch stats) ----
  {
    const int H = L.st[3].H, W = L.st[3].W, C3 = L.st[3].C, M3 = static_cast<int>(L.st[3].M), F = net->feat_dim;
    const int Kn = H * W * C3;
    RC(launch_ln_patchify(B16(L.xs[3][L.depth[3]]), batch, H, W, C3, net->head_ln_w, net->head_ln_b, 1e-6f, 1, B16(L.f),
                          F32(L.frstd), s));
    RC(launch_bn_fwd_bf16(B16(L.f), M3, C3, p->bn2_w, p->bn2_b, 1e-5f, bn_momentum, B16(L.fn), F32(L.bn2_mean), F32(L.bn2_rstd),
                          p->bn2_running_mean, p->bn2_running_var, s));
    const int tiles = ((batch + 127) / 128) * ((F + 255) / 256);
    int split = std::max(1, std::min(160, (2 * sm_count()) / std::max(1, tiles)));
    split = vdk_gemm_effective_splits(Kn, split);
    const size_t slab = static_cast<size_t>(batch) * F;
    RC(G.run(B16(L.fn), net->neck_w, F32(L.zslab), batch, F, Kn, Kn, Kn, F, VDK_EPI_NONE, nullptr, nullptr, nullptr, 0,
             VDK_DTYPE_FP32, split, split > 1 ? static_cast<long long>(slab) : 0, 0, 0));
    slab_reduce_bias_kernel<<<(batch * F + 255) / 256, 256, 0, s>>>(F32(L.zslab), split, slab, p->lin_b, batch, F, F32(L.z));
    VDK_CUDA_OK(cudaGetLastError());
    RC(launch_bn_fwd_f32(F32(L.z), batch, F, p->bn1_w, p->bn1_b, 1e-5f, bn_momentum, out_feats, F32(L.bn1_mean), F32(L.bn1_rstd),
                         p->bn1_running_mean, p->bn1_running_var, s));
  }
  return VDK_OK;
}

// The backward as a sequence of UNITS in execution order: unit 0 = neck + head LayerNorm; then per stage 3..0 one unit per
// block (last block first) followed by one unit for the stage's downsample layer (the stem for stage 0).  A caller that
// overlaps the gradient all-reduce with the backward runs [0, U) in a few consecutive ranges and reduces the gradients a
// range completed while the next one computes.
extern "C" int vdk_convnext_train_backward_units(const vdk_convnext_net* net) {
  if (!net) return 0;
  int n = 1 + 4;
  for (int st = 0; st < 4; ++st) n += net->depths[st];
  return n;
}

// A second stream for the bias-gradient column sums of dH ([tokens, 4C]: one full HBM pass over a tensor the next two GEMMs read
// anyway).  The persistent GEMM CTAs leave ~11 k registers and no shared memory per SM — enough for one 256-thread block of the
// (shared-memory-free) column-sum kernel — so the sum runs UNDER the weight- and data-gradient GEMMs of fc1 instead of in
// front of them.  Fork: the side stream waits for the event recorded after the GEMM that produced dH; join: the caller's stream
// waits for the side stream's last event before the call returns (the gradients it wrote are then ordered before anything the
// caller enqueues next: the optimizer, an all-reduce, the next forward that overwrites dH).  It is OFF unless
// VDK_TRAIN_SIDE_STREAM=1.
struct SideStream {
  cudaStream_t stream = nullptr;
  cudaEvent_t fork = nullptr, join = nullptr;
  bool ok = false, used = false;
};
static SideStream& side_stream() {
  static thread_local SideStream ss;
  static const bool enabled = [] {
    const char* e = getenv("VDK_TRAIN_SIDE_STREAM");
    return e ? atoi(e) != 0 : false;
  }();
  if (enabled && !ss.ok && ss.stream == nullptr) {
    if (cudaStreamCreateWithFlags(&ss.stream, cudaStreamNonBlocking) == cudaSuccess &&
        cudaEventCreateWithFlags(&ss.fork, cudaEventDisableTiming) == cudaSuccess &&
        cudaEventCreateWithFlags(&ss.join, cudaEventDisableTiming) == cudaSuccess)
      ss.ok = true;
    else
      cudaGetLastError();
  }
  return ss;
}

static int backward_range(const vdk_convnext_net* net, const vdk_convnext_tensors* p, const vdk_convnext_tensors* g,
                          const float* d_feats, int batch, void* workspace, size_t workspace_bytes, void* stream, int u_begin,
                          int u_end) {
  VDK_REQUIRE(net && p && g && d_feats && batch > 1, "vdk_convnext_train_backward: bad arguments");
  VDK_REQUIRE(u_begin >= 0 && u_begin < u_end && u_end <= vdk_convnext_train_backward_units(net),
              "vdk_convnext_train_backward: bad unit range [%d, %d)", u_begin, u_end);
  int u = 0;  // running unit index
  auto active = [&](int unit) { return unit >= u_begin && unit < u_end; };
  TrainLayout L;
  make_layout(net, batch, &L);
  VDK_REQUIRE(workspace && workspace_bytes >= L.total, "vdk_convnext_train_backward: workspace too small");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  auto B16 = [&](size_t off) { return reinterpret_cast<__nv_bfloat16*>(ws + off); };
  auto F32 = [&](size_t off) { return reinterpret_cast<float*>(ws + off); };
  const Gemm G{s};
  const int F = net->feat_dim;
  SideStream& side = side_stream();
  side.used = false;

  // ---- neck ----
  const int H3 = L.st[3].H, W3 = L.st[3].W, C3 = L.st[3].C, M3 = static_cast<int>(L.st[3].M), Kn = H3 * W3 * C3;
  if (active(u++)) {
    VDK_CUDA_OK(cudaMemsetAsync(F32(L.sdo), 0, static_cast<size_t>(L.n_blocks) * 2048 * 4, s));
    VDK_CUDA_OK(cudaMemsetAsync(F32(L.dw49), 0, static_cast<size_t>(L.n_blocks) * 49 * 2048 * 4, s));
    RC(launch_bn_bwd_f32(d_feats, F32(L.z), batch, F, p->bn1_w, F32(L.bn1_mean), F32(L.bn1_rstd), F32(L.dz), g->bn1_w, g->bn1_b, s));
    col_sum_f32_small_kernel<<<(F + 255) / 256, 256, 0, s>>>(F32(L.dz), batch, F, g->lin_b);
    RC(launch_cast_bf16(F32(L.dz), static_cast<int64_t>(batch) * F, B16(L.dzb), s));
    // dW[F, (h,w,c)] = dZ^T . FN  (both stored with the batch index slow), then un-permute into timm's (c, h, w) order
    RC(G.run(B16(L.dzb), B16(L.fn), F32(L.gwneck), F, Kn, batch, F, Kn, Kn, VDK_EPI_NONE, nullptr, nullptr, nullptr, 0,
             VDK_DTYPE_FP32, 1, 0, 1, 1));
    RC(launch_permute021(F32(L.gwneck), F, H3 * W3, C3, nullptr, nullptr, g->lin_w, 1, s));
    // dFN[B, Kn] = dZ . W   (W stored [F, Kn]: the contraction index F is its slow dimension)
    RC(G.run(B16(L.dzb), net->neck_w, B16(L.dfn), batch, Kn, F, F, Kn, Kn, VDK_EPI_NONE, nullptr, nullptr, nullptr, 0,
             VDK_DTYPE_BF16, 1, 0, 0, 1));
    RC(launch_bn_bwd_bf16(B16(L.dfn), B16(L.f), M3, C3, p->bn2_w, F32(L.bn2_mean), F32(L.bn2_rstd), B16(L.dy), g->bn2_w, g->bn2_b, s));
    RC(launch_ln_bwd(B16(L.dy), B16(L.f), F32(L.frstd), batch, H3, W3, C3, net->head_ln_w, net->head_ln_b, 1, B16(L.dxa), nullptr,
                     g->head_ln_w, g->head_ln_b, s));
  }
  // the gradient wrt the residual stream ping-pongs between two buffers: every block / downsample unit swaps them once
  size_t dx = L.dxa, dx_other = L.dxb;
  int k = L.n_blocks;
  for (int st = 3; st >= 0; --st) {
    const int H = L.st[st].H, W = L.st[st].W, C = L.st[st].C, M = static_cast<int>(L.st[st].M);
    int k_done_lo = -1, k_done_hi = -1;  // blocks of this stage executed by this call: [k_done_lo, k_done_hi]
    for (int j = L.depth[st] - 1; j >= 0; --j) {
      --k;
      if (!active(u++)) {
        std::swap(dx, dx_other);
        continue;
      }
      if (k_done_hi < 0) k_done_hi = k;
      k_done_lo = k;
      const vdk_convnext_block* b = &net->blocks[k];
      const vdk_convnext_block_tensors* pb = &p->blocks[k];
      const vdk_convnext_block_tensors* gb = &g->blocks[k];
      // fc2 + layer scale: G = dOut^T . h_post;  dW2 = diag(gamma) G;  dgamma, db2 from G, W2, colsum(dOut)
      float* sdo = F32(L.sdo) + static_cast<size_t>(k) * 2048;
      RC(launch_col_sum(B16(dx), M, C, C, sdo, s));
      RC(G.wgrad(B16(dx), B16(L.hpost[k]), F32(L.G), C, 4 * C, M, C, 4 * C, F32(L.wslab), false));
      RC(launch_layerscale_finalize(F32(L.G), pb->fc2_w, pb->fc2_b, pb->gamma, sdo, C, 4 * C, gb->fc2_w, gb->gamma, gb->fc2_b, s));
      // dH_pre = (dOut . diag(gamma) W2) * gelu'(h_pre)   -> overwrites the h_post buffer
      RC(G.run(B16(dx), b->fc2_wg, B16(L.hpost[k]), M, 4 * C, C, C, 4 * C, 4 * C, VDK_EPI_MUL_GELU_GRAD, nullptr, nullptr,
               B16(L.hpre[k]), 4 * C, VDK_DTYPE_BF16, 1, 0, 0, 1));
      __nv_bfloat16* dh = B16(L.hpost[k]);
      if (side.ok) {  // bias gradient of fc1 on the side stream, under the two GEMMs below
        VDK_CUDA_OK(cudaEventRecord(side.fork, s));
        VDK_CUDA_OK(cudaStreamWaitEvent(side.stream, side.fork, 0));
        RC(launch_col_sum(dh, M, 4 * C, 4 * C, gb->fc1_b, side.stream));
        side.used = true;
      } else {
        RC(launch_col_sum(dh, M, 4 * C, 4 * C, gb->fc1_b, s));
      }
      RC(G.wgrad(dh, B16(L.y[k]), gb->fc1_w, 4 * C, C, M, 4 * C, C, F32(L.wslab), true));
      RC(G.run(dh, b->fc1_w, B16(L.dy), M, C, 4 * C, 4 * C, C, C, VDK_EPI_NONE, nullptr, nullptr, nullptr, 0, VDK_DTYPE_BF16, 1, 0, 0, 1));
      // LayerNorm backward, depthwise weight gradient, depthwise data gradient (+ the residual branch)
      RC(launch_ln_bwd(B16(L.dy), B16(L.y[k]), F32(L.rstd[k]), batch, H, W, C, b->ln_w, b->ln_b, 1, B16(L.dconv), nullptr, gb->ln_w,
                       gb->ln_b, s));
      // tap gradients stay in the kernel's [49][C] layout in this block's scratch; un-permuted per stage below
      RC(launch_dwconv7_wgrad(B16(L.xs[st][j]), B16(L.dconv), batch, H, W, C, F32(L.dw49) + static_cast<size_t>(k) * 49 * 2048, gb->dw_b, s));
      RC(launch_dwconv7(1, B16(L.dconv), batch, H, W, C, b->dw_w_flip, nullptr, nullptr, nullptr, 0.f, B16(dx_other), nullptr,
                        B16(dx), s));
      std::swap(dx, dx_other);
    }
    // tap gradients of the blocks this call executed: [49][C] scratch -> += timm's [C][1][7][7], one launch per <= 32 blocks
    for (int k0 = k_done_lo; k_done_lo >= 0 && k0 <= k_done_hi; k0 += kPackTab) {
      const int nb = std::min(kPackTab, k_done_hi - k0 + 1);
      PackTab tab{};
      for (int j = 0; j < nb; ++j) {
        tab.src[j] = F32(L.dw49) + static_cast<size_t>(k0 + j) * 49 * 2048;
        tab.dst[j] = g->blocks[k0 + j].dw_w;
      }
      unpack_taps_grad_kernel<<<dim3((49 * C + 255) / 256, nb), 256, 0, s>>>(tab, C);
    }
    VDK_CUDA_OK(cudaGetLastError());
    if (st > 0 && !active(u++)) {
      std::swap(dx, dx_other);
    } else if (st > 0) {
      const vdk_convnext_down* d = &net->down[st];
      const vdk_convnext_down_tensors* gd = &g->down[st];
      const int Cin = L.st[st - 1].C;
      RC(launch_col_sum(B16(dx), M, C, C, gd->conv_b, s));
      RC(G.wgrad(B16(dx), B16(L.patch[st]), F32(L.gwc), C, 4 * Cin, M, C, 4 * Cin, F32(L.wslab), false));
      RC(launch_permute021(F32(L.gwc), C, 4, Cin, nullptr, nullptr, gd->conv_w, 1, s));  // [C][4][Cin] -> += [C][Cin][4]
      RC(G.run(B16(dx), d->conv_w, B16(L.dy), M, 4 * Cin, C, C, 4 * Cin, 4 * Cin, VDK_EPI_NONE, nullptr, nullptr, nullptr, 0,
               VDK_DTYPE_BF16, 1, 0, 0, 1));
      RC(launch_ln_bwd(B16(L.dy), B16(L.patch[st]), F32(L.prstd[st]), batch, L.st[st - 1].H, L.st[st - 1].W, Cin, d->ln_w, d->ln_b, 2,
                       B16(dx_other), nullptr, gd->ln_w, gd->ln_b, s));
      std::swap(dx, dx_other);
    }
  }
  // ---- stem ----
  if (active(u++)) {
    const int M0 = static_cast<int>(L.st[0].M), C0 = L.st[0].C;
    RC(launch_ln_bwd(B16(dx), B16(L.xs[0][0]), F32(L.rstd0), batch, L.st[0].H, L.st[0].W, C0, net->stem_ln_w, net->stem_ln_b, 1,
                     B16(L.dy), nullptr, g->stem_ln_w, g->stem_ln_b, s));
    RC(launch_col_sum(B16(L.dy), M0, C0, C0, g->stem_b, s));
    RC(G.wgrad(B16(L.dy), B16(L.p0), g->stem_w, C0, 48, M0, C0, 48, F32(L.wslab), true));
  }
  if (side.used) {  // join: everything the side stream wrote is ordered before whatever the caller enqueues next
    VDK_CUDA_OK(cudaEventRecord(side.join, side.stream));
    VDK_CUDA_OK(cudaStreamWaitEvent(s, side.join, 0));
  }
  return VDK_OK;
}

extern "C" int vdk_convnext_train_backward(const vdk_convnext_net* net, const vdk_convnext_tensors* p,
                                           const vdk_convnext_tensors* g, const float* d_feats, int batch, void* workspace,
                                           size_t workspace_bytes, void* stream) {
  VDK_REQUIRE(net, "vdk_convnext_train_backward: null net");
  return backward_range(net, p, g, d_feats, batch, workspace, workspace_bytes, stream, 0, vdk_convnext_train_backward_units(net));
}

extern "C" int vdk_convnext_train_backward_range(const vdk_convnext_net* net, const vdk_convnext_tensors* p,
                                                 const vdk_convnext_tensors* g, const float* d_feats, int batch, void* workspace,
                                                 size_t workspace_bytes, void* stream, int unit_begin, int unit_end) {
  VDK_REQUIRE(net, "vdk_convnext_train_backward_range: null net");
  return backward_range(net, p, g, d_feats, batch, workspace, workspace_bytes, stream, unit_begin, unit_end);
}
