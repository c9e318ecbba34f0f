// attention_tc.cu — softmax(Q K^T / sqrt(d)) V on the sm_90a warpgroup tensor cores (wgmma), head_dim 64, 72 or 80, bf16.
//
// Replaces timm's Attention.forward inside every ViT block of the reference's backbone
// (models/faceX/backbone/timm_wrapper.py:52 -> timm VisionTransformer blocks; SURVEY.md §2.4 K4): scores are never
// written to memory.  Input is the qkv Linear's output as stored, bf16 [B, N, 3, H, D]; output bf16 [B, N, H*D]
// (+ optionally the log2-domain log-sum-exp per row, which the training backward consumes).
//
// Head dims above 64 (SigLIP So400m: 72, CLIP ViT-H: 80): TMA sees qkv as the 4-D tensor (D, 3H, N, B), whose row pitch D*2
// bytes (144, 160) is a multiple of 16.  Every head's rows arrive as two boxes: columns 0-63 with 128-byte swizzle (the D = 64
// layout) and a 16-column remainder at column 64 with 32-byte swizzle.  At D = 72 columns 72-79 of the remainder lie outside
// dimension 0, so TMA zero-fills them: the padded k-step of S adds nothing and the next head's data is never read.
//   S = Q K^T   four k16 steps on the swizzle-128 region + one on the swizzle-32 region
//   O += P V    m64n64k16 over columns 0-63 + m64n16k16 over the remainder; only the D valid columns are stored
//
// CTAs are PERSISTENT (one per SM); an item = one (image, head) x TWO 128-query tiles (ViT-B/16's 197 tokens are exactly two),
// items strided over the grid.  288 threads:
//   warpgroup 0 (warps 0-3)   query tile 0: S = Q K^T (two wgmma m64 x 64 x 64, Q and K K-major) into registers, the
//                             softmax on the accumulator fragments (a row lives in one quad of threads), then
//                             O += P V with P taken straight from registers (bf16) and V as stored (MN-major operand)
//   warpgroup 1 (warps 4-7)   query tile 1
//   warp 8                    TMA producer: Q tile pair once per item (double-buffered: the next item's Q lands during this
//                             item), K/V tiles (64 keys) through a four-deep mbarrier ring shared by both warpgroups
// Softmax is the online recurrence in the log2 domain with a LAZY rescale: the running reference maximum only moves (and
// O / l are only rescaled) when a row's maximum grows by more than 2^8; P = exp2(s - m_ref) then stays below 256, exact in
// bf16's range, and the final O / l cancels the stale reference.
#include "vdk_host.h"
#include "vdk_ptx.cuh"

#include <algorithm>
#include <cmath>

namespace vdk {

constexpr int kAtQM = 128;        // query rows per tile (two m64 halves)
constexpr int kAtKV = 64;         // keys per tile
constexpr int kAtStages = 4;      // K/V ring
constexpr int kAtThreads = 288;

// Shared-memory layout of one head dim.  A tile is its swizzle-128 region (columns 0-63, 128-byte rows) followed, for D > 64,
// by its swizzle-32 region (columns 64-79, 32-byte rows); both stay 1024-byte aligned.
template <int D>
struct AttShape {
  static_assert(D == 64 || D == 72 || D == 80, "attention head dim");
  static constexpr bool kRem = D > 64;                      // a 16-column remainder
  static constexpr int kQMain = kAtQM * 64 * 2;             // 16 KB
  static constexpr int kQTile = kQMain + (kRem ? kAtQM * 16 * 2 : 0);   // + 4 KB
  static constexpr int kKMain = kAtKV * 64 * 2;             // 8 KB
  static constexpr int kKTile = kKMain + (kRem ? kAtKV * 16 * 2 : 0);   // + 2 KB (K or V)
  static constexpr int kSmem = 2 * 2 * kQTile + kAtStages * 2 * kKTile + 16 * 8 + 1024;  // Q double-buffered
  static_assert(kSmem <= 227 * 1024, "attention shared memory budget");
  static_assert(kQTile % 1024 == 0 && kKTile % 1024 == 0, "swizzle atoms need 1024-byte aligned tiles");
};

struct AttParams {
  int B, N, H;
  float scale_log2e;
  __nv_bfloat16* out;
  float* lse2;
  int n_qtiles, n_kvtiles;
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// maps: q / kv = columns 0-63 (128-byte swizzle, 128- / 64-row boxes); q_rem / kv_rem = columns 64-79 (32-byte swizzle), used
// only when D > 64
template <int D>
__global__ void __launch_bounds__(kAtThreads, 1)
attention_fwd_tc_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_kv,
                        const __grid_constant__ CUtensorMap map_q_rem, const __grid_constant__ CUtensorMap map_kv_rem, const AttParams p) {
  using S = AttShape<D>;
  constexpr int kAtQTile = S::kQTile, kAtKTile = S::kKTile;
  extern __shared__ uint8_t att_smem_raw[];
  uint8_t* smem = att_smem_raw + ((1024u - (smem_u32(att_smem_raw) & 1023u)) & 1023u);
  uint8_t* smem_q = smem;                                     // [2 items in flight][2 tiles][Q tile]
  uint8_t* smem_kv = smem + 2 * 2 * kAtQTile;                 // [stages][K tile | V tile]
  uint64_t* q_full = reinterpret_cast<uint64_t*>(smem_kv + kAtStages * 2 * kAtKTile);  // [2]
  uint64_t* q_empty = q_full + 2;            // [2]
  uint64_t* kv_full = q_empty + 2;           // [stages]
  uint64_t* kv_empty = kv_full + kAtStages;  // [stages]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int J = p.n_kvtiles, N = p.N;
  const int n_pairs = (p.n_qtiles + 1) / 2;
  const int n_items = n_pairs * p.H * p.B;  // persistent: this CTA takes items blockIdx.x, + gridDim.x, ...

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_q);
    prefetch_tensormap(&map_kv);
    if constexpr (S::kRem) {
      prefetch_tensormap(&map_q_rem);
      prefetch_tensormap(&map_kv_rem);
    }
    for (int i = 0; i < 2; ++i) {
      mbar_init(&q_full[i], 1);
      mbar_init(&q_empty[i], 8);  // one arrival per warp of both warpgroups
    }
    for (int i = 0; i < kAtStages; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  auto decode = [&](int item, int& pair, int& h, int& b) {
    pair = item % n_pairs;
    const int r = item / n_pairs;
    h = r % p.H;
    b = r / p.H;
  };

  if (warp == 8) {
    // ===================== TMA producer: Q of the next item and its K/V tiles run ahead of the tensor core =====================
    if (lane == 0) {
      int qc = 0, kvc = 0;  // items / K-V tiles loaded so far (barrier phases run across items)
      for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++qc) {
        int pair, h, b;
        decode(item, pair, h, b);
        const int qt0 = pair * 2, n_t = min(2, p.n_qtiles - qt0);
        const int qb = qc & 1;  // Q is double-buffered: the next item's tiles land while this item is still in its softmax
        if (qc >= 2) mbar_wait_relaxed<true>(&q_empty[qb], ((qc >> 1) - 1) & 1);  // every S = Q K^T of the item two back has retired
        mbar_arrive_expect_tx(&q_full[qb], n_t * kAtQTile);
        for (int t = 0; t < n_t; ++t) {
          uint8_t* dst = smem_q + (qb * 2 + t) * kAtQTile;
          tma_load_4d(dst, &map_q, &q_full[qb], 0, h, (qt0 + t) * kAtQM, b);
          if constexpr (S::kRem) tma_load_4d(dst + S::kQMain, &map_q_rem, &q_full[qb], 64, h, (qt0 + t) * kAtQM, b);
        }
        for (int j = 0; j < J; ++j, ++kvc) {
          const int st = kvc % kAtStages;
          if (kvc >= kAtStages) mbar_wait_relaxed<true>(&kv_empty[st], ((kvc / kAtStages) - 1) & 1);
          mbar_arrive_expect_tx(&kv_full[st], 2 * kAtKTile);  // zero-filled columns (D = 72) count as transferred bytes
          uint8_t* dst = smem_kv + st * 2 * kAtKTile;
          tma_load_4d(dst, &map_kv, &kv_full[st], 0, p.H + h, j * kAtKV, b);
          tma_load_4d(dst + kAtKTile, &map_kv, &kv_full[st], 0, 2 * p.H + h, j * kAtKV, b);
          if constexpr (S::kRem) {
            tma_load_4d(dst + S::kKMain, &map_kv_rem, &kv_full[st], 64, p.H + h, j * kAtKV, b);
            tma_load_4d(dst + kAtKTile + S::kKMain, &map_kv_rem, &kv_full[st], 64, 2 * p.H + h, j * kAtKV, b);
          }
        }
      }
    }
  } else {
    // ===================== warpgroup t: query tile t of the item =====================
    const int t = warp >> 2;
    const int wl = warp & 3;
    const int fcol = (lane & 3) * 2;  // first of this thread's two columns in every 8-column block
    int qc = 0, kvc = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++qc) {
      int pair, h, b;
      decode(item, pair, h, b);
      const int qt0 = pair * 2;
      const int qb = qc & 1;
      if (t >= min(2, p.n_qtiles - qt0)) {
        // odd tile count: this warpgroup idles for the item but still releases what the producer counts on.  Waiting for
        // each fill first keeps its arrivals in the phase they belong to.
        mbar_wait<true>(&q_full[qb], (qc >> 1) & 1);
        if (lane == 0) mbar_arrive(&q_empty[qb]);
        for (int j = 0; j < J; ++j, ++kvc) {
          const int st = kvc % kAtStages;
          mbar_wait<true>(&kv_full[st], (kvc / kAtStages) & 1);
          if (lane == 0) mbar_arrive(&kv_empty[st]);
        }
        continue;
      }
      mbar_wait<true>(&q_full[qb], (qc >> 1) & 1);
      // rows of this thread: (hm, i) -> tile row hm * 64 + wl * 16 + lane / 4 + 8 i
      float o[2][32];
      float o_rem[2][8];  // columns 64-79 (D > 64 only)
#pragma unroll
      for (int hm = 0; hm < 2; ++hm) {
#pragma unroll
        for (int i = 0; i < 32; ++i) o[hm][i] = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) o_rem[hm][i] = 0.f;
      }
      float m_ref[2][2], l[2][2];
#pragma unroll
      for (int hm = 0; hm < 2; ++hm)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          m_ref[hm][i] = -INFINITY;
          l[hm][i] = 0.f;
        }
      for (int j = 0; j < J; ++j, ++kvc) {
        const int st = kvc % kAtStages;
        mbar_wait<true>(&kv_full[st], (kvc / kAtStages) & 1);
        // ---- S = Q K^T ----
        float s[2][32];
        wgmma_fence();
#pragma unroll
        for (int hm = 0; hm < 2; ++hm) {
          const uint64_t da = wgmma_desc_k_sw128(smem_u32(smem_q + (qb * 2 + t) * kAtQTile + hm * 8192));
          const uint64_t db = wgmma_desc_k_sw128(smem_u32(smem_kv + st * 2 * kAtKTile));
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_m64n64k16_ss<true, 0, 0>(s[hm], da + 2 * k, db + 2 * k, k > 0 ? 1u : 0u);
          if constexpr (S::kRem)
            wgmma_m64n64k16_ss<true, 0, 0>(s[hm], wgmma_desc_k_sw32(smem_u32(smem_q + (qb * 2 + t) * kAtQTile + S::kQMain + hm * 2048)),
                                           wgmma_desc_k_sw32(smem_u32(smem_kv + st * 2 * kAtKTile + S::kKMain)), 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(s[0]);
        wgmma_fence_regs(s[1]);
        if (j + 1 == J && lane == 0) mbar_arrive(&q_empty[qb]);  // the item's last S MMAs have retired: its Q buffer is free
        const int valid = min(kAtKV, N - j * kAtKV);  // keys of this tile that exist
        // ---- row maxima (a row's 64 scores are spread over the 4 threads of a quad) ----
        float mx[2][2];
        bool grow = false;
#pragma unroll
        for (int hm = 0; hm < 2; ++hm)
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            float m = -INFINITY;
#pragma unroll
            for (int jb = 0; jb < 8; ++jb)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                if (valid == kAtKV || jb * 8 + fcol + e < valid) m = fmaxf(m, s[hm][4 * jb + 2 * i + e]);
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
            mx[hm][i] = m * p.scale_log2e;
            if (j > 0 && fmaxf(m_ref[hm][i], mx[hm][i]) - m_ref[hm][i] > 8.0f) grow = true;
          }
        if (j == 0) {
#pragma unroll
          for (int hm = 0; hm < 2; ++hm)
#pragma unroll
            for (int i = 0; i < 2; ++i) m_ref[hm][i] = mx[hm][i];
        } else if (__any_sync(0xffffffffu, grow)) {
          // rescale O and l of the rows of this warp (alpha = 1 for rows whose maximum did not move)
#pragma unroll
          for (int hm = 0; hm < 2; ++hm)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const float m_new = fmaxf(m_ref[hm][i], mx[hm][i]);
              const float alpha = ex2_approx(m_ref[hm][i] - m_new);
              m_ref[hm][i] = m_new;
              l[hm][i] *= alpha;
#pragma unroll
              for (int jb = 0; jb < 8; ++jb) {
                o[hm][4 * jb + 2 * i] *= alpha;
                o[hm][4 * jb + 2 * i + 1] *= alpha;
              }
              if constexpr (S::kRem) {
#pragma unroll
                for (int jb = 0; jb < 2; ++jb) {
                  o_rem[hm][4 * jb + 2 * i] *= alpha;
                  o_rem[hm][4 * jb + 2 * i + 1] *= alpha;
                }
              }
            }
        }
        // ---- P = exp2(s * c - m_ref) -> bf16 A fragments (the accumulator layout of a 64 x 16 block), row sums in fp32 ----
        uint32_t pa[2][4][4];
#pragma unroll
        for (int hm = 0; hm < 2; ++hm) {
#pragma unroll
          for (int jb = 0; jb < 8; ++jb)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              float e2[2];
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const float x = fmaf(s[hm][4 * jb + 2 * i + e], p.scale_log2e, -m_ref[hm][i]);
                // the sequence's ragged last tile: keys beyond N get P = 0 exactly (never NaN garbage)
                e2[e] = (valid == kAtKV || jb * 8 + fcol + e < valid) ? ex2_approx(x) : 0.f;
                l[hm][i] += e2[e];
              }
              pa[hm][jb >> 1][(jb & 1) * 2 + i] = pack_bf16x2(e2[0], e2[1]);
            }
        }
        // ---- O += P V ----
        wgmma_fence();
#pragma unroll
        for (int hm = 0; hm < 2; ++hm) {
          const uint64_t db = wgmma_desc_mn_sw128(smem_u32(smem_kv + st * 2 * kAtKTile + kAtKTile), 8192);
#pragma unroll
          for (int kk = 0; kk < kAtKV / 16; ++kk) wgmma_m64n64k16_rs_bf16<1>(o[hm], pa[hm][kk], db + 128u * kk, 1u);
          if constexpr (S::kRem) {
            const uint64_t dr = wgmma_desc_mn_sw32(smem_u32(smem_kv + st * 2 * kAtKTile + kAtKTile + S::kKMain));
#pragma unroll
            for (int kk = 0; kk < kAtKV / 16; ++kk) wgmma_m64n16k16_rs_bf16<1>(o_rem[hm], pa[hm][kk], dr + 32u * kk, 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(o[0]);
        wgmma_fence_regs(o[1]);
        if constexpr (S::kRem) {
          wgmma_fence_regs(o_rem[0]);
          wgmma_fence_regs(o_rem[1]);
        }
        if (lane == 0) mbar_arrive(&kv_empty[st]);  // K_j / V_j free
      }
      // ---- epilogue: O / l -> bf16 rows ----
#pragma unroll
      for (int hm = 0; hm < 2; ++hm)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float lt = l[hm][i];
          lt += __shfl_xor_sync(0xffffffffu, lt, 1);
          lt += __shfl_xor_sync(0xffffffffu, lt, 2);
          const float inv = 1.0f / lt;
          const int row = (qt0 + t) * kAtQM + hm * 64 + wl * 16 + (lane >> 2) + 8 * i;  // token index of this query
          if (row < N) {
            __nv_bfloat16* dst = p.out + (static_cast<size_t>(b) * N + row) * (static_cast<size_t>(p.H) * D) + h * D;
#pragma unroll
            for (int jb = 0; jb < 8; ++jb)
              *reinterpret_cast<uint32_t*>(dst + jb * 8 + fcol) =
                  pack_bf16x2(o[hm][4 * jb + 2 * i] * inv, o[hm][4 * jb + 2 * i + 1] * inv);
#pragma unroll
            for (int jb = 0; jb < (D - 64) / 8; ++jb)  // the remainder's valid 8-column blocks
              *reinterpret_cast<uint32_t*>(dst + 64 + jb * 8 + fcol) =
                  pack_bf16x2(o_rem[hm][4 * jb + 2 * i] * inv, o_rem[hm][4 * jb + 2 * i + 1] * inv);
            if (p.lse2 && (lane & 3) == 0) p.lse2[(static_cast<size_t>(b) * p.H + h) * N + row] = m_ref[hm][i] + log2f(lt);
          }
        }
    }
  }
}

// qkv bf16 [B, N, 3, H, D] -> out bf16 [B, N, H*D]; lse2 (optional) fp32 [B, H, N] in the log2 domain
template <int D>
static int launch_attention_tc_d(const __nv_bfloat16* qkv, int B, int N, int H, __nv_bfloat16* out, float* lse2, cudaStream_t s) {
  using S = AttShape<D>;
  static bool attr = false;
  if (!attr) {
    VDK_CUDA_OK(cudaFuncSetAttribute(attention_fwd_tc_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kSmem));
    attr = true;
  }
  // the same (D, 3H, N, B) view with 128-row (Q) and 64-row (K, V) boxes, 64 columns (128-byte swizzle) and 16 (32-byte)
  CUtensorMap map_q, map_kv, map_q_rem, map_kv_rem;
  int rc = make_tma_qkv_16bit(&map_q, qkv, D, H, N, B, 64, kAtQM);
  if (rc != VDK_OK) return rc;
  rc = make_tma_qkv_16bit(&map_kv, qkv, D, H, N, B, 64, kAtKV);
  if (rc != VDK_OK) return rc;
  if (S::kRem) {
    rc = make_tma_qkv_16bit(&map_q_rem, qkv, D, H, N, B, 16, kAtQM);
    if (rc != VDK_OK) return rc;
    rc = make_tma_qkv_16bit(&map_kv_rem, qkv, D, H, N, B, 16, kAtKV);
    if (rc != VDK_OK) return rc;
  } else {
    map_q_rem = map_q;  // unused
    map_kv_rem = map_kv;
  }
  AttParams p{};
  p.B = B; p.N = N; p.H = H;
  p.scale_log2e = 1.4426950408889634f / sqrtf(static_cast<float>(D));
  p.out = out;
  p.lse2 = lse2;
  p.n_qtiles = (N + kAtQM - 1) / kAtQM;
  p.n_kvtiles = (N + kAtKV - 1) / kAtKV;
  const long long n_items = static_cast<long long>((p.n_qtiles + 1) / 2) * H * B;
  VDK_REQUIRE(n_items < (1ll << 31), "attention: too many (image, head, tile pair) items");
  const int grid = static_cast<int>(std::min<long long>(n_items, sm_count()));  // persistent: one CTA per SM
  attention_fwd_tc_kernel<D><<<grid, kAtThreads, S::kSmem, s>>>(map_q, map_kv, map_q_rem, map_kv_rem, p);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

int launch_attention_tc(const __nv_bfloat16* qkv, int B, int N, int H, int head_dim, __nv_bfloat16* out, float* lse2, cudaStream_t s) {
  VDK_REQUIRE(B > 0 && N > 0 && H > 0 && H <= 65535 && B <= 65535, "attention: bad shape");
  switch (head_dim) {
    case 64: return launch_attention_tc_d<64>(qkv, B, N, H, out, lse2, s);
    case 72: return launch_attention_tc_d<72>(qkv, B, N, H, out, lse2, s);
    case 80: return launch_attention_tc_d<80>(qkv, B, N, H, out, lse2, s);
    default: return fail(VDK_ERR_INVALID, "attention: head_dim must be 64, 72 or 80 (got %d)", head_dim);
  }
}

}  // namespace vdk
