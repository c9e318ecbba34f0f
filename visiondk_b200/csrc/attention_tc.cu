// attention_tc.cu — softmax(Q K^T / sqrt(d)) V on the sm_90a warpgroup tensor cores (wgmma), head_dim 64, bf16.
//
// Replaces timm's Attention.forward inside every ViT block of the reference's backbone
// (models/faceX/backbone/timm_wrapper.py:52 -> timm VisionTransformer blocks; SURVEY.md §2.4 K4): scores are never
// written to memory.  Input is the qkv Linear's output as stored, bf16 [B, N, 3, H, 64]; output bf16 [B, N, H*64]
// (+ optionally the log2-domain log-sum-exp per row, which the training backward consumes).
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

constexpr int kAtD = 64;          // head dim
constexpr int kAtQM = 128;        // query rows per tile (two m64 halves)
constexpr int kAtKV = 64;         // keys per tile
constexpr int kAtStages = 4;      // K/V ring (16 KB per stage)
constexpr int kAtThreads = 288;
constexpr int kAtQTile = kAtQM * kAtD * 2;   // 16 KB: a 128 x 64 bf16 Q tile
constexpr int kAtKTile = kAtKV * kAtD * 2;   // 8 KB: a 64 x 64 bf16 tile (K, V)
constexpr int kAtSmem = 2 * 2 * kAtQTile + kAtStages * 2 * kAtKTile + 16 * 8 + 1024;  // Q double-buffered
static_assert(kAtSmem <= 227 * 1024, "attention shared memory budget");

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

__global__ void __launch_bounds__(kAtThreads, 1)
attention_fwd_tc_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_kv, const AttParams p) {
  extern __shared__ uint8_t att_smem_raw[];
  uint8_t* smem = att_smem_raw + ((1024u - (smem_u32(att_smem_raw) & 1023u)) & 1023u);
  uint8_t* smem_q = smem;                                     // [2 items in flight][2 tiles][16 KB]
  uint8_t* smem_kv = smem + 2 * 2 * kAtQTile;                 // [stages][K 8 KB | V 8 KB]
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
        for (int t = 0; t < n_t; ++t)
          tma_load_3d(smem_q + (qb * 2 + t) * kAtQTile, &map_q, &q_full[qb], h * kAtD, (qt0 + t) * kAtQM, b);
        for (int j = 0; j < J; ++j, ++kvc) {
          const int st = kvc % kAtStages;
          if (kvc >= kAtStages) mbar_wait_relaxed<true>(&kv_empty[st], ((kvc / kAtStages) - 1) & 1);
          mbar_arrive_expect_tx(&kv_full[st], 2 * kAtKTile);
          tma_load_3d(smem_kv + st * 2 * kAtKTile, &map_kv, &kv_full[st], (p.H + h) * kAtD, j * kAtKV, b);
          tma_load_3d(smem_kv + st * 2 * kAtKTile + kAtKTile, &map_kv, &kv_full[st], (2 * p.H + h) * kAtD, j * kAtKV, b);
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
#pragma unroll
      for (int hm = 0; hm < 2; ++hm)
#pragma unroll
        for (int i = 0; i < 32; ++i) o[hm][i] = 0.f;
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
          for (int k = 0; k < kAtD / 16; ++k) wgmma_m64n64k16_ss<true, 0, 0>(s[hm], da + 2 * k, db + 2 * k, k > 0 ? 1u : 0u);
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
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(o[0]);
        wgmma_fence_regs(o[1]);
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
            __nv_bfloat16* dst = p.out + (static_cast<size_t>(b) * N + row) * (static_cast<size_t>(p.H) * kAtD) + h * kAtD;
#pragma unroll
            for (int jb = 0; jb < 8; ++jb)
              *reinterpret_cast<uint32_t*>(dst + jb * 8 + fcol) =
                  pack_bf16x2(o[hm][4 * jb + 2 * i] * inv, o[hm][4 * jb + 2 * i + 1] * inv);
            if (p.lse2 && (lane & 3) == 0) p.lse2[(static_cast<size_t>(b) * p.H + h) * N + row] = m_ref[hm][i] + log2f(lt);
          }
        }
    }
  }
}

// qkv bf16 [B, N, 3, H, 64] -> out bf16 [B, N, H*64]; lse2 (optional) fp32 [B, H, N] in the log2 domain
int launch_attention_tc(const __nv_bfloat16* qkv, int B, int N, int H, __nv_bfloat16* out, float* lse2, cudaStream_t s) {
  VDK_REQUIRE(B > 0 && N > 0 && H > 0 && H <= 65535 && B <= 65535, "attention: bad shape");
  static bool attr = false;
  if (!attr) {
    VDK_CUDA_OK(cudaFuncSetAttribute(attention_fwd_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kAtSmem));
    attr = true;
  }
  CUtensorMap map_q, map_kv;  // the same [B][N][3*H*64] view with 128-row (Q) and 64-row (K, V) boxes
  const uint64_t pitch = 3ull * H * kAtD;
  int rc = make_tma_3d_16bit(&map_q, qkv, pitch, static_cast<uint64_t>(N), static_cast<uint64_t>(B), pitch, pitch * N, kAtQM);
  if (rc != VDK_OK) return rc;
  rc = make_tma_3d_16bit(&map_kv, qkv, pitch, static_cast<uint64_t>(N), static_cast<uint64_t>(B), pitch, pitch * N, kAtKV);
  if (rc != VDK_OK) return rc;
  AttParams p{};
  p.B = B; p.N = N; p.H = H;
  p.scale_log2e = 1.4426950408889634f / sqrtf(static_cast<float>(kAtD));
  p.out = out;
  p.lse2 = lse2;
  p.n_qtiles = (N + kAtQM - 1) / kAtQM;
  p.n_kvtiles = (N + kAtKV - 1) / kAtKV;
  const long long n_items = static_cast<long long>((p.n_qtiles + 1) / 2) * H * B;
  VDK_REQUIRE(n_items < (1ll << 31), "attention: too many (image, head, tile pair) items");
  const int grid = static_cast<int>(std::min<long long>(n_items, sm_count()));  // persistent: one CTA per SM
  attention_fwd_tc_kernel<<<grid, kAtThreads, kAtSmem, s>>>(map_q, map_kv, p);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

}  // namespace vdk
