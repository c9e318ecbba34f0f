// retrieval.cu — exact inner-product top-k for the CBIR path: L2-normalise -> score -> select -> re-rank.
//
// Replaces F.normalize (models/faceX/face_model.py:139), faiss GpuIndexFlat add/search
// (engine/cbir/evaluation.py:155-168,190-195; cbir_eval.py:82-95,113-118).
//
// Pipeline (all on device, nothing leaves HBM):
//   rows_prepare   fp32 rows -> canonical unit rows (fp32) + fp16 copy + per-row rounding-error norm
//   score_filter   fp16 wgmma GEMM of a 128-query tile (resident in smem) against streamed gallery tiles;
//                  the epilogue never writes the score matrix: each thread owns one query row of a staged chunk and
//                  appends only scores >= tau[row] to a segment of that row's candidate list that this CTA
//                  owns exclusively (plain stores, a register counter — no atomics on the scan path)
//   select         per query: k-th largest approximate score A_k (radix select), keep a >= A_k - 2*eps
//                  (eps bounds |approx - canonical|, so the true top-k survive) as the row's carry list and
//                  tighten tau for the next gallery range
//   rerank         after the last range: canonical re-score of the carry list (fp64, fixed order), sort by
//                  (score desc, id asc), emit k
// The gallery is scanned in geometrically growing ranges so that tau is tight when most of it streams by.
#include "vdk_host.h"
#include "vdk_ptx.cuh"
#include "score_tile.cuh"
#include "topk_keys.cuh"  // canonical arithmetic (restated in oracle/retrieval.py; the two must agree bit for bit)

#include <cfloat>
#include <cmath>

namespace vdk {

// ------------------------------------------------------------------------------------------------
// rows_prepare: one warp per row
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rows_prepare_kernel(const float* __restrict__ x, int64_t n, int dim,
                                                           int normalize, float* __restrict__ xn,
                                                           __half* __restrict__ xh, float* __restrict__ row_norm,
                                                           float* __restrict__ row_err) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (row >= n) return;
  const float* xr = x + row * dim;
  float denom = 1.0f;
  if (normalize) {
    double ss = 0.0;
    for (int i = lane; i < dim; i += 32) {
      const double v = static_cast<double>(xr[i]);
      ss = fma(v, v, ss);
    }
    ss = warp_sum_f64(ss);
    const float nrm = static_cast<float>(sqrt(ss));
    denom = fmaxf(nrm, 1e-12f);  // F.normalize eps
  }
  double s2 = 0.0, e2 = 0.0;
  for (int i = lane; i < dim; i += 32) {
    const float v = normalize ? __fdiv_rn(xr[i], denom) : xr[i];
    const __half h = __float2half_rn(v);
    const float d = v - __half2float(h);
    s2 = fma(static_cast<double>(v), static_cast<double>(v), s2);
    e2 = fma(static_cast<double>(d), static_cast<double>(d), e2);
    if (xn) xn[row * dim + i] = v;
    xh[row * dim + i] = h;
  }
  s2 = warp_sum_f64(s2);
  e2 = warp_sum_f64(e2);
  if (lane == 0) {
    // round the bounds up: they are used as upper bounds on ||xn|| and ||xn - xh||
    if (row_norm) row_norm[row] = __double2float_ru(sqrt(s2)) * 1.000001f;
    row_err[row] = __double2float_ru(sqrt(e2)) * 1.000001f + 1e-30f;
  }
}

__global__ void reduce_max_kernel(const float* __restrict__ x, int64_t n, float* out) {
  float m = -FLT_MAX;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    m = fmaxf(m, x[i]);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  // values are non-negative norms: the int ordering of their bit patterns equals the float ordering
  if ((threadIdx.x & 31) == 0 && m >= 0.f) atomicMax(reinterpret_cast<int*>(out), __float_as_int(m));
}

// ------------------------------------------------------------------------------------------------
// score_filter: fp16 wgmma GEMM with a threshold-filter epilogue
// ------------------------------------------------------------------------------------------------
constexpr int kQM = 128;          // queries per tile (two consumer warpgroups of 64 rows)
constexpr int kGN = 256;          // gallery rows per tile (wgmma N)
constexpr int kSBK = 64;          // K per smem block (128-byte swizzle row of fp16)
constexpr int kQBlockBytes = kQM * kSBK * 2;   // 16 KB
constexpr int kGStageBytes = kGN * kSBK * 2;   // 32 KB
constexpr int kGStages = 2;       // with a resident 512-dim query tile (128 KB) two gallery stages fit beside the staging buffer
constexpr int kScoreThreads = 384;  // producer warpgroup, two consumer warpgroups
constexpr int kStageLd = 64 + 1;  // fp32 pitch of the staged 128 x 64 score chunk (odd: conflict-free row reads)
constexpr int kMaxKB = 8;         // dim <= 512
constexpr int kMaxSeg = 32;       // candidate segments per query = 2 x gallery splits per range (two epilogue threads per row)
static_assert(kQM == kTileM && kGN == kTileN && kSBK == kTileKB && kQBlockBytes == kTileABlockBytes &&
                  kGStageBytes == kTileBStageBytes && kGStages == kTileStages && kStageLd == kTileStageLd,
              "score_filter_kernel runs the mainloop of score_tile.cuh");

struct ScoreParams {
  int n_query;
  int num_kb;  // dim / 64
  int64_t g_lo, g_hi;
  int n_qtiles, n_splits, tiles_per_split, n_tiles;
  const float* tau;   // per-query admission threshold (sparse mode)
  uint2* seg;         // [n_query][seg_stride] {score bits, gallery row}; writer (split s, half h) owns segment 2s+h
  int seg_stride;     // entries per query
  int seg_cap;        // entries per (query, split)
  unsigned* seg_cnt;  // [n_query][kMaxSeg] admitted count per (query, split) — may exceed seg_cap (overflow)
};

static int score_smem_bytes(int num_kb) {
  return num_kb * kQBlockBytes + kGStages * kGStageBytes + kQM * kStageLd * 4 + (2 * kGStages + 2) * 8 + 1024;
}

template <bool kDense>
__global__ void __launch_bounds__(kScoreThreads, 1)
score_filter_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_g,
                    const ScoreParams p) {
  extern __shared__ uint8_t smem_raw[];
  // align inside the dynamic smem window without a pointer->integer->pointer round trip (which would demote every
  // later access to generic LD/ST)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* smem_q = smem;
  uint8_t* smem_g = smem + p.num_kb * kQBlockBytes;
  uint32_t* stage_sm = reinterpret_cast<uint32_t*>(smem_g + kGStages * kGStageBytes);  // [128][kStageLd] score bits
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(stage_sm + kQM * kStageLd);  // 128 x 65 words: 8-byte aligned
  uint64_t* empty_bar = full_bar + kGStages;
  uint64_t* q_full = empty_bar + kGStages;
  uint64_t* q_empty = q_full + 1;

  const int n_units = p.n_qtiles * p.n_splits;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_q);
    prefetch_tensormap(&map_g);
    for (int i = 0; i < kGStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);  // one arrival per consumer warp
    }
    mbar_init(q_full, 1);
    mbar_init(q_empty, 8);
    fence_mbar_init();
  }
  __syncthreads();

  if (threadIdx.x < 128) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0, uphase = 0;
      for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
        const int qt = u % p.n_qtiles, sp = u / p.n_qtiles;
        const int t0 = sp * p.tiles_per_split;
        const int t1 = min(t0 + p.tiles_per_split, p.n_tiles);
        if (t0 >= t1) continue;
        // the query tile stays resident for the whole unit
        mbar_wait<true>(q_empty, uphase ^ 1);
        mbar_arrive_expect_tx(q_full, p.num_kb * kQBlockBytes);
        for (int kb = 0; kb < p.num_kb; ++kb)
          tma_load_2d(smem_q + kb * kQBlockBytes, &map_q, q_full, kb * kSBK, qt * kQM, kEvictLast);
        uphase ^= 1;
        tile_produce_b(smem_g, &map_g, full_bar, empty_bar, p.num_kb, static_cast<int>(p.g_lo), t0, t1, stage, phase);
      }
    }
  } else {
    // ===================== consumers: scores of 64 query rows each, then the filter =====================
    // The accumulator leaves the registers in 64-column chunks through shared memory; thread (row, half) then examines 32
    // consecutive gallery columns of one query row, so each (row, split, half) has exactly one writer thread.
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int ct = threadIdx.x - 128;
    const int cg = ct >> 7;
    const int wl = (ct >> 5) & 3, lane = ct & 31;
    const int frow = cg * 64 + wl * 16 + (lane >> 2);
    const int fcol = (lane & 3) * 2;
    const int erow = ct & 127, half = ct >> 7;
    int stage = 0;
    uint32_t phase = 0, uphase = 0;
    float acc[kGN / 2];
    for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
      const int qt = u % p.n_qtiles, sp = u / p.n_qtiles;
      const int t0 = sp * p.tiles_per_split;
      const int t1 = min(t0 + p.tiles_per_split, p.n_tiles);
      if (t0 >= t1) continue;
      mbar_wait<true>(q_full, uphase);
      uphase ^= 1;
      const int row = qt * kQM + erow;
      const bool row_ok = row < p.n_query;
      float tau = INFINITY;
      if (!kDense && row_ok) tau = p.tau[row];
      uint2* seg = p.seg + static_cast<size_t>(row_ok ? row : 0) * p.seg_stride + (kDense ? 0 : (sp * 2 + half) * p.seg_cap);
      unsigned cnt = 0;
      for (int t = t0; t < t1; ++t) {
        tile_mma(acc, smem_q, smem_g, full_bar, empty_bar, p.num_kb, cg, lane, stage, phase);
        if (lane == 0 && t + 1 == t1) mbar_arrive(q_empty);  // every MMA of this unit has retired: the query tile may be overwritten
        const int64_t gbase = p.g_lo + static_cast<int64_t>(t) * kGN;
#pragma unroll
        for (int cc = 0; cc < kGN / 64; ++cc) {
          tile_stage_chunk(stage_sm, acc, cc, frow, fcol);
          named_bar_sync(1, 256);
          uint32_t r[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) r[j] = stage_sm[erow * kStageLd + half * 32 + j];
          named_bar_sync(1, 256);  // the staging buffer may take the next chunk
          const int c = cc * 2 + half;  // 32-column chunk of the tile
          const int64_t g0 = gbase + c * 32;
          if (kDense) {
            if (row_ok && g0 < p.g_hi) {
              uint2* dst = seg + (g0 - p.g_lo);
              const int64_t rem = p.g_hi - g0;
              const int nv = rem < 32 ? static_cast<int>(rem) : 32;
              if (nv == 32) {
#pragma unroll
                for (int j = 0; j < 32; j += 2)
                  *reinterpret_cast<uint4*>(dst + j) = make_uint4(r[j], static_cast<uint32_t>(g0 + j), r[j + 1],
                                                                  static_cast<uint32_t>(g0 + j + 1));
              } else {
#pragma unroll
                for (int j = 0; j < 32; ++j)
                  if (j < nv) dst[j] = make_uint2(r[j], static_cast<uint32_t>(g0 + j));
              }
            }
          } else {
            // two-level test: group maxima first, so the common case costs ~1 instruction per score
            float gm[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              float m = __uint_as_float(r[q * 8]);
#pragma unroll
              for (int j = 1; j < 8; ++j) m = fmaxf(m, __uint_as_float(r[q * 8 + j]));
              gm[q] = m;
            }
            if (fmaxf(fmaxf(gm[0], gm[1]), fmaxf(gm[2], gm[3])) >= tau) {  // rows beyond n_query carry tau = +inf
              const uint32_t gcol = static_cast<uint32_t>(g0);
              const int64_t remv = p.g_hi - g0;
              const uint32_t nvalid = remv < 32 ? static_cast<uint32_t>(remv > 0 ? remv : 0) : 32u;
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                if (gm[q] >= tau) {
#pragma unroll
                  for (int j = q * 8; j < q * 8 + 8; ++j) {
                    if (__uint_as_float(r[j]) >= tau && static_cast<uint32_t>(j) < nvalid) {
                      if (cnt < static_cast<unsigned>(p.seg_cap)) seg[cnt] = make_uint2(r[j], gcol + j);
                      ++cnt;
                    }
                  }
                }
              }
            }
          }
        }
      }
      if (!kDense && row_ok) p.seg_cnt[static_cast<size_t>(row) * kMaxSeg + sp * 2 + half] = cnt;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// select: one CTA per query — k-th largest approximate score, admission bound, compaction of survivors
// ------------------------------------------------------------------------------------------------
constexpr int kSelThreads = 128;
constexpr unsigned kShortList = 256;  // lists up to this length are swept by a single warp

struct SelectParams {
  int n_query, k;
  const uint2* carry_in;  // [n_query][carry_cap] survivors of earlier ranges
  uint2* carry_out;       // [n_query][carry_cap]
  unsigned* carry_cnt;    // [n_query] in: entries in carry_in; out: entries in carry_out
  int carry_cap;
  const uint2* seg;       // this range's admitted candidates
  int seg_stride, seg_cap, n_seg;
  const unsigned* seg_cnt;
  int dense_n;            // > 0: the range was scored densely: seg holds dense_n entries per row
  float* tau;
  const float* eps;       // per-query bound on |approx - canonical|
  int32_t* status;        // {overflow_rows, max_candidates, max_survivors, reserved}
  int32_t* row_flag;      // [n_query] set to 1 for rows whose lists overflowed (results incomplete)
  float* kth_lb;          // [n_query] optional: lower bound of the k-th largest canonical score of this shard
  int stage_cap;          // entries of dynamic shared memory available for staging (<= kSelStage)
  const float* ext_lb;    // [n_query] optional: lower bound of the GLOBAL k-th canonical score known before this range
};

// Rows whose lists hold at most kSelStage entries in total (every sparse range in practice: ~110 carried + a few hundred
// admitted; the dense first range: 4096) are first gathered into ONE contiguous shared-memory array — every global load of the
// row is issued at once instead of 33 short dependent sweeps per radix pass — and the four radix passes and the compaction
// then run out of shared memory.  Longer rows keep sweeping the lists in place.
constexpr int kSelStage = 4096;

// kPre: the prefilter of dense ranges, entries held in registers.  Its own instantiation: the 64 registers of the entry
// array would otherwise cut the occupancy of every sparse-range launch.
template <bool kAgg, bool kPre>
__global__ void __launch_bounds__(kSelThreads) select_kernel(const SelectParams p) {
  extern __shared__ uint2 s_stage[];  // [p.stage_cap]
  __shared__ unsigned hist[256];
  __shared__ unsigned s_cnt[kMaxSeg + 1];
  __shared__ unsigned s_off[kMaxSeg + 2];
  __shared__ unsigned s_bin, s_krem, s_m, s_over, s_n2;
  __shared__ float s_floor;
  const int row = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  // entry lists of this row: list 0 = carry, lists 1.. = segments (or one dense list)
  int n_lists = 1 + (p.dense_n > 0 ? 1 : p.n_seg);
  if (tid == 0) {
    s_over = 0;
    s_m = 0;
    s_n2 = 0;
    s_cnt[0] = min(p.carry_cnt[row], static_cast<unsigned>(p.carry_cap));
  }
  if (tid >= 1 && tid < n_lists) {
    if (p.dense_n > 0) {
      s_cnt[1] = static_cast<unsigned>(p.dense_n);
    } else {
      const unsigned c = p.seg_cnt[static_cast<size_t>(row) * kMaxSeg + (tid - 1)];
      if (c > static_cast<unsigned>(p.seg_cap)) atomicOr(&s_over, 1u);
      s_cnt[tid] = min(c, static_cast<unsigned>(p.seg_cap));
    }
  }
  __syncthreads();
  if (tid == 0) {
    unsigned acc = 0;
    for (int l = 0; l < n_lists; ++l) {
      s_off[l] = acc;
      acc += s_cnt[l];
    }
    s_off[n_lists] = acc;
  }
  __syncthreads();
  const unsigned n = s_off[n_lists];
  auto list_ptr_g = [&](int l) -> const uint2* {
    if (l == 0) return p.carry_in + static_cast<size_t>(row) * p.carry_cap;
    return p.seg + static_cast<size_t>(row) * p.seg_stride + static_cast<size_t>(l - 1) * (p.dense_n > 0 ? 0 : p.seg_cap);
  };
  const bool staged = n <= static_cast<unsigned>(p.stage_cap);
  // Dense range (thousands of scores per row, all of one sign and exponent: the first radix digits barely discriminate and
  // their histogram atomics pile up on 2-3 bins).  Prefilter instead: thread t takes the maximum of
  // entries t, t + 128, ...; >= k threads hold a maximum >= F (the k-th largest of the 128 maxima), so the
  // k-th largest score of the row is >= F and only entries >= F - 2 eps can survive the select.  They (a few hundred) are
  // compacted into shared memory and the radix passes run on them.
  const bool pre = kPre && p.dense_n > 0 && staged && n >= 1024u && p.k <= kSelThreads;  // CTA-uniform
  if constexpr (kPre) {
    // every entry is read ONCE and kept (64 registers) between the maximum and the compaction
    if (pre) {
      constexpr int kPer = kSelStage / kSelThreads;
      uint2 ent[kPer];
      const uint2* c0 = list_ptr_g(0);
      const uint2* d0 = list_ptr_g(1);
      const unsigned cnt0 = s_cnt[0];
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < kPer; ++j) {
        const unsigned i = static_cast<unsigned>(j * kSelThreads + tid);
        ent[j] = make_uint2(0xff800000u, 0u);  // -inf
        if (i < n) ent[j] = i < cnt0 ? c0[i] : d0[i - cnt0];
        mx = fmaxf(mx, __uint_as_float(ent[j].x));
      }
      float* s_mx = reinterpret_cast<float*>(hist);  // re-zeroed by every radix pass
      s_mx[tid] = mx;
      __syncthreads();
      int gt = 0, ge = 0;
      for (int j = 0; j < kSelThreads; ++j) {
        const float y = s_mx[j];
        gt += y > mx ? 1 : 0;
        ge += y >= mx ? 1 : 0;
      }
      if (gt < p.k && p.k <= ge) s_floor = mx;  // the k-th largest maximum (ties write the same value)
      __syncthreads();
      const float keep_from = s_floor - 2.0f * p.eps[row];
#pragma unroll
      for (int j = 0; j < kPer; ++j) {
        const bool k_ = static_cast<unsigned>(j * kSelThreads + tid) < n && __uint_as_float(ent[j].x) >= keep_from;
        const unsigned m = __ballot_sync(0xffffffffu, k_);
        if (m != 0u) {  // warp-uniform
          unsigned base_pos = 0;
          if (lane == 0) base_pos = atomicAdd(&s_n2, static_cast<unsigned>(__popc(m)));
          base_pos = __shfl_sync(0xffffffffu, base_pos, 0);
          if (k_) s_stage[base_pos + __popc(m & ((1u << lane) - 1u))] = ent[j];
        }
      }
      __syncthreads();
      if (tid == 0) s_cnt[0] = s_n2;  // <= n <= stage_cap
      n_lists = 1;
      __syncthreads();
    }
  }
  if (!pre && staged) {
    for (int l = warp; l < n_lists; l += kSelThreads / 32) {
      const unsigned c = s_cnt[l];
      if (c > kShortList) continue;
      const uint2* e = list_ptr_g(l);
      const unsigned o = s_off[l];
      for (unsigned i = lane; i < c; i += 32) s_stage[o + i] = e[i];
    }
    for (int l = 0; l < n_lists; ++l) {
      const unsigned c = s_cnt[l];
      if (c <= kShortList) continue;
      const uint2* e = list_ptr_g(l);
      const unsigned o = s_off[l];
      for (unsigned i = tid; i < c; i += kSelThreads) s_stage[o + i] = e[i];
    }
    __syncthreads();
    if (tid == 0) s_cnt[0] = n;
    n_lists = 1;
    __syncthreads();
  }
  auto list_ptr = [&](int l) -> const uint2* { return staged ? s_stage : list_ptr_g(l); };

  // ---- radix select of the k-th largest key over all lists (4 x 8 bits, MSB first) ----
  float tau_use = -INFINITY;
  float kth_approx = -INFINITY;
  if (n >= static_cast<unsigned>(p.k)) {
    uint32_t prefix = 0, mask = 0;
    unsigned k_rem = static_cast<unsigned>(p.k);
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int i = tid; i < 256; i += kSelThreads) hist[i] = 0;
      __syncthreads();
      // long lists are swept by the whole CTA, short ones (a segment holds tens of entries) by one warp each, so that
      // 30+ nearly empty lists do not cost 30+ CTA-wide loop trips
      // warp-aggregated histogram: candidate scores share sign and exponent, so the first digit of most keys falls into a
      // handful of bins — one shared-memory atomic per (warp, distinct bin) instead of one per key (the 4096-entry dense
      // range would serialise ~1000 deep on a single bin)
      for (int l = 0; l < n_lists; ++l) {
        const unsigned c = s_cnt[l];
        if (c <= kShortList) continue;
        const uint2* e = list_ptr(l);
        for (unsigned base = 0; base < c; base += kSelThreads) {
          const unsigned i = base + tid;
          unsigned bin = 0xffffffffu;
          if (i < c) {
            const uint32_t key = ord_u32(__uint_as_float(e[i].x));
            if ((key & mask) == prefix) bin = (key >> shift) & 255u;
          }
          if (kAgg) {
            const unsigned peers = __match_any_sync(0xffffffffu, bin);
            if (bin != 0xffffffffu && lane == __ffs(peers) - 1) atomicAdd(&hist[bin], static_cast<unsigned>(__popc(peers)));
          } else if (bin != 0xffffffffu) {
            atomicAdd(&hist[bin], 1u);
          }
        }
      }
      for (int l = warp; l < n_lists; l += kSelThreads / 32) {
        const unsigned c = s_cnt[l];
        if (c > kShortList) continue;
        const uint2* e = list_ptr(l);
        for (unsigned base = 0; base < c; base += 32) {
          const unsigned i = base + lane;
          unsigned bin = 0xffffffffu;
          if (i < c) {
            const uint32_t key = ord_u32(__uint_as_float(e[i].x));
            if ((key & mask) == prefix) bin = (key >> shift) & 255u;
          }
          if (bin != 0xffffffffu) atomicAdd(&hist[bin], 1u);  // short lists: few keys per warp, nothing to aggregate
        }
      }
      __syncthreads();
      if (warp == 0) {
        // lane l owns bins 255-8l .. 248-8l (descending); find the bin where the running count reaches k_rem
        unsigned part = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) part += hist[255 - 8 * lane - j];
        unsigned incl = part;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
          const unsigned o = __shfl_up_sync(0xffffffffu, incl, off);
          if (lane >= off) incl += o;
        }
        const unsigned excl = incl - part;
        if (excl < k_rem && incl >= k_rem) {  // exactly one lane
          unsigned acc = excl;
          int b = 255 - 8 * lane;
          for (int j = 0; j < 8; ++j, --b) {
            if (acc + hist[b] >= k_rem) break;
            acc += hist[b];
          }
          s_bin = static_cast<unsigned>(b);
          s_krem = k_rem - acc;
        }
      }
      __syncthreads();
      prefix |= s_bin << shift;
      mask |= 255u << shift;
      k_rem = s_krem;
      __syncthreads();
    }
    // admission bound: everything within 2*eps below the k-th largest approximate score may be a true top-k member
    kth_approx = unord_u32(prefix);
    tau_use = kth_approx - 2.0f * p.eps[row];
  }
  // sharded search: a candidate below (global k-th canonical lower bound) - eps cannot reach the global top-k either
  if (p.ext_lb) tau_use = fmaxf(tau_use, p.ext_lb[row] - p.eps[row]);

  // ---- compaction of the survivors into the other carry buffer ----
  uint2* out = p.carry_out + static_cast<size_t>(row) * p.carry_cap;
  // survivors take consecutive slots of the carry list: one atomic per warp iteration (ballot + prefix), not one per survivor
  auto keep = [&](bool in_range, uint2 v) {
    const bool k_ = in_range && __uint_as_float(v.x) >= tau_use;
    const unsigned m = __ballot_sync(0xffffffffu, k_);
    if (m == 0u) return;
    unsigned base_pos = 0;
    if (lane == 0) base_pos = atomicAdd(&s_m, static_cast<unsigned>(__popc(m)));
    base_pos = __shfl_sync(0xffffffffu, base_pos, 0);
    if (k_) {
      const unsigned pos = base_pos + __popc(m & ((1u << lane) - 1u));
      if (pos < static_cast<unsigned>(p.carry_cap)) out[pos] = v;
    }
  };
  for (int l = 0; l < n_lists; ++l) {
    const unsigned c = s_cnt[l];
    if (c <= kShortList) continue;
    const uint2* e = list_ptr(l);
    for (unsigned base = 0; base < c; base += kSelThreads) {
      const unsigned i = base + tid;
      keep(i < c, i < c ? e[i] : make_uint2(0u, 0u));
    }
  }
  for (int l = warp; l < n_lists; l += kSelThreads / 32) {
    const unsigned c = s_cnt[l];
    if (c > kShortList) continue;
    const uint2* e = list_ptr(l);
    for (unsigned base = 0; base < c; base += 32) {
      const unsigned i = base + lane;
      keep(i < c, i < c ? e[i] : make_uint2(0u, 0u));
    }
  }
  __syncthreads();
  if (tid == 0) {
    const unsigned m = s_m;
    p.carry_cnt[row] = min(m, static_cast<unsigned>(p.carry_cap));
    p.tau[row] = tau_use;
    // a lower bound of this shard's k-th largest CANONICAL score (|approx - canonical| <= eps): what the ranks of a sharded
    // search exchange (max) to skip re-ranking candidates that cannot reach the global top-k
    if (p.kth_lb) p.kth_lb[row] = p.ext_lb ? fmaxf(kth_approx - p.eps[row], p.ext_lb[row]) : kth_approx - p.eps[row];
    if (s_over || m > static_cast<unsigned>(p.carry_cap)) {
      if (atomicExch(&p.row_flag[row], 1) == 0) atomicAdd(&p.status[0], 1);  // count each row once
    }
    atomicMax(&p.status[1], static_cast<int>(min(n, 0x7fffffffu)));
    atomicMax(&p.status[2], static_cast<int>(min(m, 0x7fffffffu)));
  }
}

// ------------------------------------------------------------------------------------------------
// rerank: canonical re-score of a row's carry list, sort by (score desc, id asc), emit k
// ------------------------------------------------------------------------------------------------
constexpr int kRerankThreads = 256;

struct RerankParams {
  int n_query, dim, k;
  const uint2* carry;
  const unsigned* carry_cnt;
  int carry_cap;
  const float* q32;
  const float* g32;
  int64_t id_offset;
  float* out_scores;
  int64_t* out_ids;
  const float* kth_lb;  // optional [n_query]: lower bound of the GLOBAL k-th canonical score (max over shards)
  const float* eps;     // per-query bound on |approx - canonical|
};

__global__ void __launch_bounds__(kRerankThreads) rerank_kernel(const RerankParams p) {
  extern __shared__ unsigned long long s_sort[];  // [pow2 >= m] sort keys, then [carry_cap] uint32 kept candidate slots
  __shared__ unsigned s_keep;
  const int row = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int nwarps = kRerankThreads / 32;
  const int m_all = static_cast<int>(min(p.carry_cnt[row], static_cast<unsigned>(p.carry_cap)));
  const uint2* e = p.carry + static_cast<size_t>(row) * p.carry_cap;
  const float* q = p.q32 + static_cast<size_t>(row) * p.dim;
  uint32_t* keep = reinterpret_cast<uint32_t*>(s_sort + p.carry_cap);
  // sharded search: a candidate whose approximate score is below (global k-th canonical lower bound) - eps cannot be in the
  // global top-k (canonical >= bound implies approx >= bound - eps), so its 2 KB row is never fetched
  const float thr = p.kth_lb ? p.kth_lb[row] - p.eps[row] : -INFINITY;
  if (tid == 0) s_keep = 0;
  __syncthreads();
  for (int c = tid; c < m_all; c += kRerankThreads)
    if (__uint_as_float(e[c].x) >= thr) keep[atomicAdd(&s_keep, 1u)] = static_cast<uint32_t>(c);
  __syncthreads();
  const int m = static_cast<int>(s_keep);
  // two candidates per warp iteration: their row loads are independent, which hides the gather latency
  for (int c = warp * 2; c < m; c += nwarps * 2) {
    const uint32_t gi0 = e[keep[c]].y;
    const bool has1 = c + 1 < m;
    const uint32_t gi1 = has1 ? e[keep[c + 1]].y : gi0;
    const float* g0 = p.g32 + static_cast<size_t>(gi0) * p.dim;
    const float* g1 = p.g32 + static_cast<size_t>(gi1) * p.dim;
    double a0 = 0.0, a1 = 0.0;
    for (int i = lane; i < p.dim; i += 32) {
      const double qv = static_cast<double>(q[i]);
      a0 = fma(qv, static_cast<double>(g0[i]), a0);
      a1 = fma(qv, static_cast<double>(g1[i]), a1);
    }
    a0 = warp_sum_f64(a0);
    a1 = warp_sum_f64(a1);
    if (lane == 0) {
      s_sort[c] = (static_cast<unsigned long long>(ord_u32(static_cast<float>(a0))) << 32) | static_cast<unsigned long long>(~gi0);
      if (has1)
        s_sort[c + 1] = (static_cast<unsigned long long>(ord_u32(static_cast<float>(a1))) << 32) | static_cast<unsigned long long>(~gi1);
    }
  }
  int m2 = 1;
  while (m2 < m) m2 <<= 1;
  for (int i = m + tid; i < m2; i += kRerankThreads) s_sort[i] = 0ull;  // below every real key
  __syncthreads();
  // bitonic sort, descending: key = (ordered score, ~id) so equal scores order by ascending id
  for (int size = 2; size <= m2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = tid; i < (m2 >> 1); i += kRerankThreads) {
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool desc = ((lo & size) == 0);
        const unsigned long long a = s_sort[lo], b = s_sort[hi];
        if ((a < b) == desc) {
          s_sort[lo] = b;
          s_sort[hi] = a;
        }
      }
      __syncthreads();
    }
  }
  for (int j = tid; j < p.k; j += kRerankThreads) {
    float sc = -FLT_MAX;  // faiss pads inner-product results with lowest() and id -1
    int64_t id = -1;
    if (j < m) {
      const unsigned long long key = s_sort[j];
      sc = unord_u32(static_cast<uint32_t>(key >> 32));
      id = static_cast<int64_t>(~static_cast<uint32_t>(key & 0xffffffffull)) + p.id_offset;
    }
    p.out_scores[static_cast<size_t>(row) * p.k + j] = sc;
    p.out_ids[static_cast<size_t>(row) * p.k + j] = id;
  }
}

__global__ void eps_kernel(const float* __restrict__ q_norm, const float* __restrict__ q_err,
                           const float* __restrict__ g_norm_max, const float* __restrict__ g_err_max, int n,
                           float* __restrict__ eps, float* __restrict__ tau, unsigned* __restrict__ carry_cnt,
                           float* __restrict__ kth_lb) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float gn = g_norm_max ? *g_norm_max : 0.f, ge = g_err_max ? *g_err_max : 0.f;
  const float qn = q_norm[i] + q_err[i];
  // |approx - canonical| <= |dq.g| + |qh.dg| + tensor-core accumulation error (DESIGN.md, "error bound")
  const float e = q_err[i] * gn + qn * ge + 1.220703125e-4f /*2^-13*/ * qn * (gn + ge);
  eps[i] = e * 1.0001f + 1e-30f;
  tau[i] = -INFINITY;
  carry_cnt[i] = 0;
  kth_lb[i] = -INFINITY;
}

// ------------------------------------------------------------------------------------------------
// merge of per-shard lists, and brute-force pair scores for verification
// ------------------------------------------------------------------------------------------------
// Lists as separate (scores, ids) arrays.
__global__ void topk_merge_kernel(const float* __restrict__ scores, const int64_t* __restrict__ ids, int n_lists, int64_t n_query,
                                  int k, float* __restrict__ out_scores, int64_t* __restrict__ out_ids) {
  // one warp per query; lists are individually ordered, so a k-step tournament over n_lists heads suffices
  const int lane = threadIdx.x & 31;
  const int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (row >= n_query) return;
  int head = 0;  // lane l owns list l (n_lists <= 32)
  const size_t list_stride = static_cast<size_t>(n_query) * k;
  for (int j = 0; j < k; ++j) {
    float sc = -FLT_MAX;
    int64_t id = -1;
    if (lane < n_lists && head < k) {
      sc = scores[lane * list_stride + row * k + head];
      id = ids[lane * list_stride + row * k + head];
    }
    // best = max score, then smallest non-negative id
    float bs = sc;
    int64_t bid = id;
    int bl = lane;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float os = __shfl_xor_sync(0xffffffffu, bs, off);
      const int64_t oid = __shfl_xor_sync(0xffffffffu, bid, off);
      const int ol = __shfl_xor_sync(0xffffffffu, bl, off);
      const bool o_valid = oid >= 0, b_valid = bid >= 0;
      bool take;
      if (o_valid != b_valid) take = o_valid;
      else if (os != bs) take = os > bs;
      else if (oid != bid) take = oid < bid;
      else take = ol < bl;
      if (take) {
        bs = os;
        bid = oid;
        bl = ol;
      }
    }
    if (lane == 0) {
      out_scores[row * k + j] = bid >= 0 ? bs : -FLT_MAX;
      out_ids[row * k + j] = bid;
    }
    if (lane == bl && bid >= 0) ++head;
  }
}

// Lists PACKED as one 64-bit word per entry (score bits << 32 | uint32 id, id -1 = 0xffffffff), the form the ranks of the
// sharded search exchange in ONE all-gather: one query per GROUP of `group` = pow2 >= n_lists lanes (4 queries per warp on 8
// shards).  Lane l of a group walks list l and holds its head as ONE 64-bit key (order-preserving score bits << 32 | ~id: larger
// is better — score desc, id asc; 0 = list exhausted) with the next entry already loaded, so a step is log2(group) 64-bit
// max-shuffles and the winner's register move: no load on the critical path (the general kernel above re-loads 32 heads and
// runs a five-round three-field tournament per step).
__global__ void __launch_bounds__(256) topk_merge_packed_kernel(const unsigned long long* __restrict__ packed, int n_lists,
                                                                int group, int64_t n_query, int k,
                                                                float* __restrict__ out_scores, int64_t* __restrict__ out_ids) {
  const int lane = threadIdx.x & 31;
  const int sub = lane & (group - 1);
  const int64_t warp_id = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int64_t row = warp_id * (32 / group) + lane / group;
  const bool row_ok = row < n_query;  // lanes of rows past the end keep shuffling (full-mask warp), they never load or store
  const bool has_list = row_ok && sub < n_lists;
  const unsigned long long* src = packed + (has_list ? static_cast<size_t>(sub) * n_query * k + static_cast<size_t>(row) * k : 0);
  auto key_of = [](unsigned long long w) -> unsigned long long {
    const uint32_t lo = static_cast<uint32_t>(w);
    if (lo == 0xffffffffu) return 0ull;  // padding (id -1): the list ends here
    uint32_t u = static_cast<uint32_t>(w >> 32);
    if (u == 0x80000000u) u = 0u;  // -0.0 ties with +0.0 under the float comparison of the tie rule
    return (static_cast<unsigned long long>(ord_u32(__uint_as_float(u))) << 32) | static_cast<unsigned long long>(~lo);
  };
  unsigned long long cur_w = has_list ? src[0] : ~0ull, nxt_w = (has_list && k > 1) ? src[1] : ~0ull;  // ~0: padding word
  unsigned long long cur = key_of(cur_w);
  int head = 0;
  for (int j = 0; j < k; ++j) {
    unsigned long long best = cur;
    for (int off = group >> 1; off > 0; off >>= 1) {
      const unsigned long long o = __shfl_xor_sync(0xffffffffu, best, off);
      best = o > best ? o : best;
    }
    if (best == 0ull) {  // every list exhausted
      if (sub == 0 && row_ok) {
        out_scores[row * k + j] = -FLT_MAX;
        out_ids[row * k + j] = -1;
      }
    } else if (cur == best) {  // keys are unique (shards hold disjoint ids): exactly one lane wins, emits its entry, advances
      out_scores[row * k + j] = __uint_as_float(static_cast<uint32_t>(cur_w >> 32));  // the original bits (-0.0 stays -0.0)
      out_ids[row * k + j] = static_cast<int64_t>(static_cast<uint32_t>(cur_w));
      ++head;
      cur_w = nxt_w;
      cur = key_of(cur_w);
      nxt_w = head + 1 < k ? src[head + 1] : ~0ull;
    }
  }
}

__global__ void topk_pack_kernel(const float* __restrict__ scores, const int64_t* __restrict__ ids, int64_t n,
                                 unsigned long long* __restrict__ out) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t id = ids[i];
  out[i] = (static_cast<unsigned long long>(__float_as_uint(scores[i])) << 32) |
           static_cast<unsigned long long>(id < 0 ? 0xffffffffu : static_cast<uint32_t>(id));
}

__global__ void exact_pairs_kernel(const float* __restrict__ q32, const float* __restrict__ g32, int dim,
                                   const int64_t* __restrict__ qi, const int64_t* __restrict__ gi, int64_t n,
                                   float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t w = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (w >= n) return;
  const float* q = q32 + qi[w] * dim;
  const float* g = g32 + gi[w] * dim;
  double acc = 0.0;
  for (int i = lane; i < dim; i += 32) acc = fma(static_cast<double>(q[i]), static_cast<double>(g[i]), acc);
  acc = warp_sum_f64(acc);
  if (lane == 0) out[w] = static_cast<float>(acc);
}

// ------------------------------------------------------------------------------------------------
// exhaustive path: canonical scores of a few queries against EVERY gallery row, exact selection on 64-bit keys.
// Taken only for rows whose candidate lists overflowed even on the all-dense plan (thousands of exact duplicates of
// a top-k member): faiss' flat search never fails on such galleries (engine/cbir/evaluation.py:193), so neither may
// this one.  No approximate pass, no capacity: key = (ordered canonical score, ~row), unique per row, so the k-th
// largest key is found exactly by an 8 x 8-bit radix select and the k survivors are sorted.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) exhaustive_scores_kernel(const float* __restrict__ q32, int nq, const float* __restrict__ g32,
                                                                int64_t ng, int dim, unsigned long long* __restrict__ keys) {
  extern __shared__ float ex_q[];  // [nq][dim]
  for (int i = threadIdx.x; i < nq * dim; i += blockDim.x) ex_q[i] = q32[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
  for (int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; row < ng; row += warps) {
    float s[kExQ];
    canonical_scores_x8(ex_q, nq, g32 + row * dim, dim, lane, s);
#pragma unroll
    for (int j = 0; j < kExQ; ++j)
      if (j < nq && lane == 0) keys[static_cast<size_t>(j) * ng + row] = score_key(s[j], static_cast<uint32_t>(row));
  }
}

__global__ void __launch_bounds__(kExThreads) exhaustive_select_kernel(const unsigned long long* __restrict__ keys, int64_t ng, int k,
                                                                       int64_t id_offset, float* __restrict__ out_scores,
                                                                       int64_t* __restrict__ out_ids) {
  select_topk_keys(keys + static_cast<size_t>(blockIdx.x) * ng, ng, k, id_offset, out_scores + static_cast<size_t>(blockIdx.x) * k,
                   out_ids + static_cast<size_t>(blockIdx.x) * k);
}

static int pow2_ceil(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

struct TopkWorkspace {
  uint2* seg;
  uint2* carry[2];
  unsigned* seg_cnt;
  unsigned* carry_cnt;
  float* tau;
  float* eps;
  int32_t* row_flag;
  float* kth_lb;
};
static size_t align256(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }
static size_t workspace_bytes(int64_t nq, int seg_stride, int carry_cap) {
  const size_t n = static_cast<size_t>(nq);
  return align256(n * seg_stride * sizeof(uint2)) + 2 * align256(n * carry_cap * sizeof(uint2)) +
         align256(n * kMaxSeg * sizeof(unsigned)) + 5 * align256(n * sizeof(float)) + 256;
}
static TopkWorkspace carve_workspace(void* workspace, int64_t nq, int seg_stride, int carry_cap) {
  const size_t n = static_cast<size_t>(nq);
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  TopkWorkspace w;
  w.seg = reinterpret_cast<uint2*>(ws);
  ws += align256(n * seg_stride * sizeof(uint2));
  for (int i = 0; i < 2; ++i) {
    w.carry[i] = reinterpret_cast<uint2*>(ws);
    ws += align256(n * carry_cap * sizeof(uint2));
  }
  w.seg_cnt = reinterpret_cast<unsigned*>(ws);
  ws += align256(n * kMaxSeg * sizeof(unsigned));
  w.carry_cnt = reinterpret_cast<unsigned*>(ws);
  ws += align256(n * sizeof(float));
  w.tau = reinterpret_cast<float*>(ws);
  ws += align256(n * sizeof(float));
  w.eps = reinterpret_cast<float*>(ws);
  ws += align256(n * sizeof(float));
  w.row_flag = reinterpret_cast<int32_t*>(ws);
  ws += align256(n * sizeof(float));
  w.kth_lb = reinterpret_cast<float*>(ws);
  return w;
}

struct RangeLaunch {
  int n_splits, seg_cap;
};

// One gallery range [lo, hi) of the scan: the launch both vdk_ip_topk and vdk_score_range use.
static int launch_score_range(const CUtensorMap& mq, const CUtensorMap& mg, int nq, int dim, int64_t lo, int64_t hi,
                              bool dense, const TopkWorkspace& w, int seg_stride, RangeLaunch* info, cudaStream_t s) {
  static bool score_attr = false;
  if (!score_attr) {
    VDK_CUDA_OK(cudaFuncSetAttribute(score_filter_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     score_smem_bytes(kMaxKB)));
    VDK_CUDA_OK(cudaFuncSetAttribute(score_filter_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     score_smem_bytes(kMaxKB)));
    score_attr = true;
  }
  VDK_REQUIRE(lo % kGN == 0, "score range must start on a multiple of %d", kGN);
  if (dense) VDK_REQUIRE(hi - lo <= seg_stride, "dense first range exceeds candidate capacity");
  const int sms = sm_count();
  ScoreParams p{};
  p.n_query = nq;
  p.num_kb = dim / kSBK;
  p.g_lo = lo;
  p.g_hi = hi;
  p.n_qtiles = (nq + kQM - 1) / kQM;
  p.n_tiles = static_cast<int>((hi - lo + kGN - 1) / kGN);
  // (query tile, gallery split) units are statically dealt to the persistent CTAs: pick the split count (at most
  // kMaxSeg/2, one candidate segment per split, query and epilogue half) whose unit count fills whole waves best
  const int max_splits = std::max(1, std::min(kMaxSeg / 2, p.n_tiles));
  int best = 1;
  double best_eff = -1.0;
  for (int sp = 1; sp <= max_splits; ++sp) {
    const int tps = (p.n_tiles + sp - 1) / sp;
    const int nsp = (p.n_tiles + tps - 1) / tps;
    const long long units = static_cast<long long>(p.n_qtiles) * nsp;
    const long long waves = (units + sms - 1) / sms;
    // work is quantised in tiles per unit: the busiest CTA runs `waves` units of `tps` tiles
    const double eff = static_cast<double>(p.n_qtiles) * p.n_tiles / (static_cast<double>(waves) * sms * tps);
    if (eff > best_eff + 1e-9 || (eff > best_eff - 1e-9 && nsp > best)) {
      best_eff = eff;
      best = nsp;
    }
  }
  p.tiles_per_split = (p.n_tiles + best - 1) / best;
  p.n_splits = (p.n_tiles + p.tiles_per_split - 1) / p.tiles_per_split;
  p.tau = w.tau;
  p.seg = w.seg;
  p.seg_stride = seg_stride;
  p.seg_cap = seg_stride / (2 * p.n_splits);
  p.seg_cnt = w.seg_cnt;
  if (info) {
    info->n_splits = p.n_splits;
    info->seg_cap = p.seg_cap;
  }
  const int units = p.n_qtiles * p.n_splits;
  const int grid = std::min(units, sms);
  const int smem = score_smem_bytes(p.num_kb);
  ProfScope prof(kProfScoreFilter, 2.0 * dim * static_cast<double>(nq) * static_cast<double>(hi - lo),
                 2.0 * dim * (static_cast<double>(hi - lo) + static_cast<double>(nq) * p.n_splits), s);
  if (dense)
    score_filter_kernel<true><<<grid, kScoreThreads, smem, s>>>(mq, mg, p);
  else
    score_filter_kernel<false><<<grid, kScoreThreads, smem, s>>>(mq, mg, p);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

}  // namespace vdk

using namespace vdk;

extern "C" int vdk_rows_prepare(const float* x, int64_t n, int dim, int normalize, float* xn, void* xh,
                                float* row_norm, float* row_err, void* stream) {
  VDK_REQUIRE(x && xh && row_err, "vdk_rows_prepare: x, xh and row_err are required");
  VDK_REQUIRE(n >= 0 && dim > 0, "vdk_rows_prepare: bad shape n=%lld dim=%d", (long long)n, dim);
  if (n == 0) return VDK_OK;
  const int64_t warps_per_block = 256 / 32;
  const int64_t blocks = (n + warps_per_block - 1) / warps_per_block;
  VDK_REQUIRE(blocks < (1ll << 31), "vdk_rows_prepare: too many rows");
  rows_prepare_kernel<<<static_cast<unsigned>(blocks), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, n, dim, normalize, xn, reinterpret_cast<__half*>(xh), row_norm, row_err);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_reduce_max(const float* x, int64_t n, float* out, void* stream) {
  VDK_REQUIRE(x && out && n >= 0, "vdk_reduce_max: bad arguments");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  VDK_CUDA_OK(cudaMemsetAsync(out, 0, sizeof(float), s));
  if (n == 0) return VDK_OK;
  const int blocks = static_cast<int>(std::min<int64_t>((n + 255) / 256, 1184));
  reduce_max_kernel<<<blocks, 256, 0, s>>>(x, n, out);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_topk_plan_default(vdk_topk_plan* plan, int64_t n_query, int64_t n_gallery, int dim, int k) {
  VDK_REQUIRE(plan, "vdk_topk_plan_default: null plan");
  VDK_REQUIRE(n_query >= 0 && n_gallery >= 0 && n_gallery < (1ll << 31), "vdk_topk_plan_default: bad sizes");
  VDK_REQUIRE(dim > 0 && dim % 64 == 0 && dim <= 64 * kMaxKB, "vdk_topk_plan_default: dim must be a multiple of 64, <= 512 (got %d)", dim);
  VDK_REQUIRE(k >= 1 && k <= 1024, "vdk_topk_plan_default: k must be in [1,1024] (got %d)", k);
  plan->n_query = n_query;
  plan->n_gallery = n_gallery;
  plan->dim = dim;
  plan->k = k;
  plan->cand_capacity = pow2_ceil(std::max(16384, 16 * k));  // per-range admitted candidates per query
  plan->carry_capacity = pow2_ceil(std::max(2048, 4 * k));  // survivors carried between ranges
  plan->dense_mask = 1;                                     // only the first range is scored densely
  // first range is scored densely (no threshold yet); each later range is 8x the prefix before it, so the
  // expected number of admitted candidates per range stays near 7k.
  int64_t end = std::min<int64_t>(n_gallery, std::max(4096, 4 * k));
  end = (end + kGN - 1) / kGN * kGN;
  if (end > plan->cand_capacity) end = plan->cand_capacity;
  int s = 0;
  for (; s < 8; ++s) {
    if (end >= n_gallery || s == 7) {
      plan->stage_end[s] = n_gallery;
      ++s;
      break;
    }
    plan->stage_end[s] = end;
    end *= 8;
  }
  plan->n_stages = s;
  for (int i = s; i < 8; ++i) plan->stage_end[i] = n_gallery;
  return VDK_OK;
}

extern "C" size_t vdk_topk_workspace_bytes(const vdk_topk_plan* plan) {
  if (!plan) return 0;
  return workspace_bytes(plan->n_query, plan->cand_capacity, plan->carry_capacity);
}

static int check_plan(const vdk_topk_plan* plan) {
  VDK_REQUIRE(plan, "null plan");
  const int dim = plan->dim, k = plan->k;
  VDK_REQUIRE(dim > 0 && dim % 64 == 0 && dim <= 64 * kMaxKB, "unsupported dim %d", dim);
  VDK_REQUIRE(k >= 1 && k <= 1024, "k must be in [1,1024]");
  VDK_REQUIRE(plan->cand_capacity >= 2 * k && plan->cand_capacity % kMaxSeg == 0, "bad cand_capacity");
  VDK_REQUIRE(plan->carry_capacity >= 2 * k && plan->carry_capacity <= 4096, "carry_capacity must be in [2k, 4096]");
  VDK_REQUIRE(plan->n_stages >= 1 && plan->n_stages <= 8 && plan->stage_end[plan->n_stages - 1] == plan->n_gallery,
              "stage table must end at n_gallery");
  VDK_REQUIRE(plan->n_query < (1ll << 31) - kQM && plan->n_gallery < (1ll << 31), "sizes exceed 32-bit tiling");
  VDK_REQUIRE(plan->dense_mask >= 0 && plan->dense_mask < 256, "bad dense_mask");
  return VDK_OK;
}

// The scan half of vdk_ip_topk: thresholds, gallery ranges, selects.  Leaves every query's surviving candidates in the
// workspace (carry list) and, if `kth_lb_out` is given, a lower bound of the shard's k-th largest canonical score per query.
// tau[row] = max(tau[row], ext_lb[row] - eps[row]): a lower bound of the GLOBAL k-th canonical score (max over shards) tightens
// this shard's admission threshold before its next range
__global__ void tighten_kernel(float* __restrict__ tau, const float* __restrict__ ext_lb, const float* __restrict__ eps, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) tau[i] = fmaxf(tau[i], ext_lb[i] - eps[i]);
}

// Stages [stage_begin, stage_end) of the scan: thresholds, gallery ranges, selects.  Leaves every query's surviving candidates
// in the workspace (carry list) and, per query, a lower bound of the shard's k-th largest canonical score (w.kth_lb).
static int topk_filter(const vdk_topk_plan* plan, const void* qh, const float* q_norm, const float* q_err, const void* gh,
                       const float* g_norm_max, const float* g_err_max, int32_t* status, void* workspace, size_t workspace_bytes,
                       cudaStream_t s, int stage_begin = 0, int stage_end = 8, const float* ext_lb = nullptr) {
  int rc = check_plan(plan);
  if (rc != VDK_OK) return rc;
  VDK_REQUIRE(status, "vdk_ip_topk: null status");
  const int64_t nq = plan->n_query, ng = plan->n_gallery;
  const int dim = plan->dim, k = plan->k, seg_stride = plan->cand_capacity, carry_cap = plan->carry_capacity;
  if (stage_end > plan->n_stages) stage_end = plan->n_stages;
  VDK_REQUIRE(stage_begin >= 0 && stage_begin <= stage_end, "vdk_ip_topk: bad stage range [%d, %d)", stage_begin, stage_end);
  if (stage_begin == 0) VDK_CUDA_OK(cudaMemsetAsync(status, 0, 4 * sizeof(int32_t), s));
  if (nq == 0) return VDK_OK;
  VDK_REQUIRE(qh && q_norm && q_err, "vdk_ip_topk: null query operand");
  VDK_REQUIRE(workspace && workspace_bytes >= vdk_topk_workspace_bytes(plan), "vdk_ip_topk: workspace too small");
  VDK_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "vdk_ip_topk: workspace must be 256-byte aligned");
  if (ng > 0) VDK_REQUIRE(gh && g_norm_max && g_err_max, "vdk_ip_topk: null gallery operand");

  const TopkWorkspace w = carve_workspace(workspace, nq, seg_stride, carry_cap);
  if (stage_begin == 0) {
    VDK_CUDA_OK(cudaMemsetAsync(w.row_flag, 0, static_cast<size_t>(nq) * sizeof(int32_t), s));
    eps_kernel<<<(static_cast<int>(nq) + 255) / 256, 256, 0, s>>>(q_norm, q_err, ng > 0 ? g_norm_max : nullptr,
                                                                   ng > 0 ? g_err_max : nullptr, static_cast<int>(nq),
                                                                   w.eps, w.tau, w.carry_cnt, w.kth_lb);
    VDK_CUDA_OK(cudaGetLastError());
  }
  if (ext_lb) {
    tighten_kernel<<<(static_cast<int>(nq) + 255) / 256, 256, 0, s>>>(w.tau, ext_lb, w.eps, static_cast<int>(nq));
    VDK_CUDA_OK(cudaGetLastError());
  }
  static bool sel_attr = false;
  if (!sel_attr) {
    VDK_CUDA_OK(cudaFuncSetAttribute(select_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSelStage * sizeof(uint2)));
    VDK_CUDA_OK(cudaFuncSetAttribute(select_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSelStage * sizeof(uint2)));
    VDK_CUDA_OK(cudaFuncSetAttribute(select_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSelStage * sizeof(uint2)));
    sel_attr = true;
  }
  int cur = 0;  // carry buffer holding the current survivors
  if (ng > 0) {
    CUtensorMap mq, mg;
    rc = make_tma_2d_16bit(&mq, qh, static_cast<uint64_t>(nq), dim, dim, kQM, kSBK);
    if (rc != VDK_OK) return rc;
    rc = make_tma_2d_16bit(&mg, gh, static_cast<uint64_t>(ng), dim, dim, kGN, kSBK);
    if (rc != VDK_OK) return rc;
    int64_t lo = 0;
    for (int st = 0; st < stage_end; ++st) {
      const int64_t hi = plan->stage_end[st];
      VDK_REQUIRE(hi > lo || (hi == lo && st > 0), "vdk_ip_topk: stage table must be increasing");
      if (hi == lo) continue;
      if (st < stage_begin) {  // executed by an earlier call: only the carry parity and the range start move
        cur ^= 1;
        lo = hi;
        continue;
      }
      const bool dense = (st == 0) || ((plan->dense_mask >> st) & 1);
      RangeLaunch info{};
      rc = launch_score_range(mq, mg, static_cast<int>(nq), dim, lo, hi, dense, w, seg_stride, &info, s);
      if (rc != VDK_OK) return rc;
      SelectParams sp{};
      sp.n_query = static_cast<int>(nq);
      sp.k = k;
      sp.carry_in = w.carry[cur];
      sp.carry_out = w.carry[cur ^ 1];
      sp.carry_cnt = w.carry_cnt;
      sp.carry_cap = carry_cap;
      sp.seg = w.seg;
      sp.seg_stride = seg_stride;
      sp.seg_cap = info.seg_cap;
      sp.n_seg = 2 * info.n_splits;
      sp.seg_cnt = w.seg_cnt;
      sp.dense_n = dense ? static_cast<int>(hi - lo) : 0;
      sp.tau = w.tau;
      sp.eps = w.eps;
      sp.status = status;
      sp.row_flag = w.row_flag;
      sp.kth_lb = w.kth_lb;
      sp.ext_lb = ext_lb;
      // staging area: the dense first range needs room for every score of the range, a sparse range for a few hundred
      sp.stage_cap = dense ? kSelStage : kSelStage / 2;
      // dense ranges: the prefilter where it applies (what is left after it needs no aggregation), else warp-aggregated
      // histogram atomics, which pay on thousands of keys whose first digit collides; sparse ranges: the plain select
      if (dense && k <= kSelThreads)
        select_kernel<false, true><<<static_cast<unsigned>(nq), kSelThreads, sp.stage_cap * sizeof(uint2), s>>>(sp);
      else if (dense)
        select_kernel<true, false><<<static_cast<unsigned>(nq), kSelThreads, sp.stage_cap * sizeof(uint2), s>>>(sp);
      else
        select_kernel<false, false><<<static_cast<unsigned>(nq), kSelThreads, sp.stage_cap * sizeof(uint2), s>>>(sp);
      VDK_CUDA_OK(cudaGetLastError());
      cur ^= 1;
      lo = hi;
    }
  }
  return VDK_OK;
}

// carry buffer that holds the survivors after the first `stages_done` stages of this plan ran
static int carry_after(const vdk_topk_plan* plan, int stages_done) {
  int cur = 0;
  int64_t lo = 0;
  if (plan->n_gallery > 0)
    for (int st = 0; st < plan->n_stages && st < stages_done; ++st) {
      const int64_t hi = plan->stage_end[st];
      if (hi == lo) continue;
      cur ^= 1;
      lo = hi;
    }
  return cur;
}
static int final_carry(const vdk_topk_plan* plan) { return carry_after(plan, plan->n_stages); }

// ------------------------------------------------------------------------------------------------
// Sharded search: what the shards tell each other between gallery ranges.
//
// The k-th bound of ONE shard says little about the k-th score of the union when every shard holds a share of a query's
// neighbours (max over W shards of "100th of my 4096 rows" is still the 100th-of-4096 quantile, not the 100th of 32768).  So a
// shard reports a RANK SKETCH: lower bounds of its canonical scores at ranks k, k/2, k/4, ... (>= r_i of its rows score at least
// sketch[i]).  Shards hold disjoint rows, so for any threshold t the union holds at least sum_s max{r_i : sketch_s[i] >= t}
// rows scoring >= t; the largest reported t whose sum reaches k is a lower bound of the GLOBAL k-th canonical score.  With
// neighbours spread evenly it is the ceil(k/W)-th score of the weakest shard (~ the k-th of the union); with all neighbours in
// one shard it is that shard's k-th (the old max).
// ------------------------------------------------------------------------------------------------
constexpr int kSketchMaxRanks = 8;
constexpr int kSketchCap = 512;  // survivors per query the rank count handles; longer lists (massive ties) report rank k only

struct SketchParams {
  int n_query, k, n_ranks;
  int ranks[kSketchMaxRanks];
  const uint2* carry;
  const unsigned* carry_cnt;
  int carry_cap;
  const float* eps;
  const float* kth_lb;
  float* out;  // [n_query][n_ranks]
};

__global__ void __launch_bounds__(128) rank_sketch_kernel(const SketchParams p) {
  __shared__ float s_val[4][kSketchCap];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * 4 + warp;
  if (row >= p.n_query) return;  // warps are independent from here on (no CTA-wide barrier below)
  const unsigned m = min(p.carry_cnt[row], static_cast<unsigned>(p.carry_cap));
  float res[kSketchMaxRanks];
#pragma unroll
  for (int r = 0; r < kSketchMaxRanks; ++r) res[r] = -INFINITY;
  if (m <= static_cast<unsigned>(kSketchCap)) {
    const uint2* e = p.carry + static_cast<size_t>(row) * p.carry_cap;
    float* v = s_val[warp];
    for (unsigned i = lane; i < m; i += 32) v[i] = __uint_as_float(e[i].x);
    __syncwarp();
    // the survivors are every scanned row at or above the admission bound: the r-th largest of them is the r-th largest of
    // the shard so far.  Rank of a value by counting (m ~ k + a few): v is the r-th largest iff #{x > v} < r <= #{x >= v}
    // four values per lane share one sweep over the list (one shared-memory read per four rank updates)
    for (unsigned base = 0; base < m; base += 128) {
      float x[4];
      int gt[4] = {0, 0, 0, 0}, ge[4] = {0, 0, 0, 0};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const unsigned i = base + q * 32 + lane;
        x[q] = i < m ? v[i] : INFINITY;  // +inf: never matches a rank (#{y >= inf} = 0)
      }
      for (unsigned j = 0; j < m; ++j) {
        const float y = v[j];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          gt[q] += y > x[q] ? 1 : 0;
          ge[q] += y >= x[q] ? 1 : 0;
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int r = 0; r < kSketchMaxRanks; ++r)
          if (r < p.n_ranks && gt[q] < p.ranks[r] && p.ranks[r] <= ge[q]) res[r] = x[q];
    }
  }
#pragma unroll
  for (int r = 0; r < kSketchMaxRanks; ++r) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) res[r] = fmaxf(res[r], __shfl_xor_sync(0xffffffffu, res[r], off));
  }
  if (lane == 0) {
    const float eps = p.eps[row];
#pragma unroll
    for (int r = 0; r < kSketchMaxRanks; ++r)
      if (r < p.n_ranks)
        // rank k: the select's own bound (it also carries the global bound this shard already knew, which is as good a claim:
        // a threshold below a valid global bound is a valid global bound)
        p.out[static_cast<size_t>(row) * p.n_ranks + r] = p.ranks[r] == p.k ? p.kth_lb[row] : res[r] - eps;
  }
}

struct BoundParams {
  const float* sketches;  // [n_shards][n_query][n_ranks]
  int n_shards, n_query, n_ranks, k;
  int ranks[kSketchMaxRanks];
  float* bound;  // [n_query] in/out: max(bound, best threshold the sketches prove)
};

__global__ void __launch_bounds__(128) sketch_bound_kernel(const BoundParams p) {
  extern __shared__ float s_sk[];  // [4][n_shards * n_ranks]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * 4 + warp;
  if (row >= p.n_query) return;
  const int nc = p.n_shards * p.n_ranks;
  float* v = s_sk + warp * nc;
  for (int c = lane; c < nc; c += 32) {
    const int sh = c / p.n_ranks, i = c - sh * p.n_ranks;
    v[c] = p.sketches[(static_cast<size_t>(sh) * p.n_query + row) * p.n_ranks + i];
  }
  __syncwarp();
  float best = -INFINITY;
  for (int c = lane; c < nc; c += 32) {
    const float t = v[c];
    if (!(t > -INFINITY)) continue;
    int cnt = 0;
    for (int sh = 0; sh < p.n_shards; ++sh) {
      int cs = 0;
      for (int i = 0; i < p.n_ranks; ++i)
        if (v[sh * p.n_ranks + i] >= t) cs = max(cs, p.ranks[i]);
      cnt += cs;
    }
    if (cnt >= p.k) best = fmaxf(best, t);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) best = fmaxf(best, __shfl_xor_sync(0xffffffffu, best, off));
  if (lane == 0) p.bound[row] = fmaxf(p.bound[row], best);
}

static int topk_rerank(const vdk_topk_plan* plan, const float* q32, const float* g32, int64_t id_offset, const float* kth_lb_global,
                       float* out_scores, int64_t* out_ids, void* workspace, size_t workspace_bytes, cudaStream_t s) {
  int rc = check_plan(plan);
  if (rc != VDK_OK) return rc;
  VDK_REQUIRE(out_scores && out_ids, "vdk_ip_topk: null output");
  const int64_t nq = plan->n_query;
  if (nq == 0) return VDK_OK;
  VDK_REQUIRE(q32 && (g32 || plan->n_gallery == 0), "vdk_ip_topk: null fp32 rows");
  VDK_REQUIRE(workspace && workspace_bytes >= vdk_topk_workspace_bytes(plan), "vdk_ip_topk: workspace too small");
  const int carry_cap = plan->carry_capacity;
  const TopkWorkspace w = carve_workspace(workspace, nq, plan->cand_capacity, carry_cap);
  RerankParams rp{};
  rp.n_query = static_cast<int>(nq);
  rp.dim = plan->dim;
  rp.k = plan->k;
  rp.carry = w.carry[final_carry(plan)];
  rp.carry_cnt = w.carry_cnt;
  rp.carry_cap = carry_cap;
  rp.q32 = q32;
  rp.g32 = g32;
  rp.id_offset = id_offset;
  rp.out_scores = out_scores;
  rp.out_ids = out_ids;
  rp.kth_lb = kth_lb_global;
  rp.eps = w.eps;
  static bool rr_attr = false;
  if (!rr_attr) {  // carry_capacity up to 4096: 48 KB of sort keys + kept slots, above the default dynamic limit
    VDK_CUDA_OK(cudaFuncSetAttribute(rerank_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     4096 * static_cast<int>(sizeof(unsigned long long) + sizeof(uint32_t))));
    rr_attr = true;
  }
  rerank_kernel<<<static_cast<unsigned>(nq), kRerankThreads, carry_cap * (sizeof(unsigned long long) + sizeof(uint32_t)), s>>>(rp);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_ip_topk(const vdk_topk_plan* plan, const float* q32, const void* qh, const float* q_norm,
                           const float* q_err, const float* g32, const void* gh, const float* g_norm_max,
                           const float* g_err_max, int64_t id_offset, float* out_scores, int64_t* out_ids,
                           int32_t* status, void* workspace, size_t workspace_bytes, void* stream) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  VDK_REQUIRE(out_scores && out_ids && status, "vdk_ip_topk: null output");
  int rc = topk_filter(plan, qh, q_norm, q_err, gh, g_norm_max, g_err_max, status, workspace, workspace_bytes, s);
  if (rc != VDK_OK) return rc;
  return topk_rerank(plan, q32, g32, id_offset, nullptr, out_scores, out_ids, workspace, workspace_bytes, s);
}

extern "C" int vdk_ip_topk_filter(const vdk_topk_plan* plan, const void* qh, const float* q_norm, const float* q_err,
                                  const void* gh, const float* g_norm_max, const float* g_err_max, float* kth_lb_out,
                                  int32_t* status, void* workspace, size_t workspace_bytes, void* stream) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  int rc = topk_filter(plan, qh, q_norm, q_err, gh, g_norm_max, g_err_max, status, workspace, workspace_bytes, s);
  if (rc != VDK_OK) return rc;
  if (kth_lb_out && plan->n_query > 0) {
    const TopkWorkspace w = carve_workspace(workspace, plan->n_query, plan->cand_capacity, plan->carry_capacity);
    VDK_CUDA_OK(cudaMemcpyAsync(kth_lb_out, w.kth_lb, static_cast<size_t>(plan->n_query) * sizeof(float), cudaMemcpyDeviceToDevice, s));
  }
  return VDK_OK;
}

extern "C" int vdk_ip_topk_filter_stages(const vdk_topk_plan* plan, const void* qh, const float* q_norm, const float* q_err,
                                         const void* gh, const float* g_norm_max, const float* g_err_max, int stage_begin,
                                         int stage_end, const float* ext_lb, float* kth_lb_out, int32_t* status, void* workspace,
                                         size_t workspace_bytes, void* stream) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  int rc = topk_filter(plan, qh, q_norm, q_err, gh, g_norm_max, g_err_max, status, workspace, workspace_bytes, s, stage_begin,
                       stage_end, ext_lb);
  if (rc != VDK_OK) return rc;
  if (kth_lb_out && plan->n_query > 0) {
    const TopkWorkspace w = carve_workspace(workspace, plan->n_query, plan->cand_capacity, plan->carry_capacity);
    VDK_CUDA_OK(cudaMemcpyAsync(kth_lb_out, w.kth_lb, static_cast<size_t>(plan->n_query) * sizeof(float), cudaMemcpyDeviceToDevice, s));
  }
  return VDK_OK;
}

extern "C" int vdk_ip_topk_rerank(const vdk_topk_plan* plan, const float* q32, const float* g32, int64_t id_offset,
                                  const float* kth_lb_global, float* out_scores, int64_t* out_ids, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  return topk_rerank(plan, q32, g32, id_offset, kth_lb_global, out_scores, out_ids, workspace, workspace_bytes,
                     reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vdk_ip_topk_rank_sketch(const vdk_topk_plan* plan, int stages_done, const int32_t* ranks, int n_ranks,
                                       float* sketch_out, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_plan(plan);
  if (rc != VDK_OK) return rc;
  VDK_REQUIRE(ranks && sketch_out, "vdk_ip_topk_rank_sketch: null operand");
  VDK_REQUIRE(n_ranks >= 1 && n_ranks <= kSketchMaxRanks, "vdk_ip_topk_rank_sketch: n_ranks must be in [1,%d]", kSketchMaxRanks);
  VDK_REQUIRE(stages_done >= 1, "vdk_ip_topk_rank_sketch: no stage has run");
  const int64_t nq = plan->n_query;
  if (nq == 0) return VDK_OK;
  VDK_REQUIRE(workspace && workspace_bytes >= vdk_topk_workspace_bytes(plan), "vdk_ip_topk_rank_sketch: workspace too small");
  const TopkWorkspace w = carve_workspace(workspace, nq, plan->cand_capacity, plan->carry_capacity);
  SketchParams sp{};
  sp.n_query = static_cast<int>(nq);
  sp.k = plan->k;
  sp.n_ranks = n_ranks;
  for (int i = 0; i < n_ranks; ++i) {
    VDK_REQUIRE(ranks[i] >= 1 && ranks[i] <= plan->k, "vdk_ip_topk_rank_sketch: rank %d outside [1,k]", ranks[i]);
    sp.ranks[i] = ranks[i];
  }
  sp.carry = w.carry[carry_after(plan, stages_done)];
  sp.carry_cnt = w.carry_cnt;
  sp.carry_cap = plan->carry_capacity;
  sp.eps = w.eps;
  sp.kth_lb = w.kth_lb;
  sp.out = sketch_out;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  rank_sketch_kernel<<<static_cast<unsigned>((nq + 3) / 4), 128, 0, s>>>(sp);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_topk_bound_from_sketches(const float* sketches, int n_shards, int64_t n_query, const int32_t* ranks,
                                            int n_ranks, int k, float* bound_inout, void* stream) {
  VDK_REQUIRE(sketches && ranks && bound_inout, "vdk_topk_bound_from_sketches: null operand");
  VDK_REQUIRE(n_ranks >= 1 && n_ranks <= kSketchMaxRanks, "vdk_topk_bound_from_sketches: n_ranks must be in [1,%d]", kSketchMaxRanks);
  VDK_REQUIRE(n_shards >= 1 && n_shards <= 256 && k >= 1 && n_query >= 0, "vdk_topk_bound_from_sketches: n_shards must be in [1,256]");
  if (n_query == 0) return VDK_OK;
  BoundParams bp{};
  bp.sketches = sketches;
  bp.n_shards = n_shards;
  bp.n_query = static_cast<int>(n_query);
  bp.n_ranks = n_ranks;
  bp.k = k;
  for (int i = 0; i < n_ranks; ++i) bp.ranks[i] = ranks[i];
  bp.bound = bound_inout;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  sketch_bound_kernel<<<static_cast<unsigned>((n_query + 3) / 4), 128, 4 * n_shards * n_ranks * sizeof(float), s>>>(bp);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_topk_merge(const float* scores, const int64_t* ids, int n_lists, int64_t n_query, int k,
                              float* out_scores, int64_t* out_ids, void* stream) {
  VDK_REQUIRE(scores && ids && out_scores && out_ids, "vdk_topk_merge: null operand");
  VDK_REQUIRE(n_lists >= 1 && n_lists <= 32 && k >= 1 && n_query >= 0, "vdk_topk_merge: n_lists must be in [1,32]");
  if (n_query == 0) return VDK_OK;
  const int64_t blocks = (n_query + 7) / 8;
  topk_merge_kernel<<<static_cast<unsigned>(blocks), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      scores, ids, n_lists, n_query, k, out_scores, out_ids);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_topk_pack(const float* scores, const int64_t* ids, int64_t n, void* packed, void* stream) {
  VDK_REQUIRE(scores && ids && packed && n >= 0, "vdk_topk_pack: bad arguments");
  if (n == 0) return VDK_OK;
  topk_pack_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      scores, ids, n, reinterpret_cast<unsigned long long*>(packed));
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_topk_merge_packed(const void* packed, int n_lists, int64_t n_query, int k, float* out_scores,
                                     int64_t* out_ids, void* stream) {
  VDK_REQUIRE(packed && out_scores && out_ids, "vdk_topk_merge_packed: null operand");
  VDK_REQUIRE(n_lists >= 1 && n_lists <= 32 && k >= 1 && n_query >= 0, "vdk_topk_merge_packed: n_lists must be in [1,32]");
  if (n_query == 0) return VDK_OK;
  const int group = pow2_ceil(n_lists);
  const int64_t warps = (n_query + 32 / group - 1) / (32 / group);
  topk_merge_packed_kernel<<<static_cast<unsigned>((warps + 7) / 8), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const unsigned long long*>(packed), n_lists, group, n_query, k, out_scores, out_ids);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_ip_exact_pairs(const float* q32, const float* g32, int dim, const int64_t* qi, const int64_t* gi,
                                  int64_t n, float* out, void* stream) {
  VDK_REQUIRE(q32 && g32 && qi && gi && out && dim > 0 && n >= 0, "vdk_ip_exact_pairs: bad arguments");
  if (n == 0) return VDK_OK;
  const int64_t blocks = (n + 7) / 8;
  exact_pairs_kernel<<<static_cast<unsigned>(blocks), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      q32, g32, dim, qi, gi, n, out);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_score_range(const vdk_topk_plan* plan, const void* qh, const void* gh, int64_t lo, int64_t hi,
                               int dense, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_plan(plan);
  if (rc != VDK_OK) return rc;
  VDK_REQUIRE(qh && gh && workspace, "vdk_score_range: null operand");
  VDK_REQUIRE(workspace_bytes >= vdk_topk_workspace_bytes(plan), "vdk_score_range: workspace too small");
  VDK_REQUIRE(lo >= 0 && hi > lo && hi <= plan->n_gallery, "vdk_score_range: bad range");
  const TopkWorkspace w = carve_workspace(workspace, plan->n_query, plan->cand_capacity, plan->carry_capacity);
  CUtensorMap mq, mg;
  rc = make_tma_2d_16bit(&mq, qh, static_cast<uint64_t>(plan->n_query), plan->dim, plan->dim, kQM, kSBK);
  if (rc != VDK_OK) return rc;
  rc = make_tma_2d_16bit(&mg, gh, static_cast<uint64_t>(plan->n_gallery), plan->dim, plan->dim, kGN, kSBK);
  if (rc != VDK_OK) return rc;
  return launch_score_range(mq, mg, static_cast<int>(plan->n_query), plan->dim, lo, hi, dense != 0, w,
                            plan->cand_capacity, nullptr, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vdk_topk_row_flags(const vdk_topk_plan* plan, const void* workspace, size_t workspace_bytes,
                                  const int32_t** row_flags) {
  int rc = check_plan(plan);
  if (rc != VDK_OK) return rc;
  VDK_REQUIRE(workspace && row_flags && workspace_bytes >= vdk_topk_workspace_bytes(plan), "vdk_topk_row_flags: bad arguments");
  const TopkWorkspace w = carve_workspace(const_cast<void*>(workspace), plan->n_query, plan->cand_capacity, plan->carry_capacity);
  *row_flags = w.row_flag;
  return VDK_OK;
}

extern "C" size_t vdk_ip_topk_exhaustive_workspace_bytes(int64_t n_gallery) {
  return static_cast<size_t>(kExQ) * static_cast<size_t>(n_gallery > 0 ? n_gallery : 1) * sizeof(unsigned long long);
}

extern "C" int vdk_ip_topk_exhaustive(const float* q32, int64_t n_query, const float* g32, int64_t n_gallery, int dim, int k,
                                      int64_t id_offset, float* out_scores, int64_t* out_ids, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  VDK_REQUIRE(out_scores && out_ids, "vdk_ip_topk_exhaustive: null output");
  VDK_REQUIRE(n_query >= 0 && n_gallery >= 0 && n_gallery < (1ll << 32) && dim > 0, "vdk_ip_topk_exhaustive: bad sizes");
  VDK_REQUIRE(k >= 1 && k <= 1024, "vdk_ip_topk_exhaustive: k must be in [1,1024]");
  VDK_REQUIRE(static_cast<size_t>(kExQ) * dim * sizeof(float) <= 96 * 1024, "vdk_ip_topk_exhaustive: dim too large (%d)", dim);
  if (n_query == 0) return VDK_OK;
  VDK_REQUIRE(q32 && (g32 || n_gallery == 0), "vdk_ip_topk_exhaustive: null operand");
  VDK_REQUIRE(workspace && workspace_bytes >= vdk_ip_topk_exhaustive_workspace_bytes(n_gallery),
              "vdk_ip_topk_exhaustive: workspace too small");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(workspace);
  static bool attr = false;
  if (!attr) {
    VDK_CUDA_OK(cudaFuncSetAttribute(exhaustive_scores_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    attr = true;
  }
  for (int64_t q0 = 0; q0 < n_query; q0 += kExQ) {
    const int nq = static_cast<int>(std::min<int64_t>(kExQ, n_query - q0));
    if (n_gallery > 0) {
      const int blocks = static_cast<int>(std::min<int64_t>((n_gallery + 7) / 8, 8 * sm_count()));
      exhaustive_scores_kernel<<<blocks, 256, static_cast<size_t>(nq) * dim * sizeof(float), s>>>(
          q32 + q0 * dim, nq, g32, n_gallery, dim, keys);
      VDK_CUDA_OK(cudaGetLastError());
    }
    exhaustive_select_kernel<<<nq, kExThreads, 0, s>>>(keys, n_gallery, k, id_offset, out_scores + q0 * k, out_ids + q0 * k);
    VDK_CUDA_OK(cudaGetLastError());
  }
  return VDK_OK;
}
