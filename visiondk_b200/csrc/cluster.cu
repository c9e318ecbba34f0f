// cluster.cu — DBSCAN with metric="cosine" over unit rows, without ever writing the Gram matrix.
//
// Replaces DBSCAN(eps, min_samples, metric="cosine").fit(X) of the reference's tools/clustering.py.  Semantics (DESIGN §3c,
// restated by oracle/cluster.py): j is a neighbour of i iff i == j or the canonical score s_ij >= T, where T is the least fp32
// score that scikit-learn's float32 distance test passes (computed on the host).  Three passes over 128 x 256 tiles of the Gram
// matrix, fp16 wgmma with fp32 accumulation fed by TMA, as in retrieval.cu's score kernel:
//   count   all rows x all rows, upper triangle: neighbour counts (a pair counts for both rows)
//   union   core x core, upper triangle: lock-free union-find, the larger root hooked under the smaller
//   border  non-core x core: atomicMin of the core neighbour's final label
// The tile epilogue decides a pair from the tensor-core score a when |a - T| exceeds retrieval's error bound eps_i; the pairs
// in between go to a boundary buffer and are decided by the canonical fp64 score.  A row band whose boundary pairs did not fit
// the buffer is redone (boundary pairs only, in column pieces small enough to fit), so no pair is ever left undecided.
#include "vdk_host.h"
#include "score_tile.cuh"
#include "topk_keys.cuh"

#include <algorithm>
#include <climits>
#include <cmath>
#include <vector>

namespace vdk {
namespace {

constexpr int kRM = kTileM;       // rows per tile (two consumer warpgroups of 64) = rows per band
constexpr int kCN = kTileN;       // columns per tile (wgmma N)
constexpr int kBK = kTileKB;      // K per smem block (128-byte swizzle row of fp16)
constexpr int kABlockBytes = kTileABlockBytes;
constexpr int kBStageBytes = kTileBStageBytes;
constexpr int kStages = kTileStages;
constexpr int kThreads = 384;     // producer warpgroup + two consumer warpgroups
constexpr int kLd = kTileStageLd; // fp32 pitch of the staged 128 x 64 chunk
constexpr int kMaxKB = 8;         // dim <= 512
constexpr int kTilesPerUnit = 16; // column tiles per CTA: the row block's A tile is loaded once per 4096 columns
// One CTA per (128-row block, 4096-column unit): the count pass launches ceil(n/128) * ceil(n/4096) CTAs, which must stay
// below 2^31.  2^25 - 4096 rows keeps it there (and every row and column index in int32).
constexpr int64_t kMaxRows = (1ll << 25) - 4096;

enum { kCount = 0, kUnion = 1, kBorder = 2 };

struct GramParams {
  int n_a, n_b, num_kb;
  int sym;                  // rows and columns are the same set: only pairs with column > row
  int rb0, ct0, ct1, n_cu;  // row blocks rb0 + blockIdx.x / n_cu, column tiles [ct0, ct1) in units of kTilesPerUnit
  int boundary_only;        // redo of an overflowed band: collect the boundary pairs, decide nothing else
  const int32_t* idx_a;     // local row -> global row (nullptr: identity)
  const float* hi;          // [n] global: a >= hi[i] -> neighbour
  const float* lo;          // [n] global: a < lo[i] -> not a neighbour
  int32_t* counts;          // count pass (global rows)
  int32_t* parent;          // union pass (core-local)
  const int32_t* clabel;    // border pass: label of a core-local column
  int32_t* labels;          // border pass (global rows)
  uint2* buf;               // boundary pairs {local row, local column}
  unsigned long long cap;
  unsigned long long* buf_cnt;  // appends attempted; > cap: some pairs were dropped
  int32_t* band_flag;       // [row blocks] set when a pair of the band was dropped
};

int gram_smem_bytes(int num_kb) {
  return num_kb * kABlockBytes + kStages * kBStageBytes + kRM * kLd * 4 + kCN * 4 + (2 * kStages + 1) * 8 + 1024;
}

// Union-find over core-local indices.  parent[x] <= x always: hooks put the larger root under the smaller and path halving
// only ever writes an ancestor, so a component's root is its smallest index.  Loads go through L2 (volatile): another SM's
// hook must be seen.
__device__ __forceinline__ int uf_find(int32_t* parent, int x) {
  volatile int32_t* par = parent;
  while (true) {
    const int p = par[x];
    if (p == x) return x;
    const int gp = par[p];
    if (gp != p) par[x] = gp;
    x = gp;
  }
}

__device__ __forceinline__ void uf_unite(int32_t* parent, int a, int b) {
  while (true) {
    a = uf_find(parent, a);
    b = uf_find(parent, b);
    if (a == b) return;
    if (a > b) {
      const int t = a;
      a = b;
      b = t;
    }
    const int old = atomicCAS(&parent[b], b, a);
    if (old == b) return;
    b = old;  // b stopped being a root: retry from what it was hooked under
  }
}

template <int kPass>
__global__ void __launch_bounds__(kThreads, 1)
gram_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const GramParams p) {
  const int rb = p.rb0 + static_cast<int>(blockIdx.x) / p.n_cu;
  int t_lo = p.ct0 + (static_cast<int>(blockIdx.x) % p.n_cu) * kTilesPerUnit;
  const int t_hi = min(t_lo + kTilesPerUnit, p.ct1);
  if (p.sym) t_lo = max(t_lo, rb * kRM / kCN);  // first column tile holding a column above the block's first row
  if (t_lo >= t_hi) return;  // CTA-uniform

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + p.num_kb * kABlockBytes;
  uint32_t* stage_sm = reinterpret_cast<uint32_t*>(smem_b + kStages * kBStageBytes);
  int32_t* s_col = reinterpret_cast<int32_t*>(stage_sm + kRM * kLd);  // [kCN] column counts of the tile
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_col + kCN);
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* a_full = empty_bar + kStages;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_a);
    prefetch_tensormap(&map_b);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);  // one arrival per consumer warp
    }
    mbar_init(a_full, 1);
    fence_mbar_init();
  }
  for (int i = threadIdx.x; i < kCN; i += kThreads) s_col[i] = 0;
  __syncthreads();

  if (threadIdx.x < 128) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(a_full, p.num_kb * kABlockBytes);
      for (int kb = 0; kb < p.num_kb; ++kb)
        tma_load_2d(smem_a + kb * kABlockBytes, &map_a, a_full, kb * kBK, rb * kRM, kEvictLast);
      int stage = 0;
      uint32_t phase = 0;
      tile_produce_b(smem_b, &map_b, full_bar, empty_bar, p.num_kb, 0, t_lo, t_hi, stage, phase);
    }
  } else {
    // ===================== consumers: 64 rows x 256 columns each, then the classification =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int ct = threadIdx.x - 128;
    const int cg = ct >> 7;
    const int wl = (ct >> 5) & 3, lane = ct & 31;
    const int frow = cg * 64 + wl * 16 + (lane >> 2);
    const int fcol = (lane & 3) * 2;
    const int erow = ct & 127, half = ct >> 7;
    const int row = rb * kRM + erow;
    const bool row_ok = row < p.n_a;
    const int grow = row_ok ? (p.idx_a ? p.idx_a[row] : row) : 0;
    const float hi = row_ok ? p.hi[grow] : INFINITY;
    const float lo = row_ok ? p.lo[grow] : INFINITY;
    int cnt = 0;
    int mlab = INT_MAX;
    int rroot = -1;
    int stage = 0;
    uint32_t phase = 0;
    float acc[kCN / 2];
    mbar_wait<true>(a_full, 0);
    for (int t = t_lo; t < t_hi; ++t) {
      tile_mma(acc, smem_a, smem_b, full_bar, empty_bar, p.num_kb, cg, lane, stage, phase);
#pragma unroll
      for (int cc = 0; cc < kCN / 64; ++cc) {
        tile_stage_chunk(stage_sm, acc, cc, frow, fcol);
        named_bar_sync(1, 256);
        // this thread's 32 columns of the chunk that are in (a >= hi) and in the band (lo <= a < hi), as bit masks; only their
        // set bits are walked (rare for sparse neighbourhoods)
        uint32_t in_mask = 0, band_mask = 0;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const float a = __uint_as_float(stage_sm[erow * kLd + half * 32 + j]);
          in_mask |= a >= hi ? 1u << j : 0u;
          band_mask |= (a >= lo && a < hi) ? 1u << j : 0u;
        }
        named_bar_sync(1, 256);
        if ((in_mask | band_mask) != 0u) {
          const int c0 = (cc * 2 + half) * 32;
          const int col0 = t * kCN + c0;
          const int nv = min(max(p.n_b - col0, 0), 32);              // columns past n_b
          uint32_t ok = nv == 32 ? 0xffffffffu : (1u << nv) - 1u;
          if (p.sym) {                                                 // columns at or left of the diagonal
            const int first = min(max(row - col0 + 1, 0), 32);
            ok &= first == 32 ? 0u : 0xffffffffu << first;
          }
          in_mask &= p.boundary_only ? 0u : ok;
          band_mask &= ok;
          while (in_mask) {
            const int j = __ffs(in_mask) - 1;
            in_mask &= in_mask - 1;
            const int col = col0 + j;
            if (kPass == kCount) {
              ++cnt;
              atomicAdd(&s_col[c0 + j], 1);
            } else if (kPass == kUnion) {
              // rroot: a root the row had, hence an ancestor of it for good.  If the column's current root is rroot the
              // edge is already inside one set: one find per edge instead of two, and no CAS, once a cluster is merged
              if (rroot < 0) rroot = uf_find(p.parent, row);
              const int cr = uf_find(p.parent, col);
              if (cr != rroot) {
                uf_unite(p.parent, rroot, cr);
                rroot = uf_find(p.parent, rroot);
              }
            } else {
              mlab = min(mlab, p.clabel[col]);
            }
          }
          while (band_mask) {
            const int j = __ffs(band_mask) - 1;
            band_mask &= band_mask - 1;
            const unsigned long long pos = atomicAdd(p.buf_cnt, 1ull);
            if (pos < p.cap) p.buf[pos] = make_uint2(static_cast<uint32_t>(row), static_cast<uint32_t>(col0 + j));
            else p.band_flag[rb] = 1;
          }
        }
      }
      if (kPass == kCount) {  // the tile's column counts, one global atomic per column
        named_bar_sync(1, 256);
        const int col = t * kCN + ct;
        const int v = s_col[ct];
        if (v != 0) {
          atomicAdd(&p.counts[col], v);
          s_col[ct] = 0;
        }
        named_bar_sync(1, 256);
      }
    }
    if (kPass == kCount && cnt != 0) atomicAdd(&p.counts[grow], cnt);
    if (kPass == kBorder && mlab != INT_MAX) atomicMin(&p.labels[grow], mlab);
  }
}

struct ResolveParams {
  const float* x32;
  int dim;
  float threshold;
  const uint2* buf;
  unsigned long long cap;
  const unsigned long long* buf_cnt;
  const int32_t* band_flag;  // nullptr: resolve every pair (a redo)
  const int32_t* idx_a;
  const int32_t* idx_b;
  int32_t* counts;
  int32_t* parent;
  const int32_t* clabel;
  int32_t* labels;
  unsigned long long* rechecked;
};

// Boundary pairs: one warp per pair, the canonical score of the two fp32 unit rows (topk_keys.cuh's fixed order).
template <int kPass>
__global__ void __launch_bounds__(256) resolve_kernel(const ResolveParams p) {
  const int lane = threadIdx.x & 31;
  const unsigned long long n = min(*p.buf_cnt, p.cap);
  const unsigned long long warps = (static_cast<unsigned long long>(gridDim.x) * blockDim.x) >> 5;
  unsigned local = 0;
  for (unsigned long long w = (static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; w < n; w += warps) {
    const uint2 e = p.buf[w];
    if (p.band_flag && p.band_flag[e.x / kRM]) continue;  // the band is redone as a whole
    const int ga = p.idx_a ? p.idx_a[e.x] : static_cast<int>(e.x);
    const int gb = p.idx_b ? p.idx_b[e.y] : static_cast<int>(e.y);
    float s[kExQ];
    canonical_scores_x8(p.x32 + static_cast<int64_t>(ga) * p.dim, 1, p.x32 + static_cast<int64_t>(gb) * p.dim, p.dim, lane, s);
    ++local;
    if (lane == 0 && s[0] >= p.threshold) {
      if (kPass == kCount) {
        atomicAdd(&p.counts[ga], 1);
        atomicAdd(&p.counts[gb], 1);
      } else if (kPass == kUnion) {
        uf_unite(p.parent, static_cast<int>(e.x), static_cast<int>(e.y));
      } else {
        atomicMin(&p.labels[ga], p.clabel[e.y]);
      }
    }
  }
  if (lane == 0 && local != 0) atomicAdd(p.rechecked, static_cast<unsigned long long>(local));
}

// Per-row decision band: |a - s| <= e_i for every column (retrieval's per-query bound, DESIGN §3, with the gallery maxima of
// the row norm and the fp16 rounding-error norm); a >= T + e_i proves s >= T, a < T - e_i proves s < T.
__global__ void bounds_kernel(const float* __restrict__ norm, const float* __restrict__ err, const float* __restrict__ norm_max,
                              const float* __restrict__ err_max, int n, float threshold, float* __restrict__ hi,
                              float* __restrict__ lo, int32_t* __restrict__ counts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float gn = *norm_max, ge = *err_max;
  const float qn = norm[i] + err[i];
  const float e = (err[i] * gn + qn * ge + 1.220703125e-4f /*2^-13*/ * qn * (gn + ge)) * 1.0001f + 1e-30f;
  hi[i] = __fadd_ru(threshold, e);
  lo[i] = __fsub_rd(threshold, e);
  counts[i] = 1;  // the row itself
}

// One CTA: stable split of [0, n) by a predicate into order[0, m) (true, ascending) and order[m, n) (false, ascending); m to
// *m_out.  kind 0: counts[i] >= min_samples (core rows); kind 1: parent[i] == i (roots), order then holds each root's rank.
constexpr int kScanThreads = 1024;
template <int kKind>
__global__ void __launch_bounds__(kScanThreads) split_kernel(const int32_t* __restrict__ v, int n, int min_samples,
                                                             int32_t* __restrict__ out, int32_t* __restrict__ m_out) {
  __shared__ int s_sum[kScanThreads];
  const int tid = threadIdx.x;
  const int per = (n + kScanThreads - 1) / kScanThreads;
  const int b0 = min(n, tid * per), b1 = min(n, b0 + per);
  auto pred = [&](int i) { return kKind == 0 ? v[i] >= min_samples : v[i] == i; };
  int c = 0;
  for (int i = b0; i < b1; ++i) c += pred(i) ? 1 : 0;
  s_sum[tid] = c;
  __syncthreads();
  for (int off = 1; off < kScanThreads; off <<= 1) {
    const int add = tid >= off ? s_sum[tid - off] : 0;
    __syncthreads();
    s_sum[tid] += add;
    __syncthreads();
  }
  const int total = s_sum[kScanThreads - 1];
  int t_pos = s_sum[tid] - c;
  int f_pos = total + (b0 - t_pos);
  for (int i = b0; i < b1; ++i) {
    if (kKind == 0) {
      if (pred(i)) out[t_pos++] = i;
      else out[f_pos++] = i;
    } else if (pred(i)) {
      out[i] = t_pos++;  // rank of root i
    }
  }
  if (tid == 0) *m_out = total;
}

// Gathered fp16 rows (order[0, n_core) the core rows, then the others) and the union-find's initial forest.
__global__ void gather_kernel(const __half* __restrict__ xh, const int32_t* __restrict__ order, int n, int dim, int n_core,
                              __half* __restrict__ xg, int32_t* __restrict__ parent, int32_t* __restrict__ labels) {
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int per_row = dim / 8;  // 16-byte vectors
  if (t >= static_cast<int64_t>(n) * per_row) return;
  const int r = static_cast<int>(t / per_row), c = static_cast<int>(t % per_row);
  const int g = order[r];
  reinterpret_cast<uint4*>(xg)[t] = reinterpret_cast<const uint4*>(xh)[static_cast<int64_t>(g) * per_row + c];
  if (c == 0) {
    if (r < n_core) parent[r] = r;
    labels[g] = INT_MAX;
  }
}

// The forest is final here and nothing writes it any more: each row walks READ-ONLY to its root (parent[x] < x off the root,
// so the walk ends).  Compressing in place instead would race: a halving store of another row's walk can land after a row
// stored its root and leave it pointing at a non-root, whose rank is undefined.
__global__ void core_labels_kernel(const int32_t* __restrict__ parent, const int32_t* __restrict__ rank,
                                   const int32_t* __restrict__ order, int n_core, int32_t* __restrict__ clabel,
                                   int32_t* __restrict__ labels) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_core) return;
  int r = i;
  for (int p = parent[r]; p != r; p = parent[r]) r = p;
  const int lab = rank[r];
  clabel[i] = lab;
  labels[order[i]] = lab;
}

__global__ void noise_kernel(int32_t* labels, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && labels[i] == INT_MAX) labels[i] = -1;
}

size_t align256(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }

struct Workspace {
  int32_t *order, *parent, *rank, *clabel, *band_flag;
  float *hi, *lo;
  __half* xg;
  uint2* buf;
  unsigned long long* u64;  // {buf_cnt, rechecked}
  int32_t* i32;             // {n_core, n_roots}
};

size_t workspace_size(int64_t n, int dim, int64_t cap, Workspace* w, uint8_t* base) {
  const size_t nn = static_cast<size_t>(n);
  const size_t bands = (nn + kRM - 1) / kRM;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    uint8_t* p = base ? base + off : nullptr;
    off += align256(bytes);
    return p;
  };
  uint8_t* order = take(nn * 4);
  uint8_t* parent = take(nn * 4);
  uint8_t* rank = take(nn * 4);
  uint8_t* clabel = take(nn * 4);
  uint8_t* band_flag = take(bands * 4);
  uint8_t* hi = take(nn * 4);
  uint8_t* lo = take(nn * 4);
  uint8_t* xg = take(nn * dim * 2);
  uint8_t* buf = take(static_cast<size_t>(cap) * sizeof(uint2));
  uint8_t* u64 = take(2 * sizeof(unsigned long long));
  uint8_t* i32 = take(2 * sizeof(int32_t));
  if (w) {
    w->order = reinterpret_cast<int32_t*>(order);
    w->parent = reinterpret_cast<int32_t*>(parent);
    w->rank = reinterpret_cast<int32_t*>(rank);
    w->clabel = reinterpret_cast<int32_t*>(clabel);
    w->band_flag = reinterpret_cast<int32_t*>(band_flag);
    w->hi = reinterpret_cast<float*>(hi);
    w->lo = reinterpret_cast<float*>(lo);
    w->xg = reinterpret_cast<__half*>(xg);
    w->buf = reinterpret_cast<uint2*>(buf);
    w->u64 = reinterpret_cast<unsigned long long*>(u64);
    w->i32 = reinterpret_cast<int32_t*>(i32);
  }
  return off;
}

// CUDA events around the phases and the Gram kernels (only when the caller asks for timing).
struct Timer {
  bool on;
  cudaStream_t s;
  std::vector<std::pair<int, std::pair<cudaEvent_t, cudaEvent_t>>> spans;  // slot: 0..3 phases, 4..6 Gram kernels
  cudaEvent_t begin(int) {
    if (!on) return nullptr;
    cudaEvent_t e;
    cudaEventCreate(&e);
    cudaEventRecord(e, s);
    return e;
  }
  void end(int slot, cudaEvent_t b) {
    if (!on) return;
    cudaEvent_t e;
    cudaEventCreate(&e);
    cudaEventRecord(e, s);
    spans.push_back({slot, {b, e}});
  }
  void collect(vdk_dbscan_stats* st) {
    for (auto& sp : spans) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, sp.second.first, sp.second.second);
      if (sp.first < 4) st->phase_ms[sp.first] += ms;
      else st->gram_ms[sp.first - 4] += ms;
      cudaEventDestroy(sp.second.first);
      cudaEventDestroy(sp.second.second);
    }
    spans.clear();
  }
};

struct PassSpec {
  int pass;
  const void* a;
  int n_a;
  const int32_t* idx_a;
  const void* b;
  int n_b;
  const int32_t* idx_b;
  bool sym;
};

int launch_gram(const PassSpec& ps, int dim, const Workspace& w, int32_t* counts, int32_t* labels, int64_t cap, int rb0, int n_rb,
                int ct0, int ct1, bool boundary_only, cudaStream_t s) {
  CUtensorMap ma, mb;
  int rc = make_tma_2d_16bit(&ma, ps.a, static_cast<uint64_t>(ps.n_a), dim, dim, kRM, kBK);
  if (rc != VDK_OK) return rc;
  rc = make_tma_2d_16bit(&mb, ps.b, static_cast<uint64_t>(ps.n_b), dim, dim, kCN, kBK);
  if (rc != VDK_OK) return rc;
  GramParams p{};
  p.n_a = ps.n_a;
  p.n_b = ps.n_b;
  p.num_kb = dim / kBK;
  p.sym = ps.sym ? 1 : 0;
  p.rb0 = rb0;
  p.ct0 = ct0;
  p.ct1 = ct1;
  p.n_cu = (ct1 - ct0 + kTilesPerUnit - 1) / kTilesPerUnit;
  p.boundary_only = boundary_only ? 1 : 0;
  p.idx_a = ps.idx_a;
  p.hi = w.hi;
  p.lo = w.lo;
  p.counts = counts;
  p.parent = w.parent;
  p.clabel = w.clabel;
  p.labels = labels;
  p.buf = w.buf;
  p.cap = static_cast<unsigned long long>(cap);
  p.buf_cnt = w.u64;
  p.band_flag = w.band_flag;
  const int64_t grid = static_cast<int64_t>(n_rb) * p.n_cu;
  VDK_REQUIRE(grid < (1ll << 31), "vdk_dbscan: too many tiles");
  const int smem = gram_smem_bytes(p.num_kb);
  ProfScope prof(kProfOther, 2.0 * dim * static_cast<double>(ps.n_a) * ps.n_b * (ps.sym ? 0.5 : 1.0), 0.0, s);
  if (ps.pass == kCount) gram_kernel<kCount><<<static_cast<unsigned>(grid), kThreads, smem, s>>>(ma, mb, p);
  else if (ps.pass == kUnion) gram_kernel<kUnion><<<static_cast<unsigned>(grid), kThreads, smem, s>>>(ma, mb, p);
  else gram_kernel<kBorder><<<static_cast<unsigned>(grid), kThreads, smem, s>>>(ma, mb, p);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

int launch_resolve(const PassSpec& ps, const float* x32, int dim, float threshold, const Workspace& w, int32_t* counts,
                   int32_t* labels, int64_t cap, bool redo, cudaStream_t s) {
  ResolveParams r{};
  r.x32 = x32;
  r.dim = dim;
  r.threshold = threshold;
  r.buf = w.buf;
  r.cap = static_cast<unsigned long long>(cap);
  r.buf_cnt = w.u64;
  r.band_flag = redo ? nullptr : w.band_flag;
  r.idx_a = ps.idx_a;
  r.idx_b = ps.idx_b;
  r.counts = counts;
  r.parent = w.parent;
  r.clabel = w.clabel;
  r.labels = labels;
  r.rechecked = w.u64 + 1;
  const int grid = 8 * sm_count();
  if (ps.pass == kCount) resolve_kernel<kCount><<<grid, 256, 0, s>>>(r);
  else if (ps.pass == kUnion) resolve_kernel<kUnion><<<grid, 256, 0, s>>>(r);
  else resolve_kernel<kBorder><<<grid, 256, 0, s>>>(r);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

// One pass over the whole Gram block, then the overflowed bands again, boundary pairs only, in column pieces that fit.
int run_pass(const PassSpec& ps, const float* x32, int dim, float threshold, const Workspace& w, int32_t* counts, int32_t* labels,
             int64_t cap, Timer& timer, int64_t* redone, cudaStream_t s) {
  if (ps.n_a == 0 || ps.n_b == 0) return VDK_OK;
  const int n_rb = (ps.n_a + kRM - 1) / kRM;
  const int n_ct = (ps.n_b + kCN - 1) / kCN;
  VDK_CUDA_OK(cudaMemsetAsync(w.u64, 0, sizeof(unsigned long long), s));
  VDK_CUDA_OK(cudaMemsetAsync(w.band_flag, 0, static_cast<size_t>(n_rb) * sizeof(int32_t), s));
  cudaEvent_t g0 = timer.begin(4 + ps.pass);
  int rc = launch_gram(ps, dim, w, counts, labels, cap, 0, n_rb, 0, n_ct, false, s);
  if (rc != VDK_OK) return rc;
  timer.end(4 + ps.pass, g0);
  rc = launch_resolve(ps, x32, dim, threshold, w, counts, labels, cap, false, s);
  if (rc != VDK_OK) return rc;
  unsigned long long appended = 0;
  VDK_CUDA_OK(cudaMemcpyAsync(&appended, w.u64, sizeof(appended), cudaMemcpyDeviceToHost, s));
  VDK_CUDA_OK(cudaStreamSynchronize(s));
  if (appended <= static_cast<unsigned long long>(cap)) return VDK_OK;
  std::vector<int32_t> flags(n_rb);
  VDK_CUDA_OK(cudaMemcpy(flags.data(), w.band_flag, flags.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
  for (int b = 0; b < n_rb; ++b) {
    if (!flags[b]) continue;
    ++*redone;
    std::vector<std::pair<int, int>> pieces{{ps.sym ? b * kRM / kCN : 0, n_ct}};
    while (!pieces.empty()) {
      const auto pc = pieces.back();
      pieces.pop_back();
      VDK_CUDA_OK(cudaMemsetAsync(w.u64, 0, sizeof(unsigned long long), s));
      cudaEvent_t r0 = timer.begin(4 + ps.pass);
      rc = launch_gram(ps, dim, w, counts, labels, cap, b, 1, pc.first, pc.second, true, s);
      if (rc != VDK_OK) return rc;
      timer.end(4 + ps.pass, r0);
      VDK_CUDA_OK(cudaMemcpyAsync(&appended, w.u64, sizeof(appended), cudaMemcpyDeviceToHost, s));
      VDK_CUDA_OK(cudaStreamSynchronize(s));
      if (appended > static_cast<unsigned long long>(cap)) {
        // a single tile holds kRM x kCN <= cap pairs, so halving always ends
        const int mid = pc.first + (pc.second - pc.first) / 2;
        pieces.push_back({mid, pc.second});
        pieces.push_back({pc.first, mid});
        continue;
      }
      rc = launch_resolve(ps, x32, dim, threshold, w, counts, labels, cap, true, s);
      if (rc != VDK_OK) return rc;
    }
  }
  return VDK_OK;
}

}  // namespace
}  // namespace vdk

using namespace vdk;

extern "C" size_t vdk_dbscan_workspace_bytes(int64_t n, int dim, int64_t boundary_capacity) {
  if (n < 1 || n > kMaxRows || dim < kBK || dim > kBK * kMaxKB || dim % kBK != 0 || boundary_capacity < kRM * kCN)
    return 0;
  return workspace_size(n, dim, boundary_capacity, nullptr, nullptr);
}

extern "C" int vdk_dbscan(const float* x32, const void* xh, const float* row_norm, const float* row_err, const float* norm_max,
                          const float* err_max, int64_t n, int dim, float threshold, int min_samples, int64_t boundary_capacity,
                          int32_t* labels, int32_t* counts, vdk_dbscan_stats* stats, int timing, void* workspace,
                          size_t workspace_bytes, void* stream) {
  VDK_REQUIRE(x32 && xh && row_norm && row_err && norm_max && err_max, "vdk_dbscan: null row operand");
  VDK_REQUIRE(labels && counts && stats, "vdk_dbscan: null output");
  VDK_REQUIRE(n >= 1 && n <= kMaxRows, "vdk_dbscan: n must be in [1, %lld] (got %lld)", (long long)kMaxRows, (long long)n);
  VDK_REQUIRE(dim >= kBK && dim <= kBK * kMaxKB && dim % kBK == 0, "vdk_dbscan: dim must be a multiple of 64, <= 512 (got %d)", dim);
  VDK_REQUIRE(min_samples >= 1, "vdk_dbscan: min_samples must be >= 1 (got %d)", min_samples);
  VDK_REQUIRE(!std::isnan(threshold), "vdk_dbscan: threshold is NaN");
  VDK_REQUIRE(boundary_capacity >= kRM * kCN, "vdk_dbscan: boundary_capacity must be >= %d pairs (one tile)", kRM * kCN);
  const size_t need = workspace_size(n, dim, boundary_capacity, nullptr, nullptr);
  VDK_REQUIRE(workspace && workspace_bytes >= need, "vdk_dbscan: workspace too small (%zu < %zu bytes)", workspace_bytes, need);
  VDK_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "vdk_dbscan: workspace must be 256-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  static bool attr = false;
  if (!attr) {
    VDK_CUDA_OK(cudaFuncSetAttribute(gram_kernel<kCount>, cudaFuncAttributeMaxDynamicSharedMemorySize, gram_smem_bytes(kMaxKB)));
    VDK_CUDA_OK(cudaFuncSetAttribute(gram_kernel<kUnion>, cudaFuncAttributeMaxDynamicSharedMemorySize, gram_smem_bytes(kMaxKB)));
    VDK_CUDA_OK(cudaFuncSetAttribute(gram_kernel<kBorder>, cudaFuncAttributeMaxDynamicSharedMemorySize, gram_smem_bytes(kMaxKB)));
    attr = true;
  }
  *stats = vdk_dbscan_stats{};
  Workspace w;
  workspace_size(n, dim, boundary_capacity, &w, reinterpret_cast<uint8_t*>(workspace));
  const int nn = static_cast<int>(n);
  const int blocks = (nn + 255) / 256;
  Timer timer{timing != 0, s, {}};
  int rc;

  // ---- count ----
  cudaEvent_t t0 = timer.begin(0);
  VDK_CUDA_OK(cudaMemsetAsync(w.u64 + 1, 0, sizeof(unsigned long long), s));
  bounds_kernel<<<blocks, 256, 0, s>>>(row_norm, row_err, norm_max, err_max, nn, threshold, w.hi, w.lo, counts);
  VDK_CUDA_OK(cudaGetLastError());
  const PassSpec count_pass{kCount, xh, nn, nullptr, xh, nn, nullptr, true};
  rc = run_pass(count_pass, x32, dim, threshold, w, counts, labels, boundary_capacity, timer, &stats->redone_bands, s);
  if (rc != VDK_OK) return rc;
  timer.end(0, t0);

  // ---- union ----
  cudaEvent_t t1 = timer.begin(1);
  split_kernel<0><<<1, kScanThreads, 0, s>>>(counts, nn, min_samples, w.order, w.i32);
  VDK_CUDA_OK(cudaGetLastError());
  int32_t n_core = 0;
  VDK_CUDA_OK(cudaMemcpyAsync(&n_core, w.i32, sizeof(n_core), cudaMemcpyDeviceToHost, s));
  VDK_CUDA_OK(cudaStreamSynchronize(s));
  const int64_t vec = n * (dim / 8);
  gather_kernel<<<static_cast<unsigned>((vec + 255) / 256), 256, 0, s>>>(reinterpret_cast<const __half*>(xh), w.order, nn, dim,
                                                                          n_core, w.xg, w.parent, labels);
  VDK_CUDA_OK(cudaGetLastError());
  const PassSpec union_pass{kUnion, w.xg, n_core, w.order, w.xg, n_core, w.order, true};
  rc = run_pass(union_pass, x32, dim, threshold, w, counts, labels, boundary_capacity, timer, &stats->redone_bands, s);
  if (rc != VDK_OK) return rc;
  timer.end(1, t1);

  // ---- finalise (components -> labels numbered by their smallest core index) ----
  cudaEvent_t t2 = timer.begin(3);
  int32_t n_roots = 0;
  if (n_core > 0) {
    split_kernel<1><<<1, kScanThreads, 0, s>>>(w.parent, n_core, 0, w.rank, w.i32 + 1);
    VDK_CUDA_OK(cudaGetLastError());
    core_labels_kernel<<<(n_core + 255) / 256, 256, 0, s>>>(w.parent, w.rank, w.order, n_core, w.clabel, labels);
    VDK_CUDA_OK(cudaGetLastError());
    VDK_CUDA_OK(cudaMemcpyAsync(&n_roots, w.i32 + 1, sizeof(n_roots), cudaMemcpyDeviceToHost, s));
  }
  timer.end(3, t2);

  // ---- border ----
  cudaEvent_t t3 = timer.begin(2);
  const PassSpec border_pass{kBorder, w.xg + static_cast<int64_t>(n_core) * dim, nn - n_core, w.order + n_core, w.xg, n_core,
                             w.order, false};
  rc = run_pass(border_pass, x32, dim, threshold, w, counts, labels, boundary_capacity, timer, &stats->redone_bands, s);
  if (rc != VDK_OK) return rc;
  timer.end(2, t3);

  cudaEvent_t t4 = timer.begin(3);
  noise_kernel<<<blocks, 256, 0, s>>>(labels, nn);
  VDK_CUDA_OK(cudaGetLastError());
  timer.end(3, t4);
  unsigned long long rechecked = 0;
  VDK_CUDA_OK(cudaMemcpyAsync(&rechecked, w.u64 + 1, sizeof(rechecked), cudaMemcpyDeviceToHost, s));
  VDK_CUDA_OK(cudaStreamSynchronize(s));
  stats->n_core = n_core;
  stats->n_clusters = n_roots;
  stats->rechecked_pairs = static_cast<int64_t>(rechecked);
  timer.collect(stats);
  return VDK_OK;
}
