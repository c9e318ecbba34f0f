// ivf.cu — inverted-file indexes for the CBIR path: IVF-Flat and IVF-PQ (8-bit codes by residual), inner product.
//
// The faiss index_factory strings "IVF<nlist>,Flat" and "IVF<nlist>,PQ<M>[x8]" of engine/cbir/evaluation.py:110,155.
// faiss is not vendored, so the arithmetic is ours, fixed-order and restated bit for bit in oracle/ivf.py:
//   kmeans_update   per-centroid fp64 sum of its members in ascending row order -> fp32(sum / count); empty clusters take
//                   a copy of the largest one, the two copies scaled by 1 +- 1/1024 on alternate dimensions
//   pq_encode       r = fl32(x - c); per sub-space argmin_j of the sequential fp64 sum of (r_t - cw_jt)^2, ties -> lowest j
//   pq_lut          LUT[m][j] = fp32(sequential fp64 sum of q_t * cw_jt)
//   ivf_flat_scan   one CTA per (list, <= 8 queries probing it): canonical scores (canonical_scores_x8) of the list's rows
//   ivf_pq_scan     one CTA per query, LUT in shared memory, one thread per code: s = coarse; s = fl32(s + LUT[m][code_m])
//   select          the exact (score desc, id asc) selection on 64-bit keys of the exhaustive flat path (select_topk_keys)
// Coarse assignment and probing use the flat index (vdk_ip_topk) over the centroids; list building is a stable sort.
#include "vdk_host.h"
#include "topk_keys.cuh"

#include <cfloat>
#include <cmath>

namespace vdk {

constexpr float kSplitEps = 1.0f / 1024.0f;

__global__ void __launch_bounds__(128) kmeans_update_kernel(const float* __restrict__ x, int64_t ld, int dim, int k,
                                                            const int64_t* __restrict__ order, const int64_t* __restrict__ offsets,
                                                            float* __restrict__ centroids) {
  const int g = blockIdx.x;
  const int s = g / k;
  const int64_t lo = offsets[g], hi = offsets[g + 1];
  if (hi == lo) return;  // empty: filled by the split
  const double cnt = static_cast<double>(hi - lo);
  for (int t = threadIdx.x; t < dim; t += blockDim.x) {
    double acc = 0.0;
    for (int64_t i = lo; i < hi; ++i) acc = __dadd_rn(acc, static_cast<double>(x[order[i] * ld + static_cast<int64_t>(s) * dim + t]));
    centroids[static_cast<int64_t>(g) * dim + t] = static_cast<float>(__ddiv_rn(acc, cnt));
  }
}

// One CTA per sub-space: empty clusters in ascending order each split the then-largest cluster (lowest index on ties).
__global__ void __launch_bounds__(256) kmeans_split_kernel(int dim, int k, int64_t* __restrict__ counts, float* __restrict__ centroids) {
  __shared__ int64_t s_val[256];
  __shared__ int s_idx[256];
  int64_t* cnt = counts + static_cast<int64_t>(blockIdx.x) * k;
  float* c = centroids + static_cast<int64_t>(blockIdx.x) * k * dim;
  const int tid = threadIdx.x;
  for (int ci = 0; ci < k; ++ci) {
    if (cnt[ci] != 0) continue;  // uniform: cnt was last written before a __syncthreads
    int64_t bv = -1;
    int bi = 0;
    for (int j = tid; j < k; j += blockDim.x)
      if (cnt[j] > bv) bv = cnt[j], bi = j;
    s_val[tid] = bv;
    s_idx[tid] = bi;
    __syncthreads();
    for (int w = blockDim.x / 2; w > 0; w >>= 1) {
      if (tid < w) {
        const int64_t ov = s_val[tid + w];
        const int oi = s_idx[tid + w];
        if (ov > s_val[tid] || (ov == s_val[tid] && oi < s_idx[tid])) s_val[tid] = ov, s_idx[tid] = oi;
      }
      __syncthreads();
    }
    const int cj = s_idx[0];
    for (int t = tid; t < dim; t += blockDim.x) {
      const float v = c[static_cast<int64_t>(cj) * dim + t];
      const float up = 1.0f + kSplitEps, down = 1.0f - kSplitEps;
      c[static_cast<int64_t>(ci) * dim + t] = __fmul_rn(v, (t & 1) ? down : up);
      c[static_cast<int64_t>(cj) * dim + t] = __fmul_rn(v, (t & 1) ? up : down);
    }
    __syncthreads();
    if (tid == 0) {
      cnt[ci] = cnt[cj] / 2;
      cnt[cj] -= cnt[ci];
    }
    __syncthreads();
  }
}

// One thread per (row, sub-space).  The codewords of a sub-space are read by every lane of a warp at once (broadcast).
__global__ void __launch_bounds__(256) pq_encode_kernel(const float* __restrict__ x, int64_t n, int d, const float* __restrict__ coarse,
                                                        const int64_t* __restrict__ list_of_row, int M,
                                                        const float* __restrict__ codebooks, float* __restrict__ residual,
                                                        uint8_t* __restrict__ codes) {
  const int64_t row = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int m = blockIdx.y;
  if (row >= n) return;
  const int dsub = d / M;
  const float* xr = x + row * d + m * dsub;
  const float* cr = coarse + list_of_row[row] * d + m * dsub;
  float* rr = residual + row * d + m * dsub;
  for (int t = 0; t < dsub; ++t) rr[t] = __fsub_rn(xr[t], cr[t]);
  double best = INFINITY;
  int bj = 0;
  for (int j = 0; j < 256; ++j) {
    const float* cw = codebooks + (static_cast<int64_t>(m) * 256 + j) * dsub;
    double acc = 0.0;
    for (int t = 0; t < dsub; ++t) {
      const double df = __dsub_rn(static_cast<double>(rr[t]), static_cast<double>(__ldg(cw + t)));
      acc = __dadd_rn(acc, __dmul_rn(df, df));
    }
    if (acc < best) best = acc, bj = j;
  }
  codes[row * M + m] = static_cast<uint8_t>(bj);
}

// One thread per (query, sub-space, codeword).
__global__ void __launch_bounds__(256) pq_lut_kernel(const float* __restrict__ q, int64_t nq, int d, int M,
                                                     const float* __restrict__ codebooks, float* __restrict__ lut) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= nq * M * 256) return;
  const int j = static_cast<int>(i & 255);
  const int m = static_cast<int>((i >> 8) % M);
  const int64_t qi = (i >> 8) / M;
  const int dsub = d / M;
  const float* qr = q + qi * d + m * dsub;
  const float* cw = codebooks + (static_cast<int64_t>(m) * 256 + j) * dsub;
  double acc = 0.0;
  for (int t = 0; t < dsub; ++t) acc = fma(static_cast<double>(qr[t]), static_cast<double>(cw[t]), acc);  // exact products
  lut[i] = static_cast<float>(acc);
}

constexpr int kScanThreads = 256;

// items[i] = {list, first pair, pair count <= kExQ}: the pairs [first, first + count) of the list-sorted (query, list) pairs.
__global__ void __launch_bounds__(kScanThreads) ivf_flat_scan_kernel(const float* __restrict__ q32, int dim, const int32_t* __restrict__ items,
                                                                     const int32_t* __restrict__ pair_query, const int64_t* __restrict__ pair_out,
                                                                     const int64_t* __restrict__ offsets, const float* __restrict__ rows,
                                                                     const int64_t* __restrict__ ids, unsigned long long* __restrict__ keys) {
  extern __shared__ float sq[];  // [nq][dim]
  __shared__ int64_t s_out[kExQ];
  const int list = items[3 * blockIdx.x], first = items[3 * blockIdx.x + 1], nq = items[3 * blockIdx.x + 2];
  for (int i = threadIdx.x; i < nq * dim; i += blockDim.x) {
    const int j = i / dim;
    sq[i] = q32[static_cast<int64_t>(pair_query[first + j]) * dim + (i - j * dim)];
  }
  if (threadIdx.x < nq) s_out[threadIdx.x] = pair_out[first + threadIdx.x];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t lo = offsets[list], n = offsets[list + 1] - lo;
  for (int64_t r = threadIdx.x >> 5; r < n; r += kScanThreads / 32) {
    float s[kExQ];
    canonical_scores_x8(sq, nq, rows + (lo + r) * dim, dim, lane, s);
    const uint32_t id = static_cast<uint32_t>(ids[lo + r]);
#pragma unroll
    for (int j = 0; j < kExQ; ++j)
      if (j < nq && lane == j) keys[s_out[j] + r] = score_key(s[j], id);
  }
}

__global__ void __launch_bounds__(kScanThreads) ivf_pq_scan_kernel(int nprobe, const int64_t* __restrict__ probe_lists,
                                                                   const float* __restrict__ probe_scores, const int64_t* __restrict__ pair_out,
                                                                   const int64_t* __restrict__ offsets, const uint8_t* __restrict__ codes, int M,
                                                                   const int64_t* __restrict__ ids, const float* __restrict__ lut,
                                                                   unsigned long long* __restrict__ keys) {
  extern __shared__ float s_lut[];  // [M][256]
  const int64_t q = blockIdx.x;
  const float4* src = reinterpret_cast<const float4*>(lut + q * M * 256);
  for (int i = threadIdx.x; i < M * 64; i += blockDim.x) reinterpret_cast<float4*>(s_lut)[i] = src[i];
  __syncthreads();
  for (int p = 0; p < nprobe; ++p) {
    const int64_t list = probe_lists[q * nprobe + p];
    if (list < 0) continue;
    const float coarse = probe_scores[q * nprobe + p];
    const int64_t lo = offsets[list], n = offsets[list + 1] - lo;
    unsigned long long* out = keys + pair_out[q * nprobe + p];
    for (int64_t r = threadIdx.x; r < n; r += blockDim.x) {
      const uint8_t* c = codes + (lo + r) * M;
      float s = coarse;
      if ((M & 3) == 0) {
        for (int m = 0; m < M; m += 4) {
          const uint32_t w = *reinterpret_cast<const uint32_t*>(c + m);
          s = __fadd_rn(s, s_lut[(m + 0) * 256 + (w & 255u)]);
          s = __fadd_rn(s, s_lut[(m + 1) * 256 + ((w >> 8) & 255u)]);
          s = __fadd_rn(s, s_lut[(m + 2) * 256 + ((w >> 16) & 255u)]);
          s = __fadd_rn(s, s_lut[(m + 3) * 256 + (w >> 24)]);
        }
      } else {
        for (int m = 0; m < M; ++m) s = __fadd_rn(s, s_lut[m * 256 + c[m]]);
      }
      out[r] = score_key(s, static_cast<uint32_t>(ids[lo + r]));
    }
  }
}

__global__ void __launch_bounds__(kExThreads) select_keys_kernel(const unsigned long long* __restrict__ keys,
                                                                 const int64_t* __restrict__ offsets, const int64_t* __restrict__ counts,
                                                                 int k, float* __restrict__ out_scores, int64_t* __restrict__ out_ids) {
  const int64_t q = blockIdx.x;
  select_topk_keys(keys + offsets[q], counts[q], k, 0, out_scores + q * k, out_ids + q * k);
}

}  // namespace vdk

using namespace vdk;

extern "C" int vdk_kmeans_update(const float* x, int64_t ld, int dim, int n_sub, int k, const int64_t* order, const int64_t* offsets,
                                 int64_t* counts, float* centroids, void* stream) {
  VDK_REQUIRE(x && order && offsets && counts && centroids, "vdk_kmeans_update: null operand");
  VDK_REQUIRE(dim > 0 && n_sub > 0 && k > 0 && ld >= static_cast<int64_t>(n_sub) * dim && static_cast<int64_t>(n_sub) * k < (1ll << 31),
              "vdk_kmeans_update: bad sizes (dim %d, n_sub %d, k %d, ld %lld)", dim, n_sub, k, static_cast<long long>(ld));
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  kmeans_update_kernel<<<n_sub * k, 128, 0, s>>>(x, ld, dim, k, order, offsets, centroids);
  VDK_CUDA_OK(cudaGetLastError());
  kmeans_split_kernel<<<n_sub, 256, 0, s>>>(dim, k, counts, centroids);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_pq_encode(const float* x, int64_t n, int d, const float* coarse, const int64_t* list_of_row, int M,
                             const float* codebooks, float* residual, uint8_t* codes, void* stream) {
  VDK_REQUIRE(d > 0 && M > 0 && M <= 128 && d % M == 0 && n >= 0, "vdk_pq_encode: bad sizes (d %d, M %d)", d, M);
  if (n == 0) return VDK_OK;
  VDK_REQUIRE(x && coarse && list_of_row && codebooks && residual && codes, "vdk_pq_encode: null operand");
  const dim3 grid(static_cast<unsigned>((n + 255) / 256), static_cast<unsigned>(M));
  pq_encode_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, n, d, coarse, list_of_row, M, codebooks, residual, codes);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_pq_lut(const float* q, int64_t n_query, int d, int M, const float* codebooks, float* lut, void* stream) {
  VDK_REQUIRE(d > 0 && M > 0 && M <= 128 && d % M == 0 && n_query >= 0, "vdk_pq_lut: bad sizes (d %d, M %d)", d, M);
  if (n_query == 0) return VDK_OK;
  VDK_REQUIRE(q && codebooks && lut, "vdk_pq_lut: null operand");
  const int64_t total = n_query * M * 256;
  pq_lut_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(q, n_query, d, M,
                                                                                                               codebooks, lut);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_ivf_flat_scan(const float* q32, int dim, const int32_t* items, int64_t n_items, const int32_t* pair_query,
                                 const int64_t* pair_out, const int64_t* list_offsets, const float* list_rows, const int64_t* list_ids,
                                 void* keys, void* stream) {
  VDK_REQUIRE(dim > 0 && static_cast<size_t>(kExQ) * dim * sizeof(float) <= 96 * 1024 && n_items >= 0 && n_items < (1ll << 31),
              "vdk_ivf_flat_scan: bad sizes (dim %d)", dim);
  if (n_items == 0) return VDK_OK;
  VDK_REQUIRE(q32 && items && pair_query && pair_out && list_offsets && list_rows && list_ids && keys, "vdk_ivf_flat_scan: null operand");
  static bool attr = false;
  if (!attr) {
    VDK_CUDA_OK(cudaFuncSetAttribute(ivf_flat_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    attr = true;
  }
  ivf_flat_scan_kernel<<<static_cast<unsigned>(n_items), kScanThreads, static_cast<size_t>(kExQ) * dim * sizeof(float),
                         reinterpret_cast<cudaStream_t>(stream)>>>(q32, dim, items, pair_query, pair_out, list_offsets, list_rows,
                                                                   list_ids, reinterpret_cast<unsigned long long*>(keys));
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_ivf_pq_scan(int64_t n_query, int nprobe, const int64_t* probe_lists, const float* probe_scores, const int64_t* pair_out,
                               const int64_t* list_offsets, const uint8_t* codes, int M, const int64_t* list_ids, const float* lut,
                               void* keys, void* stream) {
  VDK_REQUIRE(n_query >= 0 && n_query < (1ll << 31) && nprobe > 0 && M > 0 && M <= 128, "vdk_ivf_pq_scan: bad sizes (nprobe %d, M %d)",
              nprobe, M);
  if (n_query == 0) return VDK_OK;
  VDK_REQUIRE(probe_lists && probe_scores && pair_out && list_offsets && codes && list_ids && lut && keys, "vdk_ivf_pq_scan: null operand");
  static bool attr = false;
  if (!attr) {
    VDK_CUDA_OK(cudaFuncSetAttribute(ivf_pq_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 256 * 4));
    attr = true;
  }
  ivf_pq_scan_kernel<<<static_cast<unsigned>(n_query), kScanThreads, static_cast<size_t>(M) * 256 * sizeof(float),
                       reinterpret_cast<cudaStream_t>(stream)>>>(nprobe, probe_lists, probe_scores, pair_out, list_offsets, codes, M,
                                                                 list_ids, lut, reinterpret_cast<unsigned long long*>(keys));
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_topk_select_keys(const void* keys, const int64_t* offsets, const int64_t* counts, int64_t n_query, int k,
                                    float* out_scores, int64_t* out_ids, void* stream) {
  VDK_REQUIRE(k >= 1 && k <= 1024 && n_query >= 0 && n_query < (1ll << 31), "vdk_topk_select_keys: bad sizes (k %d)", k);
  if (n_query == 0) return VDK_OK;
  VDK_REQUIRE(keys && offsets && counts && out_scores && out_ids, "vdk_topk_select_keys: null operand");
  select_keys_kernel<<<static_cast<unsigned>(n_query), kExThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const unsigned long long*>(keys), offsets, counts, k, out_scores, out_ids);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}
