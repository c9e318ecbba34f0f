// topk_keys.cuh — the canonical fp64 score loop and the exact key selection shared by the exhaustive flat search
// (retrieval.cu) and the IVF list scans (ivf.cu).  The arithmetic is restated in oracle/retrieval.py; the two must
// agree bit for bit.
#pragma once
#include <cfloat>
#include <cstdint>

namespace vdk {

// Fixed-order fp64 dot: lane l accumulates elements l, l+32, ... in order, then a 16/8/4/2/1 xor butterfly.
// Products of two fp32 values are exact in fp64, so fma(a,b,acc) and acc + a*b round identically.
__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

__device__ __forceinline__ uint32_t ord_u32(float f) {  // order-preserving float -> uint32
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float unord_u32(uint32_t o) {
  const uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
  return __uint_as_float(u);
}

// Selection key of a (score, id) pair: larger key = better under (score desc, id asc).  Unique per id (id < 2^32).
__device__ __forceinline__ unsigned long long score_key(float s, uint32_t id) {
  return (static_cast<unsigned long long>(ord_u32(s)) << 32) | static_cast<unsigned long long>(~id);
}

constexpr int kExQ = 8;  // queries scored per pass over a gallery row

// Canonical scores of nq <= kExQ queries (shared memory, [nq][dim]) against the row g, computed by one warp.  Every lane
// returns all nq scores in out[0..nq).  nq must be uniform across the warp.
__device__ __forceinline__ void canonical_scores_x8(const float* qs, int nq, const float* __restrict__ g, int dim, int lane,
                                                    float (&out)[kExQ]) {
  double acc[kExQ];
#pragma unroll
  for (int j = 0; j < kExQ; ++j) acc[j] = 0.0;
  for (int i = lane; i < dim; i += 32) {  // the canonical order: lane l takes l, l+32, ... then the xor butterfly
    const double gv = static_cast<double>(g[i]);
#pragma unroll
    for (int j = 0; j < kExQ; ++j)
      if (j < nq) acc[j] = fma(static_cast<double>(qs[j * dim + i]), gv, acc[j]);
  }
#pragma unroll
  for (int j = 0; j < kExQ; ++j)
    if (j < nq) out[j] = static_cast<float>(warp_sum_f64(acc[j]));
}

constexpr int kExThreads = 1024;

// One CTA of kExThreads threads: the k best of n unique keys e[0..n) (score_key), written as (score desc, id asc) to
// out_scores / out_ids [k], padded with (-FLT_MAX, -1).  The k-th largest key is found exactly by an 8 x 8-bit radix
// select, and the survivors (exactly min(n, k) <= 1024 of them, keys being unique) are bitonic-sorted in shared memory.
__device__ __forceinline__ void select_topk_keys(const unsigned long long* __restrict__ e, int64_t ng, int k, int64_t id_offset,
                                                 float* __restrict__ out_scores, int64_t* __restrict__ out_ids) {
  __shared__ unsigned hist[256];
  __shared__ unsigned long long s_sort[1024];
  __shared__ unsigned s_bin, s_krem, s_m;
  const int tid = threadIdx.x;
  const int kk = static_cast<int>(ng < k ? ng : k);
  unsigned long long prefix = 0ull, mask = 0ull;
  unsigned k_rem = static_cast<unsigned>(kk);
  if (kk > 0 && ng > kk) {
    for (int shift = 56; shift >= 0; shift -= 8) {
      for (int i = tid; i < 256; i += kExThreads) hist[i] = 0;
      __syncthreads();
      for (int64_t i = tid; i < ng; i += kExThreads) {
        const unsigned long long key = e[i];
        if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255ull], 1u);
      }
      __syncthreads();
      if (tid == 0) {
        unsigned acc = 0;
        int b = 255;
        for (; b > 0; --b) {
          if (acc + hist[b] >= k_rem) break;
          acc += hist[b];
        }
        s_bin = static_cast<unsigned>(b);
        s_krem = k_rem - acc;
      }
      __syncthreads();
      prefix |= static_cast<unsigned long long>(s_bin) << shift;
      mask |= 255ull << shift;
      k_rem = s_krem;
      __syncthreads();
    }
  }
  // keys are unique: exactly kk keys are >= the k-th largest (prefix); with ng <= k every key survives (prefix = 0)
  if (tid == 0) s_m = 0;
  for (int i = tid; i < 1024; i += kExThreads) s_sort[i] = 0ull;
  __syncthreads();
  for (int64_t i = tid; i < ng; i += kExThreads) {
    const unsigned long long key = e[i];
    if (key >= prefix) {
      const unsigned pos = atomicAdd(&s_m, 1u);
      if (pos < 1024u) s_sort[pos] = key;
    }
  }
  __syncthreads();
  for (int size = 2; size <= 1024; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = tid; i < 512; i += kExThreads) {
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
  for (int j = tid; j < k; j += kExThreads) {
    float sc = -FLT_MAX;
    int64_t id = -1;
    if (j < kk) {
      const unsigned long long key = s_sort[j];
      sc = unord_u32(static_cast<uint32_t>(key >> 32));
      id = static_cast<int64_t>(~static_cast<uint32_t>(key & 0xffffffffull)) + id_offset;
    }
    out_scores[j] = sc;
    out_ids[j] = id;
  }
}

}  // namespace vdk
