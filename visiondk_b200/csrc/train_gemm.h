// train_gemm.h — the GEMM forms of the training paths (convnext_train.cu, vit_train.cu) on top of gemm_run.
#pragma once
#include <algorithm>

#include "vdk_host.h"

namespace vdk {

// dst[i] (+)= sum over slabs, fixed order (convnext_train.cu)
int launch_slab_reduce(const float* slabs, int n_slabs, size_t stride, int64_t n4, float* dst, int accumulate, cudaStream_t s);
// out[r, c] = bias[c] (0 when bias is null) + sum over slabs, fixed order: the split-K neck Linear (convnext_train.cu)
int launch_slab_reduce_bias(const float* slabs, int n_slabs, size_t stride, const float* bias, int rows, int cols, float* out,
                            cudaStream_t s);
// out[c] += sum_r x[r, c], one thread per column: the neck Linear's bias gradient over a small batch (convnext_train.cu)
int launch_col_sum_f32_small(const float* x, int rows, int cols, float* out, cudaStream_t s);

// split count for a weight-gradient GEMM (few output tiles, very long contraction): at least two, so that vdk_gemm
// takes its raw-partials output mode; every split stores its own fp32 slab, which a reduction kernel then adds in a
// fixed order (deterministic, and no atomics on the few hot output addresses).
inline int wgrad_splits(int M, int N, size_t K) {
  const int tiles = ((M + 127) / 128) * ((N + 255) / 256);
  const int want = std::max(2, (2 * sm_count()) / std::max(1, tiles));
  return vdk_gemm_effective_splits(static_cast<int>(K), want);
}
// the dW slabs [splits][M][N], then the column-sum slabs [splits][M] of a bias gradient
inline size_t wgrad_slab_bytes(int M, int N, size_t K) {
  return static_cast<size_t>(std::max(2, wgrad_splits(M, N, K))) * M * (static_cast<size_t>(N) + 1) * 4;
}

// one buffer of a train workspace: its byte offset, which the kernels index with, and its size (vdk_*_train_buffer)
struct WsRange {
  size_t off = 0, bytes = 0;
  operator size_t() const { return off; }
};

struct Gemm {
  cudaStream_t s;
  int run(const void* A, const void* B, void* D, int M, int N, int K, int lda, int ldb, int ldd, int epi, const float* bias,
          const float* gamma, const void* res, int ldr, int out_dtype, int split, long long stride, int ta, int tb,
          void* aux_out = nullptr, float* a_col_sums = nullptr) const {
    vdk_gemm_desc g{};
    g.A = A; g.B = B; g.D = D;
    g.M = M; g.N = N; g.K = K; g.lda = lda; g.ldb = ldb; g.ldd = ldd;
    g.in_dtype = VDK_DTYPE_BF16; g.out_dtype = out_dtype; g.epilogue = epi;
    g.bias = bias; g.gamma = gamma; g.residual = res; g.ldr = ldr;
    g.ln_eps = 1e-6f; g.split_k = split; g.split_stride = stride; g.trans_a = ta; g.trans_b = tb; g.aux_out = aux_out;
    g.a_col_sums = a_col_sums;
    return gemm_run(g, s);
  }
  // data gradient dY = A . B^T (B stored [K,N]) through a LayerNorm of width `group` whose saved output is y [M,N]:
  // dx = LayerNorm_backward(bf16(dY)) into D (wo > 0: the 2x2 patch rows of an image of width 2 wo, written to its NHWC
  // pixels), dgamma / dbeta +=.  slab: 2 N sm_count() floats of scratch.
  int ln_bwd(const void* A, const void* B, void* D, int M, int N, int K, const void* y, const float* rstd, const float* ln_w,
             const float* ln_b, int group, int wo, float* dgamma, float* dbeta, float* slab) const {
    vdk_gemm_desc g{};
    g.A = A; g.B = B; g.D = D;
    g.M = M; g.N = N; g.K = K; g.lda = K; g.ldb = N; g.ldd = N;
    g.in_dtype = VDK_DTYPE_BF16; g.out_dtype = VDK_DTYPE_BF16; g.epilogue = VDK_EPI_LN_BWD;
    g.gamma = ln_w; g.beta = ln_b; g.residual = y; g.ldr = N;
    g.split_k = 1; g.trans_b = 1;
    g.ln_rstd = rstd; g.ln_dgamma = dgamma; g.ln_dbeta = dbeta; g.ln_slab = slab; g.ln_group = group; g.ln_wo = wo;
    return gemm_run(g, s);
  }
  // weight gradient D[M,N] (+)= A^T B over a long K (A stored [K,M], B stored [K,N]): split-K partial slabs + fixed-order
  // reduction.  bias_grad (optional): += the column sums of A, sum_k A[k,m] (the bias gradient of the layer whose output
  // gradient A is), which the GEMM computes from the A tiles it streams and which are reduced over the splits the same way.
  int wgrad(const void* A, const void* B, float* D, int M, int N, int K, int lda, int ldb, float* slabs, bool accumulate,
            float* bias_grad = nullptr) const {
    VDK_REQUIRE((static_cast<size_t>(M) * N) % 4 == 0, "wgrad: M*N must be a multiple of 4");
    const int split = wgrad_splits(M, N, static_cast<size_t>(K));
    const size_t stride = static_cast<size_t>(M) * N;
    float* col_slabs = bias_grad ? slabs + static_cast<size_t>(split) * stride : nullptr;
    int rc = run(A, B, slabs, M, N, K, lda, ldb, N, VDK_EPI_NONE, nullptr, nullptr, nullptr, 0, VDK_DTYPE_FP32, std::max(2, split),
                 static_cast<long long>(stride), 1, 1, nullptr, col_slabs);
    if (rc != VDK_OK) return rc;
    rc = launch_slab_reduce(slabs, split, stride, static_cast<int64_t>(stride / 4), D, accumulate ? 1 : 0, s);
    if (rc != VDK_OK || !bias_grad) return rc;
    return launch_slab_reduce(col_slabs, split, static_cast<size_t>(M), M / 4, bias_grad, 1, s);
  }
};

#define RC(expr)                   \
  do {                             \
    int _rc = (expr);              \
    if (_rc != VDK_OK) return _rc; \
  } while (0)

}  // namespace vdk
