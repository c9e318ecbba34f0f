// optim.cu — the optimizer half of the faceX train step as two HBM-bound sweeps over flat fp32 buffers.
//
// Replaces Trainer.update (engine/procedure/train.py:203-215): clip_grad_norm_(max_norm=10) -> SGD(momentum,
// weight_decay) step (engine/optimizer.py:119-121 = torch.optim.SGD) -> optimizer.zero_grad() -> ModelEMA.update
// (models/ema.py:28-37), which the reference runs as ~1400 small ATen launches per step (GradScaler is a no-op in
// fp32).  Here: one reduction (sum of squared gradients, deterministic two-level order) and one fused update pass
// that reads p, g, momentum, ema and writes p, momentum, ema, g(=0): 32 bytes per parameter.
#include "vdk_host.h"

#include <cuda_runtime.h>

namespace vdk {

constexpr int kRedThreads = 256;
constexpr int kRedBlocksMax = 1184;  // fixed partial count: the order of the final sum does not depend on the device

__global__ void __launch_bounds__(kRedThreads) sumsq_partial_kernel(const float* __restrict__ g, int64_t n,
                                                                     double* __restrict__ partial) {
  // fixed assignment of elements to threads and a fixed in-block tree: bitwise reproducible run to run
  double s = 0.0;
  const int64_t n4 = n / 4;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kRedThreads + threadIdx.x; i < n4;
       i += static_cast<int64_t>(gridDim.x) * kRedThreads) {
    const float4 v = g4[i];
    s += static_cast<double>(v.x) * v.x + static_cast<double>(v.y) * v.y + static_cast<double>(v.z) * v.z +
         static_cast<double>(v.w) * v.w;
  }
  if (blockIdx.x == 0 && threadIdx.x < static_cast<int>(n - n4 * 4)) {
    const float v = g[n4 * 4 + threadIdx.x];
    s += static_cast<double>(v) * v;
  }
  __shared__ double red[kRedThreads];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int off = kRedThreads / 2; off > 0; off >>= 1) {
    if (threadIdx.x < off) red[threadIdx.x] += red[threadIdx.x + off];
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[blockIdx.x] = red[0];
}

__global__ void sumsq_final_kernel(const double* __restrict__ partial, int nblocks, double* __restrict__ acc, int accumulate) {
  __shared__ double red[kRedThreads];
  double s = 0.0;
  for (int i = threadIdx.x; i < nblocks; i += kRedThreads) s += partial[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int off = kRedThreads / 2; off > 0; off >>= 1) {
    if (threadIdx.x < off) red[threadIdx.x] += red[threadIdx.x + off];
    __syncthreads();
  }
  if (threadIdx.x == 0) *acc = (accumulate ? *acc : 0.0) + red[0];
}

struct StepArgs {
  float* p;
  float* g;
  float* mom;
  float* ema;  // may be null
  int64_t n;
  const double* total_sumsq;  // device scalar: sum of squared gradients over ALL parameters (all groups)
  float max_norm, lr, momentum, weight_decay, ema_decay, ema_one_minus_decay;
  int first_step, zero_grad;
};

__global__ void __launch_bounds__(256) sgd_clip_ema_kernel(const StepArgs a) {
  // torch.nn.utils.clip_grad_norm_: coef = max_norm / (total_norm + 1e-6), clamped to 1
  const float total_norm = static_cast<float>(sqrt(*a.total_sumsq));
  const float coef = fminf(a.max_norm / (total_norm + 1e-6f), 1.0f);
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < a.n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float p = a.p[i];
    float g = a.g[i] * coef;
    if (a.weight_decay != 0.f) g = fmaf(a.weight_decay, p, g);  // torch SGD: grad = grad + wd * param
    float buf = a.first_step ? g : fmaf(a.momentum, a.mom[i], g);
    if (a.momentum == 0.f) buf = g;
    p = fmaf(-a.lr, buf, p);
    a.p[i] = p;
    a.mom[i] = buf;
    // ema.py:35-36: v *= d; v += (1-d) * msd[k]  (three separately rounded fp32 operations, as in the reference)
    if (a.ema) a.ema[i] = __fadd_rn(__fmul_rn(a.ema[i], a.ema_decay), __fmul_rn(a.ema_one_minus_decay, p));
    if (a.zero_grad) a.g[i] = 0.f;
  }
}

__global__ void __launch_bounds__(256) ema_only_kernel(float* __restrict__ ema, const float* __restrict__ src, int64_t n, float d,
                                                       float omd) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    ema[i] = __fadd_rn(__fmul_rn(ema[i], d), __fmul_rn(omd, src[i]));
}

}  // namespace vdk

using namespace vdk;

extern "C" size_t vdk_grad_sumsq_workspace_bytes(void) { return kRedBlocksMax * sizeof(double); }

extern "C" int vdk_grad_sumsq(const float* grads, int64_t n, double* total_sumsq, int accumulate, void* workspace,
                              size_t workspace_bytes, void* stream) {
  VDK_REQUIRE(grads && total_sumsq && n >= 0, "vdk_grad_sumsq: bad arguments");
  VDK_REQUIRE(workspace && workspace_bytes >= vdk_grad_sumsq_workspace_bytes(), "vdk_grad_sumsq: workspace too small");
  VDK_REQUIRE((reinterpret_cast<uintptr_t>(grads) & 15) == 0, "vdk_grad_sumsq: grads must be 16-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int blocks = static_cast<int>(std::max<int64_t>(1, std::min<int64_t>((n / 4 + kRedThreads - 1) / kRedThreads, kRedBlocksMax)));
  sumsq_partial_kernel<<<blocks, kRedThreads, 0, s>>>(grads, n, reinterpret_cast<double*>(workspace));
  sumsq_final_kernel<<<1, kRedThreads, 0, s>>>(reinterpret_cast<double*>(workspace), blocks, total_sumsq, accumulate);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_sgd_clip_ema_step(float* params, float* grads, float* momentum_buf, float* ema, int64_t n,
                                     const double* total_sumsq, float max_norm, float lr, float momentum,
                                     float weight_decay, int first_step, float ema_decay, float ema_one_minus_decay,
                                     int zero_grad, void* stream) {
  VDK_REQUIRE(params && grads && momentum_buf && total_sumsq && n >= 0, "vdk_sgd_clip_ema_step: null operand");
  VDK_REQUIRE(max_norm > 0.f && lr >= 0.f, "vdk_sgd_clip_ema_step: bad hyper-parameters");
  if (n == 0) return VDK_OK;
  StepArgs a{params, grads, momentum_buf, ema, n, total_sumsq, max_norm, lr, momentum, weight_decay, ema_decay,
             ema_one_minus_decay, first_step, zero_grad};
  const int blocks = static_cast<int>(std::min<int64_t>((n + 255) / 256, 132 * 16));
  sgd_clip_ema_kernel<<<blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

extern "C" int vdk_ema_update(float* ema, const float* src, int64_t n, float decay, float one_minus_decay, void* stream) {
  VDK_REQUIRE(ema && src && n >= 0, "vdk_ema_update: null operand");
  if (n == 0) return VDK_OK;
  const int blocks = static_cast<int>(std::min<int64_t>((n + 255) / 256, 132 * 16));
  ema_only_kernel<<<blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(ema, src, n, decay, one_minus_decay);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}
