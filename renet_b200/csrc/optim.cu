// Optimiser step of the reference training loop on flat parameter / gradient buffers
// (reference train.py:140-142: clip_grad_norm_(parameters, grad_norm) -> Adam(lr, weight_decay).step()).
//
// The data-parallel engine (renet_b200/parallel.py) keeps every parameter and every gradient of the model as a view
// into one flat fp32 buffer each (the gradient buffer is what NCCL all-reduces), so the whole optimiser step is two
// HBM-bound launches over 20.2 M floats instead of ~17 x 6 foreach launches:
//   grad_sumsq_kernel : sum of squares of the (already all-reduced) gradient -> one device float (fixed-order
//                       two-level reduction, no float atomics: reproducible)
//   adam_step_kernel  : clip coefficient from that float (torch.nn.utils.clip_grad_norm_: max_norm / (norm + 1e-6),
//                       clamped to 1), L2 weight decay folded into the gradient (torch.optim.Adam, not AdamW),
//                       bias-corrected moments, in-place parameter update.  7 x 4 bytes of traffic per parameter.
#include <math.h>

#include "common.cuh"

namespace renet {
namespace {

constexpr int kRedThreads = 256;
constexpr int kRedBlocks = 592;   // 4 CTAs per SM

__global__ void __launch_bounds__(kRedThreads)
grad_sumsq_partial_kernel(const float* __restrict__ g, int64_t n, float* __restrict__ partial) {
  const int64_t n4 = n >> 2;
  float s = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * kRedThreads + threadIdx.x; i < n4; i += (int64_t)gridDim.x * kRedThreads) {
    const float4 v = ldg_f4(g + 4 * i);
    s = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, fmaf(v.w, v.w, s))));
  }
  if (blockIdx.x == 0)
    for (int64_t i = 4 * n4 + threadIdx.x; i < n; i += kRedThreads) s = fmaf(g[i], g[i], s);
  __shared__ float sm[kRedThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < kRedThreads / 32; ++w) t += sm[w];
    partial[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(1024)
grad_sumsq_final_kernel(const float* __restrict__ partial, int nblk, float* __restrict__ out, int accumulate) {
  __shared__ float sm[32];
  float s = 0.f;
  for (int i = threadIdx.x; i < nblk; i += 1024) s += partial[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = sm[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0) out[0] = accumulate ? out[0] + t : t;
  }
}

struct AdamArgs {
  float lr, beta1, beta2, eps, weight_decay, bc1, bc2_sqrt, max_norm, grad_scale;
};

__device__ __forceinline__ float adam_one(float& p, float g, float& m, float& v, const AdamArgs& a, float coef) {
  g = fmaf(a.weight_decay, p, g * coef);
  m = fmaf(a.beta1, m, (1.f - a.beta1) * g);
  v = fmaf(a.beta2, v, (1.f - a.beta2) * g * g);
  const float denom = sqrtf(v) / a.bc2_sqrt + a.eps;
  p -= (a.lr / a.bc1) * (m / denom);
  return p;
}

__global__ void __launch_bounds__(256)
adam_step_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                 int64_t n, AdamArgs a, const float* __restrict__ sumsq) {
  float coef = a.grad_scale;
  if (sumsq != nullptr && a.max_norm > 0.f) {
    const float norm = sqrtf(__ldg(sumsq)) * a.grad_scale;
    coef *= fminf(1.f, a.max_norm / (norm + 1e-6f));
  }
  const int64_t n4 = n >> 2;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n4; i += (int64_t)gridDim.x * 256) {
    float4 pp = *reinterpret_cast<const float4*>(p + 4 * i), mm = *reinterpret_cast<const float4*>(m + 4 * i),
           vv = *reinterpret_cast<const float4*>(v + 4 * i);
    const float4 gg = ldg_f4(g + 4 * i);
    adam_one(pp.x, gg.x, mm.x, vv.x, a, coef); adam_one(pp.y, gg.y, mm.y, vv.y, a, coef);
    adam_one(pp.z, gg.z, mm.z, vv.z, a, coef); adam_one(pp.w, gg.w, mm.w, vv.w, a, coef);
    st_f4(p + 4 * i, pp); st_f4(m + 4 * i, mm); st_f4(v + 4 * i, vv);
  }
  if (blockIdx.x == 0)
    for (int64_t i = 4 * n4 + threadIdx.x; i < n; i += 256) adam_one(p[i], g[i], m[i], v[i], a, coef);
}

}  // namespace
}  // namespace renet

using namespace renet;

extern "C" {

int64_t renet_grad_sumsq_workspace_bytes(void) { return kRedBlocks * (int64_t)sizeof(float); }

int renet_grad_sumsq(const float* grad, int64_t n, float* out, int32_t accumulate, void* workspace,
                     int64_t workspace_bytes, void* stream) {
  RENET_CHECK_ARG(n >= 0 && out != nullptr, "renet_grad_sumsq: bad arguments");
  RENET_CHECK_ARG(n == 0 || (grad != nullptr && workspace != nullptr && workspace_bytes >= renet_grad_sumsq_workspace_bytes()),
                  "renet_grad_sumsq: null pointer / workspace too small");
  RENET_CHECK_ARG((reinterpret_cast<uintptr_t>(grad) & 15) == 0, "renet_grad_sumsq: grad must be 16-byte aligned");
  // n == 0 may come with a NULL workspace: no partial block runs, and the final kernel (nblk = 0) writes 0 or keeps out
  int64_t want = (n / 4 + kRedThreads - 1) / kRedThreads;
  const int nblk = n == 0 ? 0 : (int)(want < 1 ? 1 : (want > kRedBlocks ? kRedBlocks : want));
  if (nblk > 0) {
    grad_sumsq_partial_kernel<<<nblk, kRedThreads, 0, (cudaStream_t)stream>>>(grad, n, (float*)workspace);
    RENET_CHECK_LAUNCH("grad_sumsq_partial_kernel");
  }
  grad_sumsq_final_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>((const float*)workspace, nblk, out, accumulate);
  RENET_CHECK_LAUNCH("grad_sumsq_final_kernel");
  return RENET_OK;
}

int renet_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                    float beta1, float beta2, float eps, float weight_decay, int64_t step, const float* sumsq,
                    float max_norm, float grad_scale, void* stream) {
  RENET_CHECK_ARG(n >= 0 && step >= 1, "renet_adam_step: bad arguments (step counts from 1)");
  if (n == 0) return RENET_OK;
  RENET_CHECK_ARG(param && grad && exp_avg && exp_avg_sq, "renet_adam_step: null pointer");
  RENET_CHECK_ARG(((reinterpret_cast<uintptr_t>(param) | reinterpret_cast<uintptr_t>(grad) |
                    reinterpret_cast<uintptr_t>(exp_avg) | reinterpret_cast<uintptr_t>(exp_avg_sq)) & 15) == 0,
                  "renet_adam_step: buffers must be 16-byte aligned");
  AdamArgs a;
  a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.weight_decay = weight_decay;
  a.bc1 = (float)(1.0 - pow((double)beta1, (double)step));
  a.bc2_sqrt = (float)sqrt(1.0 - pow((double)beta2, (double)step));
  a.max_norm = max_norm; a.grad_scale = grad_scale;
  const int64_t want = (n / 4 + 255) / 256;
  const unsigned grid = (unsigned)(want < 1 ? 1 : (want > kNumSMs * 8 ? kNumSMs * 8 : want));
  adam_step_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(param, grad, exp_avg, exp_avg_sq, n, a, sumsq);
  RENET_CHECK_LAUNCH("adam_step_kernel");
  return RENET_OK;
}

}  // extern "C"
