// Per-graph pooling of node features over a batched graph: dgl.max_nodes / dgl.mean_nodes of the reference's global
// aggregator (Aggregator.py:58-61, 101-104) -- one row per batched graph (timestamp) out of all its nodes' layer-2 features.
// HBM-bound: every node row is read once (forward) / written once (backward).
#include <math.h>

#include "common.cuh"

namespace renet {
namespace {

// one CTA per (segment, feature block of 128); thread = feature; rows of the segment are walked 4 at a time
template <bool MAX>
__global__ void __launch_bounds__(128)
segment_pool_fwd_kernel(const float* __restrict__ H, const int32_t* __restrict__ seg_ptr, int d, float* __restrict__ out,
                        int32_t* __restrict__ argmax) {
  const int g = blockIdx.x, c = blockIdx.y * 128 + threadIdx.x;
  if (c >= d) return;
  const int r0 = __ldg(seg_ptr + g), r1 = __ldg(seg_ptr + g + 1);
  float best = MAX ? -INFINITY : 0.f;      // an all -inf segment gives -inf (arg = its first row), as torch.max does
  int arg = r0;
  for (int r = r0; r < r1; ++r) {
    const float v = __ldg(H + (int64_t)r * d + c);
    if (MAX) { if (v > best) { best = v; arg = r; } }      // first maximum wins, like torch.max
    else best += v;
  }
  if (MAX) {
    out[(int64_t)g * d + c] = r1 > r0 ? best : 0.f;
    argmax[(int64_t)g * d + c] = arg;
  } else {
    out[(int64_t)g * d + c] = r1 > r0 ? best / (float)(r1 - r0) : 0.f;
  }
}

__global__ void segment_max_bwd_kernel(const float* __restrict__ dout, const int32_t* __restrict__ argmax,
                                       const int32_t* __restrict__ seg_ptr, int64_t G, int d, float* __restrict__ dH) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G * d) return;
  const int g = (int)(i / d), c = (int)(i % d);
  if (__ldg(seg_ptr + g + 1) > __ldg(seg_ptr + g)) dH[(int64_t)argmax[i] * d + c] = dout[i];   // one writer per (g, c)
}

__global__ void __launch_bounds__(128)
segment_mean_bwd_kernel(const float* __restrict__ dout, const int32_t* __restrict__ seg_ptr, int d, float* __restrict__ dH) {
  const int g = blockIdx.x, c = blockIdx.y * 128 + threadIdx.x;
  if (c >= d) return;
  const int r0 = __ldg(seg_ptr + g), r1 = __ldg(seg_ptr + g + 1);
  if (r1 <= r0) return;
  const float v = dout[(int64_t)g * d + c] / (float)(r1 - r0);
  for (int r = r0; r < r1; ++r) dH[(int64_t)r * d + c] = v;
}

}  // namespace
}  // namespace renet

using namespace renet;

extern "C" {

int renet_segment_pool_fwd(const float* H, const int32_t* seg_ptr, int64_t G, int32_t d, int32_t mode, float* out,
                           int32_t* argmax, void* stream) {
  RENET_CHECK_ARG(G >= 0 && d > 0 && (mode == 0 || mode == 1), "renet_segment_pool_fwd: bad arguments");
  if (G == 0) return RENET_OK;
  RENET_CHECK_ARG(H && seg_ptr && out && (mode == 0 || argmax), "renet_segment_pool_fwd: null pointer");
  dim3 grid((unsigned)G, (unsigned)((d + 127) / 128));
  if (mode == 1) segment_pool_fwd_kernel<true><<<grid, 128, 0, (cudaStream_t)stream>>>(H, seg_ptr, d, out, argmax);
  else segment_pool_fwd_kernel<false><<<grid, 128, 0, (cudaStream_t)stream>>>(H, seg_ptr, d, out, argmax);
  RENET_CHECK_LAUNCH("segment_pool_fwd_kernel");
  return RENET_OK;
}

int renet_segment_pool_bwd(const float* dout, const int32_t* seg_ptr, const int32_t* argmax, int64_t G, int64_t N,
                           int32_t d, int32_t mode, float* dH, void* stream) {
  RENET_CHECK_ARG(G >= 0 && N >= 0 && d > 0 && (mode == 0 || mode == 1), "renet_segment_pool_bwd: bad arguments");
  if (N == 0) return RENET_OK;
  RENET_CHECK_ARG(dH != nullptr, "renet_segment_pool_bwd: null pointer");
  RENET_CHECK_CUDA(cudaMemsetAsync(dH, 0, (size_t)N * d * sizeof(float), (cudaStream_t)stream));
  if (G == 0) return RENET_OK;
  RENET_CHECK_ARG(dout && seg_ptr && (mode == 0 || argmax), "renet_segment_pool_bwd: null pointer");
  if (mode == 1) {
    segment_max_bwd_kernel<<<(unsigned)((G * d + 255) / 256), 256, 0, (cudaStream_t)stream>>>(dout, argmax, seg_ptr, G, d, dH);
    RENET_CHECK_LAUNCH("segment_max_bwd_kernel");
  } else {
    dim3 grid((unsigned)G, (unsigned)((d + 127) / 128));
    segment_mean_bwd_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(dout, seg_ptr, d, dH);
    RENET_CHECK_LAUNCH("segment_mean_bwd_kernel");
  }
  return RENET_OK;
}

}  // extern "C"
