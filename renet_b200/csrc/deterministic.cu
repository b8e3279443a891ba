// Deterministic mode (renet_set_deterministic) and the fixed-order reductions it shares between translation units.
//
// With the mode on, no gradient of the training step is summed by float atomics: every producer writes partial sums to a
// buffer indexed by something the inputs and shapes fix (a K chunk, a row chunk, an edge run), and a second pass adds
// them in index order.  The buffers live in one stream-ordered block per (device, stream), so no entry point's signature
// or workspace size depends on the mode.  That per-(device, stream) allocator (stream_block) serves the GEMM engine too.
#include <cub/device/device_radix_sort.cuh>

#include <atomic>
#include <mutex>
#include <vector>

#include "common.cuh"

namespace renet {

static std::atomic<int> g_deterministic{0};
bool deterministic() { return g_deterministic.load(std::memory_order_relaxed) != 0; }
int set_deterministic(int on) { return g_deterministic.exchange(on ? 1 : 0); }

namespace {

struct StreamBlocks {
  int device;
  cudaStream_t stream;
  StreamBlock kind[kNumBlockKinds];
};
std::mutex g_blocks_mu;
std::vector<StreamBlocks> g_blocks;
constexpr int kMaxStreams = 8;
constexpr int64_t kBlockStep = int64_t(8) << 20;

inline int64_t align256(int64_t x) { return (x + 255) & ~int64_t(255); }

// out[r * ldo + c] (+)= sum_s parts[s * stride + r * cols + c]
__global__ void sum_partials_kernel(const float* __restrict__ parts, int n_parts, int64_t stride, int64_t rows, int cols,
                                    float* __restrict__ out, int64_t ldo, int accumulate) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  float* o = out + (i / cols) * ldo + i % cols;
  float s = accumulate ? *o : 0.f;
  for (int k = 0; k < n_parts; ++k) s += parts[(int64_t)k * stride + i];
  *o = s;
}

__global__ void scatter_keys_kernel(const int32_t* __restrict__ index, const int32_t* __restrict__ outer,
                                    int32_t* __restrict__ keys, int32_t* __restrict__ pos, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t k = __ldg(index + i);
  keys[i] = outer != nullptr ? __ldg(outer + k) : k;
  pos[i] = (int32_t)i;
}

// One warp per sorted position that starts a run of equal keys: dst[key] += the run's rows, summed in run order (= ascending
// source row, the sort being stable), 256 columns at a time in registers.
__global__ void scatter_add_rows_sorted_kernel(const float* __restrict__ src, int64_t ld, const int32_t* __restrict__ keys,
                                               const int32_t* __restrict__ pos, float* __restrict__ dst, int64_t n, int d) {
  const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const int32_t key = __ldg(keys + w);
  if (w > 0 && __ldg(keys + w - 1) == key) return;
  int64_t end = w + 1;
  while (end < n && __ldg(keys + end) == key) ++end;
  float* out = dst + (int64_t)key * d;
  for (int c0 = 0; c0 < d; c0 += 256) {
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    for (int64_t j = w; j < end; ++j) {
      const float* row = src + (int64_t)__ldg(pos + j) * ld + c0 + lane;
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (c0 + lane + 32 * k < d) acc[k] += __ldg(row + 32 * k);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k)
      if (c0 + lane + 32 * k < d) out[c0 + lane + 32 * k] += acc[k];
  }
}

}  // namespace

int stream_block(StreamBlockKind kind, int64_t bytes, cudaStream_t stream, StreamBlock* out) {
  std::lock_guard<std::mutex> lk(g_blocks_mu);
  int dev = 0;
  RENET_CHECK_CUDA(cudaGetDevice(&dev));
  StreamBlocks* s = nullptr;
  for (auto& e : g_blocks)
    if (e.device == dev && e.stream == stream) s = &e;
  if (s == nullptr) {
    if ((int)g_blocks.size() >= kMaxStreams) {     // bounded: drop the oldest (its stream may be gone: free synchronously)
      RENET_CHECK_CUDA(cudaDeviceSynchronize());
      for (const StreamBlock& b : g_blocks.front().kind)
        if (b.p) RENET_CHECK_CUDA(cudaFree(b.p));
      g_blocks.erase(g_blocks.begin());
    }
    g_blocks.push_back(StreamBlocks{dev, stream, {}});
    s = &g_blocks.back();
  }
  StreamBlock& b = s->kind[kind];
  if (bytes > b.bytes) {
    const int64_t grown = (bytes + kBlockStep - 1) / kBlockStep * kBlockStep;
    if (b.p) RENET_CHECK_CUDA(cudaFreeAsync(b.p, stream));
    b = StreamBlock{};
    RENET_CHECK_CUDA(cudaMallocAsync(&b.p, (size_t)grown, stream));
    b.bytes = grown;
  }
  *out = b;
  ++b.uses;
  return RENET_OK;
}

int det_scratch(int64_t bytes, cudaStream_t stream, void** out) {
  StreamBlock b;
  const int rc = stream_block(kBlockDeterministic, bytes, stream, &b);
  if (rc) return rc;
  *out = b.p;
  return RENET_OK;
}

int launch_sum_partials(const float* parts, int n_parts, int64_t stride, int64_t rows, int cols, float* out, int64_t ldo,
                        bool accumulate, cudaStream_t stream) {
  const int64_t n = rows * cols;
  if (n == 0) return RENET_OK;
  sum_partials_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(parts, n_parts, stride, rows, cols, out, ldo, accumulate);
  RENET_CHECK_LAUNCH("sum_partials_kernel");
  return RENET_OK;
}

int scatter_add_rows_det(const float* src, int64_t ld, const int32_t* index, const int32_t* outer, float* dst, int64_t n_rows,
                         int d, cudaStream_t stream) {
  if (n_rows == 0) return RENET_OK;
  if (n_rows >= (int64_t(1) << 31)) {
    set_error("scatter_add_rows: %lld rows exceed the int32 sort", (long long)n_rows);
    return RENET_ERR_INVALID_ARG;
  }
  size_t cub_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const int32_t*)nullptr, (int32_t*)nullptr, (const int32_t*)nullptr,
                                  (int32_t*)nullptr, (int)n_rows);
  const int64_t arr = align256(n_rows * 4);
  void* base = nullptr;
  int rc = det_scratch(4 * arr + (int64_t)cub_bytes, stream, &base);
  if (rc) return rc;
  char* p = static_cast<char*>(base);
  int32_t* keys_in = (int32_t*)p;
  int32_t* pos_in = (int32_t*)(p + arr);
  int32_t* keys = (int32_t*)(p + 2 * arr);
  int32_t* pos = (int32_t*)(p + 3 * arr);
  const unsigned nb = (unsigned)((n_rows + 255) / 256);
  scatter_keys_kernel<<<nb, 256, 0, stream>>>(index, outer, keys_in, pos_in, n_rows);
  RENET_CHECK_LAUNCH("scatter_keys_kernel");
  RENET_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(p + 4 * arr, cub_bytes, keys_in, keys, pos_in, pos, (int)n_rows, 0,
                                                   (int)(sizeof(int32_t) * 8), stream));
  count_launch(3);
  scatter_add_rows_sorted_kernel<<<(unsigned)((n_rows * 32 + 255) / 256), 256, 0, stream>>>(src, ld, keys, pos, dst, n_rows, d);
  RENET_CHECK_LAUNCH("scatter_add_rows_sorted_kernel");
  return RENET_OK;
}

}  // namespace renet
