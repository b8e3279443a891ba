// Shared helpers for librenet_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#include "../../include/renet_b200.h"

namespace renet {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);
// every dense-GEMM launcher records which kernel (renet_gemm_kernel) it ran; renet_debug_gemm reports it
void note_gemm_kernel(int kernel);
int last_gemm_kernel();

#define RENET_CHECK_ARG(cond, ...)                  \
  do {                                              \
    if (!(cond)) {                                  \
      ::renet::set_error(__VA_ARGS__);              \
      return RENET_ERR_INVALID_ARG;                 \
    }                                               \
  } while (0)

#define RENET_CHECK_CUDA(expr)                                                        \
  do {                                                                                \
    cudaError_t _e = (expr);                                                          \
    if (_e != cudaSuccess) {                                                          \
      ::renet::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),     \
                         __FILE__, __LINE__);                                         \
      return RENET_ERR_CUDA;                                                          \
    }                                                                                 \
  } while (0)

#define RENET_CHECK_LAUNCH(name)                                                      \
  do {                                                                                \
    cudaError_t _e = cudaGetLastError();                                              \
    if (_e != cudaSuccess) {                                                          \
      ::renet::set_error("launch of %s failed: %s", name, cudaGetErrorString(_e));    \
      return RENET_ERR_CUDA;                                                          \
    }                                                                                 \
    ::renet::count_launch();                                                          \
  } while (0)

constexpr int kNumSMs = 132;  // H100 SXM: one persistent CTA per SM

__device__ __forceinline__ float4 ldg_f4(const float* p) {
  return __ldg(reinterpret_cast<const float4*>(p));
}
// streaming 128-bit load that does not allocate in L1 (keeps L1 for the relation-weight table)
__device__ __forceinline__ float4 ldg_f4_stream(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void st_f4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

// 128-bit vector reduction to global memory (sm_90+): one RED for four floats.
__device__ __forceinline__ void red_add_f4(float* p, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}

// deterministic mode (renet_set_deterministic): every gradient reduction of the training step sums in an order that depends
// only on the inputs and shapes -- no float atomics, no order set by CTA scheduling (DESIGN §4)
bool deterministic();
int set_deterministic(int on);
// Stream-ordered device blocks the library keeps for itself: one per (device, stream, kind), allocated with cudaMallocAsync
// on first use and grown on demand in 8 MB steps, the old block freed behind the work already queued on that stream.  The
// work of one stream is ordered, so a block is only ever used by its own stream's calls.  *out holds at least `bytes` for
// work enqueued on `stream` until the next call of the same kind on that stream.
enum StreamBlockKind { kBlockPackedB, kBlockDedupKeys, kBlockDedupRows, kBlockDeterministic, kNumBlockKinds };
struct StreamBlock {
  void* p;
  int64_t bytes;   // the block's size: at least the bytes asked for
  int64_t uses;    // earlier calls that returned this block: 0 = allocated by this call (contents undefined)
};
int stream_block(StreamBlockKind kind, int64_t bytes, cudaStream_t stream, StreamBlock* out);
// The block of the deterministic reductions' partial sums and sort keys
int det_scratch(int64_t bytes, cudaStream_t stream, void** out);
// out[r * ldo + c] (+)= sum over s = 0, 1, ..., n_parts - 1 of parts[s * stride + r * cols + c]   (r < rows, c < cols)
int launch_sum_partials(const float* parts, int n_parts, int64_t stride, int64_t rows, int cols, float* out, int64_t ldo,
                        bool accumulate, cudaStream_t stream);
// dst[key_i] += src[i * ld ...][0 .. d) for i < n_rows, key_i = outer ? outer[index[i]] : index[i]; the rows of each key are
// added in ascending i (stable radix sort by key, then one warp per distinct key)
int scatter_add_rows_det(const float* src, int64_t ld, const int32_t* index, const int32_t* outer, float* dst, int64_t n_rows,
                         int d, cudaStream_t stream);

// internal (non-exported) launchers shared between translation units -------------------------------
// C[M,N] (ldc) = A[M,K] (rows optionally through a_index; lda) @ B[K,N] (ldb) [+ bias[N]] [+ C if accumulate].
// b_cacheable: B is a weight, so the tensor-core engine may key its packed image on B's address (packed_cache_lookup).
// Pass false for a B that lives in a per-call workspace: another call of the same weight generation can hold a different
// matrix at that address, and a cached image would be stale.
int sgemm_nn(const float* A, const int32_t* a_index, int64_t lda, const float* B, int64_t ldb, float* C,
             int64_t ldc, const float* bias, int64_t M, int32_t N, int32_t K, bool accumulate,
             cudaStream_t stream, bool b_cacheable = true);
// The FFMA engine of sgemm_nn: the register-tiled kernel where sgemm_nn_tiled_ok holds (and naive is false), else one thread
// per output
bool sgemm_nn_tiled_ok(const float* A, int64_t lda, const float* B, int64_t ldb, const float* C, int64_t ldc,
                       const float* bias, int32_t N, int32_t K);
int sgemm_nn_ffma(const float* A, const int32_t* a_index, int64_t lda, const float* B, int64_t ldb, float* C,
                  int64_t ldc, const float* bias, int64_t M, int32_t N, int32_t K, bool accumulate, bool naive,
                  cudaStream_t stream);
// C[M,N] += / = A^T B with A [K,M] (rows of A optionally through a_index), B [K,N]:  C = A^T @ B
// (split-K tiled kernel where sgemm_tn_tiled_ok holds and naive is false, else one thread per output)
bool sgemm_tn_tiled_ok(const float* A, int64_t lda, const float* B, int64_t ldb, const float* C, int64_t ldc, int32_t M,
                       int32_t N);
int sgemm_tn(const float* A, const int32_t* a_index, int64_t lda, const float* B, int64_t ldb, float* C,
             int64_t ldc, int32_t M, int32_t N, int64_t K, bool accumulate, cudaStream_t stream, bool naive = false);
// C[M,N] = A[M,K] @ B^T with B [N,K]
int sgemm_nt(const float* A, int64_t lda, const float* B, int64_t ldb, float* C, int64_t ldc,
             int64_t M, int32_t N, int32_t K, bool accumulate, cudaStream_t stream);

// 0 = automatic, 1 = tile, 3 = stream (RENET_GATHER_KERNEL=tile|stream; rgcn_fwd.cu)
int gather_kernel_choice();
constexpr int64_t kStreamMinEdges = 16384;   // below this a persistent one-CTA-per-SM launch costs more than the tile kernel
constexpr int64_t kStreamMinNodes = 16384;   // graphs with indexed input rows (layer 1) and the backward dH
constexpr int64_t kStreamMinPlainNodes = 2048;   // forward with plain input rows (layer 2's read-out sub-graph)
constexpr int64_t kStreamMaxNodes = 40960;    // 33 MB of fp32 features (2/3 of the 50 MB L2): beyond this the source rows come from HBM
// forward: indexed_input = the input rows come through an index (h_index); the backward passes true (its threshold is
// kStreamMinNodes)
bool gather_use_stream(int64_t E, int64_t N, bool indexed_input);
void set_stream_debug_buffer(long long* p);   // debug: per-warp time stamps of the stream kernel (rgcn_fwd.cu)          // the stream kernel (rgcn_stream.cuh) serves this edge count

// tensor-core (wgmma) GEMM engine building blocks (umma_gemm.cu); gemm_mode() == 1 selects the engine
int gemm_mode();
// An indexed wgmma product of at least this many rows (EPI 0, no accumulate, resident panel) computes each distinct index
// once and copies the rows out (umma_gemm_dedup).  Layer 1's self-loop (N ~ 33 k nodes, ~20 % distinct entities) is above
// it; layer 2's read-out rows (S ~ 8.5 k, all distinct) are below, where the extra passes would be pure cost (DESIGN §5).
constexpr int64_t kDedupMinRows = 16384;
int64_t umma_packed_bytes(int N, int K);
void set_gemm_debug_buffer(long long* p);     // debug: per-warpgroup time stamps of the packed GEMM kernels (umma_gemm.cu)
// packed-weight cache (umma_gemm.cu): persistent device buffer for this key, or nullptr when caching is off; *hit says
// whether it already holds the image for the current weight generation
void set_weight_generation(int64_t g);
void* packed_cache_lookup(const void* const* keys, int nkeys, int64_t bytes, bool* hit);
bool umma_shape_ok(int N, int K);
int umma_pack_b(const float* B, int64_t sk, int64_t sn, int N, int K, void* Bp, int tile_offset, cudaStream_t stream);
// fused epilogues of the packed wgmma GEMM (umma_gemm.cu): see the comment there
struct EpiArgs {
  const int32_t* target;   // [M] class of every row
  const float* lse;        // [M] (EPI 2)
  float* pmax;             // [2 * n_tiles, M] (EPI 1)
  float* psum;             // [2 * n_tiles, M] (EPI 1)
  float* tlogit;           // [M] (EPI 1): written by the one thread that sees the target column
  float* dT;               // [N, ldT] (EPI 2): the same gradient transposed (A operand of dW = dlogits^T @ X)
  int64_t ldT;
  float scale;             // (EPI 2, 4)
  const float* dscale;     // (EPI 2, 4) optional device scalar multiplied into scale (the upstream gradient, no host read)
  // soft targets (EPI 3, 4): P[row * ldp + col], rows need not sum to 1
  const float* soft;
  int64_t ldp;
  float* pdot;             // [2 * n_tiles, M] (EPI 3): sum of P * logit over the (row, half column tile)
  float* pmass;            // [2 * n_tiles, M] (EPI 3): sum of P over the same
  const float* rowmass;    // [M] (EPI 4): sum of P over the whole row
  // grouped top-k selection (EPI 5): rows come in groups of sel_R; p = row_w[row] * exp(logit - lse[row]) with
  // p >= tau[group] is appended as (p, (row % sel_R) * N + col) to that group's candidate buffer of sel_cap entries
  const float* row_w;
  const float* tau;
  int32_t* sel_count;      // [G] candidates found per group (counts past sel_cap: the capacity the call needs)
  float* sel_val;          // [G, sel_cap]
  int32_t* sel_idx;        // [G, sel_cap]
  int sel_R, sel_cap;
  // rank counting (EPI 6): every logit of row `row` is compared with tlogit[row] (the label's logit from the EPI 1 pass),
  // and rank_counts[rank_ld * row + {0, 1}] += {#greater, #equal} (integer atomics).  Per exclusion list j < n_lists (0..2):
  // the sigmoid, with the columns of excl_col[excl_begin[j * M + row] .. excl_end[j * M + row]) (sorted; the lists share
  // excl_col) other than target[row] set to 0, is compared with the label's, and rank_counts[rank_ld * row + 2 + 2 * j +
  // {0, 1}] += {#greater, #equal}.  rank_ld >= 2 + 2 * n_lists; the columns past the lists' are not written.
  const int32_t* excl_col;
  const int32_t* excl_begin;
  const int32_t* excl_end;
  int32_t* rank_counts;
  int n_lists;
  int rank_ld;
};
// p = w * exp(z - lse), rounded the same way wherever the grouped top-k forms it (decoder.cu, umma_gemm.cu)
__device__ __forceinline__ float topk_prob(float z, float lse, float w) { return __fmul_rn(w, expf(__fsub_rn(z, lse))); }
// torch.sigmoid of a CUDA float tensor, bit for bit: 1 / (1 + exp(-z)) with the accurate expf and an IEEE division.  In fp32
// it rounds to exactly 1 above z ~ 17 and to exactly 0 once exp(-z) overflows, and filtered ranks count those ties.
__device__ __forceinline__ float torch_sigmoid(float z) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-z))); }
int umma_gemm_prepacked_ex(const float* A, const int32_t* a_index, int64_t lda, const void* Bp, float* C, int64_t ldc,
                           const float* bias, int64_t M, int N, int K, bool accumulate, int batch, int64_t batch_a,
                           int64_t batch_bp, int64_t batch_c, int epi_mode, const EpiArgs& epi, int k_splits, int64_t split_c,
                           cudaStream_t stream);
int umma_gemm_prepacked(const float* A, const int32_t* a_index, int64_t lda, const void* Bp, float* C, int64_t ldc,
                        const float* bias, int64_t M, int N, int K, bool accumulate, int batch, int64_t batch_a,
                        int64_t batch_bp, int64_t batch_c, cudaStream_t stream);
// renet_debug_gemm without its kernel id (umma_gemm.cu)
int debug_gemm(int form, int kernel, const float* A, const int32_t* a_index, int64_t lda, const float* B, int64_t ldb, float* C,
               int64_t ldc, const float* bias, int64_t M, int N, int64_t K, bool accumulate, int batch, int64_t batch_a,
               int64_t batch_b, int64_t batch_c, void* ws, int64_t ws_bytes, cudaStream_t stream);

}  // namespace renet
