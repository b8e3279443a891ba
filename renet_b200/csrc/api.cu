// extern "C" entry points of librenet_b200.so (declared in include/renet_b200.h).
#include <cub/device/device_radix_sort.cuh>

#include <atomic>
#include <mutex>
#include <string.h>
#include <vector>

#include "common.cuh"

namespace renet {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
static thread_local int g_last_gemm_kernel = 0;
void note_gemm_kernel(int kernel) { g_last_gemm_kernel = kernel; }
int last_gemm_kernel() { return g_last_gemm_kernel; }

// launchers defined in the other translation units
int launch_rgcn_gather(const float* H, const int32_t* h_index, const float* W, const int32_t* row_ptr,
                       const int32_t* col_src, const int32_t* col_type, const float* norm, float* Hout,
                       int64_t N, int64_t E, int d_in, int d_out, int nb, int relu, int has_loop,
                       cudaStream_t stream, int R2 = -1, const int32_t* hot_rel = nullptr, int n_hot = 0);
int launch_rgcn_bwd(const float* H, const int32_t* h_index, const float* W, const float* Wloop,
                    const int32_t* t_row_ptr, const int32_t* t_col_dst, const int32_t* t_col_type,
                    const int32_t* rel_ptr, const int32_t* rel_src, const int32_t* rel_dst, const float* norm,
                    const float* Hout, const float* dHout, float* dH, float* dW, float* dWloop, float* G_ws,
                    int64_t N, int64_t E, int d_in, int d_out, int nb, int R2, int relu, cudaStream_t stream,
                    int64_t N_dst = -1);
int launch_selfloop_bwd(const float* H, const int32_t* h_index, const float* Wloop, const float* dLoop, float* dH,
                        float* dWloop, float* WloopT_ws, int64_t N, int d_in, int d_out, cudaStream_t stream);
int launch_scatter_add_rows(const float* src, const int32_t* index, float* dst, int64_t n_rows, int d,
                            cudaStream_t stream);
int64_t gru_workspace_floats(int64_t S, int64_t Q, int64_t T, int h, bool dropout = false, int max_len = 0);
int launch_gru_fwd(const float* H2, const int32_t* readout, const int32_t* row_glob, const float* glob,
                   const float* ent, const float* rel, const int32_t* seq_s, const int32_t* seq_r,
                   const int32_t* seq_len, const int32_t* seq_start, const int32_t* host_batch_sizes,
                   int max_len, const float* w_ih4, const float* w_hh4, const float* b_ih4, const float* b_hh4,
                   const float* w_ih3, const float* w_hh3, const float* b_ih3, const float* b_hh3, float* hn4,
                   float* hn3, int64_t S, int64_t Q, int64_t T, int h, float* ws_base, cudaStream_t stream, float p_drop = 0.f,
                   uint64_t seed = 0, const int32_t* row_seq = nullptr, const float* ext_X4 = nullptr, int k4 = 0,
                   const float* ext_X3 = nullptr, int k3 = 0, int phase = 0);
int64_t gru_bwd_workspace_floats(int64_t S, int64_t Q, int64_t T, int h, bool dropout = false, int max_len = 0);
int launch_dropout_mask(uint64_t seed, uint64_t offset, int64_t n, float p, float* out, cudaStream_t stream);
int launch_gru_bwd(const float* H2, const int32_t* readout, const int32_t* row_glob, const float* glob,
                   const float* ent, const float* rel, const int32_t* seq_s, const int32_t* seq_r,
                   const int32_t* seq_len, const int32_t* seq_start, const int32_t* host_batch_sizes, int max_len,
                   const float* w_ih4, const float* w_hh4, const float* w_ih3, const float* w_hh3,
                   const float* dhn4, const float* dhn3, float* dH2, float* d_ent, float* d_rel, float* d_glob,
                   float* dw_ih4, float* dw_hh4, float* db_ih4, float* db_hh4, float* dw_ih3, float* dw_hh3,
                   float* db_ih3, float* db_hh3, int64_t N, int64_t S, int64_t Q, int64_t T, int h,
                   const float* fwd_ws, float* bwd_ws, cudaStream_t stream, float p_drop = 0.f, uint64_t seed = 0,
                   const int32_t* row_seq = nullptr, const float* ext_X4 = nullptr, int k4 = 0, const float* ext_X3 = nullptr,
                   int k3 = 0, float* out_dX4 = nullptr, float* out_dX3 = nullptr);
int launch_pack_inputs(const float* H2, const int32_t* readout, const int32_t* row_glob, const float* glob,
                       const float* ent, const float* rel, const int32_t* row_seq, const int32_t* seq_s,
                       const int32_t* seq_r, const int32_t* packed_row, float* X4, float* X3, int64_t S, int h,
                       cudaStream_t stream);

int gemm_mode();
int set_gemm_mode(int m);

namespace {

__global__ void iota_kernel(int32_t* p, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = (int32_t)i;
}

// sorted keys -> row_ptr (handles empty rows), and gather the payload columns through perm
__global__ void csr_finish_kernel(const int32_t* __restrict__ keys, const int32_t* __restrict__ perm,
                                  const int32_t* __restrict__ src, const int32_t* __restrict__ etype,
                                  int32_t* __restrict__ row_ptr, int32_t* __restrict__ col_src,
                                  int32_t* __restrict__ col_type, int64_t N, int64_t E) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > E) return;
  const int64_t prev = (i == 0) ? -1 : keys[i - 1];
  const int64_t cur = (i == E) ? N : keys[i];
  for (int64_t k = prev + 1; k <= cur; ++k) row_ptr[k] = (int32_t)i;
  if (i < E) {
    const int32_t p = perm[i];
    col_src[i] = src[p];
    if (etype != nullptr) col_type[i] = etype[p];
  }
}

inline int64_t align256(int64_t x) { return (x + 255) & ~int64_t(255); }

int key_bits(int64_t N) {
  int b = 1;
  while ((int64_t(1) << b) < N && b < 31) ++b;
  return b;
}

}  // namespace
}  // namespace renet

using namespace renet;

namespace renet {
namespace {
// seq_s[q] = triplets[s_idx[q]][col_s], seq_r[q] = triplets[s_idx[q]][1] (model.py:81-84: samples in history-length
// order) and row_graph[i] = comp_graph[row_comp[i]] (utils.py:224-225: the timestamp of every read-out row), one launch
__global__ void prepare_sequences_kernel(const int64_t* __restrict__ triplets, int ld, int col_s, const int32_t* __restrict__ s_idx,
                                         int Q, const int32_t* __restrict__ comp_graph,
                                         const int32_t* __restrict__ row_comp, int S, int32_t* __restrict__ seq_s,
                                         int32_t* __restrict__ seq_r, int32_t* __restrict__ row_graph) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < Q) {
    const int64_t* t = triplets + ld * (int64_t)s_idx[i];
    seq_s[i] = (int32_t)t[col_s];
    seq_r[i] = (int32_t)t[1];
  }
  if (i < S) row_graph[i] = comp_graph[row_comp[i]];
}

// renet_encode_fwd's fork / join: one side stream per device, one event pair per (device, caller stream), so that calls on
// several devices, or from several host threads on their own streams, never record or wait on another call's event.  The
// pair table is bounded like stream_block's; an entry is only dropped while no call holds it (busy == 0), and dropping it
// needs no synchronisation (cudaEventDestroy releases a pending event once it completes).
struct EncodeFork {
  int device;
  cudaStream_t caller;
  cudaEvent_t fork, join;
  int busy;
};
std::mutex g_fork_mu;
std::vector<cudaStream_t> g_side;       // indexed by device
std::vector<EncodeFork> g_forks;
constexpr int kMaxForks = 8;

int fork_acquire(cudaStream_t caller, cudaStream_t* side, cudaEvent_t* fork, cudaEvent_t* join) {
  std::lock_guard<std::mutex> lk(g_fork_mu);
  int dev = 0;
  RENET_CHECK_CUDA(cudaGetDevice(&dev));
  if ((int)g_side.size() <= dev) g_side.resize(dev + 1, nullptr);
  if (g_side[dev] == nullptr) RENET_CHECK_CUDA(cudaStreamCreateWithFlags(&g_side[dev], cudaStreamNonBlocking));
  EncodeFork* f = nullptr;
  for (auto& e : g_forks)
    if (e.device == dev && e.caller == caller) f = &e;
  if (f == nullptr) {
    if ((int)g_forks.size() >= kMaxForks) {
      for (size_t i = 0; i < g_forks.size(); ++i)
        if (g_forks[i].busy == 0) {            // the oldest idle entry
          cudaEventDestroy(g_forks[i].fork);
          cudaEventDestroy(g_forks[i].join);
          g_forks.erase(g_forks.begin() + i);
          break;
        }
    }
    EncodeFork e{dev, caller, nullptr, nullptr, 0};
    RENET_CHECK_CUDA(cudaEventCreateWithFlags(&e.fork, cudaEventDisableTiming));
    RENET_CHECK_CUDA(cudaEventCreateWithFlags(&e.join, cudaEventDisableTiming));
    g_forks.push_back(e);
    f = &g_forks.back();
  }
  ++f->busy;
  *side = g_side[dev];
  *fork = f->fork;
  *join = f->join;
  return RENET_OK;
}

void fork_release(cudaStream_t caller) {
  std::lock_guard<std::mutex> lk(g_fork_mu);
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return;
  for (auto& e : g_forks)
    if (e.device == dev && e.caller == caller && e.busy > 0) --e.busy;
}

struct ForkLease {
  cudaStream_t caller;
  bool held = false;
  ~ForkLease() {
    if (held) fork_release(caller);
  }
};
}  // namespace
}  // namespace renet


extern "C" {

int renet_version(void) { return 100; /* 0.1.0 */ }
const char* renet_last_error(void) { return g_err; }
int64_t renet_launch_count(void) { return g_launches.load(); }
int renet_set_gemm_engine(int engine) { return set_gemm_mode(engine); }
int renet_get_gemm_engine(void) { return gemm_mode(); }
int renet_set_deterministic(int on) { return set_deterministic(on); }
int renet_get_deterministic(void) { return deterministic() ? 1 : 0; }
int renet_set_weight_generation(int64_t generation) { renet::set_weight_generation(generation); return RENET_OK; }

int64_t renet_csr_workspace_bytes(int64_t N, int64_t E) {
  size_t cub_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const int32_t*)nullptr, (int32_t*)nullptr,
                                  (const int32_t*)nullptr, (int32_t*)nullptr, (int)E, 0, key_bits(N));
  return align256((int64_t)cub_bytes) + 3 * align256(E * 4) + 256;
}

int renet_build_csr(const int32_t* dst, const int32_t* src, const int32_t* etype, int64_t N, int64_t E,
                    int32_t* row_ptr, int32_t* col_src, int32_t* col_type, int32_t* perm, void* workspace,
                    int64_t workspace_bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  RENET_CHECK_ARG(N >= 0 && E >= 0 && E < (int64_t(1) << 31) && N < (int64_t(1) << 31), "renet_build_csr: bad N/E");
  RENET_CHECK_ARG(row_ptr != nullptr, "renet_build_csr: row_ptr is null");
  if (E == 0) {
    RENET_CHECK_CUDA(cudaMemsetAsync(row_ptr, 0, (N + 1) * sizeof(int32_t), stream));
    return RENET_OK;
  }
  RENET_CHECK_ARG(dst && src && col_src && workspace, "renet_build_csr: null pointer");
  RENET_CHECK_ARG(etype == nullptr || col_type != nullptr, "renet_build_csr: col_type is null");
  RENET_CHECK_ARG(workspace_bytes >= renet_csr_workspace_bytes(N, E), "renet_build_csr: workspace too small");
  char* ws = (char*)workspace;
  int32_t* keys_out = (int32_t*)ws;            ws += align256(E * 4);
  int32_t* vals_in = (int32_t*)ws;             ws += align256(E * 4);
  int32_t* vals_out = perm ? perm : (int32_t*)ws;  ws += align256(E * 4);
  size_t cub_bytes = (size_t)(workspace_bytes - (ws - (char*)workspace));
  const unsigned nb = (unsigned)((E + 256) / 256);
  iota_kernel<<<nb, 256, 0, stream>>>(vals_in, E);
  RENET_CHECK_LAUNCH("iota_kernel");
  RENET_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(ws, cub_bytes, dst, keys_out, vals_in, vals_out, (int)E, 0,
                                                   key_bits(N), stream));
  count_launch(3);
  csr_finish_kernel<<<nb, 256, 0, stream>>>(keys_out, vals_out, src, etype, row_ptr, col_src, col_type, N, E);
  RENET_CHECK_LAUNCH("csr_finish_kernel");
  return RENET_OK;
}

static int check_layer_args(const char* fn, const void* H, const void* W, const void* row_ptr, const void* norm,
                            const void* Hout, int64_t N, int64_t E, int d_in, int d_out, int nb, int R2) {
  RENET_CHECK_ARG(N >= 0 && E >= 0 && N < (int64_t(1) << 31) && E < (int64_t(1) << 31), "%s: bad N/E", fn);
  RENET_CHECK_ARG(d_in > 0 && d_out > 0 && nb > 0 && d_in % nb == 0 && d_out % nb == 0,
                  "%s: d_in=%d d_out=%d must be positive multiples of num_bases=%d", fn, d_in, d_out, nb);
  RENET_CHECK_ARG(R2 > 0, "%s: R2 must be positive", fn);
  if (N > 0) RENET_CHECK_ARG(H && W && row_ptr && norm && Hout, "%s: null pointer", fn);
  RENET_CHECK_ARG(E > 0 || d_in == d_out, "%s: a graph without edges needs d_in == d_out", fn);
  return RENET_OK;
}

int renet_selfloop_gemm(const float* H, const int32_t* h_index, const float* Wloop, float* Hout, int64_t N,
                        int32_t d_in, int32_t d_out, void* stream) {
  RENET_CHECK_ARG(N >= 0 && d_in > 0 && d_out > 0, "renet_selfloop_gemm: bad shape");
  if (N == 0) return RENET_OK;
  RENET_CHECK_ARG(H && Wloop && Hout, "renet_selfloop_gemm: null pointer");
  return sgemm_nn(H, h_index, d_in, Wloop, d_out, Hout, d_out, nullptr, N, d_out, d_in, false,
                  (cudaStream_t)stream);
}

int renet_rgcn_gather(const float* H, const int32_t* h_index, const float* W, const int32_t* row_ptr,
                      const int32_t* col_src, const int32_t* col_type, const float* norm, float* Hout, int64_t N,
                      int64_t E, int32_t d_in, int32_t d_out, int32_t num_bases, int32_t R2, int32_t relu,
                      int32_t has_loop, void* stream) {
  int rc = check_layer_args("renet_rgcn_gather", H, W, row_ptr, norm, Hout, N, E, d_in, d_out, num_bases, R2);
  if (rc) return rc;
  RENET_CHECK_ARG(E == 0 || (col_src && col_type), "renet_rgcn_gather: null edge arrays");
  return launch_rgcn_gather(H, h_index, W, row_ptr, col_src, col_type, norm, Hout, N, E, d_in, d_out, num_bases,
                            relu, has_loop, (cudaStream_t)stream, R2);
}

int renet_rgcn_gather_hot(const float* H, const int32_t* h_index, const float* W, const int32_t* row_ptr,
                          const int32_t* col_src, const int32_t* col_type, const float* norm, float* Hout, int64_t N,
                          int64_t E, int32_t d_in, int32_t d_out, int32_t num_bases, int32_t R2, int32_t relu,
                          int32_t has_loop, const int32_t* hot_rel, int32_t n_hot, void* stream) {
  int rc = check_layer_args("renet_rgcn_gather_hot", H, W, row_ptr, norm, Hout, N, E, d_in, d_out, num_bases, R2);
  if (rc) return rc;
  RENET_CHECK_ARG(E == 0 || (col_src && col_type), "renet_rgcn_gather_hot: null edge arrays");
  RENET_CHECK_ARG(n_hot >= 0 && (n_hot == 0 || hot_rel != nullptr), "renet_rgcn_gather_hot: bad hot-relation list");
  return launch_rgcn_gather(H, h_index, W, row_ptr, col_src, col_type, norm, Hout, N, E, d_in, d_out, num_bases,
                            relu, has_loop, (cudaStream_t)stream, R2, n_hot > 0 ? hot_rel : nullptr, n_hot);
}

int renet_debug_stream_timing(void* buffer) {
  set_stream_debug_buffer(static_cast<long long*>(buffer));
  return RENET_OK;
}

int renet_debug_gemm_timing(void* buffer) {
  set_gemm_debug_buffer(static_cast<long long*>(buffer));
  return RENET_OK;
}

int renet_debug_gemm(int32_t form, int32_t kernel, const float* A, const int32_t* a_index, int64_t lda, const float* B,
                     int64_t ldb, float* C, int64_t ldc, const float* bias, int64_t M, int32_t N, int64_t K, int32_t accumulate,
                     int32_t batch, int64_t batch_a, int64_t batch_b, int64_t batch_c, void* workspace, int64_t workspace_bytes,
                     void* stream) {
  note_gemm_kernel(0);
  const int rc = debug_gemm(form, kernel, A, a_index, lda, B, ldb, C, ldc, bias, M, N, K, accumulate != 0, batch, batch_a,
                            batch_b, batch_c, workspace, workspace_bytes, (cudaStream_t)stream);
  return rc ? rc : last_gemm_kernel();
}

int renet_rgcn_block_fwd(const float* H, const int32_t* h_index, const float* W, const float* Wloop,
                         const int32_t* row_ptr, const int32_t* col_src, const int32_t* col_type,
                         const float* norm, float* Hout, int64_t N, int64_t E, int32_t d_in, int32_t d_out,
                         int32_t num_bases, int32_t R2, int32_t relu, void* stream) {
  int rc = check_layer_args("renet_rgcn_block_fwd", H, W, row_ptr, norm, Hout, N, E, d_in, d_out, num_bases, R2);
  if (rc) return rc;
  RENET_CHECK_ARG(E == 0 || (col_src && col_type), "renet_rgcn_block_fwd: null edge arrays");
  if (N == 0) return RENET_OK;
  if (Wloop != nullptr) {
    rc = sgemm_nn(H, h_index, d_in, Wloop, d_out, Hout, d_out, nullptr, N, d_out, d_in, false, (cudaStream_t)stream);
    if (rc) return rc;
  }
  return launch_rgcn_gather(H, h_index, W, row_ptr, col_src, col_type, norm, Hout, N, E, d_in, d_out, num_bases,
                            relu, Wloop != nullptr, (cudaStream_t)stream, R2);
}

int renet_rgcn_block_bwd(const float* H, const int32_t* h_index, const float* W, const float* Wloop,
                         const int32_t* t_row_ptr, const int32_t* t_col_dst, const int32_t* t_col_type,
                         const int32_t* rel_ptr, const int32_t* rel_src, const int32_t* rel_dst, const float* norm,
                         const float* Hout, const float* dHout, float* dH, float* dW, float* dWloop, float* G_ws,
                         int64_t N, int64_t E, int32_t d_in, int32_t d_out, int32_t num_bases, int32_t R2,
                         int32_t relu, void* stream) {
  int rc = check_layer_args("renet_rgcn_block_bwd", H, W, t_row_ptr, norm, dHout, N, E, d_in, d_out, num_bases, R2);
  if (rc) return rc;
  RENET_CHECK_ARG(E > 0 || N == 0, "renet_rgcn_block_bwd: graphs without edges are not supported in backward");
  RENET_CHECK_ARG(dH && dW && G_ws && (Wloop == nullptr || dWloop != nullptr), "renet_rgcn_block_bwd: null output");
  RENET_CHECK_ARG(!relu || Hout != nullptr, "renet_rgcn_block_bwd: relu backward needs Hout");
  RENET_CHECK_ARG(t_col_dst && t_col_type && rel_ptr && rel_src && rel_dst, "renet_rgcn_block_bwd: null edge arrays");
  if (N == 0) return RENET_OK;
  return launch_rgcn_bwd(H, h_index, W, Wloop, t_row_ptr, t_col_dst, t_col_type, rel_ptr, rel_src, rel_dst, norm,
                         Hout, dHout, dH, dW, dWloop, G_ws, N, E, d_in, d_out, num_bases, R2, relu,
                         (cudaStream_t)stream);
}

int renet_rgcn_bipartite_bwd(const float* H, const float* W, const int32_t* t_row_ptr, const int32_t* t_col_dst,
                             const int32_t* t_col_type, const int32_t* rel_ptr, const int32_t* rel_src, const int32_t* rel_dst,
                             const float* norm, const float* Hout, const float* dHout, float* dH, float* dW, float* G_ws,
                             int64_t N_src, int64_t N_dst, int64_t E, int32_t d_in, int32_t d_out, int32_t num_bases, int32_t R2,
                             int32_t relu, void* stream) {
  int rc = check_layer_args("renet_rgcn_bipartite_bwd", H, W, t_row_ptr, norm, dHout, N_src, E, d_in, d_out, num_bases, R2);
  if (rc) return rc;
  RENET_CHECK_ARG(N_dst >= 0 && N_dst < (int64_t(1) << 31), "renet_rgcn_bipartite_bwd: bad N_dst");
  RENET_CHECK_ARG(dH && dW && G_ws, "renet_rgcn_bipartite_bwd: null output");
  RENET_CHECK_ARG(!relu || Hout != nullptr, "renet_rgcn_bipartite_bwd: relu backward needs Hout");
  if (N_src == 0) return RENET_OK;
  if (E == 0 || N_dst == 0) {       // no edge reaches a destination: dH = 0, dW unchanged
    RENET_CHECK_CUDA(cudaMemsetAsync(dH, 0, (size_t)N_src * d_in * sizeof(float), (cudaStream_t)stream));
    return RENET_OK;
  }
  RENET_CHECK_ARG(t_col_dst && t_col_type && rel_ptr && rel_src && rel_dst, "renet_rgcn_bipartite_bwd: null edge arrays");
  return launch_rgcn_bwd(H, nullptr, W, nullptr, t_row_ptr, t_col_dst, t_col_type, rel_ptr, rel_src, rel_dst, norm, Hout, dHout,
                         dH, dW, nullptr, G_ws, N_src, E, d_in, d_out, num_bases, R2, relu, (cudaStream_t)stream, N_dst);
}

int renet_selfloop_gemm_bwd(const float* H, const int32_t* h_index, const float* Wloop, const float* dLoop,
                            float* dH, float* dWloop, float* ws, int64_t N, int32_t d_in, int32_t d_out,
                            void* stream) {
  RENET_CHECK_ARG(N >= 0 && d_in > 0 && d_out > 0, "renet_selfloop_gemm_bwd: bad shape");
  if (N == 0) return RENET_OK;
  RENET_CHECK_ARG(H && Wloop && dLoop && dH && dWloop && ws, "renet_selfloop_gemm_bwd: null pointer");
  return launch_selfloop_bwd(H, h_index, Wloop, dLoop, dH, dWloop, ws, N, d_in, d_out, (cudaStream_t)stream);
}

int renet_scatter_add_rows(const float* src, const int32_t* index, float* dst, int64_t n_rows, int32_t d,
                           void* stream) {
  RENET_CHECK_ARG(n_rows >= 0 && d > 0, "renet_scatter_add_rows: bad shape");
  if (n_rows == 0) return RENET_OK;
  RENET_CHECK_ARG(src && index && dst, "renet_scatter_add_rows: null pointer");
  return launch_scatter_add_rows(src, index, dst, n_rows, d, (cudaStream_t)stream);
}

int64_t renet_gru_workspace_bytes(int64_t S, int64_t Q, int64_t T, int32_t h) {
  return gru_workspace_floats(S, Q, T, h) * (int64_t)sizeof(float);
}
int64_t renet_gru_workspace_bytes_len(int64_t S, int64_t Q, int64_t T, int32_t h, int32_t max_len) {
  return gru_workspace_floats(S, Q, T, h, false, max_len) * (int64_t)sizeof(float);
}

int renet_gru_fwd(const float* H2, const int32_t* readout, const int32_t* row_glob, const float* glob,
                  const float* ent, const float* rel, const int32_t* seq_s, const int32_t* seq_r,
                  const int32_t* seq_len, const int32_t* seq_start, const int32_t* host_batch_sizes,
                  int32_t max_len, const float* w_ih4, const float* w_hh4, const float* b_ih4, const float* b_hh4,
                  const float* w_ih3, const float* w_hh3, const float* b_ih3, const float* b_hh3, float* hn4,
                  float* hn3, int64_t S, int64_t Q, int64_t T, int32_t h, void* workspace, int64_t workspace_bytes,
                  void* stream) {
  RENET_CHECK_ARG(S >= 0 && Q >= 0 && T >= 0 && h > 0 && max_len >= 0, "renet_gru_fwd: bad shape");
  if (S == 0 || Q == 0) return RENET_OK;
  RENET_CHECK_ARG(H2 && readout && row_glob && glob && ent && rel && seq_s && seq_r && seq_len && seq_start &&
                      host_batch_sizes && w_ih4 && w_hh4 && b_ih4 && b_hh4 && w_ih3 && w_hh3 && b_ih3 && b_hh3 &&
                      hn4 && hn3 && workspace,
                  "renet_gru_fwd: null pointer");
  RENET_CHECK_ARG(workspace_bytes >= renet_gru_workspace_bytes_len(S, Q, T, h, max_len),
                  "renet_gru_fwd: workspace of %lld bytes too small for max_len %d (needs %lld)", (long long)workspace_bytes,
                  max_len, (long long)renet_gru_workspace_bytes_len(S, Q, T, h, max_len));
  RENET_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 15) == 0, "renet_gru_fwd: workspace must be 16-byte aligned");
  return launch_gru_fwd(H2, readout, row_glob, glob, ent, rel, seq_s, seq_r, seq_len, seq_start, host_batch_sizes,
                        max_len, w_ih4, w_hh4, b_ih4, b_hh4, w_ih3, w_hh3, b_ih3, b_hh3, hn4, hn3, S, Q, T, h,
                        (float*)workspace, (cudaStream_t)stream);
}

int64_t renet_gru_bwd_workspace_bytes(int64_t S, int64_t Q, int64_t T, int32_t h) {
  return gru_bwd_workspace_floats(S, Q, T, h) * (int64_t)sizeof(float);
}
int64_t renet_gru_bwd_workspace_bytes_len(int64_t S, int64_t Q, int64_t T, int32_t h, int32_t max_len) {
  return gru_bwd_workspace_floats(S, Q, T, h, false, max_len) * (int64_t)sizeof(float);
}

int renet_gru_bwd(const float* H2, const int32_t* readout, const int32_t* row_glob, const float* glob,
                  const float* ent, const float* rel, const int32_t* seq_s, const int32_t* seq_r,
                  const int32_t* seq_len, const int32_t* seq_start, const int32_t* host_batch_sizes,
                  int32_t max_len, const float* w_ih4, const float* w_hh4, const float* w_ih3, const float* w_hh3,
                  const float* dhn4, const float* dhn3, float* dH2, float* d_ent, float* d_rel, float* d_glob,
                  float* dw_ih4, float* dw_hh4, float* db_ih4, float* db_hh4, float* dw_ih3, float* dw_hh3,
                  float* db_ih3, float* db_hh3, int64_t N, int64_t S, int64_t Q, int64_t T, int32_t h,
                  const void* fwd_workspace, void* bwd_workspace, int64_t bwd_workspace_bytes, void* stream) {
  RENET_CHECK_ARG(N >= 0 && S >= 0 && Q >= 0 && T >= 0 && h > 0 && max_len >= 0, "renet_gru_bwd: bad shape");
  if (S == 0 || Q == 0) return RENET_OK;
  RENET_CHECK_ARG(H2 && readout && row_glob && glob && ent && rel && seq_s && seq_r && seq_len && seq_start &&
                      host_batch_sizes && w_ih4 && w_hh4 && w_ih3 && w_hh3 && dhn4 && dhn3 && dH2 && d_ent &&
                      d_rel && dw_ih4 && dw_hh4 && db_ih4 && db_hh4 && dw_ih3 && dw_hh3 && db_ih3 && db_hh3 &&
                      fwd_workspace && bwd_workspace,
                  "renet_gru_bwd: null pointer");
  RENET_CHECK_ARG(bwd_workspace_bytes >= renet_gru_bwd_workspace_bytes_len(S, Q, T, h, max_len),
                  "renet_gru_bwd: workspace of %lld bytes too small for max_len %d (needs %lld)", (long long)bwd_workspace_bytes,
                  max_len, (long long)renet_gru_bwd_workspace_bytes_len(S, Q, T, h, max_len));
  RENET_CHECK_ARG((reinterpret_cast<uintptr_t>(bwd_workspace) & 15) == 0, "renet_gru_bwd: workspace must be 16-byte aligned");
  return launch_gru_bwd(H2, readout, row_glob, glob, ent, rel, seq_s, seq_r, seq_len, seq_start, host_batch_sizes,
                        max_len, w_ih4, w_hh4, w_ih3, w_hh3, dhn4, dhn3, dH2, d_ent, d_rel, d_glob, dw_ih4, dw_hh4,
                        db_ih4, db_hh4, dw_ih3, dw_hh3, db_ih3, db_hh3, N, S, Q, T, h, (const float*)fwd_workspace,
                        (float*)bwd_workspace, (cudaStream_t)stream);
}

int64_t renet_gru_dropout_workspace_bytes(int64_t S, int64_t Q, int64_t T, int32_t h) {
  return gru_workspace_floats(S, Q, T, h, true) * (int64_t)sizeof(float);
}
int64_t renet_gru_bwd_dropout_workspace_bytes(int64_t S, int64_t Q, int64_t T, int32_t h) {
  return gru_bwd_workspace_floats(S, Q, T, h, true) * (int64_t)sizeof(float);
}
int64_t renet_gru_dropout_workspace_bytes_len(int64_t S, int64_t Q, int64_t T, int32_t h, int32_t max_len) {
  return gru_workspace_floats(S, Q, T, h, true, max_len) * (int64_t)sizeof(float);
}
int64_t renet_gru_bwd_dropout_workspace_bytes_len(int64_t S, int64_t Q, int64_t T, int32_t h, int32_t max_len) {
  return gru_bwd_workspace_floats(S, Q, T, h, true, max_len) * (int64_t)sizeof(float);
}

int renet_gru_fwd_dropout(const float* H2, const int32_t* readout, const int32_t* row_glob, const float* glob,
                          const float* ent, const float* rel, const int32_t* row_seq, const int32_t* seq_s,
                          const int32_t* seq_r, const int32_t* seq_len, const int32_t* seq_start,
                          const int32_t* host_batch_sizes, int32_t max_len, const float* w_ih4, const float* w_hh4,
                          const float* b_ih4, const float* b_hh4, const float* w_ih3, const float* w_hh3, const float* b_ih3,
                          const float* b_hh3, float* hn4, float* hn3, int64_t S, int64_t Q, int64_t T, int32_t h, float p,
                          uint64_t seed, void* workspace, int64_t workspace_bytes, void* stream) {
  RENET_CHECK_ARG(S >= 0 && Q >= 0 && T >= 0 && h > 0 && max_len >= 0, "renet_gru_fwd_dropout: bad shape");
  RENET_CHECK_ARG(p > 0.f && p < 1.f, "renet_gru_fwd_dropout: p must be in (0, 1); use renet_gru_fwd for p = 0");
  if (S == 0 || Q == 0) return RENET_OK;
  RENET_CHECK_ARG(H2 && readout && row_glob && glob && ent && rel && row_seq && seq_s && seq_r && seq_len && seq_start &&
                      host_batch_sizes && w_ih4 && w_hh4 && b_ih4 && b_hh4 && w_ih3 && w_hh3 && b_ih3 && b_hh3 && hn4 &&
                      hn3 && workspace, "renet_gru_fwd_dropout: null pointer");
  RENET_CHECK_ARG(workspace_bytes >= renet_gru_dropout_workspace_bytes_len(S, Q, T, h, max_len),
                  "renet_gru_fwd_dropout: workspace of %lld bytes too small for max_len %d (needs %lld)", (long long)workspace_bytes,
                  max_len, (long long)renet_gru_dropout_workspace_bytes_len(S, Q, T, h, max_len));
  RENET_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 127) == 0, "renet_gru_fwd_dropout: workspace must be 128-byte aligned");
  return launch_gru_fwd(H2, readout, row_glob, glob, ent, rel, seq_s, seq_r, seq_len, seq_start, host_batch_sizes, max_len,
                        w_ih4, w_hh4, b_ih4, b_hh4, w_ih3, w_hh3, b_ih3, b_hh3, hn4, hn3, S, Q, T, h, (float*)workspace,
                        (cudaStream_t)stream, p, seed, row_seq);
}

int renet_gru_bwd_dropout(const float* H2, const int32_t* readout, const int32_t* row_glob, const float* glob,
                          const float* ent, const float* rel, const int32_t* row_seq, const int32_t* seq_s,
                          const int32_t* seq_r, const int32_t* seq_len, const int32_t* seq_start,
                          const int32_t* host_batch_sizes, int32_t max_len, const float* w_ih4, const float* w_hh4,
                          const float* w_ih3, const float* w_hh3, const float* dhn4, const float* dhn3, float* dH2,
                          float* d_ent, float* d_rel, float* d_glob, float* dw_ih4, float* dw_hh4, float* db_ih4,
                          float* db_hh4, float* dw_ih3, float* dw_hh3, float* db_ih3, float* db_hh3, int64_t N, int64_t S,
                          int64_t Q, int64_t T, int32_t h, float p, uint64_t seed, const void* fwd_workspace,
                          void* bwd_workspace, int64_t bwd_workspace_bytes, void* stream) {
  RENET_CHECK_ARG(N >= 0 && S >= 0 && Q >= 0 && T >= 0 && h > 0 && max_len >= 0, "renet_gru_bwd_dropout: bad shape");
  RENET_CHECK_ARG(p > 0.f && p < 1.f, "renet_gru_bwd_dropout: p must be in (0, 1)");
  if (S == 0 || Q == 0) return RENET_OK;
  RENET_CHECK_ARG(H2 && readout && row_glob && glob && ent && rel && row_seq && seq_s && seq_r && seq_len && seq_start &&
                      host_batch_sizes && w_ih4 && w_hh4 && w_ih3 && w_hh3 && dhn4 && dhn3 && dH2 && d_ent && d_rel && dw_ih4 &&
                      dw_hh4 && db_ih4 && db_hh4 && dw_ih3 && dw_hh3 && db_ih3 && db_hh3 && fwd_workspace && bwd_workspace,
                  "renet_gru_bwd_dropout: null pointer");
  RENET_CHECK_ARG(bwd_workspace_bytes >= renet_gru_bwd_dropout_workspace_bytes_len(S, Q, T, h, max_len),
                  "renet_gru_bwd_dropout: workspace of %lld bytes too small for max_len %d (needs %lld)",
                  (long long)bwd_workspace_bytes, max_len, (long long)renet_gru_bwd_dropout_workspace_bytes_len(S, Q, T, h, max_len));
  return launch_gru_bwd(H2, readout, row_glob, glob, ent, rel, seq_s, seq_r, seq_len, seq_start, host_batch_sizes, max_len, w_ih4,
                        w_hh4, w_ih3, w_hh3, dhn4, dhn3, dH2, d_ent, d_rel, d_glob, dw_ih4, dw_hh4, db_ih4, db_hh4, dw_ih3,
                        dw_hh3, db_ih3, db_hh3, N, S, Q, T, h, (const float*)fwd_workspace, (float*)bwd_workspace,
                        (cudaStream_t)stream, p, seed, row_seq);
}

int renet_gru_dense_fwd(const float* X4, int32_t k4, const float* X3, int32_t k3, const int32_t* seq_len,
                        const int32_t* seq_start, const int32_t* host_batch_sizes, int32_t max_len, const float* w_ih4,
                        const float* w_hh4, const float* b_ih4, const float* b_hh4, const float* w_ih3, const float* w_hh3,
                        const float* b_ih3, const float* b_hh3, float* hn4, float* hn3, int64_t S, int64_t Q, int32_t h,
                        void* workspace, int64_t workspace_bytes, void* stream) {
  RENET_CHECK_ARG(S >= 0 && Q >= 0 && h > 0 && max_len >= 0, "renet_gru_dense_fwd: bad shape");
  if (S == 0 || Q == 0) return RENET_OK;
  RENET_CHECK_ARG(X4 && seq_len && seq_start && host_batch_sizes && w_ih4 && w_hh4 && b_ih4 && b_hh4 && hn4 && hn3 && workspace,
                  "renet_gru_dense_fwd: null pointer");
  RENET_CHECK_ARG(X3 == nullptr || (w_ih3 && w_hh3 && b_ih3 && b_hh3), "renet_gru_dense_fwd: second encoder needs its weights");
  RENET_CHECK_ARG(workspace_bytes >= renet_gru_dropout_workspace_bytes_len(S, Q, 1, h, max_len),
                  "renet_gru_dense_fwd: workspace of %lld bytes too small for max_len %d (needs %lld)", (long long)workspace_bytes,
                  max_len, (long long)renet_gru_dropout_workspace_bytes_len(S, Q, 1, h, max_len));
  RENET_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 127) == 0, "renet_gru_dense_fwd: workspace must be 128-byte aligned");
  return launch_gru_fwd(nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, seq_len, seq_start,
                        host_batch_sizes, max_len, w_ih4, w_hh4, b_ih4, b_hh4, w_ih3, w_hh3, b_ih3, b_hh3, hn4, hn3, S, Q, 1, h,
                        (float*)workspace, (cudaStream_t)stream, 0.f, 0, nullptr, X4, k4, X3, k3);
}

int renet_gru_dense_bwd(const float* X4, int32_t k4, const float* X3, int32_t k3, const int32_t* seq_len,
                        const int32_t* seq_start, const int32_t* host_batch_sizes, int32_t max_len, const float* w_ih4,
                        const float* w_hh4, const float* w_ih3, const float* w_hh3, const float* dhn4, const float* dhn3,
                        float* dX4, float* dX3, float* dw_ih4, float* dw_hh4, float* db_ih4, float* db_hh4, float* dw_ih3,
                        float* dw_hh3, float* db_ih3, float* db_hh3, int64_t S, int64_t Q, int32_t h,
                        const void* fwd_workspace, void* bwd_workspace, int64_t bwd_workspace_bytes, void* stream) {
  RENET_CHECK_ARG(S >= 0 && Q >= 0 && h > 0 && max_len >= 0, "renet_gru_dense_bwd: bad shape");
  if (S == 0 || Q == 0) return RENET_OK;
  RENET_CHECK_ARG(X4 && seq_len && seq_start && host_batch_sizes && w_ih4 && w_hh4 && dhn4 && dhn3 && dX4 && dw_ih4 && dw_hh4 &&
                      db_ih4 && db_hh4 && fwd_workspace && bwd_workspace, "renet_gru_dense_bwd: null pointer");
  RENET_CHECK_ARG(X3 == nullptr || (w_ih3 && w_hh3 && dX3 && dw_ih3 && dw_hh3 && db_ih3 && db_hh3),
                  "renet_gru_dense_bwd: second encoder needs its weights and gradient buffers");
  RENET_CHECK_ARG(bwd_workspace_bytes >= renet_gru_bwd_dropout_workspace_bytes_len(S, Q, 1, h, max_len),
                  "renet_gru_dense_bwd: workspace of %lld bytes too small for max_len %d (needs %lld)",
                  (long long)bwd_workspace_bytes, max_len, (long long)renet_gru_bwd_dropout_workspace_bytes_len(S, Q, 1, h, max_len));
  return launch_gru_bwd(nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, seq_len, seq_start,
                        host_batch_sizes, max_len, w_ih4, w_hh4, w_ih3, w_hh3, dhn4, dhn3, nullptr, nullptr, nullptr, nullptr,
                        dw_ih4, dw_hh4, db_ih4, db_hh4, dw_ih3, dw_hh3, db_ih3, db_hh3, 0, S, Q, 1, h,
                        (const float*)fwd_workspace, (float*)bwd_workspace, (cudaStream_t)stream, 0.f, 0, nullptr, X4, k4, X3, k3,
                        dX4, dX3);
}

int renet_dropout_mask(uint64_t seed, uint64_t offset, int64_t n, float p, float* out, void* stream) {
  RENET_CHECK_ARG(n >= 0 && p >= 0.f && p < 1.f, "renet_dropout_mask: bad arguments");
  if (n == 0) return RENET_OK;
  RENET_CHECK_ARG(out != nullptr, "renet_dropout_mask: null pointer");
  return launch_dropout_mask(seed, offset, n, p, out, (cudaStream_t)stream);
}

int renet_encode_fwd(const float* ent, const int32_t* node_ent, const int32_t* row_ptr, const int32_t* col_src,
                     const int32_t* col_type, const float* norm, const float* W1, const float* Wloop1, const float* W2,
                     const float* Wloop2, float* H1, float* H2, int64_t N, int64_t E, int32_t R2, const int32_t* readout,
                     const int32_t* row_glob, const float* glob, const float* rel, const int32_t* seq_s,
                     const int32_t* seq_r, const int32_t* seq_len, const int32_t* seq_start,
                     const int32_t* host_batch_sizes, int32_t max_len, const float* w_ih4, const float* w_hh4,
                     const float* b_ih4, const float* b_hh4, const float* w_ih3, const float* w_hh3, const float* b_ih3,
                     const float* b_hh3, float* hn4, float* hn3, int64_t S, int64_t Q, int64_t T, int32_t h,
                     int32_t num_bases, const int32_t* sub_uniq, const int32_t* sub_readout, const int32_t* sub_row_ptr,
                     const int32_t* sub_col_src, const int32_t* sub_col_type, const float* sub_norm, const int32_t* hot_rel,
                     int32_t n_hot, void* workspace, int64_t workspace_bytes, void* stream) {
  RENET_CHECK_ARG(n_hot >= 0 && (n_hot == 0 || hot_rel != nullptr), "renet_encode_fwd: bad hot-relation list");
  if (n_hot == 0) hot_rel = nullptr;
  // a history graph without edges would pass h through both layers (DGL); layer 2 runs on the read-out sub-graph, where
  // that pass-through is not implemented, so such a batch is refused (RGCNAggregator rejects it before it gets here)
  RENET_CHECK_ARG(N == 0 || E > 0, "renet_encode_fwd: the history graph has no edges");
  // The part of the GRU that does not depend on the RGCN output -- weight packing, bias rows, the per-sequence and
  // per-timestamp input projections: four small launches, latency-bound, a handful of CTAs -- runs on a side stream
  // underneath the two RGCN layers (fork / join by events: the side stream is the device's, the event pair the caller
  // stream's, both created on first use, fork_acquire).
  cudaStream_t side = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  ForkLease lease{(cudaStream_t)stream};
  const bool gru_args_ok = S > 0 && Q > 0 && readout && row_glob && glob && rel && seq_s && seq_r && seq_len && seq_start &&
                           host_batch_sizes && w_ih4 && w_hh4 && b_ih4 && b_hh4 && w_ih3 && w_hh3 && b_ih3 && b_hh3 && hn4 && hn3 &&
                           workspace && workspace_bytes >= renet_gru_workspace_bytes_len(S, Q, T, h, max_len) &&
                           (reinterpret_cast<uintptr_t>(workspace) & 15) == 0 && max_len >= 0 && T >= 0;
  bool forked = false;
  if (gru_args_ok) {
    const int rc0 = fork_acquire((cudaStream_t)stream, &side, &ev_fork, &ev_join);
    if (rc0) return rc0;
    lease.held = true;
    RENET_CHECK_CUDA(cudaEventRecord(ev_fork, (cudaStream_t)stream));
    RENET_CHECK_CUDA(cudaStreamWaitEvent(side, ev_fork, 0));
    int rc1 = launch_gru_fwd(nullptr, readout, row_glob, glob, ent, rel, seq_s, seq_r, seq_len, seq_start, host_batch_sizes, max_len,
                             w_ih4, w_hh4, b_ih4, b_hh4, w_ih3, w_hh3, b_ih3, b_hh3, hn4, hn3, S, Q, T, h, (float*)workspace, side,
                             0.f, 0, nullptr, nullptr, 0, nullptr, 0, 1);
    RENET_CHECK_CUDA(cudaEventRecord(ev_join, side));
    if (rc1) return rc1;
    forked = true;
  }
  // layer 1 (embedding lookup fused through node_ent, ReLU), layer 2 (linear), then read-out + both GRUs
  int rc = check_layer_args("renet_encode_fwd", ent, W1, row_ptr, norm, H1, N, E, h, h, num_bases, R2);
  if (rc) return rc;
  RENET_CHECK_ARG(E == 0 || (col_src && col_type), "renet_encode_fwd: null edge arrays");
  if (N > 0) {
    if (Wloop1 != nullptr) {
      rc = sgemm_nn(ent, node_ent, h, Wloop1, h, H1, h, nullptr, N, h, h, false, (cudaStream_t)stream);
      if (rc) return rc;
    }
    rc = launch_rgcn_gather(ent, node_ent, W1, row_ptr, col_src, col_type, norm, H1, N, E, h, h, num_bases, 1,
                            Wloop1 != nullptr, (cudaStream_t)stream, R2, hot_rel, n_hot);
    if (rc) return rc;
  }
  if (sub_uniq != nullptr) {
    // layer 2 on the read-out sub-graph (renet_readout_subgraph): S compact destinations, sources = rows of H1
    RENET_CHECK_ARG(sub_readout && sub_row_ptr && sub_col_src && sub_col_type && sub_norm,
                    "renet_encode_fwd: incomplete read-out sub-graph");
    if (S > 0) {
      if (Wloop2 != nullptr) {
        rc = sgemm_nn(H1, sub_uniq, h, Wloop2, h, H2, h, nullptr, S, h, h, false, (cudaStream_t)stream);
        if (rc) return rc;
      }
      rc = launch_rgcn_gather(H1, nullptr, W2, sub_row_ptr, sub_col_src, sub_col_type, sub_norm, H2, S, E, h, h,
                              num_bases, 0, Wloop2 != nullptr, (cudaStream_t)stream, R2, hot_rel, n_hot);
      if (rc) return rc;
    }
    readout = sub_readout;
  } else {
    rc = renet_rgcn_block_fwd(H1, nullptr, W2, Wloop2, row_ptr, col_src, col_type, norm, H2, N, E, h, h, num_bases, R2, 0,
                              stream);
    if (rc) return rc;
  }
  if (forked) RENET_CHECK_CUDA(cudaStreamWaitEvent((cudaStream_t)stream, ev_join, 0));
  if (forked)
    return launch_gru_fwd(H2, readout, row_glob, glob, ent, rel, seq_s, seq_r, seq_len, seq_start, host_batch_sizes, max_len, w_ih4,
                          w_hh4, b_ih4, b_hh4, w_ih3, w_hh3, b_ih3, b_hh3, hn4, hn3, S, Q, T, h, (float*)workspace,
                          (cudaStream_t)stream, 0.f, 0, nullptr, nullptr, 0, nullptr, 0, 2);
  return renet_gru_fwd(H2, readout, row_glob, glob, ent, rel, seq_s, seq_r, seq_len, seq_start, host_batch_sizes, max_len,
                       w_ih4, w_hh4, b_ih4, b_hh4, w_ih3, w_hh3, b_ih3, b_hh3, hn4, hn3, S, Q, T, h, workspace,
                       workspace_bytes, stream);
}

int renet_prepare_sequences(const int64_t* triplets, int32_t ld, int32_t col_s, const int32_t* s_idx, int64_t Q,
                             const int32_t* comp_graph, const int32_t* row_comp, int64_t S, int32_t* seq_s,
                             int32_t* seq_r, int32_t* row_graph, void* stream) {
  RENET_CHECK_ARG(Q >= 0 && S >= 0 && (col_s == 0 || col_s == 2) && ld >= 3, "renet_prepare_sequences: bad arguments");
  const int64_t n = Q > S ? Q : S;
  if (n == 0) return RENET_OK;
  RENET_CHECK_ARG((Q == 0 || (triplets && s_idx && seq_s && seq_r)) && (S == 0 || (comp_graph && row_comp && row_graph)),
                  "renet_prepare_sequences: null pointer");
  renet::prepare_sequences_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      triplets, ld, col_s, s_idx, (int)Q, comp_graph, row_comp, (int)S, seq_s, seq_r, row_graph);
  RENET_CHECK_LAUNCH("prepare_sequences_kernel");
  return RENET_OK;
}

int renet_pack_inputs(const float* H2, const int32_t* readout, const int32_t* row_glob, const float* glob,
                      const float* ent, const float* rel, const int32_t* row_seq, const int32_t* seq_s,
                      const int32_t* seq_r, const int32_t* packed_row, float* X4, float* X3, int64_t S, int32_t h,
                      void* stream) {
  RENET_CHECK_ARG(S >= 0 && h > 0, "renet_pack_inputs: bad shape");
  if (S == 0) return RENET_OK;
  RENET_CHECK_ARG(H2 && readout && row_glob && glob && ent && rel && row_seq && seq_s && seq_r && packed_row &&
                      X4 && X3,
                  "renet_pack_inputs: null pointer");
  return launch_pack_inputs(H2, readout, row_glob, glob, ent, rel, row_seq, seq_s, seq_r, packed_row, X4, X3, S, h,
                            (cudaStream_t)stream);
}

}  // extern "C"
