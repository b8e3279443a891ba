// Decoder of RE-Net: logits = X @ W^T + b followed by cross-entropy (reference model.py:89-91 object prediction
// [B, 3h] x [3h, |E|]; model.py:97-100 relation prediction [B, 2h] x [2h, R]) -- SURVEY.md section 8(f) row 3.
//
// Forward: the wgmma 3xTF32 GEMM (umma_gemm.cu) with a fused epilogue: every (row, half column tile) reduces its
// logits to a running (max, sum of exp) pair and the target's logit, so the [B, |E|] logits (94 MB at ICEWS18) never
// reach memory; ce_reduce_kernel combines the 2*ceil(|E|/200) partials per row into logsumexp and the per-row loss.
// Backward: the logits are recomputed by the same GEMM with the gradient epilogue
//     dlogits = (softmax - onehot) * scale          (written row-major AND transposed)
// and the three gradients are tensor-core GEMMs / a row sum over it:
//     dX = dlogits @ W   (long K = |E|, 12 output tiles: split-K over the grid + partial sum)
//     dW += dlogits^T @ X,   db += rowsum(dlogits^T).
//
// Soft targets (reference utils.py:287-290, the global model's loss; renet_decoder_soft_ce_*): rows of P [M, N] are
// distributions that need not sum to 1.  The forward epilogue also reduces sum(P * logit) and sum(P) per (row, half
// column tile); soft_ce_reduce_kernel combines a row's partials in fp64 in a fixed order:
//     loss_i = lse_i * sum_c P_ic - sum_c P_ic z_ic,     dlogits_ic = (sum_c' P_ic' * softmax_ic - P_ic) * scale
// and the backward pass runs the same three products on that dlogits.  No float atomics: every sum has a fixed order.
//
// Grouped top-k (renet_decoder_group_topk; the test-time roll-over's candidate scoring, reference model.py:222-279 with
// pred_r_rank2, model.py:168-213): rows come in G groups of R, row m carries a weight w_m, and
//     p[m, n] = w_m * exp(z[m, n] - lse_m)
// is the joint probability of the reference's joint = p_e * p_o * p_r.  Per group, the k largest p and their flat indices
// r * N + n, without ever writing the [G*R, N] logits:
//   1. the EPI 1 pass without a target gives every (row, half column tile) partial max / sum of exp, then lse;
//   2. every partial max is an actual logit, so the k-th largest of w_m * exp(pmax - lse_m) over a group's R * n_part
//      partials is a lower bound tau_g of the group's k-th p (topk_tau_kernel, a block-wide radix select; 0 when the group
//      has fewer than k partials);
//   3. the EPI 5 pass recomputes the logits and appends every p >= tau_g to the group's candidate buffer; a group that
//      finds more candidates than the buffer holds is reported through *needed and nothing of the call is valid;
//   4. topk_final_kernel radix-selects the k-th (p descending, index ascending) candidate, so ties at the k-th value go to
//      the lower index, and bitonic-sorts the k winners into the output order in shared memory.
// Every step is either a fixed-order computation or an integer count, so the output is bitwise reproducible.
//
// Per-row top-k with exclusion lists (renet_decoder_topk; the forecast of RENet.forecast): the same four steps with R = 1
// and row weight 1, through the EXCL instantiations of the tau and final kernels.  Step 2 takes the (k + L_m)-th partial
// maximum of row m, L_m the length of its exclusion list, so that at least k admissible columns pass; step 4 drops the
// listed columns before the select.  The softmax stays over all N columns.
//
// Rank counts (test-time scoring, reference model.py:365-419): per row, the label's rank among the row's logits, raw and
// filtered against each of 0-2 exclusion lists (the static and the time-aware filter of evaluate_stream(time_aware=True)),
// by the tie rule #greater + (#equal - 1) / 2 + 1, without writing the [M, N] logits.  One rank pass (rank_counts below):
//   1. the EPI 1 pass with the label as target gives the partials and the label's logit tlogit; ce_reduce_kernel turns
//      them into lse and loss_rows;
//   2. the EPI 6 pass recomputes the logits with the same packed W, bias and tile mapping, so the label's own logit equals
//      tlogit bit for bit, and counts the logits above / equal to it and, per list, the sigmoids above / equal to the
//      label's with that list zeroed (the sigmoid of each logit computed once for all lists).  The counts are integers
//      added with integer atomics: the output is reproducible.
// Two entry points run it: renet_decoder_rank with at most one list and rows of 4 counts, renet_decoder_rank_multi with
// 0-2 lists and rows of 2 + 2 * n_lists.
#include "common.cuh"

namespace renet {
namespace {

inline int64_t align256(int64_t x) { return (x + 255) & ~int64_t(255); }
constexpr int kSplits = 12;

__global__ void ce_reduce_kernel(const float* __restrict__ pmax, const float* __restrict__ psum,
                                 const float* __restrict__ tlogit, int n_part, int64_t M, float* __restrict__ lse,
                                 float* __restrict__ loss_rows) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= M) return;
  float m = -3.0e38f;
  for (int i = 0; i < n_part; ++i) m = fmaxf(m, pmax[(int64_t)i * M + r]);
  float s = 0.f;
  for (int i = 0; i < n_part; ++i) s += psum[(int64_t)i * M + r] * expf(pmax[(int64_t)i * M + r] - m);
  const float l = m + logf(s);
  lse[r] = l;
  if (loss_rows != nullptr) loss_rows[r] = l - tlogit[r];
}

__global__ void soft_ce_reduce_kernel(const float* __restrict__ pmax, const float* __restrict__ psum,
                                      const float* __restrict__ pdot, const float* __restrict__ pmass, int n_part, int64_t M,
                                      float* __restrict__ lse, float* __restrict__ loss_rows, float* __restrict__ mass) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= M) return;
  double m = -3.0e38;
  for (int i = 0; i < n_part; ++i) m = fmax(m, (double)pmax[(int64_t)i * M + r]);
  double s = 0.0, pz = 0.0, pm = 0.0;
  for (int i = 0; i < n_part; ++i) {
    const int64_t j = (int64_t)i * M + r;
    s += (double)psum[j] * exp((double)pmax[j] - m);
    pz += (double)pdot[j];
    pm += (double)pmass[j];
  }
  const double l = m + log(s);
  lse[r] = (float)l;
  loss_rows[r] = (float)(l * pm - pz);
  mass[r] = (float)pm;
}

// db[c] += sum_r dT[c, r]   (one warp per class)
__global__ void rowsum_accum_kernel(const float* __restrict__ dT, int64_t ldT, int64_t M, int N, float* __restrict__ db) {
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (c >= N) return;
  float s = 0.f;
  for (int64_t r = lane; r < M; r += 32) s += dT[(int64_t)c * ldT + r];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) db[c] += s;
}

struct DecWs {
  uint8_t* Wp;      // packed W^T (B operand of the logits GEMM): logical B[k][n] = W[n*K + k]
  float *pmax, *psum, *tlogit;
  float *pdot, *pmass;   // soft targets only
  int64_t wp_bytes, total;
};
DecWs carve_fwd(void* base, int64_t M, int N, int K, bool soft = false) {
  DecWs w;
  char* p = (char*)base;
  int64_t off = 0;
  auto take = [&](int64_t bytes) { char* q = base ? p + off : nullptr; off += align256(bytes); return q; };
  const int n_part = 2 * ((N + 199) / 200);
  w.wp_bytes = umma_packed_bytes(N, K);
  w.Wp = (uint8_t*)take(w.wp_bytes);
  w.pmax = (float*)take((int64_t)n_part * M * 4);
  w.psum = (float*)take((int64_t)n_part * M * 4);
  w.tlogit = soft ? nullptr : (float*)take(M * 4);
  w.pdot = soft ? (float*)take((int64_t)n_part * M * 4) : nullptr;
  w.pmass = soft ? (float*)take((int64_t)n_part * M * 4) : nullptr;
  w.total = off;
  return w;
}
struct DecBwdWs {
  uint8_t *Wp, *Wkp, *Xp;   // W^T packed (logits), W packed as [K=|E|][N=K] (dX), X packed as [K=B][N=K] (dW)
  float *dlog, *dT, *parts;
  int64_t ldE, ldT, total;
};
DecBwdWs carve_bwd(void* base, int64_t M, int N, int K) {
  DecBwdWs w;
  char* p = (char*)base;
  int64_t off = 0;
  auto take = [&](int64_t bytes) { char* q = base ? p + off : nullptr; off += align256(bytes); return q; };
  w.ldE = (N + 3) / 4 * 4;
  w.ldT = (M + 3) / 4 * 4;
  w.Wp = (uint8_t*)take(umma_packed_bytes(N, K));
  w.Wkp = (uint8_t*)take(umma_packed_bytes(K, N));
  w.Xp = (uint8_t*)take(umma_packed_bytes(K, (int)M));
  w.dlog = (float*)take(M * w.ldE * 4);
  w.dT = (float*)take((int64_t)N * w.ldT * 4);
  w.parts = (float*)take((int64_t)kSplits * M * K * 4);
  w.total = off;
  return w;
}

// Steps 2-4 of the backward pass, shared by the hard- and soft-target decoders: dlogits (w.dlog, row-major) and its
// transpose (w.dT) are in the workspace.
int grad_products(const float* X, const float* W, float* dX, float* dW, float* dbias, int64_t M, int N, int K,
                  const DecBwdWs& w, cudaStream_t stream) {
  int rc;
  // 2. dX = dlogits @ W: A = dlogits [M, |E|], B[k][n] = W[k*K + n]; split-K partials, then their sum
  if ((rc = umma_pack_b(W, K, 1, K, N, w.Wkp, 0, stream))) return rc;
  EpiArgs none{};
  const int used = umma_gemm_prepacked_ex(w.dlog, nullptr, w.ldE, w.Wkp, w.parts, K, nullptr, M, K, N, false, 1, 0, 0, 0, 0, none,
                                          kSplits, M * (int64_t)K, stream);
  if (used < 0) return used;
  if ((rc = launch_sum_partials(w.parts, used, M * (int64_t)K, M, K, dX, K, false, stream))) return rc;
  // 3. dW += dlogits^T @ X: A = dT [|E|, M], B[k][n] = X[k*K + n]
  if ((rc = umma_pack_b(X, K, 1, K, (int)M, w.Xp, 0, stream))) return rc;
  rc = umma_gemm_prepacked_ex(w.dT, nullptr, w.ldT, w.Xp, dW, K, nullptr, N, K, (int)M, true, 1, 0, 0, 0, 0, none, 1, 0, stream);
  if (rc < 0) return rc;
  // 4. db += rowsum(dlogits^T)
  if (dbias != nullptr) {
    rowsum_accum_kernel<<<(unsigned)(((int64_t)N * 32 + 255) / 256), 256, 0, stream>>>(w.dT, w.ldT, M, N, dbias);
    RENET_CHECK_LAUNCH("rowsum_accum_kernel");
  }
  return RENET_OK;
}

// Step 1 of the backward pass: the pad columns / rows of dlogits and its transpose are zeroed (the GEMMs read them)
int zero_grad_pads(const DecBwdWs& w, int64_t M, int N, cudaStream_t stream) {
  if (w.ldE > N) RENET_CHECK_CUDA(cudaMemsetAsync(w.dlog, 0, (size_t)M * w.ldE * 4, stream));
  if (w.ldT > M) RENET_CHECK_CUDA(cudaMemsetAsync(w.dT, 0, (size_t)N * w.ldT * 4, stream));
  return RENET_OK;
}

// ---- grouped top-k ---------------------------------------------------------------------------------------------------
// Bits of a probability as an order-preserving unsigned key (p >= 0; -0 counts as +0)
__device__ __forceinline__ uint32_t prob_bits(float p) { return p > 0.f ? __float_as_uint(p) : 0u; }

// The k-th largest (1-based, k <= n) of the n keys key(0 .. n-1), block-wide: a radix select over 8-bit digits, most
// significant first.  Every thread gets the result.  hist: 256 ints of shared memory.
template <typename KeyT, typename F>
__device__ KeyT block_kth_largest(int64_t n, int64_t k, F key, int* hist) {
  __shared__ KeyT s_prefix;
  __shared__ int64_t s_rank;
  KeyT prefix = 0, mask = 0;
  int64_t rank = k;                                   // the rank still wanted among the keys that match prefix
  for (int shift = (int)sizeof(KeyT) * 8 - 8; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
      const KeyT v = key(i);
      if ((v & mask) == prefix) atomicAdd(hist + (int)((v >> shift) & 255), 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int64_t above = 0;
      int d = 255;
      for (; d > 0 && above + hist[d] < rank; --d) above += hist[d];
      s_prefix = prefix | ((KeyT)d << shift);
      s_rank = rank - above;
    }
    __syncthreads();
    prefix = s_prefix;
    rank = s_rank;
    mask |= (KeyT)255 << shift;
  }
  return prefix;
}

// tau[g] = the k-th largest of w_m * exp(pmax[i, m] - lse_m) over the rows m of group g and the partials i (0 when the
// group has fewer than k partials).  One block per group.
// EXCL (renet_decoder_topk): R = 1, every row weight is 1 (the kernel writes it to ones_out[g] for the EPI 5 pass), and
// row g has the exclusion list [excl_begin[g], excl_end[g]) (no lists when excl_begin is null).  The rank taken is k + L_g,
// L_g the list's length: each partial max is a real logit of its (row, half tile) unit and each excluded column lies in one
// unit, so at most L_g of the k + L_g largest partial maxima are excluded columns, and at least k admissible columns have
// p >= tau.
template <bool EXCL>
__global__ void __launch_bounds__(256) topk_tau_kernel(const float* __restrict__ pmax, const float* __restrict__ lse,
                                                       const float* __restrict__ row_w, int n_part, int R, int64_t M, int k,
                                                       float* __restrict__ tau, const int32_t* __restrict__ excl_begin = nullptr,
                                                       const int32_t* __restrict__ excl_end = nullptr,
                                                       float* __restrict__ ones_out = nullptr) {
  __shared__ int hist[256];
  const int64_t g = blockIdx.x;
  const int64_t n = (int64_t)R * n_part;
  int64_t rank = k;
  if constexpr (EXCL) {
    if (threadIdx.x == 0) ones_out[g] = 1.f;
    if (excl_begin != nullptr) rank += max(0, __ldg(excl_end + g) - __ldg(excl_begin + g));
  }
  if (n < rank) {
    if (threadIdx.x == 0) tau[g] = 0.f;
    return;
  }
  const int64_t m0 = g * R;
  auto key = [&](int64_t i) -> uint32_t {
    const int64_t part = i / R, m = m0 + (i - part * R);
    return prob_bits(topk_prob(__ldg(pmax + part * M + m), __ldg(lse + m), EXCL ? 1.f : __ldg(row_w + m)));
  };
  const uint32_t t = block_kth_largest<uint32_t>(n, rank, key, hist);
  if (threadIdx.x == 0) tau[g] = __uint_as_float(t);
}

constexpr int kTopkFinalThreads = 512;

// One block per group: the k best candidates by (p descending, index ascending), written in the caller's order.
// sort_n = the power of two >= k the shared-memory sort runs over.
// EXCL (renet_decoder_topk): R = 1, and the candidates in row g's exclusion list excl_col[excl_begin[g] .. excl_end[g])
// (ascending; no lists when excl_col is null) are dropped before the select.  When fewer than k candidates remain, the
// slots past them get index -1 and value 0.
template <bool EXCL>
__global__ void __launch_bounds__(kTopkFinalThreads) topk_final_kernel(const float* __restrict__ cand_val,
                                                                       const int32_t* __restrict__ cand_idx,
                                                                       const int32_t* __restrict__ count, int cap, int k,
                                                                       int order, int sort_n, float* __restrict__ values,
                                                                       int32_t* __restrict__ indices, int32_t* __restrict__ needed,
                                                                       const int32_t* __restrict__ excl_col = nullptr,
                                                                       const int32_t* __restrict__ excl_begin = nullptr,
                                                                       const int32_t* __restrict__ excl_end = nullptr) {
  extern __shared__ unsigned long long s_keys[];      // [sort_n]
  __shared__ int hist[256];
  __shared__ int s_fill;
  const int64_t g = blockIdx.x;
  const int n = count[g];
  if (n > cap) {                                       // the candidates did not fit: the caller retries with *needed
    if (threadIdx.x == 0) atomicMax(needed, n);
    return;
  }
  const float* cv = cand_val + g * cap;
  const int32_t* ci = cand_idx + g * cap;
  int xb = 0, xe = 0;
  if constexpr (EXCL) {
    if (excl_col != nullptr) {
      xb = __ldg(excl_begin + g);
      xe = __ldg(excl_end + g);
    }
  }
  auto excluded = [&](int32_t c) -> bool {            // binary search of the row's ascending list
    int lo = xb, hi = xe;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (__ldg(excl_col + mid) < c) lo = mid + 1; else hi = mid;
    }
    return lo < xe && __ldg(excl_col + lo) == c;
  };
  // larger key = better: p descending, then index ascending; keys are distinct because indices are.  EXCL: an excluded
  // candidate has key 0, below every real key (whose low word ~index is >= 2^31)
  auto key = [&](int64_t i) -> unsigned long long {
    if constexpr (EXCL) {
      if (xb < xe && excluded(ci[i])) return 0ull;
    }
    return ((unsigned long long)prob_bits(cv[i]) << 32) | (uint32_t)~(uint32_t)ci[i];
  };
  int kk = k;                                          // the winners: min(k, admissible candidates)
  if constexpr (EXCL) {
    if (threadIdx.x == 0) s_fill = 0;
    __syncthreads();
    int adm = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) adm += key(i) != 0ull;
    if (adm) atomicAdd(&s_fill, adm);
    __syncthreads();
    kk = min(k, s_fill);
    __syncthreads();
  }
  unsigned long long kth;
  if constexpr (EXCL) kth = kk > 0 ? block_kth_largest<unsigned long long>(n, kk, key, hist) : ~0ull;   // ~0: no real key
  else kth = block_kth_largest<unsigned long long>(n, k, key, hist);
  const uint32_t kth_p = (uint32_t)(kth >> 32);
  if (threadIdx.x == 0) s_fill = 0;
  __syncthreads();
  // the k winners, each as an ascending sort key of the output order:
  //   order 1: p descending, ties by index ascending
  //   order 0: index ascending among the p above the k-th p, then index ascending among those equal to it
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const unsigned long long v = key(i);
    if (v < kth) continue;
    const uint32_t p = (uint32_t)(v >> 32), idx = ~(uint32_t)v;
    const unsigned long long sk = order == 1 ? ((unsigned long long)~p << 32) | idx
                                             : ((unsigned long long)(p == kth_p) << 63) | ((unsigned long long)idx << 32) | p;
    s_keys[atomicAdd(&s_fill, 1)] = sk;
  }
  for (int i = kk + threadIdx.x; i < sort_n; i += blockDim.x) s_keys[i] = ~0ull;
  __syncthreads();
  for (int size = 2; size <= sort_n; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < sort_n / 2; i += blockDim.x) {
        const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
        const unsigned long long a = s_keys[lo], b = s_keys[hi];
        if ((a > b) == ((lo & size) == 0)) {
          s_keys[lo] = b;
          s_keys[hi] = a;
        }
      }
      __syncthreads();
    }
  }
  for (int j = threadIdx.x; j < k; j += blockDim.x) {
    if constexpr (EXCL) {
      if (j >= kk) {
        values[g * k + j] = 0.f;
        indices[g * k + j] = -1;
        continue;
      }
    }
    const unsigned long long sk = s_keys[j];
    uint32_t p, idx;
    if (order == 1) {
      p = ~(uint32_t)(sk >> 32);
      idx = (uint32_t)sk;
    } else {
      p = (uint32_t)sk;
      idx = (uint32_t)(sk >> 32) & 0x7fffffffu;
    }
    values[g * k + j] = __uint_as_float(p);
    indices[g * k + j] = (int32_t)idx;
  }
}

struct TopkWs {
  uint8_t* Wp;
  float *pmax, *psum, *lse, *tau, *cand_val;
  int32_t *count, *cand_idx;
  int64_t total;
};
TopkWs carve_topk(void* base, int64_t G, int R, int N, int K, int cap) {
  TopkWs w;
  char* p = (char*)base;
  int64_t off = 0;
  auto take = [&](int64_t bytes) { char* q = base ? p + off : nullptr; off += align256(bytes); return q; };
  const int64_t M = G * R;
  const int n_part = 2 * ((N + 199) / 200);
  w.Wp = (uint8_t*)take(umma_packed_bytes(N, K));
  w.pmax = (float*)take((int64_t)n_part * M * 4);
  w.psum = (float*)take((int64_t)n_part * M * 4);
  w.lse = (float*)take(M * 4);
  w.tau = (float*)take(G * 4);
  w.count = (int32_t*)take(G * 4);
  w.cand_val = (float*)take(G * cap * 4);
  w.cand_idx = (int32_t*)take(G * cap * 4);
  w.total = off;
  return w;
}

struct RankWs {
  DecWs fwd;
  float* lse;
  int64_t total;
};
RankWs carve_rank(void* base, int64_t M, int N, int K) {
  RankWs w;
  w.fwd = carve_fwd(base, M, N, K);
  w.lse = base ? (float*)((char*)base + w.fwd.total) : nullptr;
  w.total = w.fwd.total + align256(M * 4);
  return w;
}

// The rank pass of both rank entry points, after their argument checks: loss_rows, and counts [M, rank_ld] zeroed, then
// the raw pair and one filtered pair per list added (the columns past 2 + 2 * n_lists stay 0)
int rank_counts(const float* X, const float* W, const float* bias, const int32_t* label, int n_lists, const int32_t* excl_col,
                const int32_t* excl_begin, const int32_t* excl_end, float* loss_rows, int32_t* counts, int rank_ld, int64_t M,
                int N, int K, void* workspace, cudaStream_t stream) {
  void* base = (void*)(((uintptr_t)workspace + 255) & ~uintptr_t(255));
  RankWs w = carve_rank(base, M, N, K);
  RENET_CHECK_CUDA(cudaMemsetAsync(counts, 0, (size_t)M * rank_ld * 4, stream));
  // 1. lse, loss and the label's logit: the cross-entropy forward epilogue
  int rc = umma_pack_b(W, 1, K, N, K, w.fwd.Wp, 0, stream);          // logical B[k][n] = W[n*K + k]
  if (rc) return rc;
  EpiArgs epi{};
  epi.target = label; epi.pmax = w.fwd.pmax; epi.psum = w.fwd.psum; epi.tlogit = w.fwd.tlogit;
  rc = umma_gemm_prepacked_ex(X, nullptr, K, w.fwd.Wp, nullptr, 0, bias, M, N, K, false, 1, 0, 0, 0, 1, epi, 1, 0, stream);
  if (rc < 0) return rc;
  const int n_part = 2 * ((N + 199) / 200);
  ce_reduce_kernel<<<(unsigned)((M + 127) / 128), 128, 0, stream>>>(w.fwd.pmax, w.fwd.psum, w.fwd.tlogit, n_part, M, w.lse,
                                                                      loss_rows);
  RENET_CHECK_LAUNCH("ce_reduce_kernel");
  // 2. the counts against the label's logit, one filtered pair per list
  EpiArgs cnt{};
  cnt.target = label; cnt.tlogit = w.fwd.tlogit; cnt.excl_col = excl_col; cnt.excl_begin = excl_begin; cnt.excl_end = excl_end;
  cnt.rank_counts = counts; cnt.n_lists = n_lists; cnt.rank_ld = rank_ld;
  rc = umma_gemm_prepacked_ex(X, nullptr, K, w.fwd.Wp, nullptr, 0, bias, M, N, K, false, 1, 0, 0, 0, 6, cnt, 1, 0, stream);
  if (rc < 0) return rc;
  return RENET_OK;
}

}  // namespace
}  // namespace renet

using namespace renet;

extern "C" {

int64_t renet_decoder_ce_workspace_bytes(int64_t M, int32_t N, int32_t K) { return carve_fwd(nullptr, M, N, K).total + 256; }
int64_t renet_decoder_ce_bwd_workspace_bytes(int64_t M, int32_t N, int32_t K) { return carve_bwd(nullptr, M, N, K).total + 256; }

int renet_decoder_ce_fwd(const float* X, const float* W, const float* bias, const int32_t* target, float* loss_rows,
                         float* lse, int64_t M, int32_t N, int32_t K, void* workspace, int64_t workspace_bytes,
                         void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  RENET_CHECK_ARG(M >= 0 && N > 0 && K > 0 && K % 4 == 0, "renet_decoder_ce_fwd: bad shape (K must be a multiple of 4)");
  if (M == 0) return RENET_OK;
  RENET_CHECK_ARG(X && W && target && loss_rows && lse && workspace, "renet_decoder_ce_fwd: null pointer");
  RENET_CHECK_ARG(workspace_bytes >= renet_decoder_ce_workspace_bytes(M, N, K), "renet_decoder_ce_fwd: workspace too small");
  RENET_CHECK_ARG(((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(W)) & 15) == 0,
                  "renet_decoder_ce_fwd: X and W must be 16-byte aligned");
  void* base = (void*)(((uintptr_t)workspace + 255) & ~uintptr_t(255));
  DecWs w = carve_fwd(base, M, N, K);
  int rc = umma_pack_b(W, 1, K, N, K, w.Wp, 0, stream);          // logical B[k][n] = W[n*K + k]
  if (rc) return rc;
  EpiArgs epi{};
  epi.target = target; epi.pmax = w.pmax; epi.psum = w.psum; epi.tlogit = w.tlogit;
  rc = umma_gemm_prepacked_ex(X, nullptr, K, w.Wp, nullptr, 0, bias, M, N, K, false, 1, 0, 0, 0, 1, epi, 1, 0, stream);
  if (rc < 0) return rc;
  const int n_part = 2 * ((N + 199) / 200);
  ce_reduce_kernel<<<(unsigned)((M + 127) / 128), 128, 0, stream>>>(w.pmax, w.psum, w.tlogit, n_part, M, lse, loss_rows);
  RENET_CHECK_LAUNCH("ce_reduce_kernel");
  return RENET_OK;
}

int renet_decoder_ce_bwd(const float* X, const float* W, const float* bias, const int32_t* target, const float* lse,
                         float scale, const float* d_scale, float* dX, float* dW, float* dbias, int64_t M, int32_t N, int32_t K, void* workspace,
                         int64_t workspace_bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  RENET_CHECK_ARG(M >= 0 && N > 0 && K > 0 && K % 4 == 0, "renet_decoder_ce_bwd: bad shape (K must be a multiple of 4)");
  if (M == 0) return RENET_OK;
  RENET_CHECK_ARG(X && W && target && lse && dX && dW && workspace, "renet_decoder_ce_bwd: null pointer");
  RENET_CHECK_ARG(workspace_bytes >= renet_decoder_ce_bwd_workspace_bytes(M, N, K), "renet_decoder_ce_bwd: workspace too small");
  RENET_CHECK_ARG(((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(W)) & 15) == 0,
                  "renet_decoder_ce_bwd: X and W must be 16-byte aligned");
  void* base = (void*)(((uintptr_t)workspace + 255) & ~uintptr_t(255));
  DecBwdWs w = carve_bwd(base, M, N, K);
  int rc;
  // 1. recompute the logits, write dlogits (row-major, ld = ldE) and its transpose (ld = ldT)
  if ((rc = umma_pack_b(W, 1, K, N, K, w.Wp, 0, stream))) return rc;
  if ((rc = zero_grad_pads(w, M, N, stream))) return rc;
  EpiArgs epi{};
  epi.target = target; epi.lse = lse; epi.scale = scale; epi.dscale = d_scale; epi.dT = w.dT; epi.ldT = w.ldT;
  rc = umma_gemm_prepacked_ex(X, nullptr, K, w.Wp, w.dlog, w.ldE, bias, M, N, K, false, 1, 0, 0, 0, 2, epi, 1, 0, stream);
  if (rc < 0) return rc;
  return grad_products(X, W, dX, dW, dbias, M, N, K, w, stream);
}

int64_t renet_decoder_soft_ce_workspace_bytes(int64_t M, int32_t N, int32_t K) {
  return carve_fwd(nullptr, M, N, K, true).total + 256;
}
int64_t renet_decoder_soft_ce_bwd_workspace_bytes(int64_t M, int32_t N, int32_t K) { return carve_bwd(nullptr, M, N, K).total + 256; }

int renet_decoder_soft_ce_fwd(const float* X, const float* W, const float* bias, const float* P, int64_t ldp, float* loss_rows,
                              float* lse, float* psum, int64_t M, int32_t N, int32_t K, void* workspace, int64_t workspace_bytes,
                              void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  RENET_CHECK_ARG(M >= 0 && N > 0 && K > 0 && K % 4 == 0 && ldp >= N,
                  "renet_decoder_soft_ce_fwd: bad shape (K must be a multiple of 4, ldp >= N)");
  if (M == 0) return RENET_OK;
  RENET_CHECK_ARG(X && W && P && loss_rows && lse && psum && workspace, "renet_decoder_soft_ce_fwd: null pointer");
  RENET_CHECK_ARG(workspace_bytes >= renet_decoder_soft_ce_workspace_bytes(M, N, K), "renet_decoder_soft_ce_fwd: workspace too small");
  RENET_CHECK_ARG(((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(W)) & 15) == 0,
                  "renet_decoder_soft_ce_fwd: X and W must be 16-byte aligned");
  void* base = (void*)(((uintptr_t)workspace + 255) & ~uintptr_t(255));
  DecWs w = carve_fwd(base, M, N, K, true);
  int rc = umma_pack_b(W, 1, K, N, K, w.Wp, 0, stream);          // logical B[k][n] = W[n*K + k]
  if (rc) return rc;
  EpiArgs epi{};
  epi.pmax = w.pmax; epi.psum = w.psum; epi.soft = P; epi.ldp = ldp; epi.pdot = w.pdot; epi.pmass = w.pmass;
  rc = umma_gemm_prepacked_ex(X, nullptr, K, w.Wp, nullptr, 0, bias, M, N, K, false, 1, 0, 0, 0, 3, epi, 1, 0, stream);
  if (rc < 0) return rc;
  const int n_part = 2 * ((N + 199) / 200);
  soft_ce_reduce_kernel<<<(unsigned)((M + 127) / 128), 128, 0, stream>>>(w.pmax, w.psum, w.pdot, w.pmass, n_part, M, lse,
                                                                          loss_rows, psum);
  RENET_CHECK_LAUNCH("soft_ce_reduce_kernel");
  return RENET_OK;
}

int renet_decoder_soft_ce_bwd(const float* X, const float* W, const float* bias, const float* P, int64_t ldp, const float* lse,
                              const float* psum, float scale, const float* d_scale, float* dX, float* dW, float* dbias, int64_t M,
                              int32_t N, int32_t K, void* workspace, int64_t workspace_bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  RENET_CHECK_ARG(M >= 0 && N > 0 && K > 0 && K % 4 == 0 && ldp >= N,
                  "renet_decoder_soft_ce_bwd: bad shape (K must be a multiple of 4, ldp >= N)");
  if (M == 0) return RENET_OK;
  RENET_CHECK_ARG(X && W && P && lse && psum && dX && dW && workspace, "renet_decoder_soft_ce_bwd: null pointer");
  RENET_CHECK_ARG(workspace_bytes >= renet_decoder_soft_ce_bwd_workspace_bytes(M, N, K),
                  "renet_decoder_soft_ce_bwd: workspace too small");
  RENET_CHECK_ARG(((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(W)) & 15) == 0,
                  "renet_decoder_soft_ce_bwd: X and W must be 16-byte aligned");
  void* base = (void*)(((uintptr_t)workspace + 255) & ~uintptr_t(255));
  DecBwdWs w = carve_bwd(base, M, N, K);
  int rc;
  // 1. recompute the logits, write dlogits (row-major, ld = ldE) and its transpose (ld = ldT)
  if ((rc = umma_pack_b(W, 1, K, N, K, w.Wp, 0, stream))) return rc;
  if ((rc = zero_grad_pads(w, M, N, stream))) return rc;
  EpiArgs epi{};
  epi.lse = lse; epi.scale = scale; epi.dscale = d_scale; epi.dT = w.dT; epi.ldT = w.ldT;
  epi.soft = P; epi.ldp = ldp; epi.rowmass = psum;
  rc = umma_gemm_prepacked_ex(X, nullptr, K, w.Wp, w.dlog, w.ldE, bias, M, N, K, false, 1, 0, 0, 0, 4, epi, 1, 0, stream);
  if (rc < 0) return rc;
  return grad_products(X, W, dX, dW, dbias, M, N, K, w, stream);
}

int64_t renet_decoder_group_topk_workspace_bytes(int64_t G, int32_t R, int32_t N, int32_t K, int32_t capacity) {
  return carve_topk(nullptr, G, R, N, K, capacity).total + 256;
}

int renet_decoder_group_topk(const float* X, const float* W, const float* bias, const float* row_weight, int64_t G, int32_t R,
                             int32_t N, int32_t K, int32_t k, int32_t order, int32_t capacity, float* values, int32_t* indices,
                             int32_t* needed, void* workspace, int64_t workspace_bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  RENET_CHECK_ARG(G >= 0 && R > 0 && N > 0 && K > 0 && K % 4 == 0 && (int64_t)R * N < (int64_t(1) << 31),
                  "renet_decoder_group_topk: bad shape (K must be a multiple of 4, R * N < 2^31)");
  RENET_CHECK_ARG(k >= 1 && (int64_t)k <= (int64_t)R * N, "renet_decoder_group_topk: k = %d outside [1, R * N = %lld]", k,
                  (long long)R * N);
  RENET_CHECK_ARG(k <= RENET_TOPK_MAX_K, "renet_decoder_group_topk: k = %d above RENET_TOPK_MAX_K = %d", k, RENET_TOPK_MAX_K);
  RENET_CHECK_ARG(order == RENET_TOPK_ORDER_INDEX || order == RENET_TOPK_ORDER_VALUE, "renet_decoder_group_topk: unknown order %d",
                  order);
  RENET_CHECK_ARG(capacity >= k, "renet_decoder_group_topk: capacity %d < k = %d", capacity, k);
  RENET_CHECK_ARG(needed != nullptr, "renet_decoder_group_topk: null pointer");
  if (G == 0) return RENET_OK;
  RENET_CHECK_ARG(X && W && row_weight && values && indices && workspace, "renet_decoder_group_topk: null pointer");
  RENET_CHECK_ARG(workspace_bytes >= renet_decoder_group_topk_workspace_bytes(G, R, N, K, capacity),
                  "renet_decoder_group_topk: workspace too small");
  RENET_CHECK_ARG(((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(W)) & 15) == 0,
                  "renet_decoder_group_topk: X and W must be 16-byte aligned");
  static bool attr = false;
  if (!attr) {
    RENET_CHECK_CUDA(cudaFuncSetAttribute(topk_final_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, RENET_TOPK_MAX_K * 8));
    attr = true;
  }
  void* base = (void*)(((uintptr_t)workspace + 255) & ~uintptr_t(255));
  TopkWs w = carve_topk(base, G, R, N, K, capacity);
  const int64_t M = G * R;
  const int n_part = 2 * ((N + 199) / 200);
  RENET_CHECK_CUDA(cudaMemsetAsync(needed, 0, 4, stream));
  RENET_CHECK_CUDA(cudaMemsetAsync(w.count, 0, (size_t)G * 4, stream));
  // 1. lse of every row: the cross-entropy forward epilogue without a target
  int rc = umma_pack_b(W, 1, K, N, K, w.Wp, 0, stream);          // logical B[k][n] = W[n*K + k]
  if (rc) return rc;
  EpiArgs epi{};
  epi.pmax = w.pmax; epi.psum = w.psum;
  rc = umma_gemm_prepacked_ex(X, nullptr, K, w.Wp, nullptr, 0, bias, M, N, K, false, 1, 0, 0, 0, 1, epi, 1, 0, stream);
  if (rc < 0) return rc;
  ce_reduce_kernel<<<(unsigned)((M + 127) / 128), 128, 0, stream>>>(w.pmax, w.psum, nullptr, n_part, M, w.lse, nullptr);
  RENET_CHECK_LAUNCH("ce_reduce_kernel");
  // 2. per-group threshold from the partial maxima
  topk_tau_kernel<false><<<(unsigned)G, 256, 0, stream>>>(w.pmax, w.lse, row_weight, n_part, R, M, k, w.tau);
  RENET_CHECK_LAUNCH("topk_tau_kernel");
  // 3. the candidates at or above it
  EpiArgs sel{};
  sel.lse = w.lse; sel.row_w = row_weight; sel.tau = w.tau; sel.sel_count = w.count; sel.sel_val = w.cand_val;
  sel.sel_idx = w.cand_idx; sel.sel_R = R; sel.sel_cap = capacity;
  rc = umma_gemm_prepacked_ex(X, nullptr, K, w.Wp, nullptr, 0, bias, M, N, K, false, 1, 0, 0, 0, 5, sel, 1, 0, stream);
  if (rc < 0) return rc;
  // 4. the k best of each group's candidates, in the requested order
  int sort_n = 2;
  while (sort_n < k) sort_n <<= 1;
  topk_final_kernel<false><<<(unsigned)G, kTopkFinalThreads, (size_t)sort_n * 8, stream>>>(w.cand_val, w.cand_idx, w.count,
                                                                                            capacity, k, order, sort_n, values,
                                                                                            indices, needed);
  RENET_CHECK_LAUNCH("topk_final_kernel");
  return RENET_OK;
}

int64_t renet_decoder_topk_workspace_bytes(int64_t M, int32_t N, int32_t K, int32_t capacity) {
  return carve_topk(nullptr, M, 1, N, K, capacity).total + align256(M * 4) + 256;
}

int renet_decoder_topk(const float* X, const float* W, const float* bias, const int32_t* excl_col, const int32_t* excl_begin,
                       const int32_t* excl_end, int64_t M, int32_t N, int32_t K, int32_t k, int32_t capacity, float* values,
                       int32_t* indices, int32_t* needed, void* workspace, int64_t workspace_bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  RENET_CHECK_ARG(M >= 0 && N > 0 && K > 0 && K % 4 == 0, "renet_decoder_topk: bad shape (K must be a multiple of 4)");
  RENET_CHECK_ARG(k >= 1 && k <= N, "renet_decoder_topk: k = %d outside [1, N = %d]", k, N);
  RENET_CHECK_ARG(k <= RENET_TOPK_MAX_K, "renet_decoder_topk: k = %d above RENET_TOPK_MAX_K = %d", k, RENET_TOPK_MAX_K);
  RENET_CHECK_ARG(capacity >= k, "renet_decoder_topk: capacity %d < k = %d", capacity, k);
  RENET_CHECK_ARG(excl_col == nullptr || (excl_begin != nullptr && excl_end != nullptr),
                  "renet_decoder_topk: exclusion lists need excl_begin and excl_end");
  RENET_CHECK_ARG(needed != nullptr, "renet_decoder_topk: null pointer");
  if (M == 0) return RENET_OK;
  RENET_CHECK_ARG(X && W && values && indices && workspace, "renet_decoder_topk: null pointer");
  RENET_CHECK_ARG(workspace_bytes >= renet_decoder_topk_workspace_bytes(M, N, K, capacity), "renet_decoder_topk: workspace too small");
  RENET_CHECK_ARG(((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(W)) & 15) == 0,
                  "renet_decoder_topk: X and W must be 16-byte aligned");
  static bool attr = false;
  if (!attr) {
    RENET_CHECK_CUDA(cudaFuncSetAttribute(topk_final_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, RENET_TOPK_MAX_K * 8));
    attr = true;
  }
  void* base = (void*)(((uintptr_t)workspace + 255) & ~uintptr_t(255));
  TopkWs w = carve_topk(base, M, 1, N, K, capacity);
  float* ones = (float*)((char*)base + w.total);                 // every row's weight, 1: the EPI 5 pass reads it
  const int32_t* xb = excl_col != nullptr ? excl_begin : nullptr;
  const int32_t* xe = excl_col != nullptr ? excl_end : nullptr;
  const int n_part = 2 * ((N + 199) / 200);
  RENET_CHECK_CUDA(cudaMemsetAsync(needed, 0, 4, stream));
  RENET_CHECK_CUDA(cudaMemsetAsync(w.count, 0, (size_t)M * 4, stream));
  // 1. lse of every row (k_splits = 1: a row's logits and partials do not depend on the other rows)
  int rc = umma_pack_b(W, 1, K, N, K, w.Wp, 0, stream);          // logical B[k][n] = W[n*K + k]
  if (rc) return rc;
  EpiArgs epi{};
  epi.pmax = w.pmax; epi.psum = w.psum;
  rc = umma_gemm_prepacked_ex(X, nullptr, K, w.Wp, nullptr, 0, bias, M, N, K, false, 1, 0, 0, 0, 1, epi, 1, 0, stream);
  if (rc < 0) return rc;
  ce_reduce_kernel<<<(unsigned)((M + 127) / 128), 128, 0, stream>>>(w.pmax, w.psum, nullptr, n_part, M, w.lse, nullptr);
  RENET_CHECK_LAUNCH("ce_reduce_kernel");
  // 2. per-row threshold at rank k + L_m of the partial maxima, and the row weights of 1
  topk_tau_kernel<true><<<(unsigned)M, 256, 0, stream>>>(w.pmax, w.lse, nullptr, n_part, 1, M, k, w.tau, xb, xe, ones);
  RENET_CHECK_LAUNCH("topk_tau_kernel");
  // 3. every p >= tau, excluded columns included
  EpiArgs sel{};
  sel.lse = w.lse; sel.row_w = ones; sel.tau = w.tau; sel.sel_count = w.count; sel.sel_val = w.cand_val;
  sel.sel_idx = w.cand_idx; sel.sel_R = 1; sel.sel_cap = capacity;
  rc = umma_gemm_prepacked_ex(X, nullptr, K, w.Wp, nullptr, 0, bias, M, N, K, false, 1, 0, 0, 0, 5, sel, 1, 0, stream);
  if (rc < 0) return rc;
  // 4. the k best admissible candidates of each row, p descending
  int sort_n = 2;
  while (sort_n < k) sort_n <<= 1;
  topk_final_kernel<true><<<(unsigned)M, kTopkFinalThreads, (size_t)sort_n * 8, stream>>>(
      w.cand_val, w.cand_idx, w.count, capacity, k, RENET_TOPK_ORDER_VALUE, sort_n, values, indices, needed, excl_col, xb, xe);
  RENET_CHECK_LAUNCH("topk_final_kernel");
  return RENET_OK;
}

int64_t renet_decoder_rank_workspace_bytes(int64_t M, int32_t N, int32_t K) { return carve_rank(nullptr, M, N, K).total + 256; }

int renet_decoder_rank(const float* X, const float* W, const float* bias, const int32_t* label, const int32_t* excl_col,
                       const int32_t* excl_begin, const int32_t* excl_end, float* loss_rows, int32_t* counts, int64_t M, int32_t N,
                       int32_t K, void* workspace, int64_t workspace_bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  RENET_CHECK_ARG(M >= 0 && N > 0 && K > 0 && K % 4 == 0, "renet_decoder_rank: bad shape (K must be a multiple of 4)");
  if (M == 0) return RENET_OK;
  RENET_CHECK_ARG(X && W && label && loss_rows && counts && workspace, "renet_decoder_rank: null pointer");
  RENET_CHECK_ARG(excl_col == nullptr || (excl_begin != nullptr && excl_end != nullptr),
                  "renet_decoder_rank: exclusion lists need excl_begin and excl_end");
  RENET_CHECK_ARG(workspace_bytes >= renet_decoder_rank_workspace_bytes(M, N, K), "renet_decoder_rank: workspace too small");
  RENET_CHECK_ARG(((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(W)) & 15) == 0,
                  "renet_decoder_rank: X and W must be 16-byte aligned");
  // always 4 counts per row: without a list the filtered pair stays 0
  return rank_counts(X, W, bias, label, excl_col != nullptr ? 1 : 0, excl_col, excl_begin, excl_end, loss_rows, counts, 4, M, N,
                     K, workspace, stream);
}

int renet_decoder_rank_multi(const float* X, const float* W, const float* bias, const int32_t* label, int32_t n_lists,
                             const int32_t* excl_col, const int32_t* excl_begin, const int32_t* excl_end, float* loss_rows,
                             int32_t* counts, int64_t M, int32_t N, int32_t K, void* workspace, int64_t workspace_bytes,
                             void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  RENET_CHECK_ARG(M >= 0 && N > 0 && K > 0 && K % 4 == 0, "renet_decoder_rank_multi: bad shape (K must be a multiple of 4)");
  RENET_CHECK_ARG(n_lists >= 0 && n_lists <= 2, "renet_decoder_rank_multi: n_lists = %d outside 0..2", n_lists);
  RENET_CHECK_ARG(n_lists == 0 || excl_col != nullptr, "renet_decoder_rank_multi: n_lists = %d needs excl_col", n_lists);
  RENET_CHECK_ARG(n_lists == 0 || (excl_begin != nullptr && excl_end != nullptr),
                  "renet_decoder_rank_multi: n_lists = %d needs excl_begin and excl_end", n_lists);
  if (M == 0) return RENET_OK;
  RENET_CHECK_ARG(X && W && label && loss_rows && counts && workspace, "renet_decoder_rank_multi: null pointer");
  RENET_CHECK_ARG(workspace_bytes >= renet_decoder_rank_workspace_bytes(M, N, K), "renet_decoder_rank_multi: workspace too small");
  RENET_CHECK_ARG(((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(W)) & 15) == 0,
                  "renet_decoder_rank_multi: X and W must be 16-byte aligned");
  return rank_counts(X, W, bias, label, n_lists, excl_col, excl_begin, excl_end, loss_rows, counts, 2 + 2 * n_lists, M, N, K,
                     workspace, stream);
}

}  // extern "C"
