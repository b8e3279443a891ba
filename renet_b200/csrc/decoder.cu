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
  loss_rows[r] = l - tlogit[r];
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
  int64_t wp_bytes, total;
};
DecWs carve_fwd(void* base, int64_t M, int N, int K) {
  DecWs w;
  char* p = (char*)base;
  int64_t off = 0;
  auto take = [&](int64_t bytes) { char* q = base ? p + off : nullptr; off += align256(bytes); return q; };
  const int n_part = 2 * ((N + 199) / 200);
  w.wp_bytes = umma_packed_bytes(N, K);
  w.Wp = (uint8_t*)take(w.wp_bytes);
  w.pmax = (float*)take((int64_t)n_part * M * 4);
  w.psum = (float*)take((int64_t)n_part * M * 4);
  w.tlogit = (float*)take(M * 4);
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
  void* base = (void*)(((uintptr_t)workspace + 255) & ~uintptr_t(255));
  DecBwdWs w = carve_bwd(base, M, N, K);
  int rc;
  // 1. recompute the logits, write dlogits (row-major, ld = ldE) and its transpose (ld = ldT)
  if ((rc = umma_pack_b(W, 1, K, N, K, w.Wp, 0, stream))) return rc;
  if (w.ldE > N) RENET_CHECK_CUDA(cudaMemsetAsync(w.dlog, 0, (size_t)M * w.ldE * 4, stream));     // zero the pad columns
  if (w.ldT > M) RENET_CHECK_CUDA(cudaMemsetAsync(w.dT, 0, (size_t)N * w.ldT * 4, stream));
  EpiArgs epi{};
  epi.target = target; epi.lse = lse; epi.scale = scale; epi.dscale = d_scale; epi.dT = w.dT; epi.ldT = w.ldT;
  rc = umma_gemm_prepacked_ex(X, nullptr, K, w.Wp, w.dlog, w.ldE, bias, M, N, K, false, 1, 0, 0, 0, 2, epi, 1, 0, stream);
  if (rc < 0) return rc;
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

}  // extern "C"
