// Persistent tensor-core GRU recurrence (both encoders, all time steps, ONE cooperative launch).
//
// The reference runs nn.GRU / cuDNN over packed sequences (model.py:86,94).  Per time step the work is tiny
// (n_act <= 1024 sequences x 200 x 1200), so separate GEMM + gate launches are pure latency.  Here:
//   * CTA (encoder e, unit slice j of 32 hidden units, 128-sequence tile) keeps ITS slice of W_hh -- the r, z and n
//     rows of its 32 units, split hi/lo for 3xTF32, K-major, 128-byte swizzled: 172 KB -- resident in shared memory
//     for the whole kernel;
//   * every step it stages its 128 x 200 tile of h_{t-1} (ld.global.cg: written by other SMs one step earlier),
//     issues 84 wgmma per warpgroup (M=64 rows each, N=96, K=8) into register accumulators, and the epilogue adds the
//     pre-computed input projections GI[row] + PQ[q] + PT[timestamp], applies the gate math and writes h_t (and the
//     recurrent pre-activations GH, which the backward pass re-uses);
//   * steps are separated by a grid-wide barrier (atomic counter; the launch is cooperative so all CTAs are resident).
// Outputs match gru.cu's step-by-step path bit-for-bit in layout: Hs [(L+1), Q, 2h], GH [L, Q, 6h], hn4, hn3.
#include <algorithm>

#include "common.cuh"
#include "umma.cuh"

namespace renet {
namespace {

constexpr int RU = 32;                    // hidden units per CTA
constexpr int RN = 3 * RU;                // 96 accumulator columns: r | z | n of the slice
constexpr int R_BK = 32;
constexpr int R_THREADS = 256;
constexpr int R_A_BYTES = 128 * 128;      // one 32-wide K chunk of the 128-row h tile (hi or lo plane)
constexpr int R_B_PLANE = RN * 128;       // 12288
constexpr int R_MAX_CHUNKS = 7;           // h <= 224
constexpr int R_SMEM = R_MAX_CHUNKS * 2 * R_B_PLANE + 2 * R_A_BYTES + 1024 + 128;
constexpr int R_MAX_LEN = 64;             // longest call the kernel takes: its per-step active counts go by value (256 B)

struct StepCounts { int n[R_MAX_LEN]; };

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float4 ldcg_f4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }

__device__ __forceinline__ void grid_barrier(unsigned int* counter, unsigned int target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1u);
    int spins = 0;
    while (*reinterpret_cast<volatile unsigned int*>(counter) < target) {
      if (++spins > (1 << 24)) __trap();       // never hang the GPU
    }
    __threadfence();
  }
  __syncthreads();
}

__global__ void __launch_bounds__(R_THREADS, 1)
gru_recur_kernel(const float* __restrict__ GI, const float* __restrict__ PQ, const float* __restrict__ PT,
                 const float* __restrict__ bhh, const int32_t* __restrict__ row_glob,
                 const int32_t* __restrict__ seq_start, const int32_t* __restrict__ seq_len,
                 const float* __restrict__ w_hh4, const float* __restrict__ w_hh3, float* __restrict__ Hs,
                 float* __restrict__ GH, float* __restrict__ hn4, float* __restrict__ hn3, unsigned int* barrier_counter,
                 StepCounts counts, int max_len, int Q, int h) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024 - (raw & 1023)) & 1023);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int enc = blockIdx.y, slice = blockIdx.x;
  const int u0 = slice * RU;
  const int nu = min(RU, h - u0);                       // valid units in this slice
  const int n_chunks = (h + R_BK - 1) / R_BK;
  uint8_t* sB = smem;                                   // [chunk][hi,lo][96 rows x 128 B]
  uint8_t* sA = smem + R_MAX_CHUNKS * 2 * R_B_PLANE;    // [hi,lo][128 rows x 128 B]
  const uint32_t smem_base = smem_u32(smem);
  const int wg = tid >> 7;                              // warpgroup: accumulator rows [64 wg, 64 wg + 64) of the tile
  // ---- W_hh slice -> shared memory (once): row n' = g*32 + ul  <-  w_hh[g*h + u0 + ul][k] ----------------------------
  const float* w_hh = enc == 0 ? w_hh4 : w_hh3;
  for (int task = tid; task < RN * 8 * n_chunks; task += R_THREADS) {
    const int c = task / (RN * 8), rem = task % (RN * 8);
    const int n = rem >> 3, j = rem & 7;
    const int g = n / RU, ul = n % RU;
    const int k = c * R_BK + 4 * j;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ul < nu && k < h) v = ldg_f4(w_hh + (int64_t)(g * h + u0 + ul) * h + k);
    float4 hi, lo;
    split4(v, hi, lo);
    const uint32_t off = sw128_offset(n, j);
    *reinterpret_cast<float4*>(sB + (size_t)c * 2 * R_B_PLANE + off) = hi;
    *reinterpret_cast<float4*>(sB + (size_t)c * 2 * R_B_PLANE + R_B_PLANE + off) = lo;
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  const unsigned int n_ctas = gridDim.x * gridDim.y * gridDim.z;
  const int n_mtiles = (Q + 127) / 128;
  const int64_t hs_stride = (int64_t)Q * 2 * h;
  float acc[RN / 2];
#pragma unroll
  for (int i = 0; i < RN / 2; ++i) acc[i] = 0.f;
  int a_uses = 0;

  for (int t = 0; t < max_len; ++t) {
    const int n_act = counts.n[t];
    if (n_act <= 0) break;
    const float* Hprev = Hs + (int64_t)t * hs_stride;
    float* Hnext = Hs + (int64_t)(t + 1) * hs_stride;
    float* GHt = GH + (int64_t)t * Q * 6 * h;
    for (int mt = blockIdx.z; mt < n_mtiles && mt * 128 < n_act; mt += gridDim.z) {
      const int q0 = mt * 128;
      // ---- (1) everything that does not depend on the MMAs is fetched first: all K chunks of this tile's h_{t-1} rows
      //          (registers) and the input-projection sums GI[row] + PQ[q] + PT[timestamp] + b_hh of the thread's 16 units
      float4 areg[R_MAX_CHUNKS][4];
      if (t > 0) {
#pragma unroll
        for (int c = 0; c < R_MAX_CHUNKS; ++c) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int task = tid + i * R_THREADS;
            const int r = task >> 3, j = task & 7;
            const int qq = q0 + r, k = c * R_BK + 4 * j;
            areg[c][i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (c < n_chunks && qq < n_act && k < h) areg[c][i] = ldcg_f4(Hprev + (int64_t)qq * 2 * h + enc * h + k);
          }
        }
      }
      if (t > 0) {
        // ---- (2) gh = h_{t-1}[tile] @ W_hh_slice^T on the tensor cores: per chunk only split + store + 12 MMAs ----------
#pragma unroll
        for (int c = 0; c < R_MAX_CHUNKS; ++c) {
          if (c < n_chunks) {
            if (a_uses > 0) {                                  // previous MMAs (both warpgroups) have read sA
              wgmma_wait<0>();
              acc_fence(acc);
              __syncthreads();
            }
            ++a_uses;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int task = tid + i * R_THREADS;
              const int r = task >> 3, j = task & 7;
              float4 hi, lo;
              split4(areg[c][i], hi, lo);
              const uint32_t off = sw128_offset(r, j);
              *reinterpret_cast<float4*>(sA + off) = hi;
              *reinterpret_cast<float4*>(sA + R_A_BYTES + off) = lo;
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncthreads();
            const uint32_t a_hi = smem_base + R_MAX_CHUNKS * 2 * R_B_PLANE + wg * 64 * 128, a_lo = a_hi + R_A_BYTES;
            const uint32_t b_hi = smem_base + c * 2 * R_B_PLANE, b_lo = b_hi + R_B_PLANE;
            wgmma_fence();
            acc_fence(acc);
#pragma unroll
            for (int ks = 0; ks < R_BK / 8; ++ks) {
              const uint32_t ko = ks * 32;
              const uint64_t dAh = make_desc_sw128(a_hi + ko), dAl = make_desc_sw128(a_lo + ko);
              const uint64_t dBh = make_desc_sw128(b_hi + ko), dBl = make_desc_sw128(b_lo + ko);
              wgmma_tf32_n96(acc, dAh, dBh, (c | ks) != 0);
              wgmma_tf32_n96(acc, dAl, dBh, 1);
              wgmma_tf32_n96(acc, dAh, dBl, 1);
            }
            wgmma_commit();
          }
        }
        wgmma_wait<0>();
        acc_fence(acc);
        __syncthreads();                                       // sA is free: it holds the epilogue tile below
      }
      // ---- (3) epilogue.  The accumulator fragments are spread over the warpgroup's threads, but all global operands are
      //      row-major: the tile goes through shared memory (the free A buffer, two halves of 64 rows) and is then
      //      processed one row per warp with lane = hidden unit, so every global access is a coalesced 128-byte segment
      //      (the strided version moved 2.4x the bytes).
      constexpr int TS = RN + 4;                           // padded row stride: conflict-free 16-byte stores
      float* sT = reinterpret_cast<float*>(sA);            // [64 rows][100] floats = 25.6 KB
#pragma unroll 1
      for (int half_rows = 0; half_rows < 2; ++half_rows) {
        if (t > 0 && wg == half_rows) acc_store(acc, sT, TS, tid & 127);   // warpgroup g holds rows [64 g, 64 g + 64)
        __syncthreads();
        const int u = u0 + lane;
        float* hn = enc == 0 ? hn4 : hn3;
        if (u < h) {
          const float b_r = __ldg(bhh + enc * 3 * h + u), b_z = __ldg(bhh + enc * 3 * h + h + u),
                      b_n = __ldg(bhh + enc * 3 * h + 2 * h + u);
          // 8 rows per warp and half (row = warp + 8 i), lane = unit.  Index chains (seq_start -> row -> row_glob) are
          // resolved for all rows first, then the operand loads of 4 rows at a time are in flight together.
          int64_t rowi[8], gli[8];
          int qi[8], leni[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            qi[i] = q0 + half_rows * 64 + warp + 8 * i;
            const int qc = min(qi[i], n_act - 1);
            rowi[i] = (int64_t)__ldg(seq_start + qc) + t;
            leni[i] = __ldg(seq_len + qc);
          }
#pragma unroll
          for (int i = 0; i < 8; ++i) gli[i] = (int64_t)__ldg(row_glob + rowi[i]);
#pragma unroll
          for (int b4 = 0; b4 < 8; b4 += 4) {
            float i_r[4], i_z[4], i_n[4], hp[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int x = b4 + i;
              const int qc = min(qi[x], n_act - 1);
              const float* gi = GI + rowi[x] * 6 * h + enc * 3 * h + u;
              const float* pq = PQ + (int64_t)qc * 6 * h + enc * 3 * h + u;
              const float* pt = PT + gli[x] * 6 * h + enc * 3 * h + u;
              i_r[i] = __ldg(gi) + __ldg(pq) + __ldg(pt);
              i_z[i] = __ldg(gi + h) + __ldg(pq + h) + __ldg(pt + h);
              i_n[i] = __ldg(gi + 2 * h) + __ldg(pq + 2 * h) + __ldg(pt + 2 * h);
              hp[i] = t > 0 ? __ldcg(Hprev + (int64_t)qc * 2 * h + enc * h + u) : 0.f;
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int x = b4 + i;
              const int q = qi[x];
              if (q < n_act) {
                const int rr = warp + 8 * x;
                float g_r = 0.f, g_z = 0.f, g_n = 0.f;
                if (t > 0) {
                  g_r = sT[rr * TS + lane]; g_z = sT[rr * TS + RU + lane]; g_n = sT[rr * TS + 2 * RU + lane];
                  if (GH != nullptr) {                     // recurrent pre-activations (without bias), kept for backward
                    float* gh = GHt + (int64_t)q * 6 * h + enc * 3 * h + u;
                    gh[0] = g_r; gh[h] = g_z; gh[2 * h] = g_n;
                  }
                }
                const float r = sigm(i_r[i] + g_r + b_r);
                const float z = sigm(i_z[i] + g_z + b_z);
                const float n = tanhf(i_n[i] + r * (g_n + b_n));
                const float o = (1.f - z) * n + z * hp[i];
                Hnext[(int64_t)q * 2 * h + enc * h + u] = o;
                if (t == leni[x] - 1) hn[(int64_t)q * h + u] = o;
              }
            }
          }
        }
        __syncthreads();
      }
    }
    if (t + 1 < max_len && counts.n[t + 1] > 0) grid_barrier(barrier_counter, (unsigned int)(t + 1) * n_ctas);
  }
}

}  // namespace

// Returns 1 when the recurrence ran on this kernel, 0 when the shape is not supported (caller falls back), <0 on error.
int launch_gru_recur(const float* GI, const float* PQ, const float* PT, const float* bhh, const int32_t* row_glob,
                     const int32_t* seq_start, const int32_t* seq_len, const float* w_hh4, const float* w_hh3, float* Hs,
                     float* GH, float* hn4, float* hn3, unsigned int* barrier_counter, const int32_t* host_batch_sizes,
                     int max_len, int64_t Q, int h, cudaStream_t stream) {
  if (h % 4 != 0 || h > R_MAX_CHUNKS * R_BK || max_len > R_MAX_LEN || Q <= 0) return 0;
  static int coop = -1, sms = 0;
  if (coop < 0) {
    int dev = 0;
    RENET_CHECK_CUDA(cudaGetDevice(&dev));
    RENET_CHECK_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    RENET_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    RENET_CHECK_CUDA(cudaFuncSetAttribute(gru_recur_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, R_SMEM));
  }
  if (!coop) return 0;
  const int slices = (h + RU - 1) / RU;
  const int n_mtiles = (int)((Q + 127) / 128);
  const int gz = std::max(1, std::min(n_mtiles, sms / (slices * 2)));
  if (slices * 2 > sms) return 0;
  StepCounts counts;
  for (int t = 0; t < R_MAX_LEN; ++t) counts.n[t] = t < max_len ? host_batch_sizes[t] : 0;
  RENET_CHECK_CUDA(cudaMemsetAsync(barrier_counter, 0, sizeof(unsigned int), stream));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(slices, 2, gz);
  cfg.blockDim = dim3(R_THREADS);
  cfg.dynamicSmemBytes = R_SMEM;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int iQ = (int)Q;
  RENET_CHECK_CUDA(cudaLaunchKernelEx(&cfg, gru_recur_kernel, GI, PQ, PT, bhh, row_glob, seq_start, seq_len, w_hh4, w_hh3,
                                      Hs, GH, hn4, hn3, barrier_counter, counts, max_len, iQ, h));
  count_launch();
  return 1;
}

}  // namespace renet
