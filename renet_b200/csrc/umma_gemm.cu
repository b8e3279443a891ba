// fp32-accurate GEMM on the Hopper tensor cores (wgmma): C[M,N] = A[M,K] @ B[K,N] (+bias) (+C)
//
// RE-Net's dense work on the hot path -- the self-loop H @ W_loop (RGCN.py:35) and the GRU input /
// recurrent projections (model.py:86,94) -- must match a CPU fp32 oracle to 1e-4, which single-pass
// TF32 (10-bit mantissa, ~3e-4 on K=200) does not.  This kernel issues wgmma .tf32 with the
// 3xTF32 split:  a = a_hi + a_lo,  b = b_hi + b_lo  (hi = top 19 bits, lo = a - a_hi exactly),
//     D += a_hi*b_hi + a_lo*b_hi + a_hi*b_lo        (fp32 accumulation in registers)
// which recovers ~fp32 accuracy (dropped term a_lo*b_lo ~ 2^-22 relative) at 1/3 of TF32 peak -- still
// several times the FFMA roofline.
//
// Structure (one CTA per 128-row tile of A x one <=200-column tile of B, 256 threads = two warpgroups):
//   * operands are staged by the threads themselves (not TMA): A rows may be gathered through an index
//     (fused embedding lookup / read-out), B is row-major [K,N] and has to be transposed to K-major,
//     and both need the hi/lo split, so a register pass is required anyway;
//   * smem holds two stages of {A_hi, A_lo [128 x 40], B_hi, B_lo [208 x 40]} in the canonical
//     no-swizzle K-major layout (8-row x 16-byte core matrices; LBO = one 4-column slab, SBO = 128 B);
//   * warpgroup g issues 15 wgmma (5 k-steps x 3 split products, M=64 rows [64g, 64g+64), N=208, K=8) per stage;
//     the staging of chunk c+1 overlaps the MMAs of chunk c (at most one wgmma group in flight);
//   * accumulator: 104 fp32 registers per thread; the epilogue goes through shared memory (thread = row) and
//     writes C with bias / accumulate applied.
#include "common.cuh"
#include <mutex>
#include <vector>

#include "umma.cuh"

namespace renet {
namespace {

constexpr int UM = 128;          // rows per CTA tile
constexpr int UN = 200;          // logical columns per CTA tile
constexpr int UNP = 208;         // padded to a multiple of 16 for the MMA N
constexpr int UKC = 40;          // K per stage (5 MMA k-steps of 8)
constexpr int USLABS = UKC / 4;  // 16-byte (4 x fp32) column slabs per stage
constexpr int UTHREADS = 256;
constexpr int A_SLAB_BYTES = UM * 16;    // 2048
constexpr int B_SLAB_BYTES = UNP * 16;   // 3328
constexpr int A_BYTES = USLABS * A_SLAB_BYTES;   // 20480
constexpr int B_BYTES = USLABS * B_SLAB_BYTES;   // 33280
constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;   // 107520
constexpr int NUM_STAGES = 2;
constexpr int SMEM_BYTES = NUM_STAGES * STAGE_BYTES;
constexpr int CLD = UNP + 4;     // row stride (floats) of the accumulator tile in shared memory: conflict-free float4 rows
static_assert(UM * CLD * 4 <= SMEM_BYTES, "accumulator tile reuses the operand stages");

template <bool INDEXED>
__global__ void __launch_bounds__(UTHREADS, 1)
umma_gemm_nn_kernel(const float* __restrict__ A, const int32_t* __restrict__ a_index, int64_t lda,
                    const float* __restrict__ B, int64_t ldb, float* __restrict__ C, int64_t ldc,
                    const float* __restrict__ bias, int64_t M, int N, int K, int accumulate) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  const int64_t row0 = (int64_t)blockIdx.x * UM;
  const int n0 = blockIdx.y * UN;
  const int tile_n = min(UN, N - n0);
  const uint32_t smem_base = smem_u32(smem);

  // zero the 8 padding rows (n = 200..207) of every B slab once; they are never written again
  for (int i = tid; i < NUM_STAGES * 2 * USLABS * (UNP - UN); i += UTHREADS) {
    const int r = i % (UNP - UN), sl = (i / (UNP - UN)) % USLABS, which = (i / ((UNP - UN) * USLABS)) % 2,
              st = i / ((UNP - UN) * USLABS * 2);
    float4* p = reinterpret_cast<float4*>(smem + st * STAGE_BYTES + 2 * A_BYTES + which * B_BYTES + sl * B_SLAB_BYTES +
                                          (UN + r) * 16);
    *p = make_float4(0.f, 0.f, 0.f, 0.f);
  }

  // per-thread A source rows: task = slab * 128 + row  (5 tasks per thread per chunk)
  const float* a_rows[5];
#pragma unroll
  for (int t = 0; t < 5; ++t) {
    const int task = tid + t * UTHREADS;
    const int r = task % UM;
    const int64_t gr = row0 + r;
    a_rows[t] = nullptr;
    if (gr < M) {
      const int64_t rr = INDEXED ? (int64_t)__ldg(a_index + gr) : gr;
      a_rows[t] = A + rr * lda;
    }
  }

  float acc[UNP / 2];
#pragma unroll
  for (int i = 0; i < UNP / 2; ++i) acc[i] = 0.f;
  const int nchunks = K / UKC;
  for (int c = 0; c < nchunks; ++c) {
    const int st = c % NUM_STAGES;                       // its MMAs of chunk c-2 are complete (barrier below)
    uint8_t* sA_hi = smem + st * STAGE_BYTES;
    uint8_t* sA_lo = sA_hi + A_BYTES;
    uint8_t* sB_hi = sA_lo + A_BYTES;
    uint8_t* sB_lo = sB_hi + B_BYTES;
    const int k0 = c * UKC;
    // ---- A: 128 rows x 10 slabs; thread -> (slab, row): conflict-free 16-byte smem stores ----------
#pragma unroll
    for (int t = 0; t < 5; ++t) {
      const int task = tid + t * UTHREADS;
      const int sl = task / UM, r = task % UM;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (a_rows[t] != nullptr) v = ldg_f4(a_rows[t] + k0 + 4 * sl);
      float4 hi, lo;
      split4(v, hi, lo);
      *reinterpret_cast<float4*>(sA_hi + sl * A_SLAB_BYTES + r * 16) = hi;
      *reinterpret_cast<float4*>(sA_lo + sl * A_SLAB_BYTES + r * 16) = lo;
    }
    // ---- B: [40 k] x [200 n] row-major -> K-major: 4x4 register transposes -----------------------------
    for (int task = tid; task < USLABS * (UN / 4); task += UTHREADS) {
      const int sl = task / (UN / 4), j = task % (UN / 4);
      float4 m[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        m[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (4 * j < tile_n) m[i] = ldg_f4(B + (int64_t)(k0 + 4 * sl + i) * ldb + n0 + 4 * j);
      }
      const float4 t0 = make_float4(m[0].x, m[1].x, m[2].x, m[3].x);
      const float4 t1 = make_float4(m[0].y, m[1].y, m[2].y, m[3].y);
      const float4 t2 = make_float4(m[0].z, m[1].z, m[2].z, m[3].z);
      const float4 t3 = make_float4(m[0].w, m[1].w, m[2].w, m[3].w);
      const float4 tr[4] = {t0, t1, t2, t3};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float4 hi, lo;
        split4(tr[q], hi, lo);
        *reinterpret_cast<float4*>(sB_hi + sl * B_SLAB_BYTES + (4 * j + q) * 16) = hi;
        *reinterpret_cast<float4*>(sB_lo + sl * B_SLAB_BYTES + (4 * j + q) * 16) = lo;
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> async proxy (wgmma)
    __syncthreads();
    {
      const uint32_t a_hi = smem_base + st * STAGE_BYTES + wg * 64 * 16, a_lo = a_hi + A_BYTES;   // this warpgroup's 64 rows
      const uint32_t b_hi = smem_base + st * STAGE_BYTES + 2 * A_BYTES, b_lo = b_hi + B_BYTES;
      wgmma_fence();
      acc_fence(acc);
#pragma unroll
      for (int ks = 0; ks < UKC / 8; ++ks) {
        const uint32_t ao = ks * 2 * A_SLAB_BYTES, bo = ks * 2 * B_SLAB_BYTES;
        const uint64_t dAh = make_desc(a_hi + ao, A_SLAB_BYTES, 128), dAl = make_desc(a_lo + ao, A_SLAB_BYTES, 128);
        const uint64_t dBh = make_desc(b_hi + bo, B_SLAB_BYTES, 128), dBl = make_desc(b_lo + bo, B_SLAB_BYTES, 128);
        wgmma_tf32_n208(acc, dAh, dBh, (c | ks) != 0);
        wgmma_tf32_n208(acc, dAl, dBh, 1);
        wgmma_tf32_n208(acc, dAh, dBl, 1);
      }
      wgmma_commit();
    }
    wgmma_wait<1>();             // this warpgroup's MMAs of chunk c-1 are complete
    acc_fence(acc);
    __syncthreads();             // ... and the other warpgroup's: stage (c+1) % 2 may be overwritten
  }
  wgmma_wait<0>();
  acc_fence(acc);
  __syncthreads();               // every MMA has read its operands: the stages hold the accumulator tile now

  // ---- epilogue: registers -> shared tile -> global (thread = row; warps 0-3 cols [0,104), warps 4-7 [104,208)) ---
  float* sC = reinterpret_cast<float*>(smem);
  acc_store(acc, sC + wg * 64 * CLD, CLD, tid & 127);
  __syncthreads();
  {
    const int q = warp & 3, half = warp >> 2;
    const int r = q * 32 + lane;
    const int64_t gr = row0 + r;
#pragma unroll 1
    for (int cc = half * 104; cc < half * 104 + 104; cc += 8) {
      if (gr < M && cc < tile_n) {
        const float4 a0 = *reinterpret_cast<const float4*>(sC + r * CLD + cc);
        const float4 a1 = *reinterpret_cast<const float4*>(sC + r * CLD + cc + 4);
        float o[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        float* cp = C + gr * ldc + n0 + cc;
        if (bias != nullptr) {
          const float4 b0 = ldg_f4(bias + n0 + cc), b1 = ldg_f4(bias + n0 + cc + 4);
          o[0] += b0.x; o[1] += b0.y; o[2] += b0.z; o[3] += b0.w;
          o[4] += b1.x; o[5] += b1.y; o[6] += b1.z; o[7] += b1.w;
        }
        if (accumulate) {
          const float4 c0 = *reinterpret_cast<const float4*>(cp), c1 = *reinterpret_cast<const float4*>(cp + 4);
          o[0] += c0.x; o[1] += c0.y; o[2] += c0.z; o[3] += c0.w;
          o[4] += c1.x; o[5] += c1.y; o[6] += c1.z; o[7] += c1.w;
        }
        st_f4(cp, make_float4(o[0], o[1], o[2], o[3]));
        st_f4(cp + 4, make_float4(o[4], o[5], o[6], o[7]));
      }
    }
  }
}


// ======================================================================================================
// v2: pre-packed B + TMA bulk copies + 128-byte swizzle
//
// Profiling v1 showed the tile time dominated by operand staging, not by the MMAs: every CTA re-transposed and
// re-split the same B (W_loop / GRU weights), and the no-swizzle layout forced row-strided A loads (16 useful
// bytes per 128-byte line).  v2:
//   * B is packed ONCE per GEMM by umma_pack_b_kernel into the exact shared-memory image (hi and lo planes,
//     K-major, SWIZZLE_128B, one 53 KB block per (column tile, 32-wide K chunk)); the GEMM CTAs fetch a block
//     with a single cp.async.bulk (TMA) that completes on the stage's mbarrier;
//   * A is staged by the threads with fully coalesced 128-byte row segments and conflict-free swizzled
//     16-byte stores (chunk j of row r lands at chunk j ^ (r % 8));
//   * K is processed in chunks of 32 (one swizzle atom): 4 wgmma k-steps x 3 split products per chunk and warpgroup;
//   * A and B are double-buffered: chunk c+1's bulk copy and A staging run while chunk c's MMAs do.
// ======================================================================================================
constexpr int P_BK = 32;
constexpr int P_A_BYTES = UM * 128;                  // 16384
constexpr int P_B_BYTES = UNP * 128;                 // 26624
constexpr int P_B_CHUNK = 2 * P_B_BYTES;             // hi + lo planes of one (tile, chunk)
constexpr int P_SMEM = 4 * P_A_BYTES + 2 * P_B_CHUNK + 1024 + 128;   // two stages of A (hi,lo) and of B, barriers
static_assert(UM * CLD * 4 <= 4 * P_A_BYTES + 2 * P_B_CHUNK, "accumulator tile reuses the operand stages");

// Bp[(nt * n_chunks + kc)] = {hi plane, lo plane} of B[kc*32 .. +31][nt*200 .. +207] (zero padded)
__global__ void __launch_bounds__(256)
umma_pack_b_kernel(const float* __restrict__ B, int64_t sk, int64_t sn, int N, int K, uint8_t* __restrict__ Bp,
                   int n_chunks, int tile_offset) {
  // logical B[k][n] = B[k*sk + n*sn]  (row-major [K,N]: sk = ldb, sn = 1; a [N,K] weight read transposed: sk = 1, sn = ld)
  const int nt = blockIdx.x, kc = blockIdx.y;
  const int n0 = nt * UN, k0 = kc * P_BK;
  const int tile_n = min(UN, N - n0);
  uint8_t* dst = Bp + (size_t)((nt + tile_offset) * n_chunks + kc) * P_B_CHUNK;
  for (int task = blockIdx.z * 256 + threadIdx.x; task < UNP * 8; task += 256 * gridDim.z) {
    const int j = task / UNP, n = task % UNP;      // consecutive threads -> consecutive n (coalesced reads)
    float v[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int k = k0 + 4 * j + i;
      v[i] = (n < tile_n && k < K) ? __ldg(B + (int64_t)k * sk + (int64_t)(n0 + n) * sn) : 0.f;
    }
    float4 hi, lo;
    split4(make_float4(v[0], v[1], v[2], v[3]), hi, lo);
    const uint32_t off = sw128_offset(n, j);
    *reinterpret_cast<float4*>(dst + off) = hi;
    *reinterpret_cast<float4*>(dst + P_B_BYTES + off) = lo;
  }
}

// Fused-epilogue modes of the packed kernel (the decoder of model.py:89-91,97-100: logits = X @ W^T + b, cross-entropy):
//   EPI 0  C = acc (+bias) (+C)                                   -- plain GEMM
//   EPI 1  per (row, half column tile): running max and sum of exp of the logits, and the target's logit -- the
//          [M, N] logits never reach memory; ce_reduce_kernel turns the partials into logsumexp and the loss
//   EPI 2  dlogits[row, col] = (exp(logit - lse[row]) - [col == target[row]]) * scale, written to memory for the two
//          gradient GEMMs (the backward pass recomputes the logits instead of keeping them)
template <bool INDEXED, int EPI = 0>
__global__ void __launch_bounds__(UTHREADS, 1)
umma_gemm_packed_kernel(const float* __restrict__ A, const int32_t* __restrict__ a_index, int64_t lda,
                        const uint8_t* __restrict__ Bp, float* __restrict__ C, int64_t ldc,
                        const float* __restrict__ bias, int64_t M, int N, int K, int n_chunks, int accumulate,
                        int64_t batch_a, int64_t batch_bp, int64_t batch_c, EpiArgs epi, int k_splits, int64_t split_c) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024 - (raw & 1023)) & 1023);     // swizzle atoms need 1024-byte alignment
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  // grid.z = batch x K-split.  Batched GEMMs (the two GRU encoders): per-batch operand offsets.  Split-K (long-K,
  // few-tile products such as dX = dlogits @ W of the decoder): split s owns the chunks [s*cps, (s+1)*cps) and writes its
  // partial product to C + s*split_c; the caller sums the partials.
  const int zb = blockIdx.z / k_splits, split = blockIdx.z - zb * k_splits;
  A += zb * batch_a;
  Bp += zb * batch_bp;
  C += zb * batch_c + (int64_t)split * split_c;
  if (bias != nullptr) bias += zb * (int64_t)N;
  const int cps = (n_chunks + k_splits - 1) / k_splits;
  const int c_begin = split * cps;
  const int n_local = min(cps, n_chunks - c_begin);      // >= 1: the launcher never creates an empty split
  const int64_t row_base = (int64_t)blockIdx.x * UM;
  const int nt = blockIdx.y;
  const int n0 = nt * UN;
  const int tile_n = min(UN, N - n0);
  // smem: A[2 stages][hi,lo] (4 x 16 KB), B[2 stages][hi,lo] (2 x 53 KB), barriers
  uint8_t* sA = smem;
  uint8_t* sB = smem + 4 * P_A_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sB + 2 * P_B_CHUNK);   // [0,1] B stage landed
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t bar0 = smem_u32(bars);
  if (tid == 0) {
    mbar_init(bar0, 1);
    mbar_init(bar0 + 8, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // A tasks: 128 rows x 8 sixteen-byte chunks = 1024 -> 4 per thread; 8 consecutive lanes read one
  // 128-byte row segment (coalesced), and write it to 8 distinct swizzled chunks (conflict-free)
  const float* a_rows[4];
  uint32_t a_off[4];
  int a_k[4];
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int task = tid + t * UTHREADS;
    const int r = task >> 3, j = task & 7;
    a_off[t] = sw128_offset(r, j);
    a_k[t] = 4 * j;
    const int64_t gr = row_base + r;
    a_rows[t] = nullptr;
    if (gr < M) {
      const int64_t rr = INDEXED ? (int64_t)__ldg(a_index + gr) : gr;
      a_rows[t] = A + rr * lda;
    }
  }
  const uint8_t* bp_tile = Bp + (size_t)nt * n_chunks * P_B_CHUNK;
  float4 vnext[4];
  auto load_a = [&](int c) {
    const int k0 = (c_begin + c) * P_BK;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      vnext[t] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (a_rows[t] != nullptr && k0 + a_k[t] < K) vnext[t] = ldg_f4(a_rows[t] + k0 + a_k[t]);
    }
  };
  auto store_a = [&](int s) {
    uint8_t* sA_hi = sA + s * 2 * P_A_BYTES;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      float4 hi, lo;
      split4(vnext[t], hi, lo);
      *reinterpret_cast<float4*>(sA_hi + a_off[t]) = hi;
      *reinterpret_cast<float4*>(sA_hi + P_A_BYTES + a_off[t]) = lo;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> async proxy (wgmma)
  };
  auto issue_b = [&](int c) {   // TMA: one bulk copy brings the packed B block of chunk c
    const uint32_t full = bar0 + 8 * (c & 1);
    const uint32_t dstB = smem_base + 4 * P_A_BYTES + (c & 1) * P_B_CHUNK;
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(full), "r"((uint32_t)P_B_CHUNK) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dstB),
                 "l"(bp_tile + (size_t)(c_begin + c) * P_B_CHUNK), "r"((uint32_t)P_B_CHUNK), "r"(full)
                 : "memory");
  };

  if (tid == 0) issue_b(0);
  load_a(0);
  store_a(0);
  __syncthreads();
  float acc[UNP / 2];
#pragma unroll
  for (int i = 0; i < UNP / 2; ++i) acc[i] = 0.f;
  for (int c = 0; c < n_local; ++c) {
    const int s = c & 1;
    if (c + 1 < n_local) load_a(c + 1);                 // the next chunk's global loads fly during this chunk's MMAs
    mbar_wait(bar0 + 8 * s, (c >> 1) & 1);              // B block landed
    {
      const uint32_t a_hi = smem_base + s * 2 * P_A_BYTES + wg * 64 * 128, a_lo = a_hi + P_A_BYTES;   // warpgroup's 64 rows
      const uint32_t b_hi = smem_base + 4 * P_A_BYTES + s * P_B_CHUNK, b_lo = b_hi + P_B_BYTES;
      wgmma_fence();
      acc_fence(acc);
#pragma unroll
      for (int ks = 0; ks < P_BK / 8; ++ks) {
        const uint32_t ko = ks * 32;                       // 8 fp32 = 32 bytes along the swizzled row
        const uint64_t dAh = make_desc_sw128(a_hi + ko), dAl = make_desc_sw128(a_lo + ko);
        const uint64_t dBh = make_desc_sw128(b_hi + ko), dBl = make_desc_sw128(b_lo + ko);
        wgmma_tf32_n208(acc, dAh, dBh, (c | ks) != 0);
        wgmma_tf32_n208(acc, dAl, dBh, 1);
        wgmma_tf32_n208(acc, dAh, dBl, 1);
      }
      wgmma_commit();
    }
    wgmma_wait<1>();                                     // this warpgroup's MMAs of chunk c-1 are complete
    acc_fence(acc);
    __syncthreads();                                     // ... and the other's: stage s^1 (A and B) is free
    if (c + 1 < n_local) {
      if (tid == 0) issue_b(c + 1);
      store_a(s ^ 1);
      __syncthreads();
    }
  }
  wgmma_wait<0>();
  acc_fence(acc);
  __syncthreads();                                       // every MMA has read its operands: the stages are reused below

  float* sC = reinterpret_cast<float*>(smem);
  acc_store(acc, sC + wg * 64 * CLD, CLD, tid & 127);
  __syncthreads();
  {
    // thread = accumulator row; warps 0-3 take columns [0,104), warps 4-7 [104,208), 8 at a time
    const int q = warp & 3, half = warp >> 2;
    const int r = q * 32 + lane;
    const int cbase = half * 104;
    const int64_t gr = row_base + r;
    const float* srow = sC + r * CLD;
    // EPI 1 state of this thread's (row, half tile): running max / sum of exp; EPI 2: the row's logsumexp and target
    float run_m = -3.0e38f, run_s = 0.f;
    const int tgt = (EPI != 0 && gr < M) ? __ldg(epi.target + gr) : -1;
    const float row_lse = (EPI == 2 && gr < M) ? __ldg(epi.lse + gr) : 0.f;
    const float gscale = (EPI == 2) ? epi.scale * (epi.dscale != nullptr ? __ldg(epi.dscale) : 1.f) : 0.f;
#pragma unroll 1
    for (int cc = cbase; cc < cbase + 104; cc += 8) {
      if (gr < M && cc < tile_n) {
        const float4 a0 = *reinterpret_cast<const float4*>(srow + cc), a1 = *reinterpret_cast<const float4*>(srow + cc + 4);
        float o[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        if (EPI != 0) {
          // fused cross-entropy epilogues: columns are guarded one by one (the class count need not be a multiple of 8)
          const int nv = min(8, tile_n - cc);
          float mx = -3.0e38f;
#pragma unroll
          for (int i = 0; i < 8; ++i)
            if (i < nv) {
              if (bias != nullptr) o[i] += __ldg(bias + n0 + cc + i);
              mx = fmaxf(mx, o[i]);
            }
          if (EPI == 1) {
            const float nm = fmaxf(run_m, mx);
            float add = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i)
              if (i < nv) {
                add += expf(o[i] - nm);
                if (n0 + cc + i == tgt) epi.tlogit[gr] = o[i];
              }
            run_s = run_s * expf(run_m - nm) + add;
            run_m = nm;
          } else {
            float* dp = C + gr * ldc + n0 + cc;
#pragma unroll
            for (int i = 0; i < 8; ++i)
              if (i < nv) {
                const float gv = (expf(o[i] - row_lse) - (n0 + cc + i == tgt ? 1.f : 0.f)) * gscale;
                dp[i] = gv;                                              // row-major: A of dX = dlogits @ W
                epi.dT[(int64_t)(n0 + cc + i) * epi.ldT + gr] = gv;      // transposed (lanes = consecutive rows: coalesced)
              }
          }
          continue;
        }
        float* cp = C + gr * ldc + n0 + cc;
        if (bias != nullptr) {
          const float4 b0 = ldg_f4(bias + n0 + cc), b1 = ldg_f4(bias + n0 + cc + 4);
          o[0] += b0.x; o[1] += b0.y; o[2] += b0.z; o[3] += b0.w;
          o[4] += b1.x; o[5] += b1.y; o[6] += b1.z; o[7] += b1.w;
        }
        if (accumulate) {
          const float4 c0 = *reinterpret_cast<const float4*>(cp), c1 = *reinterpret_cast<const float4*>(cp + 4);
          o[0] += c0.x; o[1] += c0.y; o[2] += c0.z; o[3] += c0.w;
          o[4] += c1.x; o[5] += c1.y; o[6] += c1.z; o[7] += c1.w;
        }
        st_f4(cp, make_float4(o[0], o[1], o[2], o[3]));
        st_f4(cp + 4, make_float4(o[4], o[5], o[6], o[7]));
      }
    }
    if (EPI == 1 && gr < M) {
      const int64_t pi = (int64_t)(nt * 2 + half) * M + gr;
      epi.pmax[pi] = run_m;
      epi.psum[pi] = run_s;
    }
  }
}

}  // namespace

// Returns 1 if the shape was taken by the tensor-core path (launch enqueued), 0 if the caller should
// fall back to the FFMA kernel, negative on error.
static uint8_t* g_scratch = nullptr;
static int64_t g_scratch_bytes = 0;
void set_scratch(void* p, int64_t bytes) { g_scratch = (uint8_t*)p; g_scratch_bytes = p ? bytes : 0; }

// ---- packed-weight cache (renet_set_weight_generation) ------------------------------------------------------------------
// Packing a weight into the tensor-core operand image is a kernel launch per weight per call.  Weights only change when the
// optimiser steps, so the caller may declare a "weight generation": while it is unchanged, a packed image made for a
// given (device, pointers, shape) key is valid and reused; a new generation invalidates every image (the buffers are
// kept and overwritten by the next pack).  generation < 0 (the default) turns the cache off.
namespace {
struct PackEntry {
  int device;
  const void* keys[6];
  int nkeys;
  int64_t bytes;
  void* buf;
  int64_t gen;
};
std::mutex g_pack_mu;
std::vector<PackEntry> g_pack_entries;
int64_t g_weight_generation = -1;
}  // namespace

void set_weight_generation(int64_t g) {
  std::lock_guard<std::mutex> lk(g_pack_mu);
  g_weight_generation = g;
}

void* packed_cache_lookup(const void* const* keys, int nkeys, int64_t bytes, bool* hit) {
  *hit = false;
  std::lock_guard<std::mutex> lk(g_pack_mu);
  if (g_weight_generation < 0 || nkeys > 6) return nullptr;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  for (auto& e : g_pack_entries) {
    if (e.device != dev || e.nkeys != nkeys || e.bytes != bytes) continue;
    bool same = true;
    for (int i = 0; i < nkeys; ++i) same &= e.keys[i] == keys[i];
    if (!same) continue;
    *hit = e.gen == g_weight_generation;
    e.gen = g_weight_generation;
    return e.buf;
  }
  if (g_pack_entries.size() >= 64) {       // bounded: drop the oldest image
    cudaFree(g_pack_entries.front().buf);
    g_pack_entries.erase(g_pack_entries.begin());
  }
  PackEntry e{};
  e.device = dev; e.nkeys = nkeys; e.bytes = bytes; e.gen = g_weight_generation;
  for (int i = 0; i < nkeys; ++i) e.keys[i] = keys[i];
  if (cudaMalloc(&e.buf, (size_t)bytes) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  g_pack_entries.push_back(e);
  return e.buf;
}

// ---- building blocks shared with gru.cu ------------------------------------------------------------------------
int64_t umma_packed_bytes(int N, int K) {
  return (int64_t)((N + UN - 1) / UN) * ((K + P_BK - 1) / P_BK) * P_B_CHUNK;
}
bool umma_shape_ok(int N, int K) { return (K % 4 == 0) && (N % 8 == 0) && N > 0 && K > 0; }

// Pack logical B[k][n] = B[k*sk + n*sn] (K x N) into tiles [tile_offset, tile_offset + ceil(N/200)) of Bp.
int umma_pack_b(const float* B, int64_t sk, int64_t sn, int N, int K, void* Bp, int tile_offset, cudaStream_t stream) {
  const int n_tiles = (N + UN - 1) / UN, n_chunks = (K + P_BK - 1) / P_BK;
  umma_pack_b_kernel<<<dim3(n_tiles, n_chunks, 7), 256, 0, stream>>>(B, sk, sn, N, K, (uint8_t*)Bp, n_chunks, tile_offset);
  RENET_CHECK_LAUNCH("umma_pack_b_kernel");
  return RENET_OK;
}

// C[b] (+)= A[b] @ Bpacked[b] (+bias[b]) for b < batch; strides in elements (A, C) / bytes (Bp).
// epi_mode 1 / 2: fused cross-entropy epilogues (EpiArgs); k_splits > 1: split-K partial products at C + s*split_c.
int umma_gemm_prepacked_ex(const float* A, const int32_t* a_index, int64_t lda, const void* Bp, float* C, int64_t ldc,
                           const float* bias, int64_t M, int N, int K, bool accumulate, int batch, int64_t batch_a,
                           int64_t batch_bp, int64_t batch_c, int epi_mode, const EpiArgs& epi, int k_splits, int64_t split_c,
                           cudaStream_t stream) {
  if (M <= 0) return RENET_OK;
  static bool attr2 = false;
  if (!attr2) {
    RENET_CHECK_CUDA(cudaFuncSetAttribute(umma_gemm_packed_kernel<true, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, P_SMEM));
    RENET_CHECK_CUDA(cudaFuncSetAttribute(umma_gemm_packed_kernel<false, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, P_SMEM));
    RENET_CHECK_CUDA(cudaFuncSetAttribute(umma_gemm_packed_kernel<false, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, P_SMEM));
    RENET_CHECK_CUDA(cudaFuncSetAttribute(umma_gemm_packed_kernel<false, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, P_SMEM));
    attr2 = true;
  }
  const int n_tiles = (N + UN - 1) / UN, n_chunks = (K + P_BK - 1) / P_BK;
  if (k_splits < 1) k_splits = 1;
  if (k_splits > n_chunks) k_splits = n_chunks;
  while (k_splits > 1 && ((n_chunks + k_splits - 1) / k_splits) * (k_splits - 1) >= n_chunks) --k_splits;   // no empty split
  dim3 grid((unsigned)((M + UM - 1) / UM), (unsigned)n_tiles, (unsigned)(batch * k_splits));
#define RENET_UMMA_LAUNCH(IDX, EP)                                                                                       \
  umma_gemm_packed_kernel<IDX, EP><<<grid, UTHREADS, P_SMEM, stream>>>(A, a_index, lda, (const uint8_t*)Bp, C, ldc, bias, M, N, K, \
                                                                      n_chunks, accumulate, batch_a, batch_bp, batch_c, epi,  \
                                                                      k_splits, split_c)
  if (epi_mode == 1) RENET_UMMA_LAUNCH(false, 1);
  else if (epi_mode == 2) RENET_UMMA_LAUNCH(false, 2);
  else if (a_index) RENET_UMMA_LAUNCH(true, 0);
  else RENET_UMMA_LAUNCH(false, 0);
#undef RENET_UMMA_LAUNCH
  RENET_CHECK_LAUNCH("umma_gemm_packed_kernel");
  return k_splits;      // > 0: the number of K-splits actually used (1 = C holds the result)
}

int umma_gemm_prepacked(const float* A, const int32_t* a_index, int64_t lda, const void* Bp, float* C, int64_t ldc,
                        const float* bias, int64_t M, int N, int K, bool accumulate, int batch, int64_t batch_a,
                        int64_t batch_bp, int64_t batch_c, cudaStream_t stream) {
  EpiArgs none{};
  const int r = umma_gemm_prepacked_ex(A, a_index, lda, Bp, C, ldc, bias, M, N, K, accumulate, batch, batch_a, batch_bp, batch_c,
                                       0, none, 1, 0, stream);
  return r < 0 ? r : RENET_OK;
}

int umma_gemm_nn_try(const float* A, const int32_t* a_index, int64_t lda, const float* B, int64_t ldb, float* C,
                     int64_t ldc, const float* bias, int64_t M, int32_t N, int32_t K, bool accumulate,
                     cudaStream_t stream) {
  const bool aligned = ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B) | reinterpret_cast<uintptr_t>(C) |
                         reinterpret_cast<uintptr_t>(bias)) & 15) == 0;
  // ---- packed path: needs the registered scratch buffer for the packed copy of B ---------------------------------
  if (aligned && umma_shape_ok(N, K) && (lda % 4 == 0) && (ldc % 4 == 0) && M >= 64 && g_scratch != nullptr &&
      umma_packed_bytes(N, K) <= g_scratch_bytes && (reinterpret_cast<uintptr_t>(g_scratch) & 127) == 0) {
    bool hit = false;
    const void* keys[4] = {B, reinterpret_cast<const void*>((intptr_t)ldb), reinterpret_cast<const void*>((intptr_t)N),
                           reinterpret_cast<const void*>((intptr_t)K)};
    void* cached = packed_cache_lookup(keys, 4, umma_packed_bytes(N, K), &hit);
    void* Bp = cached ? cached : g_scratch;
    int rc = hit ? 0 : umma_pack_b(B, ldb, 1, N, K, Bp, 0, stream);
    if (rc) return rc;
    rc = umma_gemm_prepacked(A, a_index, lda, Bp, C, ldc, bias, M, N, K, accumulate, 1, 0, 0, 0, stream);
    return rc ? rc : 1;
  }
  const bool ok = (K % UKC == 0) && K >= UKC && (N % 8 == 0) && (lda % 4 == 0) && (ldb % 4 == 0) && (ldc % 4 == 0) &&
                  M >= 64 && aligned;
  if (!ok) return 0;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e1 = cudaFuncSetAttribute(umma_gemm_nn_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    cudaError_t e2 = cudaFuncSetAttribute(umma_gemm_nn_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e1 != cudaSuccess || e2 != cudaSuccess) {
      set_error("cudaFuncSetAttribute(umma_gemm_nn_kernel) failed: %s", cudaGetErrorString(e1 != cudaSuccess ? e1 : e2));
      return RENET_ERR_CUDA;
    }
    attr_set = true;
  }
  dim3 grid((unsigned)((M + UM - 1) / UM), (unsigned)((N + UN - 1) / UN));
  if (a_index)
    umma_gemm_nn_kernel<true><<<grid, UTHREADS, SMEM_BYTES, stream>>>(A, a_index, lda, B, ldb, C, ldc, bias, M, N, K, accumulate);
  else
    umma_gemm_nn_kernel<false><<<grid, UTHREADS, SMEM_BYTES, stream>>>(A, a_index, lda, B, ldb, C, ldc, bias, M, N, K, accumulate);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("launch of umma_gemm_nn_kernel failed: %s", cudaGetErrorString(e));
    return RENET_ERR_CUDA;
  }
  count_launch();
  return 1;
}

}  // namespace renet
