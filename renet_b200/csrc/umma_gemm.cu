// fp32-accurate GEMM on the Hopper tensor cores (wgmma): C[M,N] = A[M,K] @ B[K,N] (+bias) (+C)
//
// RE-Net's dense work on the hot path -- the self-loop H @ W_loop (RGCN.py:35) and the GRU input /
// recurrent projections (model.py:86,94) -- must match a CPU fp32 oracle to 1e-4, which single-pass
// TF32 (10-bit mantissa, ~3e-4 on K=200) does not.  The kernels issue wgmma .tf32 with the
// 3xTF32 split:  a = a_hi + a_lo,  b = b_hi + b_lo  (hi = top 19 bits, lo = a - a_hi exactly),
//     D += a_hi*b_hi + a_lo*b_hi + a_hi*b_lo        (fp32 accumulation in registers)
// which recovers ~fp32 accuracy (dropped term a_lo*b_lo ~ 2^-22 relative) at 1/3 of TF32 peak -- still
// several times the FFMA roofline.
//
// Structure: B is packed once per product by umma_pack_b_kernel into the exact shared-memory image the kernels read (hi
// and lo planes, K-major, 128-byte swizzle), into an image of the packed-weight cache or into a block of the calling
// stream (stream_block, common.cuh).  A is split into hi / lo as it is staged; its rows may be gathered through an index
// (fused embedding lookup / read-out).  Two kernels consume the packed image:
//   * umma_gemm_packed_kernel ("streaming"): persistent and warp-specialised, B streamed per 128 x 104 work unit with TMA
//     bulk copies; any K, split-K and the fused epilogues;
//   * umma_gemm_resident_kernel: the whole B panel (K <= 224) resident in shared memory, A fed to wgmma from registers;
//     umma_gemm_dedup runs it over the distinct rows of an index and copies the rows out.
#include "common.cuh"
#include "launch.cuh"
#include <mutex>
#include <vector>

#include "umma.cuh"

namespace renet {
namespace {

constexpr int UM = 128;          // rows per CTA tile
constexpr int UN = 200;          // logical columns per CTA tile
constexpr int UNP = 208;         // padded to a multiple of 16 for the MMA N

// ======================================================================================================
// Streaming kernel: pre-packed B + TMA bulk copies + 128-byte swizzle, persistent and warp-specialised
//
// Operand staging, not the MMAs, dominates a tile's time when every CTA re-transposes and re-splits the same B (W_loop /
// GRU weights) and a no-swizzle layout forces row-strided A loads (16 useful bytes per 128-byte line).  So:
//   * B is packed ONCE per GEMM by umma_pack_b_kernel into the exact shared-memory image (hi and lo planes,
//     K-major, SWIZZLE_128B, one 53 KB block per (column tile, 32-wide K chunk)); rows 0-103 and 104-207 of each
//     plane are contiguous 13 KB halves (13 whole swizzle atoms), and the GEMM fetches the half it needs with two
//     cp.async.bulk (TMA) copies that complete on the stage's mbarrier;
//   * A is staged with fully coalesced 128-byte row segments and conflict-free swizzled 16-byte stores
//     (chunk j of row r lands at chunk j ^ (r % 8));
//   * K is processed in chunks of 32 (one swizzle atom); the last chunk issues only the k-steps that hold data.
//
// Work unit = 128 rows x one 104-column half of a 200-column tile (x one batch entry / K-split).  The grid has at most
// one CTA per SM and CTA b walks the units [b*U/G, (b+1)*U/G), so no SM gets more than one unit above the average:
// 34.5 k rows x 200 columns are 540 units, 4.09 per SM, at most 5.
//
// 384 threads.  Warpgroup 0 is the producer: per chunk it loads A (rows gathered through a_index), splits it into
// hi/lo, stores it swizzled and issues the B copies.  Warpgroups 1 and 2 are the consumers: each owns 64 rows of the
// unit, issues wgmma m64n104k8 (52 fp32 accumulators per thread) and runs the epilogue.  A ring of stages
// {A hi, A lo [128 x 32], B hi, B lo [104 x 32]} with a full and an empty mbarrier per stage replaces block-wide
// barriers; the producer runs up to a ring ahead across unit boundaries, so the next unit's operands land while the
// consumers finish and store the current one, and the consumers keep one wgmma group in flight across chunks.
// Each output element sees the k-steps in order and per k-step the products hi*hi, lo*hi, hi*lo.
// ======================================================================================================
constexpr int P_BK = 32;
constexpr int P_A_BYTES = UM * 128;                  // 16384: one plane of 128 rows x 32 K
constexpr int P_B_BYTES = UNP * 128;                 // 26624: one plane of 208 columns x 32 K
constexpr int P_B_CHUNK = 2 * P_B_BYTES;             // hi + lo planes of one (tile, chunk)
constexpr int P_UN = UNP / 2;                        // 104 columns per work unit
constexpr int P_BH_BYTES = P_UN * 128;               // 13312: one half of a B plane
constexpr int P_STAGE = 2 * P_A_BYTES + 2 * P_BH_BYTES;   // 59392: A hi, A lo, B hi half, B lo half
constexpr int P_THREADS = 384;
constexpr int P_CLD = P_UN + 4;                      // row stride (floats) of a consumer's staged accumulator tile
// EPI 0 stores straight from the accumulator fragments and affords 3 stages; the cross-entropy epilogues walk each row
// in column order through a staged 64 x 104 tile per consumer, which leaves room for 2.
__host__ __device__ constexpr int p_stages(int epi) { return epi == 0 ? 3 : 2; }
__host__ __device__ constexpr int p_staging_bytes(int epi) { return epi == 0 ? 0 : 2 * 64 * P_CLD * 4; }
__host__ __device__ constexpr int p_smem(int epi) { return p_stages(epi) * P_STAGE + p_staging_bytes(epi) + 1024 + 128; }
static_assert(p_smem(0) <= 232448 && p_smem(1) <= 232448, "one CTA's shared memory");
static_assert(P_STAGE % 1024 == 0 && P_BH_BYTES % 1024 == 0, "swizzle atoms stay 1024-byte aligned");

// Bp[(nt * n_chunks + kc)] = {hi plane, lo plane} of B[kc*32 .. +31][nt*200 .. +207] (zero padded)
__global__ void __launch_bounds__(256)
umma_pack_b_kernel(const float* __restrict__ B, int64_t sk, int64_t sn, int N, int K, uint8_t* __restrict__ Bp,
                   int n_chunks, int tile_offset) {
  // logical B[k][n] = B[k*sk + n*sn]  (row-major [K,N]: sk = ldb, sn = 1; a [N,K] weight read transposed: sk = 1, sn = ld)
  pdl_wait();                          // nothing before the wait: only the launch latency hides under the previous kernel
  pdl_trigger();
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

// One work unit: rows [row_base, row_base + 128), columns [n0 + 104*half, +104) of column tile nt, batch entry zb,
// K-split `split` owning the chunks [c_begin, c_begin + n_local).  Units are numbered row tile fastest, then column
// half, then batch x split (the order of the old grid's x, y, z).
struct PUnit {
  int64_t row_base;
  int nt, half, zb, split, c_begin, n_local;
};
__device__ __forceinline__ PUnit p_unit(int64_t u, int64_t n_rt, int n_tiles, int n_chunks, int k_splits) {
  PUnit w;
  const int64_t rest = u / n_rt;
  w.row_base = (u - rest * n_rt) * UM;
  const int nh = (int)(rest % (2 * n_tiles)), z = (int)(rest / (2 * n_tiles));
  w.nt = nh >> 1;
  w.half = nh & 1;
  w.zb = z / k_splits;
  w.split = z - w.zb * k_splits;
  const int cps = (n_chunks + k_splits - 1) / k_splits;
  w.c_begin = w.split * cps;
  w.n_local = min(cps, n_chunks - w.c_begin);      // >= 1: the launcher never creates an empty split
  return w;
}

// Debug timeline (renet_debug_gemm_timing, tools/gemm_timeline.py; dbg is nullptr in production): thread 0 of every
// warpgroup writes one record of 8 int64 at dbg[(blockIdx.x * 4 + warpgroup) * 8]:
//   global timer at entry and exit, SM clocks entry -> exit, SM clocks spent waiting on operand barriers (streaming
//   producer: empty; streaming consumer: full; resident: the B chunks), in wgmma.wait_group, in the epilogue, and (resident)
//   in the hi/lo split of A, which absorbs the wait for its global loads; then items done | role << 32
//   (role 0 = streaming producer, 1 = streaming consumer, 2 = resident consumer).
struct GemmStamps {
  long long* rec;
  long long g0, c0, bar, mma, epi, aop;
  int items;
  __device__ __forceinline__ GemmStamps(long long* dbg, int wg) : bar(0), mma(0), epi(0), aop(0), items(0) {
    rec = (dbg != nullptr && (threadIdx.x & 127) == 0) ? dbg + ((int64_t)blockIdx.x * 4 + wg) * 8 : nullptr;
    g0 = c0 = 0;
    if (rec) {
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g0));
      c0 = clock64();
    }
  }
  __device__ __forceinline__ long long now() const { return rec ? clock64() : 0; }
  __device__ __forceinline__ void finish(int role) const {
    if (!rec) return;
    long long g1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g1));
    rec[0] = g0; rec[1] = g1; rec[2] = clock64() - c0; rec[3] = bar; rec[4] = mma; rec[5] = epi; rec[6] = aop;
    rec[7] = (long long)items | ((long long)role << 32);
  }
};

// EPI 0 straight from a warpgroup's m64n104 fragment: thread wt holds rows r0, r0 + 8 of the 64 rows at row_base and, per
// 8-column group i, columns 8i + c0, +1 of the 104 at tile column cb; the 4 threads of a quad cover 32 contiguous bytes.
// tile_n is even (N % 4 == 0 for every caller), so each column pair is wholly inside or wholly past the tile; the pairs
// past it are skipped one by one: the decoder's gradient products have N = its K, where K % 8 == 4 ends the tile
// half-way through an 8-column group, and a store there would land on the next row's first columns.
__device__ __forceinline__ void store_fragment(const float (&acc)[P_UN / 2], float* __restrict__ Cz, int64_t ldc,
                                               const float* __restrict__ bz, int64_t row_base, int64_t M, int n0, int cb,
                                               int tile_n, int accumulate, int wt) {
  const int r0 = 16 * (wt >> 5) + ((wt & 31) >> 2), c0 = 2 * (wt & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t gr = row_base + r0 + 8 * h;
    if (gr >= M) continue;
#pragma unroll
    for (int i = 0; i < P_UN / 8; ++i) {
      const int cc = cb + 8 * i;
      if (cc + c0 >= tile_n) continue;
      float o0 = acc[4 * i + 2 * h], o1 = acc[4 * i + 2 * h + 1];
      float* cp = Cz + gr * ldc + n0 + cc + c0;
      if (bz != nullptr) {
        const float2 bv = __ldg(reinterpret_cast<const float2*>(bz + n0 + cc + c0));
        o0 += bv.x; o1 += bv.y;
      }
      if (accumulate) {
        const float2 cv = *reinterpret_cast<const float2*>(cp);
        o0 += cv.x; o1 += cv.y;
      }
      *reinterpret_cast<float2*>(cp) = make_float2(o0, o1);
    }
  }
}

// Fused-epilogue modes of the packed kernel (the decoder of model.py:89-91,97-100: logits = X @ W^T + b, cross-entropy):
//   EPI 0  C = acc (+bias) (+C)                                   -- plain GEMM
//   EPI 1  per (row, half column tile): running max and sum of exp of the logits, and the target's logit (skipped when
//          target is null) -- the [M, N] logits never reach memory; ce_reduce_kernel turns the partials into logsumexp
//          and the loss
//   EPI 2  dlogits[row, col] = (exp(logit - lse[row]) - [col == target[row]]) * scale, written to memory for the two
//          gradient GEMMs (the backward pass recomputes the logits instead of keeping them)
//   EPI 3  soft targets P (global_model.py's soft cross-entropy): EPI 1's running max and sum of exp, and the sums of
//          P * logit and of P, with P read at the logit's own position; soft_ce_reduce_kernel (decoder.cu) combines them
//   EPI 4  dlogits[row, col] = (rowmass[row] * exp(logit - lse[row]) - P[row, col]) * scale, written as in EPI 2
//   EPI 5  grouped top-k candidates (renet_decoder_group_topk): p = row_w[row] * exp(logit - lse[row]); every p at or above
//          its group's threshold is appended to the group's candidate buffer (an integer atomic picks the slot; the final
//          select sorts, so no output depends on the slot order)
//   EPI 6  rank counts (renet_decoder_rank, renet_decoder_rank_multi): every logit is compared with the label's logit that
//          the EPI 1 pass wrote to tlogit (the same tile, the same instructions: the label's own logit compares equal), raw
//          and, per exclusion list of the row (0..2), after the sigmoid with the list zeroed; each list has its own cursor,
//          the sigmoid of each logit is computed once and shared by the lists, and each (row, half tile) adds its
//          2 + 2 * n_lists counts with integer atomics
// grid.x = min(units, SMs).  Batched GEMMs (the two GRU encoders) have per-batch operand offsets.  Split-K (long-K,
// few-tile products such as dX = dlogits @ W of the decoder): split s owns the chunks [s*cps, (s+1)*cps) and writes its
// partial product to C + s*split_c; the caller sums the partials.
template <bool INDEXED, int EPI = 0>
__global__ void __launch_bounds__(P_THREADS, 1)
umma_gemm_packed_kernel(const float* __restrict__ A, const int32_t* __restrict__ a_index, int64_t lda,
                        const uint8_t* __restrict__ Bp, float* __restrict__ C, int64_t ldc,
                        const float* __restrict__ bias, int64_t M, int N, int K, int n_chunks, int accumulate,
                        int64_t batch_a, int64_t batch_bp, int64_t batch_c, EpiArgs epi, int k_splits, int64_t split_c,
                        int64_t n_units, long long* dbg) {
  constexpr int S = p_stages(EPI);
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024 - (raw & 1023)) & 1023);     // swizzle atoms need 1024-byte alignment
  const uint32_t smem_base = smem_u32(smem);
  // smem: S stages {A hi, A lo, B hi half, B lo half}, [EPI != 0: two 64 x P_CLD staging tiles], full[S], empty[S]
  const uint32_t full0 = smem_base + S * P_STAGE + p_staging_bytes(EPI);
  const uint32_t empty0 = full0 + 8 * S;
  const int tid = threadIdx.x;
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);   // warp-uniform to the compiler: the wgmma paths do not diverge
  GemmStamps ts(dbg, wg);
  if (tid == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(full0 + 8 * s, 128);     // every producer thread arrives after its A stores; the B copies add bytes
      mbar_init(empty0 + 8 * s, 8);      // lane 0 of each consumer warp arrives once its MMAs on the stage are done
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int64_t n_rt = (M + UM - 1) / UM;
  const int n_tiles = (N + UN - 1) / UN;
  const int64_t u_begin = (int64_t)blockIdx.x * n_units / gridDim.x, u_end = (int64_t)(blockIdx.x + 1) * n_units / gridDim.x;

  if (wg == 0) {
    // ---- producer.  Thread t stages 16-byte piece j = t % 8 of rows t/8 + 16 i (i < 8): 8 consecutive lanes read one
    // 128-byte row segment, and rows r and r + 16 share a swizzle phase, so row t/8 + 16 i lands at a_off + 2048 i.
    const int j = tid & 7, r0 = tid >> 3;
    const uint32_t a_off = sw128_offset(r0, j);
    // load cursor: the chunk (lu, lc) whose A is loaded next; the loads of one chunk fly while the previous is stored
    int64_t lu = u_begin;
    int lc = 0;
    PUnit lw{};
    const float* a_rows[8];
    auto set_unit = [&]() {
      lw = p_unit(lu, n_rt, n_tiles, n_chunks, k_splits);
      const float* Az = A + lw.zb * batch_a;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int64_t gr = lw.row_base + r0 + 16 * i;
        a_rows[i] = nullptr;
        if (gr < M) a_rows[i] = Az + (INDEXED ? (int64_t)__ldg(a_index + gr) : gr) * lda;
      }
    };
    auto load = [&](float4 (&v)[8], const uint8_t*& bsrc) {
      const int k = (lw.c_begin + lc) * P_BK + 4 * j;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (a_rows[i] != nullptr && k < K) v[i] = ldg_f4(a_rows[i] + k);
      }
      bsrc = Bp + lw.zb * batch_bp + ((size_t)lw.nt * n_chunks + lw.c_begin + lc) * P_B_CHUNK + lw.half * P_BH_BYTES;
      if (++lc == lw.n_local) {
        lc = 0;
        if (++lu < u_end) set_unit();
      }
    };
    auto commit = [&](const float4 (&v)[8], const uint8_t* bsrc, int q) {
      const int s = q % S;
      const uint32_t full = full0 + 8 * s, st = smem_base + s * P_STAGE;
      const long long t0 = ts.now();
      mbar_wait(empty0 + 8 * s, ((q / S) & 1) ^ 1);     // the consumers are done with the stage's previous chunk
      ts.bar += ts.now() - t0;
      ++ts.items;
      if (tid == 0) {
        mbar_expect_tx(full, 2 * P_BH_BYTES);
        bulk_copy_g2s(st + 2 * P_A_BYTES, bsrc, P_BH_BYTES, full);
        bulk_copy_g2s(st + 2 * P_A_BYTES + P_BH_BYTES, bsrc + P_B_BYTES, P_BH_BYTES, full);
      }
      uint8_t* sa = smem + s * P_STAGE;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float4 hi, lo;
        split4(v[i], hi, lo);
        *reinterpret_cast<float4*>(sa + a_off + 2048 * i) = hi;
        *reinterpret_cast<float4*>(sa + P_A_BYTES + a_off + 2048 * i) = lo;
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> async proxy (wgmma)
      mbar_arrive(full);
    };
    if (lu < u_end) {
      set_unit();
      float4 va[8], vb[8];
      const uint8_t *ba, *bb;
      load(va, ba);
      for (int q = 0;; q += 2) {
        const bool more_b = lu < u_end;
        if (more_b) load(vb, bb);
        commit(va, ba, q);
        if (!more_b) break;
        const bool more_a = lu < u_end;
        if (more_a) load(va, ba);
        commit(vb, bb, q + 1);
        if (!more_a) break;
      }
    }
    ts.finish(0);
    return;
  }

  // ---- consumers: warpgroup g = 0, 1 owns rows [64 g, 64 g + 64) of every unit
  const int g = wg - 1, wt = tid & 127, lane = tid & 31;
  float acc[P_UN / 2];
  int q = 0;
  for (int64_t u = u_begin; u < u_end; ++u) {
    const PUnit w = p_unit(u, n_rt, n_tiles, n_chunks, k_splits);
    ++ts.items;
    for (int c = 0; c < w.n_local; ++c, ++q) {
      const int s = q % S;
      long long t0 = ts.now();
      mbar_wait(full0 + 8 * s, (q / S) & 1);           // A stored and B landed
      ts.bar += ts.now() - t0;
      const uint32_t a_hi = smem_base + s * P_STAGE + g * 64 * 128, a_lo = a_hi + P_A_BYTES;
      const uint32_t b_hi = smem_base + s * P_STAGE + 2 * P_A_BYTES, b_lo = b_hi + P_BH_BYTES;
      const int nks = min(P_BK / 8, (K - (w.c_begin + c) * P_BK + 7) / 8);   // k-steps that hold data
#pragma unroll
      for (int ks = 0; ks < P_BK / 8; ++ks) {
        if (ks < nks) {
          wgmma_fence();                                 // orders the accumulator registers for this k-step's wgmma
          const uint32_t ko = ks * 32;                   // 8 fp32 = 32 bytes along the swizzled row
          const uint64_t dAh = make_desc_sw128(a_hi + ko), dAl = make_desc_sw128(a_lo + ko);
          const uint64_t dBh = make_desc_sw128(b_hi + ko), dBl = make_desc_sw128(b_lo + ko);
          wgmma_tf32_n104(acc, dAh, dBh, (c | ks) != 0);
          wgmma_tf32_n104(acc, dAl, dBh, 1);
          wgmma_tf32_n104(acc, dAh, dBl, 1);
        }
      }
      wgmma_commit();
      if (c > 0) {
        t0 = ts.now();
        wgmma_wait<1>();                                 // the previous chunk's MMAs are complete: release its stage
        ts.mma += ts.now() - t0;
        if (lane == 0) mbar_arrive(empty0 + 8 * ((q - 1) % S));
      }
    }
    long long t0 = ts.now();
    wgmma_wait<0>();
    ts.mma += ts.now() - t0;
    if (lane == 0) mbar_arrive(empty0 + 8 * ((q - 1) % S));

    const int n0 = w.nt * UN, cb = w.half * P_UN;        // tile column of the unit's column 0
    const int tile_n = min(UN, N - n0);
    float* Cz = C + w.zb * batch_c + (int64_t)w.split * split_c;
    const float* bz = bias != nullptr ? bias + w.zb * (int64_t)N : nullptr;
    if (EPI == 0) {
      t0 = ts.now();
      store_fragment(acc, Cz, ldc, bz, w.row_base + 64 * g, M, n0, cb, tile_n, accumulate, wt);
      ts.epi += ts.now() - t0;
      continue;
    }
    // cross-entropy epilogues: thread = row walks the unit's 104 columns in order, 8 at a time
    float* sC = reinterpret_cast<float*>(smem + S * P_STAGE) + g * 64 * P_CLD;
    named_bar_sync(1 + g, 128);                          // the previous unit's rows have been read
    acc_store(acc, sC, P_CLD, wt);
    named_bar_sync(1 + g, 128);
    if (wt >= 64) continue;
    constexpr bool FWD = EPI == 1 || EPI == 3, SOFT = EPI == 3 || EPI == 4, SEL = EPI == 5, RANK = EPI == 6;
    const int64_t gr = w.row_base + 64 * g + wt;
    const float* srow = sC + wt * P_CLD;
    float run_m = -3.0e38f, run_s = 0.f;               // EPI 1, 3: running max / sum of exp of this (row, half tile)
    float run_pz = 0.f, run_p = 0.f;                   // EPI 3: sums of P * logit and of P
    // EPI 1 without a target (the grouped top-k's first pass) only reduces the running max / sum of exp
    const int tgt = (!SOFT && !SEL && gr < M && epi.target != nullptr) ? __ldg(epi.target + gr) : -1;
    const int64_t sel_g = SEL ? gr / epi.sel_R : 0;
    const int sel_base = SEL ? (int)(gr - sel_g * epi.sel_R) * N : 0;     // flat index of the row's column 0 in its group
    const float row_w = (SEL && gr < M) ? __ldg(epi.row_w + gr) : 0.f;
    const float sel_tau = (SEL && gr < M) ? __ldg(epi.tau + sel_g) : 0.f;
    const float row_lse = (!FWD && !RANK && gr < M) ? __ldg(epi.lse + gr) : 0.f;
    // EPI 6: the label's logit and sigmoid and the raw pair of counts.  List j of the row is excl_col[excl_begin[j * M + row]
    // .. excl_end[j * M + row]); each list keeps a cursor (first placed at the first entry >= the unit's first column), the
    // column at the cursor in a register (0x7fffffff past the end) and a pair of counts of its own
    const float lab_z = (RANK && gr < M) ? __ldg(epi.tlogit + gr) : 0.f;
    const float lab_p = RANK ? torch_sigmoid(lab_z) : 0.f;
    int n_gt = 0, n_eq = 0;
    const int n_lists = RANK ? epi.n_lists : 0;
    int xb[2] = {0, 0}, xe[2] = {0, 0}, f_gt[2] = {0, 0}, f_eq[2] = {0, 0};
    int x_next[2] = {0x7fffffff, 0x7fffffff};
    if (RANK && gr < M) {
      const int first = n0 + cb;
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (j < n_lists) {
          int b = __ldg(epi.excl_begin + j * M + gr);
          const int e = __ldg(epi.excl_end + j * M + gr);
          for (int hi = e; b < hi;) {
            const int mid = (b + hi) >> 1;
            if (__ldg(epi.excl_col + mid) < first) b = mid + 1; else hi = mid;
          }
          xb[j] = b;
          xe[j] = e;
          if (b < e) x_next[j] = __ldg(epi.excl_col + b);
        }
    }
    const float row_mass = (EPI == 4 && gr < M) ? __ldg(epi.rowmass + gr) : 0.f;
    const float gscale = (!FWD) ? epi.scale * (epi.dscale != nullptr ? __ldg(epi.dscale) : 1.f) : 0.f;
    const float* prow = SOFT ? epi.soft + gr * epi.ldp + n0 : nullptr;   // read only for gr < M
#pragma unroll 1
    for (int lc = 0; lc < P_UN; lc += 8) {
      const int cc = cb + lc;
      if (gr < M && cc < tile_n) {
        const float4 a0 = *reinterpret_cast<const float4*>(srow + lc), a1 = *reinterpret_cast<const float4*>(srow + lc + 4);
        float o[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        // columns are guarded one by one (the class count need not be a multiple of 8)
        const int nv = min(8, tile_n - cc);
        float mx = -3.0e38f;
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (i < nv) {
            if (bz != nullptr) o[i] += __ldg(bz + n0 + cc + i);
            mx = fmaxf(mx, o[i]);
          }
        if (FWD) {
          const float nm = fmaxf(run_m, mx);
          float add = 0.f;
#pragma unroll
          for (int i = 0; i < 8; ++i)
            if (i < nv) {
              add += expf(o[i] - nm);
              if (SOFT) {
                const float p = __ldg(prow + cc + i);
                run_pz += p * o[i];
                run_p += p;
              } else if (n0 + cc + i == tgt) {
                epi.tlogit[gr] = o[i];
              }
            }
          run_s = run_s * expf(run_m - nm) + add;
          run_m = nm;
        } else if (SEL) {
#pragma unroll
          for (int i = 0; i < 8; ++i)
            if (i < nv) {
              const float p = topk_prob(o[i], row_lse, row_w);
              if (p >= sel_tau) {                                      // rare: about k per group pass the threshold
                const int slot = atomicAdd(epi.sel_count + sel_g, 1);
                if (slot < epi.sel_cap) {
                  epi.sel_val[sel_g * epi.sel_cap + slot] = p;
                  epi.sel_idx[sel_g * epi.sel_cap + slot] = sel_base + n0 + cc + i;
                }
              }
            }
        } else if (RANK) {
#pragma unroll
          for (int i = 0; i < 8; ++i)
            if (i < nv) {
              n_gt += o[i] > lab_z;
              n_eq += o[i] == lab_z;
              if (n_lists > 0) {
                const int col = n0 + cc + i;
                const float p = torch_sigmoid(o[i]);
#pragma unroll
                for (int j = 0; j < 2; ++j)
                  if (j < n_lists) {
                    while (x_next[j] < col) x_next[j] = ++xb[j] < xe[j] ? __ldg(epi.excl_col + xb[j]) : 0x7fffffff;
                    const bool zeroed = x_next[j] == col && col != tgt;
                    const float pj = zeroed ? 0.f : p;
                    f_gt[j] += pj > lab_p;
                    f_eq[j] += pj == lab_p;
                  }
              }
            }
        } else {
          float* dp = Cz + gr * ldc + n0 + cc;
#pragma unroll
          for (int i = 0; i < 8; ++i)
            if (i < nv) {
              const float gv = SOFT ? (row_mass * expf(o[i] - row_lse) - __ldg(prow + cc + i)) * gscale
                                    : (expf(o[i] - row_lse) - (n0 + cc + i == tgt ? 1.f : 0.f)) * gscale;
              dp[i] = gv;                                              // row-major: A of dX = dlogits @ W
              epi.dT[(int64_t)(n0 + cc + i) * epi.ldT + gr] = gv;      // transposed (lanes = consecutive rows: coalesced)
            }
        }
      }
    }
    if (RANK && gr < M) {
      int32_t* rc = epi.rank_counts + epi.rank_ld * gr;
      if (n_gt) atomicAdd(rc, n_gt);
      if (n_eq) atomicAdd(rc + 1, n_eq);
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (j < n_lists) {
          if (f_gt[j]) atomicAdd(rc + 2 + 2 * j, f_gt[j]);
          if (f_eq[j]) atomicAdd(rc + 3 + 2 * j, f_eq[j]);
        }
    }
    if (FWD && gr < M) {
      const int64_t pi = (int64_t)(w.nt * 2 + w.half) * M + gr;
      epi.pmax[pi] = run_m;
      epi.psum[pi] = run_s;
      if (SOFT) {
        epi.pdot[pi] = run_pz;
        epi.pmass[pi] = run_p;
      }
    }
  }
  ts.finish(1);
}

// ======================================================================================================
// Resident-panel kernel: EPI 0, no split-K, K <= 224 (the self-loop, the GRU projections)
//
// The timeline of the streaming kernel above (DESIGN §5) shows its consumers starved of operands: every 128 x 104 unit
// re-reads its 186 KB B half from L2 and has its A staged through shared memory by the producer.  Here a panel is one
// (batch entry, column tile, 104-column half) of the packed B.  The CTAs are split evenly over the panels and CTA j of a
// panel's n owns the 64-row tiles [j*R/n, (j+1)*R/n) of its R.  At entry thread 0 issues the copies of the panel's whole
// hi/lo image (n_chunks x 26 KB, one mbarrier per chunk, so chunk 0's MMAs start while the rest lands); B is never
// reloaded.  Three warpgroups, no producer: warpgroup g takes the CTA's tiles g, g + 3, ... and feeds A to wgmma from
// registers (m64n104k8, RS form).  Each thread loads its fragment's elements of rows r and r + 8 straight from global memory
// (rows gathered through a_index), the next chunk's while the current chunk's wgmma group runs, and splits them into
// hi/lo in registers.  Each output element sees the k-steps in order and per k-step the products hi*hi, lo*hi, hi*lo, with
// the same operands as in the streaming kernel.
// The row count is M, or *m_dev when m_dev is set (the deduplicated self-loop product below, whose row count is only known
// on the device): the tiles are split from it, so the work scales with the rows actually present, not with the grid.
// ======================================================================================================
constexpr int R_MAX_CHUNKS = 7;                      // K <= 224: the whole panel fits in shared memory
constexpr int R_CHUNK = 2 * P_BH_BYTES;              // 26624: hi and lo halves of one 32-wide K chunk of a panel
constexpr int R_THREADS = 384;
constexpr int R_SMEM = R_MAX_CHUNKS * R_CHUNK + 1024 + 8 * R_MAX_CHUNKS;
static_assert(R_SMEM <= 232448, "one CTA's shared memory");

template <bool INDEXED>
__global__ void __launch_bounds__(R_THREADS, 1)
umma_gemm_resident_kernel(const float* __restrict__ A, const int32_t* __restrict__ a_index, int64_t lda,
                          const uint8_t* __restrict__ Bp, float* __restrict__ C, int64_t ldc, const float* __restrict__ bias,
                          int64_t M, const int32_t* __restrict__ m_dev, int N, int K, int n_chunks, int accumulate,
                          int64_t batch_a, int64_t batch_bp, int64_t batch_c, int n_panels, int panel_before_wait,
                          long long* dbg) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t sb = raw + ((1024 - (raw & 1023)) & 1023);       // swizzle atoms need 1024-byte alignment
  const uint32_t bar0 = sb + R_MAX_CHUNKS * R_CHUNK;
  const int tid = threadIdx.x;
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);
  // panel p owns the CTAs [p*G/P, (p+1)*G/P) (G >= P: at least one each)
  const int G = gridDim.x, b = blockIdx.x;
  const int p = (int)(((int64_t)(b + 1) * n_panels - 1) / G);
  const int cta0 = (int)((int64_t)p * G / n_panels), ncta = (int)((int64_t)(p + 1) * G / n_panels) - cta0;
  int64_t t_begin, t_end;
  auto split_tiles = [&]() {
    const int64_t n_rt = (M + 63) / 64;
    t_begin = (int64_t)(b - cta0) * n_rt / ncta;
    t_end = (int64_t)(b - cta0 + 1) * n_rt / ncta;
  };
  split_tiles();
  // rows < CTAs: a CTA may have no tile, and it must not issue copies it would never wait for.  With a device row count
  // (M is an upper bound until the wait) any CTA may still get one
  const bool may_work = m_dev != nullptr || t_begin != t_end;
  const int n_tiles = (N + UN - 1) / UN;
  const int half = p & 1, nt = (p >> 1) % n_tiles, zb = (p >> 1) / n_tiles;
  GemmStamps ts(dbg, wg);
  auto copy_panel = [&]() {
    const uint8_t* src = Bp + zb * batch_bp + (size_t)nt * n_chunks * P_B_CHUNK + half * P_BH_BYTES;
    for (int c = 0; c < n_chunks; ++c) {
      const uint32_t bar = bar0 + 8 * c, dst = sb + c * R_CHUNK;
      mbar_expect_tx(bar, R_CHUNK);
      bulk_copy_g2s(dst, src + (size_t)c * P_B_CHUNK, P_BH_BYTES, bar);
      bulk_copy_g2s(dst + P_BH_BYTES, src + (size_t)c * P_B_CHUNK + P_B_BYTES, P_BH_BYTES, bar);
      mbar_arrive(bar);
    }
  };
  if (tid == 0 && may_work) {
    for (int c = 0; c < n_chunks; ++c) mbar_init(bar0 + 8 * c, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    // the packed panel is a weight image: before the wait unless the previous kernel writes it (the launcher knows:
    // a new weight generation packed it in this call)
    if (panel_before_wait) copy_panel();
  }
  // what the previous kernel produced (*m_dev, A and a_index, C when accumulating) is read after the wait; every CTA
  // reaches it (DESIGN §4)
  pdl_wait();
  pdl_trigger();
  if (!may_work) return;
  if (m_dev != nullptr) {
    M = *m_dev;
    split_tiles();
    if (t_begin == t_end) {                                       // no tile after all: the copies land before the CTA exits
      if (tid == 0 && panel_before_wait)
        for (int c = 0; c < n_chunks; ++c) mbar_wait(bar0 + 8 * c, 0);
      return;
    }
  }
  if (tid == 0 && !panel_before_wait) copy_panel();
  __syncthreads();                                                // the barriers are initialised

  const int wt = tid & 127, lane = tid & 31, tig = lane & 3;
  const int ra = 16 * (wt >> 5) + (lane >> 2);                    // this thread's fragment rows: ra, ra + 8
  const float* Az = A + zb * batch_a;
  auto row_ptr = [&](int64_t gr) -> const float* {
    return gr < M ? Az + (INDEXED ? (int64_t)__ldg(a_index + gr) : gr) * lda : nullptr;
  };
  // v[j] = A[row ra][32c + 4j + tig], v[8 + j] = the same of row ra + 8: k-step ks takes j = 2ks (a0, a1) and 2ks + 1 (a2, a3)
  auto load = [&](float (&v)[16], const float* pa, const float* pb, int c) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = c * P_BK + 4 * j + tig;
      v[j] = (pa != nullptr && k < K) ? __ldg(pa + k) : 0.f;
      v[8 + j] = (pb != nullptr && k < K) ? __ldg(pb + k) : 0.f;
    }
  };
  int64_t t = t_begin + wg;
  const float *pa = nullptr, *pb = nullptr;
  float v[16];
  if (t < t_end) {
    pa = row_ptr(t * 64 + ra);
    pb = row_ptr(t * 64 + ra + 8);
    load(v, pa, pb, 0);
  }
  const int n0 = nt * UN, cb = half * P_UN, tile_n = min(UN, N - n0);
  float* Cz = C + zb * batch_c;
  const float* bz = bias != nullptr ? bias + zb * (int64_t)N : nullptr;
  float acc[P_UN / 2];
  for (; t < t_end; t += 3) {
    ++ts.items;
    for (int c = 0; c < n_chunks; ++c) {
      long long t0 = ts.now();
      uint32_t hi[16], lo[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float h, l;
        split_tf32(v[j], h, l);
        hi[j] = __float_as_uint(h);
        lo[j] = __float_as_uint(l);
      }
      ts.aop += ts.now() - t0;
      if (c + 1 < n_chunks) {
        load(v, pa, pb, c + 1);
      } else if (t + 3 < t_end) {                                 // the next tile's first chunk
        pa = row_ptr((t + 3) * 64 + ra);
        pb = row_ptr((t + 3) * 64 + ra + 8);
        load(v, pa, pb, 0);
      }
      t0 = ts.now();
      mbar_wait(bar0 + 8 * c, 0);                                 // chunk c of the panel has landed (once per CTA)
      ts.bar += ts.now() - t0;
      const int nks = min(P_BK / 8, (K - c * P_BK + 7) / 8);      // k-steps that hold data
      const uint32_t b_hi = sb + c * R_CHUNK, b_lo = b_hi + P_BH_BYTES;
      wgmma_fence();                                              // orders the A and accumulator registers for the wgmma
#pragma unroll
      for (int ks = 0; ks < P_BK / 8; ++ks) {
        if (ks < nks) {
          const uint64_t dBh = make_desc_sw128(b_hi + ks * 32), dBl = make_desc_sw128(b_lo + ks * 32);
          const int j = 2 * ks;
          wgmma_tf32_n104_rs(acc, hi[j], hi[8 + j], hi[j + 1], hi[9 + j], dBh, (c | ks) != 0);
          wgmma_tf32_n104_rs(acc, lo[j], lo[8 + j], lo[j + 1], lo[9 + j], dBh, 1);
          wgmma_tf32_n104_rs(acc, hi[j], hi[8 + j], hi[j + 1], hi[9 + j], dBl, 1);
        }
      }
      wgmma_commit();
      t0 = ts.now();
      wgmma_wait<0>();
      ts.mma += ts.now() - t0;
      acc_fence(acc);
      reg_fence(hi);
      reg_fence(lo);
    }
    const long long t0 = ts.now();
    store_fragment(acc, Cz, ldc, bz, t * 64, M, n0, cb, tile_n, accumulate, wt);
    ts.epi += ts.now() - t0;
  }
  ts.finish(2);
}

// ======================================================================================================
// Deduplicated indexed product: C[n] = A[a_index[n]] @ B for n < M, each distinct row computed once
//
// Layer 1's self-loop row of node n is ent_embeds[node_ent[n]] @ W_loop: it depends on the node's entity only, and the batched
// graph is a disjoint union of per-timestamp components, so an entity is a node in many of them (ICEWS18: ~20 % of the
// nodes carry a distinct entity, DESIGN §3).  Three launches, no host synchronisation:
//   1. dedup_insert_kernel: inserts a_index[0..M) into an open-addressing table of 2^bits >= 2M 64-bit keys
//      (epoch << 32 | index).  The epoch changes every call, so a key of an earlier call reads as a free slot and the table
//      is never cleared.  The thread whose CAS claims a slot takes u = atomicAdd(count) and writes uniq[u] and slot_row[slot];
//      every thread records its slot in link[n].  The slot is read before the CAS, so the many inserts of a hub entity
//      mostly find the key without an atomic.  The order of the u is not deterministic; no output bit depends on it.
//   2. umma_gemm_resident_kernel over the U = count distinct rows (indexed through uniq) into a compact P[U, N], its row count
//      read from the device.  Every distinct row sees the same operands, k-steps and product order as it would undeduplicated.
//   3. dedup_expand_kernel: C[n] = P[slot_row[link[n]]], one warp per node, 128-bit loads and stores; it also zeroes count
//      for the next call (the GEMM, its only reader, has completed).
// ======================================================================================================
__device__ __forceinline__ uint32_t dedup_hash(uint32_t v, int bits) { return (v * 0x9E3779B1u) >> (32 - bits); }

__global__ void __launch_bounds__(256)
dedup_insert_kernel(const int32_t* __restrict__ a_index, int64_t M, unsigned long long* __restrict__ table, int bits,
                    uint32_t epoch, int32_t* __restrict__ slot_row, int32_t* __restrict__ uniq, int32_t* __restrict__ link,
                    int32_t* __restrict__ count) {
  pdl_wait();                          // nothing before the wait (count was zeroed by the previous call's expand)
  pdl_trigger();
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= M) return;
  const uint32_t v = (uint32_t)__ldg(a_index + n);
  const unsigned long long key = ((unsigned long long)epoch << 32) | v;
  const uint32_t mask = (1u << bits) - 1;
  uint32_t s = dedup_hash(v, bits);
  for (;;) {
    const unsigned long long cur = __ldcg(table + s);
    if (cur == key) break;
    if ((uint32_t)(cur >> 32) == epoch) {          // another index of this call: linear probing
      s = (s + 1) & mask;
      continue;
    }
    if (atomicCAS(table + s, cur, key) == cur) {   // the slot was free in this call and is ours
      const int32_t u = atomicAdd(count, 1);
      uniq[u] = (int32_t)v;
      slot_row[s] = u;
      break;
    }
    // another thread claimed the slot first: read it again
  }
  link[n] = (int32_t)s;
}

__global__ void __launch_bounds__(256)
dedup_expand_kernel(const float* __restrict__ P, const int32_t* __restrict__ slot_row, const int32_t* __restrict__ link,
                    float* __restrict__ C, int64_t ldc, int64_t M, int N, int32_t* __restrict__ count) {
  pdl_wait();                          // nothing before the wait
  pdl_trigger();
  if (blockIdx.x == 0 && threadIdx.x == 0) *count = 0;
  const int64_t n = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (n >= M) return;
  const int64_t u = __ldg(slot_row + __ldg(link + n));
  const float* src = P + u * N;
  float* dst = C + n * ldc;
  for (int j = 4 * (threadIdx.x & 31); j < N; j += 128) st_f4(dst + j, ldg_f4(src + j));
}

}  // namespace

static long long* g_gemm_dbg = nullptr;
void set_gemm_debug_buffer(long long* p) { g_gemm_dbg = p; }

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
  return launch_pdl("umma_pack_b_kernel", {}, {{Bp, (int64_t)(tile_offset + n_tiles) * n_chunks * P_B_CHUNK}},
                    umma_pack_b_kernel, dim3(n_tiles, n_chunks, 7), dim3(256), 0, stream, B, sk, sn, N, K, (uint8_t*)Bp,
                    n_chunks, tile_offset);
}

// The resident-panel kernel serves EPI 0 products without split-K whose panels fit shared memory and the grid.
static bool resident_ok(int N, int K, int batch) {
  return (K + P_BK - 1) / P_BK <= R_MAX_CHUNKS && batch * ((N + UN - 1) / UN) * 2 <= kNumSMs;
}

// M rows, or *m_dev rows (m_dev != nullptr; M is then an upper bound that sizes the grid)
static int launch_resident(const float* A, const int32_t* a_index, int64_t lda, const void* Bp, float* C, int64_t ldc,
                           const float* bias, int64_t M, const int32_t* m_dev, int N, int K, bool accumulate, int batch,
                           int64_t batch_a, int64_t batch_bp, int64_t batch_c, cudaStream_t stream) {
  static bool attr_r = false;
  if (!attr_r) {
    RENET_CHECK_CUDA(cudaFuncSetAttribute(umma_gemm_resident_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, R_SMEM));
    RENET_CHECK_CUDA(cudaFuncSetAttribute(umma_gemm_resident_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, R_SMEM));
    attr_r = true;
  }
  const int n_chunks = (K + P_BK - 1) / P_BK, n_panels = batch * ((N + UN - 1) / UN) * 2;
  // every panel gets at least one CTA; a CTA never holds more than one panel
  const int64_t n_work = (int64_t)n_panels * ((M + 63) / 64);
  const unsigned grid = (unsigned)(n_work < kNumSMs ? n_work : kNumSMs);
  // The panel copies go before the kernel's griddepcontrol.wait unless the previous kernel writes the packed image (its
  // pack ran in this call); its other inputs are read after the wait, so the launch itself always qualifies for PDL
  const int64_t bp_bytes = (int64_t)(batch - 1) * batch_bp + umma_packed_bytes(N, K);
  const int early = pdl_disjoint(stream, {{Bp, bp_bytes}}) ? 1 : 0;
  const DevSpan c_span = {C, ((int64_t)(batch - 1) * batch_c + (M - 1) * ldc + N) * 4};
  int rc;
  if (a_index)
    rc = launch_pdl("umma_gemm_resident_kernel", {}, {c_span}, umma_gemm_resident_kernel<true>, dim3(grid), dim3(R_THREADS),
                    R_SMEM, stream, A, a_index, lda, (const uint8_t*)Bp, C, ldc, bias, M, m_dev, N, K, n_chunks,
                    (int)accumulate, batch_a, batch_bp, batch_c, n_panels, early, g_gemm_dbg);
  else
    rc = launch_pdl("umma_gemm_resident_kernel", {}, {c_span}, umma_gemm_resident_kernel<false>, dim3(grid), dim3(R_THREADS),
                    R_SMEM, stream, A, a_index, lda, (const uint8_t*)Bp, C, ldc, bias, M, m_dev, N, K, n_chunks,
                    (int)accumulate, batch_a, batch_bp, batch_c, n_panels, early, g_gemm_dbg);
  if (rc) return rc;
  note_gemm_kernel(RENET_GEMM_RESIDENT);
  return RENET_OK;
}

// persistent grid: at most one CTA per SM, each walking a balanced range of 128 x 104 work units
static int launch_streaming(const float* A, const int32_t* a_index, int64_t lda, const void* Bp, float* C, int64_t ldc,
                            const float* bias, int64_t M, int N, int K, bool accumulate, int batch, int64_t batch_a,
                            int64_t batch_bp, int64_t batch_c, int epi_mode, const EpiArgs& epi, int k_splits, int64_t split_c,
                            cudaStream_t stream) {
  static bool attr2 = false;
  if (!attr2) {
    RENET_CHECK_CUDA(cudaFuncSetAttribute(umma_gemm_packed_kernel<true, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, p_smem(0)));
    RENET_CHECK_CUDA(cudaFuncSetAttribute(umma_gemm_packed_kernel<false, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, p_smem(0)));
    RENET_CHECK_CUDA(cudaFuncSetAttribute(umma_gemm_packed_kernel<false, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, p_smem(1)));
    RENET_CHECK_CUDA(cudaFuncSetAttribute(umma_gemm_packed_kernel<false, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, p_smem(2)));
    RENET_CHECK_CUDA(cudaFuncSetAttribute(umma_gemm_packed_kernel<false, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, p_smem(3)));
    RENET_CHECK_CUDA(cudaFuncSetAttribute(umma_gemm_packed_kernel<false, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, p_smem(4)));
    RENET_CHECK_CUDA(cudaFuncSetAttribute(umma_gemm_packed_kernel<false, 5>, cudaFuncAttributeMaxDynamicSharedMemorySize, p_smem(5)));
    RENET_CHECK_CUDA(cudaFuncSetAttribute(umma_gemm_packed_kernel<false, 6>, cudaFuncAttributeMaxDynamicSharedMemorySize, p_smem(6)));
    attr2 = true;
  }
  const int n_tiles = (N + UN - 1) / UN, n_chunks = (K + P_BK - 1) / P_BK;
  const int64_t n_units = (M + UM - 1) / UM * (2 * n_tiles) * batch * k_splits;
  const unsigned grid = (unsigned)(n_units < kNumSMs ? n_units : kNumSMs);
#define RENET_UMMA_LAUNCH(IDX, EP)                                                                                       \
  umma_gemm_packed_kernel<IDX, EP><<<grid, P_THREADS, p_smem(EP), stream>>>(A, a_index, lda, (const uint8_t*)Bp, C, ldc, bias, \
                                                                           M, N, K, n_chunks, accumulate, batch_a, batch_bp,  \
                                                                           batch_c, epi, k_splits, split_c, n_units, \
                                                                           g_gemm_dbg)
  if (epi_mode == 1) RENET_UMMA_LAUNCH(false, 1);
  else if (epi_mode == 2) RENET_UMMA_LAUNCH(false, 2);
  else if (epi_mode == 3) RENET_UMMA_LAUNCH(false, 3);
  else if (epi_mode == 4) RENET_UMMA_LAUNCH(false, 4);
  else if (epi_mode == 5) RENET_UMMA_LAUNCH(false, 5);
  else if (epi_mode == 6) RENET_UMMA_LAUNCH(false, 6);
  else if (a_index) RENET_UMMA_LAUNCH(true, 0);
  else RENET_UMMA_LAUNCH(false, 0);
#undef RENET_UMMA_LAUNCH
  RENET_CHECK_LAUNCH("umma_gemm_packed_kernel");
  note_gemm_kernel(RENET_GEMM_STREAMING);
  return RENET_OK;
}

// C[n] = A[a_index[n]] @ Bp (+bias) for n < M through the distinct rows of a_index (see the kernels above).  The workspace
// is two blocks of the calling stream: the keys block holds the count and the hash table and is written by nothing but
// these kernels, so it is zeroed only when it is new (epoch 0 = empty slot) or every epoch has been used; the rows block
// holds P, slot_row, uniq and link, each written by a call before that call reads it.
static int umma_gemm_dedup(const float* A, const int32_t* a_index, int64_t lda, const void* Bp, float* C, int64_t ldc,
                           const float* bias, int64_t M, int N, int K, cudaStream_t stream) {
  int bits = 1;
  while ((int64_t(1) << bits) < 2 * M) ++bits;              // the table of this call: 2^bits >= 2M slots
  const int64_t slots = int64_t(1) << bits;
  StreamBlock keys, rows;
  int rc = stream_block(kBlockDedupKeys, 256 + slots * 8, stream, &keys);
  if (!rc) rc = stream_block(kBlockDedupRows, (M * N + slots + 2 * M) * 4, stream, &rows);
  if (rc) return rc;
  const uint32_t epoch = (uint32_t)(keys.uses % 0xFFFFFFFFu) + 1;   // 1, 2, ..., 2^32 - 1, 1, ...
  if (epoch == 1) RENET_CHECK_CUDA(cudaMemsetAsync(keys.p, 0, (size_t)keys.bytes, stream));
  int32_t* count = static_cast<int32_t*>(keys.p);
  unsigned long long* table = reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(keys.p) + 256);
  float* P = static_cast<float*>(rows.p);
  int32_t* slot_row = reinterpret_cast<int32_t*>(P + M * N);
  int32_t* uniq = slot_row + slots;
  int32_t* link = uniq + M;
  const DevSpan keys_span = {keys.p, keys.bytes}, rows_span = {rows.p, rows.bytes};
  if ((rc = launch_pdl("dedup_insert_kernel", {}, {keys_span, rows_span}, dedup_insert_kernel, dim3((unsigned)((M + 255) / 256)),
                       dim3(256), 0, stream, a_index, M, table, bits, epoch, slot_row, uniq, link, count)))
    return rc;
  if ((rc = launch_resident(A, uniq, lda, Bp, P, N, bias, M, count, N, K, false, 1, 0, 0, 0, stream))) return rc;
  if ((rc = launch_pdl("dedup_expand_kernel", {}, {{C, ((M - 1) * ldc + N) * 4}, {count, 4}}, dedup_expand_kernel,
                       dim3((unsigned)((M + 7) / 8)), dim3(256), 0, stream, P, slot_row, link, C, ldc, M, N, count)))
    return rc;
  note_gemm_kernel(RENET_GEMM_DEDUP);
  return RENET_OK;
}

// C[b] (+)= A[b] @ Bpacked[b] (+bias[b]) for b < batch; strides in elements (A, C) / bytes (Bp).
// epi_mode 1-4: fused cross-entropy epilogues, 5: grouped top-k candidates, 6: rank counts (EpiArgs); k_splits > 1: split-K partial products at C + s*split_c.
int umma_gemm_prepacked_ex(const float* A, const int32_t* a_index, int64_t lda, const void* Bp, float* C, int64_t ldc,
                           const float* bias, int64_t M, int N, int K, bool accumulate, int batch, int64_t batch_a,
                           int64_t batch_bp, int64_t batch_c, int epi_mode, const EpiArgs& epi, int k_splits, int64_t split_c,
                           cudaStream_t stream) {
  if (M <= 0) return RENET_OK;
  const int n_chunks = (K + P_BK - 1) / P_BK;
  if (k_splits < 1) k_splits = 1;
  if (k_splits > n_chunks) k_splits = n_chunks;
  while (k_splits > 1 && ((n_chunks + k_splits - 1) / k_splits) * (k_splits - 1) >= n_chunks) --k_splits;   // no empty split
  if (epi_mode == 0 && k_splits == 1 && resident_ok(N, K, batch)) {
    const int rc = launch_resident(A, a_index, lda, Bp, C, ldc, bias, M, nullptr, N, K, accumulate, batch, batch_a, batch_bp,
                                   batch_c, stream);
    return rc ? rc : 1;
  }
  const int rc = launch_streaming(A, a_index, lda, Bp, C, ldc, bias, M, N, K, accumulate, batch, batch_a, batch_bp, batch_c,
                                  epi_mode, epi, k_splits, split_c, stream);
  return rc ? rc : k_splits;      // > 0: the number of K-splits actually used (1 = C holds the result)
}

int umma_gemm_prepacked(const float* A, const int32_t* a_index, int64_t lda, const void* Bp, float* C, int64_t ldc,
                        const float* bias, int64_t M, int N, int K, bool accumulate, int batch, int64_t batch_a,
                        int64_t batch_bp, int64_t batch_c, cudaStream_t stream) {
  EpiArgs none{};
  const int r = umma_gemm_prepacked_ex(A, a_index, lda, Bp, C, ldc, bias, M, N, K, accumulate, batch, batch_a, batch_bp, batch_c,
                                       0, none, 1, 0, stream);
  return r < 0 ? r : RENET_OK;
}

// Returns 1 if the shape was taken by the tensor-core path (launch enqueued), 0 if the caller should fall back to the FFMA
// kernel, negative on error.  b_cacheable: B is a weight whose packed image may be cached by address (sgemm_nn).
int umma_gemm_nn_try(const float* A, const int32_t* a_index, int64_t lda, const float* B, int64_t ldb, float* C,
                     int64_t ldc, const float* bias, int64_t M, int32_t N, int32_t K, bool accumulate,
                     cudaStream_t stream, bool b_cacheable) {
  const bool aligned = ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B) | reinterpret_cast<uintptr_t>(C) |
                         reinterpret_cast<uintptr_t>(bias)) & 15) == 0;
  if (!aligned || !umma_shape_ok(N, K) || lda % 4 != 0 || ldc % 4 != 0 || M < 64) return 0;
  // B's packed image: the cached one of this weight, or (cache off) a fresh one in the calling stream's block
  const int64_t pb = umma_packed_bytes(N, K);
  bool hit = false;
  const void* keys[4] = {B, reinterpret_cast<const void*>((intptr_t)ldb), reinterpret_cast<const void*>((intptr_t)N),
                         reinterpret_cast<const void*>((intptr_t)K)};
  void* Bp = b_cacheable ? packed_cache_lookup(keys, 4, pb, &hit) : nullptr;
  int rc = 0;
  if (Bp == nullptr) {
    StreamBlock blk;
    if ((rc = stream_block(kBlockPackedB, pb, stream, &blk))) return rc;
    Bp = blk.p;
  }
  if (!hit && (rc = umma_pack_b(B, ldb, 1, N, K, Bp, 0, stream))) return rc;
  if (a_index != nullptr && !accumulate && M >= kDedupMinRows && resident_ok(N, K, 1))
    rc = umma_gemm_dedup(A, a_index, lda, Bp, C, ldc, bias, M, N, K, stream);
  else
    rc = umma_gemm_prepacked(A, a_index, lda, Bp, C, ldc, bias, M, N, K, accumulate, 1, 0, 0, 0, stream);
  return rc ? rc : 1;
}

// renet_debug_gemm (include/renet_b200.h): every argument form of the engine, on the kernel the dispatch picks or on a forced
// one.  Every precondition is checked before anything is launched.
int debug_gemm(int form, int kernel, const float* A, const int32_t* a_index, int64_t lda, const float* B, int64_t ldb, float* C,
               int64_t ldc, const float* bias, int64_t M, int N, int64_t K, bool accumulate, int batch, int64_t batch_a,
               int64_t batch_b, int64_t batch_c, void* ws, int64_t ws_bytes, cudaStream_t stream) {
  RENET_CHECK_ARG(form >= RENET_GEMM_FORM_NN && form <= RENET_GEMM_FORM_TN, "renet_debug_gemm: unknown form %d", form);
  RENET_CHECK_ARG((kernel >= 0 && kernel <= RENET_GEMM_FFMA_NAIVE) || (kernel >= RENET_GEMM_STREAMING && kernel <= RENET_GEMM_DEDUP),
                  "renet_debug_gemm: unknown kernel %d", kernel);
  RENET_CHECK_ARG(M >= 0 && N > 0 && K > 0 && K < (int64_t(1) << 31) && lda > 0 && ldb > 0 && ldc > 0 && batch >= 1 &&
                      (batch == 1 || form == RENET_GEMM_FORM_PREPACKED),
                  "renet_debug_gemm: bad shape");
  RENET_CHECK_ARG(A && B && C, "renet_debug_gemm: null pointer");
  const bool ffma = kernel == RENET_GEMM_FFMA_TILED || kernel == RENET_GEMM_FFMA_NAIVE;
  if (form == RENET_GEMM_FORM_TN) {
    RENET_CHECK_ARG(kernel == 0 || ffma, "renet_debug_gemm: the tn form runs on the FFMA kernels only");
    RENET_CHECK_ARG(M < (int64_t(1) << 31) && bias == nullptr, "renet_debug_gemm: the tn form takes M < 2^31 and no bias");
    RENET_CHECK_ARG(kernel != RENET_GEMM_FFMA_TILED || sgemm_tn_tiled_ok(A, lda, B, ldb, C, ldc, (int)M, N),
                    "renet_debug_gemm: the tiled tn kernel needs 16-byte aligned operands and M, N, ld* multiples of 4");
    if (M == 0) return RENET_OK;
    return sgemm_tn(A, a_index, lda, B, ldb, C, ldc, (int)M, N, K, accumulate, stream, kernel == RENET_GEMM_FFMA_NAIVE);
  }
  if (form == RENET_GEMM_FORM_NN && (kernel == 0 || ffma)) {
    RENET_CHECK_ARG(kernel != RENET_GEMM_FFMA_TILED || sgemm_nn_tiled_ok(A, lda, B, ldb, C, ldc, bias, N, (int)K),
                    "renet_debug_gemm: the tiled FFMA kernel needs 16-byte aligned operands and N, K, ld* multiples of 4");
    if (M == 0) return RENET_OK;
    if (kernel == 0) return sgemm_nn(A, a_index, lda, B, ldb, C, ldc, bias, M, N, (int)K, accumulate, stream);
    return sgemm_nn_ffma(A, a_index, lda, B, ldb, C, ldc, bias, M, N, (int)K, accumulate, kernel == RENET_GEMM_FFMA_NAIVE,
                         stream);
  }
  // the packed kernels: B (batch of them) packed into the caller's workspace
  RENET_CHECK_ARG(kernel == 0 || kernel == RENET_GEMM_STREAMING || kernel == RENET_GEMM_RESIDENT ||
                      (kernel == RENET_GEMM_DEDUP && form == RENET_GEMM_FORM_NN),
                  "renet_debug_gemm: kernel %d cannot serve form %d", kernel, form);
  const bool aligned = ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(C) | reinterpret_cast<uintptr_t>(bias)) &
                        15) == 0;
  RENET_CHECK_ARG(aligned && umma_shape_ok(N, (int)K) && lda % 4 == 0 && ldc % 4 == 0 && batch_a % 4 == 0 && batch_c % 4 == 0,
                  "renet_debug_gemm: the packed kernels need 16-byte aligned A / C / bias, K %% 4 == 0, N %% 8 == 0 and "
                  "lda, ldc, batch strides multiples of 4");
  RENET_CHECK_ARG((kernel != RENET_GEMM_RESIDENT && kernel != RENET_GEMM_DEDUP) || resident_ok(N, (int)K, batch),
                  "renet_debug_gemm: the resident kernel needs K <= %d and at most %d panels", R_MAX_CHUNKS * P_BK, kNumSMs);
  RENET_CHECK_ARG(kernel != RENET_GEMM_DEDUP || (a_index != nullptr && !accumulate),
                  "renet_debug_gemm: the deduplicated product needs an index and no accumulate");
  const int64_t pb = umma_packed_bytes(N, (int)K);
  RENET_CHECK_ARG(ws != nullptr && ws_bytes >= batch * pb && (reinterpret_cast<uintptr_t>(ws) & 127) == 0,
                  "renet_debug_gemm: the workspace needs %lld bytes, 128-byte aligned", (long long)(batch * pb));
  if (M == 0) return RENET_OK;
  for (int b = 0; b < batch; ++b) {
    const int rc = umma_pack_b(B + b * batch_b, ldb, 1, N, (int)K, static_cast<uint8_t*>(ws) + b * pb, 0, stream);
    if (rc) return rc;
  }
  if (kernel == RENET_GEMM_DEDUP) return umma_gemm_dedup(A, a_index, lda, ws, C, ldc, bias, M, N, (int)K, stream);
  if (kernel == RENET_GEMM_RESIDENT)
    return launch_resident(A, a_index, lda, ws, C, ldc, bias, M, nullptr, N, (int)K, accumulate, batch, batch_a, pb, batch_c,
                           stream);
  if (kernel == RENET_GEMM_STREAMING)
    return launch_streaming(A, a_index, lda, ws, C, ldc, bias, M, N, (int)K, accumulate, batch, batch_a, pb, batch_c, 0,
                            EpiArgs{}, 1, 0, stream);
  return umma_gemm_prepacked(A, a_index, lda, ws, C, ldc, bias, M, N, (int)K, accumulate, batch, batch_a, pb, batch_c, stream);
}

}  // namespace renet
