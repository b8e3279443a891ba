// Persistent bulk-copy ("stream") gather for the RE-Net shape (d_in = d_out = 200, 100 blocks of 2x2): the kernel behind
// renet_rgcn_gather at batch scale (reference RGCN.py:79-94 + 42-48; DGL fn.sum, RGCN.py:91).
//
// Why: the tile kernel (rgcn_tile.cuh) spends about a hundred warp instructions per edge at low warp occupancy, re-fetches
// the 1600-byte relation row of most edges through L2, and every 16-destination tile pays its own dependent index chain and
// two CTA barriers.  Variants that bring source rows in with per-lane LDGs -- including a persistent one with 114 relation
// rows resident in shared memory and two rows prefetched in registers -- stop at the L1TEX request path (4 LDG.64 per
// edge, 7-8 sectors each), not at L2, HBM or the issue slots.  So the loads leave the LSU path:
//   * ONE persistent CTA per SM (32 warps).  CTA c owns the destinations [A_c, A_c+1) whose edge range is 1/gridDim of the
//     graph (node-aligned to the nearer destination start: rounds of a 256-way search in row_ptr, two at ICEWS18 scale),
//     and its warps split that EDGE range evenly at arbitrary cuts;
//   * the most frequent relation rows -- a list the caller passes (relation frequencies are a property of the dataset:
//     GraphStore computes it once), else the top of a histogram of the CTA's own edge types built in the prologue -- are
//     fetched once into shared memory by cp.async.bulk, as many as fit (82 forward: about three quarters of an ICEWS18
//     batch's edges), in 8 groups on 8 mbarriers: an edge waits only for its own group, so the edge loop does not wait for the
//     table;
//   * per edge one elected lane issues a cp.async.bulk of the 800-byte source row into a per-warp ring of D slots,
//     completing on the slot's mbarrier; the warp consumes edge i (4 x LDS.64 + 4 x LDS.128 per lane, conflict-free)
//     while the copies of the next D edges are in flight.  The 1600-byte row of a cold relation is loaded by the lanes
//     straight into the registers that a resident row would be read into (4 x LDG.128, issued before the wait for the
//     source row); the other 31 warps cover its L2 latency.  The edge indices of a block of edges are staged once in
//     shared memory, so the per-edge code has no shuffles; the ring keeps streaming across destinations.
//     On the H100 the edge loop is bound by what each edge moves from L2 (tools/stream_timeline.py: 74 SM cycles per
//     edge with cold rows in the ring and 18 resident rows, 61 with 82; the shared-memory work is about 30): so the
//     ring holds source rows only and the shared memory goes to resident relation rows;
//   * forward with HUB > 0 (layer 1): part of that memory holds "hub" source rows instead -- the CTA's most frequent
//     source nodes (star-like timestamp graphs: about half of a CTA's edges come from a few dozen nodes), chosen by a
//     histogram of its sources in the prologue; an edge from a hub issues no ring copy and reads the resident row;
//   * the running destination's sum stays in registers (edges are destination-sorted: a segmented reduction); a
//     destination that starts and ends inside the warp's range goes straight from registers through the fused
//     norm / self-loop / activation epilogue to global memory; one cut by a warp boundary is handed over through a
//     per-warp head slot + mbarrier in shared memory and finished by the warp that started it, in edge order -- no atomics,
//     bitwise reproducible (which relations are hot only changes where a row is read from, never a value).
// The same body is the backward dH kernel (BWD: reversed CSR, transposed blocks, per-edge scale norm[dst], dH += sum).
#pragma once
#include <type_traits>

#include "common.cuh"
#include "umma.cuh"

namespace renet {

constexpr int kStRpCap = 1024;           // row_ptr entries of the CTA's destinations kept in shared memory
constexpr int kStMaxR2 = 2048;           // relation-id range of the hot-row lookup table (beyond: every row comes from L2)
constexpr int kStNodeCost = 2;           // a destination (epilogue: self-loop row, norm, 800-byte store) costs about two edges
constexpr int kStSlot = 800;             // ring slot: one source row (cold relation rows are loaded into registers)
constexpr int kStHotGroups = 8;          // the resident rows land in 8 groups, one mbarrier each
constexpr int kStHubBins = 2048;         // source-node window of the hub histogram (from the CTA's smallest source node)
constexpr int kStHubScr = kStMaxR2 + 256 + 16;   // prologue scratch (ints into the ring): hub selection, after cnt + hist
// WARPS warps per CTA (>= 16), D edges in flight per warp, HOT relation rows and HUB source rows ("hubs": the CTA's most
// frequent source nodes, forward only) resident per CTA; shared memory map (bytes)
template <int WARPS, int D, int HOT, bool BWD, int HUB = 0>
struct StCfg {
  static constexpr int kWarps = WARPS, kThreads = WARPS * 32, kD = D, kHot = HOT, kHub = HUB;
  static constexpr int kHotPerGroup = (HOT + kStHotGroups - 1) / kStHotGroups;
  static constexpr int kHubPerGroup = HUB > 0 ? (HUB + kStHotGroups - 1) / kStHotGroups : 1;
  static constexpr int kBlk = (32 / D) * D;                                 // edges per index block (a multiple of D)
  static constexpr int kOffRing = 0;                                        // [warps][D][800]; prologue scratch: cnt + hist (+ hub selection)
  static constexpr int kOffHot = kOffRing + WARPS * D * kStSlot;            // [HOT][1600]
  static constexpr int kOffHub = kOffHot + HOT * 1600;                      // [HUB][800]
  static constexpr int kOffHeads = kOffHub + HUB * kStSlot;                 // [warps][200] floats
  static constexpr int kOffRp = kOffHeads + WARPS * 800;                    // [kStRpCap] ints
  static constexpr int kOffSlotOf = kOffRp + kStRpCap * 4;                  // [kStMaxR2] uint8: 1 + hot slot, 0 = cold
  static constexpr int kOffHubOf = kOffSlotOf + kStMaxR2;                   // HUB > 0: [kStHubBins] uint8: 1 + hub slot, 0 = not resident
  static constexpr int kOffIdx = kOffHubOf + (HUB > 0 ? kStHubBins : 0);    // [warps][2][32] int2 {source row, see block_stage}
  static constexpr int kOffSc = kOffIdx + WARPS * 64 * 8;                   // BWD: [warps][2][32] float edge scales
  static constexpr int kOffBars = kOffSc + (BWD ? WARPS * 64 * 4 : 0);      // mbarriers: [warps][D] ring slots, [8] hot groups, [warps] heads, HUB > 0: [8] hub groups
  static constexpr int kOffFlags = kOffBars + (WARPS * D + kStHotGroups + WARPS + (HUB > 0 ? kStHotGroups : 0)) * 8;  // [warps] (unused) + partition scratch (16) + range starts [warps + 1]
  static constexpr int kSmemBytes = kOffFlags + (2 * WARPS + 17) * 4;
  static_assert(WARPS >= 16 && WARPS <= 32, "stream gather: the partition search needs 512 threads");
  static_assert(kBlk == 32, "stream gather: index blocks are 32 edges (D = 2 or 4)");
  static_assert(kSmemBytes <= 227 * 1024, "stream gather: shared memory budget");
  static_assert(WARPS * D * kStSlot >= (kStMaxR2 + 256 + 8) * 4, "stream gather: prologue scratch lives in the ring");
  static_assert(HUB == 0 || WARPS * D * kStSlot >= (kStHubScr + 64 + kStHubBins + 256) * 4, "stream gather: hub scratch lives in the ring");
  static_assert(HOT <= 254 && (kOffHot + HOT * 1600) / 16 < 65536, "stream gather: hot rows are addressed by 16-bit offsets");
  static_assert(HUB <= 255 && (kOffHub + HUB * kStSlot) / 16 < 65536, "stream gather: hub rows are addressed by 16-bit offsets");
  static_assert(!(BWD && HUB), "stream gather: hub source rows are a forward feature");
};
// as many resident rows as fit: forward 82 (about three quarters of ICEWS18's edges with the dataset ranking), backward 77
template <bool BWD>
using StDefault = StCfg<32, 2, BWD ? 77 : 82, BWD>;
// forward on layer 1 (input rows through an index): 49 relation rows + 64 hub source rows in about the 82 rows' space
// (tools/stream_reuse_model.py: about half of a CTA's edges come from its 64 most frequent source nodes)
using StHubs = StCfg<32, 2, 49, false, 64>;

namespace {

__device__ __forceinline__ void st_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void st_cp_async4(uint32_t dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void st_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool st_elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "elect.sync _|p, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}
// first probe without bookkeeping (the copy was issued an edge or more ago: it has usually landed), bounded spin behind it
__device__ __forceinline__ void st_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  if (!done) mbar_wait(bar, parity);
}
// shared-memory loads through 32-bit shared-space addresses with the constant part as an immediate (the generic-pointer
// versions of these made ptxas recompute warp-relative bases per edge: ~25 of 110 instructions)
template <int OFF>
__device__ __forceinline__ float2 st_lds_f2(uint32_t a) {
  float2 r;
  asm volatile("ld.shared.v2.f32 {%0,%1}, [%2+%3];" : "=f"(r.x), "=f"(r.y) : "r"(a), "n"(OFF));
  return r;
}
template <int OFF>
__device__ __forceinline__ float4 st_lds_f4(uint32_t a) {
  float4 r;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4+%5];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "r"(a), "n"(OFF));
  return r;
}
__device__ __forceinline__ uint32_t st_lds_u32(uint32_t a) {
  uint32_t r;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(r) : "r"(a));
  return r;
}
__device__ __forceinline__ uint32_t st_opaque(uint32_t v) {    // keeps a loop-invariant address in a register (no rematerialisation)
  asm volatile("" : "+r"(v));
  return v;
}
__device__ __forceinline__ void st_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// one warp, over a histogram of counts (256 bins, the last one: 255 and more): the smallest threshold thr >= lo with
// #(count >= thr) <= k
__device__ __forceinline__ int st_count_threshold(const int* hist, int k, int lo, int lane) {
  int s = 0;
#pragma unroll
  for (int q = 0; q < 8; ++q) s += hist[lane * 8 + q];
  int suf = s;                                             // inclusive suffix sum over lanes (lane 31 = highest bins)
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int o = __shfl_down_sync(0xffffffffu, suf, d);
    if (lane + d < 32) suf += o;
  }
  int running = suf - s, thr = 256;                        // inside the lane's 8 bins, from the top: running = #(cnt >= bin)
#pragma unroll
  for (int q = 7; q >= 0; --q) {
    running += hist[lane * 8 + q];
    if (running <= k && lane * 8 + q >= lo) thr = lane * 8 + q;
  }
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) thr = min(thr, __shfl_xor_sync(0xffffffffu, thr, d));
  return thr;
}

}  // namespace

// BWD = false: Hout[v] = act(norm[v] * sum_e blockdiag(W[type_e]) . X[src_e] + (HAS_LOOP ? Hout[v] : 0))
// BWD = true:  Hout[u] = (HAS_LOOP ? Hout[u] : 0) + sum_e blockdiag(W[type_e])^T . (norm[col_a[e]] * X[col_a[e]])
// hot_rel [n_hot]: relations whose rows are kept in shared memory (most frequent first), or nullptr: chosen per CTA.
template <bool RELU, bool HAS_LOOP, bool INDEXED, bool BWD, class Cfg = StDefault<BWD>>
__global__ void __launch_bounds__(Cfg::kThreads, 1)
rgcn_gather_stream_kernel(const float* __restrict__ X, const int32_t* __restrict__ x_index, const float* __restrict__ W,
                          const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ col_a,
                          const int32_t* __restrict__ col_type, const float* __restrict__ norm, float* __restrict__ Hout,
                          int N, int R2, const int32_t* __restrict__ hot_rel, int n_hot_arg, int E_hint,
                          long long* __restrict__ dbg) {
  // dbg (tools/stream_timeline.py only; nullptr otherwise): 8 stamps per warp -- SM clock at entry / after the partition /
  // at the first edge / after the last edge / at exit, global timer at entry and exit, edge count
  extern __shared__ __align__(128) uint8_t st_smem[];
  // each stamp is stored when it is taken (its address from the launch parameters and special registers): no register
  // holds a stamp through the edge loop
  auto stamp = [&](int k, long long v) {
    if (dbg && (threadIdx.x & 31) == 0) dbg[((int64_t)blockIdx.x * Cfg::kWarps + (threadIdx.x >> 5)) * 8 + k] = v;
  };
  auto global_timer = []() {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
  };
  if (dbg) { stamp(0, clock64()); stamp(5, global_timer()); }
  constexpr int D = Cfg::kD, kBlk = Cfg::kBlk, kStWarps = Cfg::kWarps, kStThreads = Cfg::kThreads;
  float* heads = reinterpret_cast<float*>(st_smem + Cfg::kOffHeads);
  int32_t* s_rp = reinterpret_cast<int32_t*>(st_smem + Cfg::kOffRp);
  uint8_t* slot_of = st_smem + Cfg::kOffSlotOf;
  int* flags = reinterpret_cast<int*>(st_smem + Cfg::kOffFlags);
  int* s_part = flags + kStWarps;                                          // [16] partition / selection scratch
  int* s_e0 = s_part + 16;                                                 // [warps + 1] first edge of every warp's range
  uint64_t* bars = reinterpret_cast<uint64_t*>(st_smem + Cfg::kOffBars);
  int* cnt = reinterpret_cast<int*>(st_smem + Cfg::kOffRing);              // prologue only: [kStMaxR2] + hist[256]
  int* hist = cnt + kStMaxR2;

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);    // warp-uniform for the compiler
  // lane l owns the 2x2 blocks l, l + 32, l + 64 and -- lanes 0..3 only -- 96 + l: three full 32-lane rounds and one
  // four-lane round per row, i.e. 20 shared-memory wavefronts per edge instead of the 24 of a 25-lane x 4 mapping
  const bool tail4 = lane < 4;
  const bool use_hot = R2 > 0 && R2 <= kStMaxR2 && Cfg::kHot > 0;
  const bool given_hot = use_hot && hot_rel != nullptr;
  // The prologue is a chain of dependent reads (edge count -> two search rounds -> row_ptr slice -> edge indices -> row
  // indirection -> first rows); when the graph arrays are cold in HBM every link costs a DRAM latency.  So first thing, the grid pulls the index arrays into L2, one 128-byte line per thread: the chain then
  // pays one DRAM latency (the edge count) and L2 latencies after that.  E_hint >= E is the caller's edge count / capacity.
  {
    const int64_t gt = (int64_t)blockIdx.x * Cfg::kThreads + threadIdx.x;
    const int64_t n_rp_lines = ((int64_t)N + 1 + 31) / 32, n_e_lines = ((int64_t)E_hint + 31) / 32;
    const char* pf = nullptr;
    if (gt < n_rp_lines) pf = reinterpret_cast<const char*>(row_ptr) + gt * 128;
    else if (gt < n_rp_lines + n_e_lines) pf = reinterpret_cast<const char*>(col_a) + (gt - n_rp_lines) * 128;
    else if (gt < n_rp_lines + 2 * n_e_lines) pf = reinterpret_cast<const char*>(col_type) + (gt - n_rp_lines - n_e_lines) * 128;
    else if (INDEXED && gt < 2 * n_rp_lines + 2 * n_e_lines - 1)
      pf = reinterpret_cast<const char*>(x_index) + (gt - n_rp_lines - 2 * n_e_lines) * 128;
    if (pf) asm volatile("prefetch.global.L2 [%0];" ::"l"(pf));
  }
  const int E = __ldg(row_ptr + N);
  // CTA partition search, first round: its probe positions depend on N only, so its loads fly with the edge count's
  // (the search itself is below)
  const int half = tid >> 8, ht = tid & 255;
  const int c_idx = blockIdx.x + half;
  const bool searching = tid < 512 && c_idx > 0 && c_idx < (int)gridDim.x;
  const int probe0 = min((ht + 1) * (N / 256 + 1) - 1, N);
  const int val0 = searching ? __ldg(row_ptr + probe0) : 0;
  // the caller's hot-relation list: copied by warp 1 into the (then unused) histogram scratch now, used after the search
  // (slot table, resident-row copies).  An asynchronous copy: neither the warp nor a register waits for it meanwhile
  constexpr int kHotIters = (Cfg::kHot + 31) / 32;
  const int n_hot_given = given_hot ? min(n_hot_arg, Cfg::kHot) : 0;
  if (warp == 1) {
    for (int sl = lane; sl < n_hot_given; sl += 32) st_cp_async4(smem_u32(hist + sl), hot_rel + sl);
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  const uint32_t hot_bar0 = smem_u32(bars + kStWarps * D);   // [8]: "the resident rows of group g have landed"
  const uint32_t head_bar0 = hot_bar0 + kStHotGroups * 8;    // [warps]: "this warp's head slot is written"
  const uint32_t hub_bar0 = head_bar0 + kStWarps * 8;        // HUB > 0: [8] "the hub rows of group g have landed"

  if (tid < 16) s_part[tid] = 0;
  if (tid < kStWarps) flags[tid] = 0;
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < D; ++k) mbar_init(smem_u32(bars + warp * D + k), 1);
    mbar_init(head_bar0 + warp * 8, 1);
    if (warp == 0)
      for (int gr = 0; gr < kStHotGroups; ++gr) mbar_init(hot_bar0 + gr * 8, 1);
    if (Cfg::kHub > 0 && warp == 1)
      for (int gr = 0; gr < kStHotGroups; ++gr) mbar_init(hub_bar0 + gr * 8, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (!given_hot)
    for (int i = tid; i < kStMaxR2 + 256; i += kStThreads) cnt[i] = 0;
  for (int i = tid; i < kStMaxR2 / 4; i += kStThreads) reinterpret_cast<uint32_t*>(slot_of)[i] = 0u;
  // hub selection scratch: [0] window start (smallest source node), [1] count threshold, [2] hubs above it, [8..40)
  // per-warp tie counts, [64..) node counts [kStHubBins] + count histogram [256]
  constexpr int kHub = Cfg::kHub;
  int* hub_scr = cnt + kStHubScr;
  uint8_t* hub_of = st_smem + Cfg::kOffHubOf;
  if constexpr (kHub > 0) {
    for (int i = tid; i < 64 + kStHubBins + 256; i += kStThreads) hub_scr[i] = i == 0 ? INT_MAX : 0;
    for (int i = tid; i < kStHubBins / 4; i += kStThreads) reinterpret_cast<uint32_t*>(hub_of)[i] = 0u;
  }
  __syncthreads();
  // resident rows (slot sl = lane + 32 k holds relation row_of(k)) -> shared memory, one warp; slot sl lands on the barrier
  // of group sl / kHotPerGroup, so an edge waits only for its own group and the edge loop starts before the table is
  // complete.  Every group barrier gets its one arrival (an empty group completes at once).  Issued after the partition
  // search: the grid's 17 MB of copies (82 rows x 132 SMs) would otherwise share L2 with the search's dependent reads.
  auto load_hot = [&](int n_hot, auto row_of) {
    if (lane < kStHotGroups) {
      const int rows = min(max(n_hot - lane * Cfg::kHotPerGroup, 0), Cfg::kHotPerGroup);
      st_expect_tx(hot_bar0 + lane * 8, (uint32_t)rows * 1600u);
    }
    __syncwarp();
#pragma unroll
    for (int k = 0; k < kHotIters; ++k) {
      const int sl = lane + 32 * k;
      if (sl < n_hot)
        st_bulk_g2s(smem_u32(st_smem + Cfg::kOffHot + sl * 1600), W + (int64_t)row_of(k) * 400, 1600,
                    hot_bar0 + (sl / Cfg::kHotPerGroup) * 8);
    }
  };
  // ---- CTA partition: destinations [A, A_next) own 1/gridDim of the edges (node-aligned).  Threads 0..255 look for
  //      lower_bound(row_ptr, T_c), threads 256..511 for lower_bound(row_ptr, T_c+1).  Invariant: the answer lies in
  //      [lo, hi]; every round probes 256 evenly spaced entries of the bracket and keeps the 1/256 of it between the last
  //      probe below the target and the first one at or above it.  The number of rounds depends on N only (uniform over
  //      the CTA); the last round probes consecutive entries, so the thread that hits the answer also holds
  //      row_ptr[answer] and its left neighbour the entry before ---------------------------------------------------------------
  // work is counted in edges + kStNodeCost per destination: key(v) = row_ptr[v] + kStNodeCost * v ascends with v
  const int64_t total_cost = (int64_t)E + (int64_t)kStNodeCost * N;
  const int64_t target = ((int64_t)c_idx * total_cost) / gridDim.x;
  int lo = 0, hi = N;
  const int rounds = N < 256 ? 1 : (N < 65536 ? 2 : (N < (1 << 24) ? 3 : 4));
  for (int r = 0; r < rounds; ++r) {
    const int step = (hi - lo) / 256 + 1;
    const int p = min(lo + (ht + 1) * step - 1, hi);       // the last probes are clipped to hi, where key >= target
    const int val = r == 0 ? val0 : (searching ? __ldg(row_ptr + p) : 0);   // (round 0: loaded at entry, p == probe0)
    const bool below = searching && (int64_t)val + (int64_t)kStNodeCost * p < target;
    const unsigned m = __ballot_sync(0xffffffffu, below);
    if (lane == 0 && m) atomicAdd(&s_part[2 * r + (half & 1)], __popc(m));      // row_ptr ascends: # probes below the target
    __syncthreads();
    const int f = s_part[2 * r + (half & 1)];
    if (r == rounds - 1 && searching) {                    // step == 1: thread f probed the answer, thread f - 1 the entry before
      if (ht == f) { s_part[10 + half] = lo + f; s_part[12 + half] = val; }
      if (ht == f - 1) s_part[14 + half] = val + 1;        // + 1: 0 means "not seen"
    }
    const int new_hi = min(lo + (f + 1) * step - 1, hi);
    const int new_lo = f == 0 ? lo : min(lo + f * step - 1, hi) + 1;
    lo = new_lo; hi = new_hi;
  }
  __syncthreads();
  // ---- hot rows from the caller's list (slot table complete at the __syncthreads after the row_ptr slice) ---------------------
  if (given_hot && warp == 1) {
    asm volatile("cp.async.wait_all;" ::: "memory");      // this lane's entries of the list
    load_hot(n_hot_given, [&](int k) {
      const int sl = lane + 32 * k, r = hist[sl];
      const bool ok = r >= 0 && r < R2;                    // an id outside the table is ignored (its slot holds row 0, unused)
      if (ok) slot_of[r] = (uint8_t)(sl + 1);
      return ok ? r : 0;
    });
  }
  // the boundary goes to whichever of the two destination starts around the target is nearer (halves the imbalance a
  // heavy destination causes); both CTAs that share a boundary derive it from the same target by the same rule
  int A = 0, A_next = N, cb = 0, ce = E;
  if (blockIdx.x > 0) {
    A = s_part[10]; cb = s_part[12];
    const int64_t tgt = ((int64_t)blockIdx.x * total_cost) / gridDim.x;
    const int64_t k_hi = (int64_t)cb + (int64_t)kStNodeCost * A, k_lo = (int64_t)(s_part[14] - 1) + (int64_t)kStNodeCost * (A - 1);
    if (s_part[14] && k_hi - tgt > tgt - k_lo) { --A; cb = s_part[14] - 1; }
  }
  if (blockIdx.x + 1 < gridDim.x) {
    A_next = s_part[11]; ce = s_part[13];
    const int64_t tgt = ((int64_t)(blockIdx.x + 1) * total_cost) / gridDim.x;
    const int64_t k_hi = (int64_t)ce + (int64_t)kStNodeCost * A_next, k_lo = (int64_t)(s_part[15] - 1) + (int64_t)kStNodeCost * (A_next - 1);
    if (s_part[15] && k_hi - tgt > tgt - k_lo) { --A_next; ce = s_part[15] - 1; }
  }
  if (dbg) stamp(1, clock64());
  const int n_rp = A_next - A + 1;
  const bool rp_in_smem = n_rp <= kStRpCap;
  auto rp = [&](int v) -> int { return rp_in_smem ? s_rp[v - A] : __ldg(row_ptr + v); };   // row_ptr[v], v in [A, A_next]
  if (rp_in_smem)
    for (int i = tid; i < n_rp; i += kStThreads) s_rp[i] = __ldg(row_ptr + A + i);
  if constexpr (kHub > 0) {            // hub window start: the smallest source node of the CTA's edges
    int m = INT_MAX;
    for (int e = cb + tid; e < ce; e += kStThreads) m = min(m, __ldg(col_a + e));
    m = __reduce_min_sync(0xffffffffu, m);
    if (lane == 0 && m != INT_MAX) atomicMin(&hub_scr[0], m);
  }
  __syncthreads();
  const int hub_lo = kHub > 0 ? hub_scr[0] : 0;
  // warp ranges: the CTA's work (edges + kStNodeCost per destination) is cut into equal shares at arbitrary EDGE positions.
  // cost(v) = work before destination v; warp j starts inside the last destination whose cost(v) <= j/warps of the total
  const int64_t cta_cost = (int64_t)(ce - cb) + (int64_t)kStNodeCost * (A_next - A);
  auto range_start = [&](int j) -> int {
    const int64_t T = (cta_cost * j) / kStWarps;
    int l = A, h = A_next;
    while (l < h) {
      const int mid = (l + h + 1) >> 1;
      if ((int64_t)(rp(mid) - cb) + (int64_t)kStNodeCost * (mid - A) <= T) l = mid; else h = mid - 1;
    }
    if (l >= A_next) return ce;
    const int64_t r = T - ((int64_t)(rp(l) - cb) + (int64_t)kStNodeCost * (l - A));
    return rp(l) + (int)min(r, (int64_t)(rp(l + 1) - rp(l)));
  };
  const int e0 = range_start(warp), e1 = warp + 1 < kStWarps ? range_start(warp + 1) : ce;
  const int n = e1 - e0;
  if (lane == 0) { s_e0[warp] = e0; if (warp == kStWarps - 1) s_e0[kStWarps] = ce; }

  // ---- edge index blocks: block b = edges e0 + kBlk b .. + kBlk - 1, one per lane, staged in shared memory ------------------
  int2* my_idx = reinterpret_cast<int2*>(st_smem + Cfg::kOffIdx) + warp * 64;   // [2][32] {source row, relation | w_off16 << 16}
  float* my_sc = reinterpret_cast<float*>(st_smem + Cfg::kOffSc) + warp * 64;
  int ld_s = 0, ld_t = 0;              // block being loaded: raw indices in registers until they are staged
  float ld_sc = 1.f;
  auto block_load = [&](int b) {       // phase 1: coalesced index loads
    const int e = e0 + b * kBlk + lane;
    ld_s = 0; ld_t = 0; ld_sc = 1.f;
    if (lane < kBlk && e < e1) {
      ld_s = __ldg(col_a + e);
      ld_t = __ldg(col_type + e);
    }
  };
  auto block_gather = [&](int b) {     // phase 2: dependent loads (edge scale, row indirection)
    const int e = e0 + b * kBlk + lane;
    bool hub = false;
    if constexpr (kHub > 0) {          // residency is keyed by the source node, before the row indirection
      const unsigned w = (unsigned)(ld_s - hub_lo);
      const int hs = lane < kBlk && e < e1 && w < (unsigned)kStHubBins ? (int)hub_of[w] : 0;
      hub = hs != 0;                   // staged as 1 << 31 | its group << 16 | its row's byte offset / 16
      if (hub) ld_s = (int)(0x80000000u | (uint32_t)((hs - 1) / Cfg::kHubPerGroup) << 16 |
                            (uint32_t)((Cfg::kOffHub + (hs - 1) * kStSlot) >> 4));
    }
    if ((BWD || INDEXED) && lane < kBlk && e < e1 && !hub) {
      if (BWD) ld_sc = __ldg(norm + ld_s);
      if (INDEXED) ld_s = __ldg(x_index + ld_s);
    }
  };
  // phase 3: to shared memory.  Second word: a resident row's byte offset / 16 << 16 | its group, else the relation id.
  // First word: the source row (HUB > 0: or a resident source's hub word, see block_gather)
  auto block_stage = [&](int b) {
    const int hs = use_hot ? (int)slot_of[ld_t] : 0;
    const int woff16 = hs ? (Cfg::kOffHot + (hs - 1) * 1600) >> 4 : 0;
    my_idx[(b & 1) * 32 + lane] = make_int2(ld_s, hs ? (woff16 << 16) | ((hs - 1) / Cfg::kHotPerGroup) : ld_t);
    if (BWD) my_sc[(b & 1) * 32 + lane] = ld_sc;
    __syncwarp();
  };
  block_load(0);

  // ---- no caller list: relation histogram of the CTA's own edges -> hot rows ----------------------------------------------
  if (use_hot && !given_hot) {
    for (int e = e0 + lane; e < e1; e += 32) atomicAdd(&cnt[__ldg(col_type + e)], 1);
    __syncthreads();
    for (int r = tid; r < R2; r += kStThreads) {
      const int c = cnt[r];
      if (c > 0) atomicAdd(&hist[min(c, 255)], 1);
    }
    __syncthreads();
    if (warp == 0) {
      const int thr = st_count_threshold(hist, Cfg::kHot, 1, lane);
      if (lane == 0) s_part[8] = thr;
    }
    __syncthreads();
    const int thr = s_part[8];
    for (int r = tid; r < R2; r += kStThreads) {
      if (min(cnt[r], 255) >= thr) {                       // at most HOT relations pass
        const int slot = atomicAdd(&s_part[9], 1);
        slot_of[r] = (uint8_t)(slot + 1);
        hist[slot] = r;                                    // hist is dead: reuse as the slot -> relation list
      }
    }
    __syncthreads();
    // remaining slots: relations one count below the threshold (any of them: the choice never changes a value)
    if (thr > 1) {
      for (int r = tid; r < R2; r += kStThreads) {
        if (min(cnt[r], 255) == thr - 1) {
          const int slot = atomicAdd(&s_part[9], 1);
          if (slot < Cfg::kHot) { slot_of[r] = (uint8_t)(slot + 1); hist[slot] = r; }
        }
      }
      __syncthreads();
    }
    if (warp == 1) load_hot(min(s_part[9], Cfg::kHot), [&](int k) { return hist[lane + 32 * k]; });
  }
  // ---- hub source rows: the CTA's HUB most frequent source nodes among the kStHubBins from its smallest one (a node of at
  //      least 2 edges; ties at the threshold go to the smaller node ids).  Warp 2 fetches their rows (below) --------------
  constexpr int kHubIters = kHub > 0 ? (kHub + 31) / 32 : 1;
  int hub_row[kHubIters];
  int n_hub = 0;
  if constexpr (kHub > 0) {
    int* hcnt = hub_scr + 64;
    int* hhist = hcnt + kStHubBins;    // count histogram, then the slot -> node list
    for (int e = cb + tid; e < ce; e += kStThreads) {
      const unsigned w = (unsigned)(__ldg(col_a + e) - hub_lo);
      if (w < (unsigned)kStHubBins) atomicAdd(&hcnt[w], 1);
    }
    __syncthreads();
    for (int b = tid; b < kStHubBins; b += kStThreads) {
      const int c = hcnt[b];
      if (c >= 2) atomicAdd(&hhist[min(c, 255)], 1);
    }
    __syncthreads();
    if (warp == 0) {
      const int thr = st_count_threshold(hhist, kHub, 2, lane);
      if (lane == 0) hub_scr[1] = thr;
    }
    __syncthreads();
    // thread t owns the nodes [t kPer, (t + 1) kPer): thread order is node order, so ranking the ties is a prefix sum
    constexpr int kPer = (kStHubBins + kStThreads - 1) / kStThreads;
    const int thr = hub_scr[1];
    int ties = 0;
#pragma unroll
    for (int q = 0; q < kPer; ++q) {
      const int b = tid * kPer + q;
      if (b < kStHubBins) {
        const int c = min(hcnt[b], 255);
        if (c >= thr) {                // at most HUB nodes
          const int sl = atomicAdd(&hub_scr[2], 1);
          hub_of[b] = (uint8_t)(sl + 1);
          hhist[sl] = b;
        } else if (c == thr - 1 && c >= 2) {
          ++ties;
        }
      }
    }
    int incl = ties;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += o;
    }
    if (lane == 31) hub_scr[8 + warp] = incl;
    __syncthreads();
    const int n_above = hub_scr[2];
    int rank = n_above + __reduce_add_sync(0xffffffffu, lane < warp ? hub_scr[8 + lane] : 0) + incl - ties;
#pragma unroll
    for (int q = 0; q < kPer; ++q) {
      const int b = tid * kPer + q;
      if (b < kStHubBins && min(hcnt[b], 255) == thr - 1 && thr - 1 >= 2) {
        if (rank < kHub) { hub_of[b] = (uint8_t)(rank + 1); hhist[rank] = b; }
        ++rank;
      }
    }
    __syncthreads();                   // hub_of and the slot list are complete
    if (warp == 2) {
      n_hub = min(kHub, n_above + __reduce_add_sync(0xffffffffu, lane < kStWarps ? hub_scr[8 + lane] : 0));
#pragma unroll
      for (int k = 0; k < kHubIters; ++k) {
        const int sl = lane + 32 * k;
        hub_row[k] = sl < n_hub ? (INDEXED ? __ldg(x_index + hub_lo + hhist[sl]) : hub_lo + hhist[sl]) : 0;
      }
    }
  }
  block_gather(0);
  __syncthreads();                     // s_rp, slot_of complete; the ring (= cnt / hist) may be overwritten from here on
  block_stage(0);
  block_load(1);

  const uint32_t ring = st_opaque(smem_u32(st_smem + Cfg::kOffRing + warp * D * kStSlot));
  const uint32_t bar0 = st_opaque(smem_u32(bars + warp * D));
  const uint32_t idx_a = st_opaque(smem_u32(my_idx));        // entry of local edge k: idx_a + (k & 63) * 8
  // copy of local edge k's source row into ring slot `slot` (both warp-uniform)
  auto issue = [&](int k, int slot) {
    if (st_elect_one()) {
      const uint32_t src = st_lds_u32(idx_a + (((uint32_t)k & 63u) << 3));
      const uint32_t bar = bar0 + slot * 8;
      st_expect_tx(bar, 800u);
      st_bulk_g2s(ring + slot * kStSlot, X + (int64_t)(int)src * 200, 800, bar);
    }
  };
  // Everything above read graph structure, weights and the relation ranking only; from here on the kernel touches what
  // the previous kernel in the stream produced (the self-loop rows in Hout; layer 2's input rows).  A launcher that uses
  // programmatic stream serialisation gets the prologue overlapped with that kernel's tail; in plain stream order (what
  // the library does, see rgcn_fwd.cu) this wait returns immediately.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if constexpr (kHub > 0) {
    if (warp == 2) {                   // the hub rows, on 8 group barriers (every barrier gets its arrival)
      if (lane < kStHotGroups)
        st_expect_tx(hub_bar0 + lane * 8,
                     (uint32_t)min(max(n_hub - lane * Cfg::kHubPerGroup, 0), Cfg::kHubPerGroup) * (uint32_t)kStSlot);
      __syncwarp();
#pragma unroll
      for (int k = 0; k < kHubIters; ++k) {
        const int sl = lane + 32 * k;
        if (sl < n_hub)
          st_bulk_g2s(smem_u32(st_smem + Cfg::kOffHub + sl * kStSlot), X + (int64_t)hub_row[k] * 200, kStSlot,
                      hub_bar0 + (sl / Cfg::kHubPerGroup) * 8);
      }
    }
  } else {
#pragma unroll
    for (int k = 0; k < D; ++k)
      if (k < n) issue(k, k);
  }

  // ---- first destination of the range (binary search in the CTA's row_ptr slice while the first copies fly) -----------------
  int va;
  {
    int l = A, h = A_next;             // smallest v in [A, A_next] with rp(v) >= e0
    while (h > l) {
      const int mid = (l + h) >> 1;
      if (rp(mid) >= e0) h = mid; else l = mid + 1;
    }
    va = l;
  }
  int cur = va;
  bool continued = false;
  if (n > 0 && rp(va) > e0) { cur = va - 1; continued = true; }     // edges e0.. finish a destination an earlier warp started
  int cur_end = cur < A_next ? rp(cur + 1) : ce;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  // self-loop row (already in Hout) and norm of the running destination, fetched when it becomes the running one: its
  // epilogue comes at least one edge later, and one edge of a warp outlasts a load (32 warps take turns on the SM)
  float2 lp[4];
  float nrm = 1.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) lp[k] = make_float2(0.f, 0.f);
  auto fetch_dest = [&](int v) {
    if (v < A_next) {
      if (HAS_LOOP) {
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (k < 3 || tail4) lp[k] = *reinterpret_cast<const float2*>(Hout + (int64_t)v * 200 + 2 * (lane + 32 * k));
      }
      if (!BWD) nrm = __ldg(norm + v);
    }
  };
  auto epilogue = [&](int v) {         // registers -> global, fused norm / self-loop / activation
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (k < 3 || tail4) {
        float2 o = make_float2(acc[2 * k], acc[2 * k + 1]);
        if (!BWD) { o.x *= nrm; o.y *= nrm; }
        if (HAS_LOOP) { o.x += lp[k].x; o.y += lp[k].y; }
        if (RELU) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); }
        *reinterpret_cast<float2*>(Hout + (int64_t)v * 200 + 2 * (lane + 32 * k)) = o;
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  };
  auto publish_head = [&]() {          // partial sum of a destination an earlier warp started
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (k < 3 || tail4)
        *reinterpret_cast<float2*>(heads + warp * 200 + 2 * (lane + 32 * k)) = make_float2(acc[2 * k], acc[2 * k + 1]);
    __syncwarp();
    if (lane == 0) st_arrive(head_bar0 + warp * 8);        // release: the head slot is visible to whoever observes the phase
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  };
  // the running destination `cur` is complete (all of its edges end at or before the current position): finish it and
  // make cur + 1 the running destination
  int cur_beg = cur < A_next ? rp(cur) : ce;
  auto advance = [&]() {
    if (continued) { publish_head(); continued = false; }
    else if (cur_end > cur_beg) epilogue(cur);     // destinations without edges were written by the prologue pass
    ++cur;
    cur_beg = cur_end;
    cur_end = cur < A_next ? rp(cur + 1) : ce;
    fetch_dest(cur);                               // (rows of destinations without edges are fetched too: harmless)
  };
  if (!continued) fetch_dest(cur);

  const uint32_t ring_l8 = st_opaque(ring + 8 * lane);
  const uint32_t smem_l16 = st_opaque(smem_u32(st_smem) + 16 * lane);
  const float* w_l4 = W + 4 * lane;                         // lane's first block of a cold relation row
  uint32_t hot_seen = 0;                                     // bit g: this warp has seen hot group g complete
  const uint32_t sc_a = BWD ? st_opaque(smem_u32(my_sc)) : 0u;
  uint32_t parity = 0;
  // index blocks: load -> dependent loads -> stage, spread over the block so that no load is waited for
  constexpr int kP1 = (kBlk / D / 3) * D, kP2 = (2 * (kBlk / D) / 3) * D;
  int phase_at = kP1, phase = 0, blk = 0;
  if (dbg) stamp(2, clock64());
  if constexpr (kHub == 0) {
    for (int g = 0; g < n; g += D) {     // one pass over the ring: slot numbers are compile-time constants
      if (g == phase_at) {
        if (phase == 0) { block_gather(blk + 1); phase_at += kP2 - kP1; phase = 1; }
        else if (phase == 1) { block_stage(blk + 1); phase_at += kBlk - kP2; phase = 2; }
        else { ++blk; block_load(blk + 1); phase_at += kP1; phase = 0; }
      }
      auto do_slot = [&](auto slot_c) {
        constexpr int slot = decltype(slot_c)::value;
        const int i = g + slot;
        if (i < n) {
          while (e0 + i >= cur_end) advance();       // warp-uniform: the running destination is complete
          const uint32_t wsel = st_lds_u32(idx_a + (((uint32_t)i & 63u) << 3) + 4);
          const uint32_t woff16 = wsel >> 16;
          const float sc = BWD ? __uint_as_float(st_lds_u32(sc_a + (((uint32_t)i & 63u) << 2))) : 1.f;
          float2 h[4];
          float4 w[4];
          w[3] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (woff16) {                  // resident row: wait for its group once per warp
            const uint32_t grp = wsel & 0xffffu;
            if (!((hot_seen >> grp) & 1u)) { mbar_wait(hot_bar0 + grp * 8, 0); hot_seen |= 1u << grp; }
            const uint32_t wa = smem_l16 + (woff16 << 4);
            w[0] = st_lds_f4<0>(wa); w[1] = st_lds_f4<512>(wa); w[2] = st_lds_f4<1024>(wa);
            if (tail4) w[3] = st_lds_f4<1536>(wa);
          } else {                       // cold row: straight from L2 into registers, in flight while the source row is awaited
            const float* wr = w_l4 + (int64_t)(int)wsel * 400;
            w[0] = ldg_f4(wr); w[1] = ldg_f4(wr + 128); w[2] = ldg_f4(wr + 256);
            if (tail4) w[3] = ldg_f4(wr + 384);
          }
          st_wait(bar0 + slot * 8, parity);
          h[0] = st_lds_f2<slot * kStSlot>(ring_l8);       h[1] = st_lds_f2<slot * kStSlot + 256>(ring_l8);
          h[2] = st_lds_f2<slot * kStSlot + 512>(ring_l8);
          h[3] = make_float2(0.f, 0.f);
          if (tail4) h[3] = st_lds_f2<slot * kStSlot + 768>(ring_l8);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float x = BWD ? h[k].x * sc : h[k].x, y = BWD ? h[k].y * sc : h[k].y;
            if (!BWD) {                  // out[j] += sum_i in[i] * W[i][j]
              acc[2 * k] = fmaf(x, w[k].x, fmaf(y, w[k].z, acc[2 * k]));
              acc[2 * k + 1] = fmaf(x, w[k].y, fmaf(y, w[k].w, acc[2 * k + 1]));
            } else {                     // din[i] += sum_j W[i][j] * g[j]
              acc[2 * k] = fmaf(x, w[k].x, fmaf(y, w[k].y, acc[2 * k]));
              acc[2 * k + 1] = fmaf(x, w[k].z, fmaf(y, w[k].w, acc[2 * k + 1]));
            }
          }
          __syncwarp();                  // every lane has consumed the slot (the FMAs depend on the loads)
          if (i + D < n) issue(i + D, slot);
        }
      };
      do_slot(std::integral_constant<int, 0>{});
      do_slot(std::integral_constant<int, 1>{});
      if constexpr (D == 4) {
        do_slot(std::integral_constant<int, 2>{});
        do_slot(std::integral_constant<int, 3>{});
      }
      parity ^= 1u;
    }
  } else {
    // the ring takes the edges whose source is not resident, in edge order, D copies in flight: `iss` is the next edge to
    // look at (the staged ones: block blk + 1 from phase 2 on), `fly` the copies issued and not consumed, the oldest of
    // them in slot `rslot`.  An edge whose source is resident waits once per warp for its hub group (hot_seen bit 8 + g)
    // and reads the hub row
    int iss = 0, fly = 0, rslot = 0;
    auto top_up = [&]() {
      const int lim = min(n, (blk + (phase == 2 ? 2 : 1)) * kBlk);
      while (fly < D && iss < lim) {
        const uint32_t src = st_lds_u32(idx_a + (((uint32_t)iss & 63u) << 3));
        if (!(src >> 31)) {
          const int wslot = (rslot + fly) % D;
          if (st_elect_one()) {
            const uint32_t bar = bar0 + wslot * 8;
            st_expect_tx(bar, 800u);
            st_bulk_g2s(ring + wslot * kStSlot, X + (int64_t)(int)src * 200, 800, bar);
          }
          ++fly;
        }
        ++iss;
      }
    };
    top_up();
    const uint32_t smem_l8 = st_opaque(smem_u32(st_smem) + 8 * lane);
    for (int i = 0; i < n; ++i) {
      if (i == phase_at) {
        if (phase == 0) { block_gather(blk + 1); phase_at += kP2 - kP1; phase = 1; }
        else if (phase == 1) { block_stage(blk + 1); phase_at += kBlk - kP2; phase = 2; top_up(); }
        else { ++blk; block_load(blk + 1); phase_at += kP1; phase = 0; }
      }
      while (e0 + i >= cur_end) advance();         // warp-uniform: the running destination is complete
      const uint32_t ent = idx_a + (((uint32_t)i & 63u) << 3);
      const uint32_t src = st_lds_u32(ent), wsel = st_lds_u32(ent + 4);
      const uint32_t woff16 = wsel >> 16;
      float2 h[4];
      float4 w[4];
      w[3] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (woff16) {                    // resident relation row
        const uint32_t grp = wsel & 0xffffu;
        if (!((hot_seen >> grp) & 1u)) { mbar_wait(hot_bar0 + grp * 8, 0); hot_seen |= 1u << grp; }
        const uint32_t wa = smem_l16 + (woff16 << 4);
        w[0] = st_lds_f4<0>(wa); w[1] = st_lds_f4<512>(wa); w[2] = st_lds_f4<1024>(wa);
        if (tail4) w[3] = st_lds_f4<1536>(wa);
      } else {                         // cold relation row: from L2 into registers
        const float* wr = w_l4 + (int64_t)(int)wsel * 400;
        w[0] = ldg_f4(wr); w[1] = ldg_f4(wr + 128); w[2] = ldg_f4(wr + 256);
        if (tail4) w[3] = ldg_f4(wr + 384);
      }
      uint32_t ha;
      if (src >> 31) {                 // resident source row
        const uint32_t grp = (src >> 16) & 0x7fffu;
        if (!((hot_seen >> (8 + grp)) & 1u)) { mbar_wait(hub_bar0 + grp * 8, 0); hot_seen |= 1u << (8 + grp); }
        ha = smem_l8 + ((src & 0xffffu) << 4);
      } else {
        st_wait(bar0 + rslot * 8, parity);
        ha = ring_l8 + rslot * kStSlot;
      }
      h[0] = st_lds_f2<0>(ha); h[1] = st_lds_f2<256>(ha); h[2] = st_lds_f2<512>(ha);
      h[3] = make_float2(0.f, 0.f);
      if (tail4) h[3] = st_lds_f2<768>(ha);
#pragma unroll
      for (int k = 0; k < 4; ++k) {    // out[j] += sum_i in[i] * W[i][j]
        acc[2 * k] = fmaf(h[k].x, w[k].x, fmaf(h[k].y, w[k].z, acc[2 * k]));
        acc[2 * k + 1] = fmaf(h[k].x, w[k].y, fmaf(h[k].y, w[k].w, acc[2 * k + 1]));
      }
      if (!(src >> 31)) {
        __syncwarp();                  // every lane has consumed the slot
        --fly;
        if (++rslot == D) { rslot = 0; parity ^= 1u; }
        top_up();
      }
    }
  }
  if (dbg) stamp(3, clock64());
  // ---- end of the range ------------------------------------------------------------------------------------------------------
  if (n > 0) {
    if (cur_end <= e1) {
      advance();                       // the running destination ends exactly here
    } else if (continued) {
      publish_head();                  // the whole range lies inside one destination started earlier and finished later
      ++cur;
    } else {
      // this warp started `cur`; later warps hold the rest of its edges: add their heads in warp (= edge) order
      for (int k = warp + 1; k < kStWarps && s_e0[k] < cur_end; ++k) {
        if (s_e0[k + 1] == s_e0[k]) continue;      // empty range: no head
        mbar_wait(head_bar0 + k * 8, 0);           // acquire (bounded spin: a lost head traps instead of hanging)
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          if (q < 3 || tail4) {
            const float2 hv = *reinterpret_cast<const float2*>(heads + k * 200 + 2 * (lane + 32 * q));
            acc[2 * q] += hv.x; acc[2 * q + 1] += hv.y;
          }
        }
      }
      epilogue(cur);
      ++cur;
    }
  }
  // ---- destinations without in-edges: out = act(self-loop row) (DGL's reduce never touches them).  They are taken out of
  //      the edge-ordered main pass -- where a run of them would be one warp's serial work -- and done here, off the
  //      prologue's critical path, by all warps of the grid: 32 row_ptr entries per warp and step -----------------------------
  for (int base = (blockIdx.x * kStWarps + warp) * 32; base < N; base += gridDim.x * kStWarps * 32) {
    const int v = base + lane;
    const bool iso = v < N && __ldg(row_ptr + v) == __ldg(row_ptr + v + 1);
    unsigned m = __ballot_sync(0xffffffffu, iso);
    while (m) {
      const int u = base + __ffs(m) - 1;
      m &= m - 1;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (k < 3 || tail4) {
          float* op = Hout + (int64_t)u * 200 + 2 * (lane + 32 * k);
          float2 o = make_float2(0.f, 0.f);
          if (HAS_LOOP) o = *reinterpret_cast<const float2*>(op);
          if (RELU) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); }
          if (RELU || !HAS_LOOP) *reinterpret_cast<float2*>(op) = o;
        }
      }
    }
  }
  if (dbg) { stamp(4, clock64()); stamp(6, global_timer()); stamp(7, n); }
}

}  // namespace renet
