// CTA-cooperative fused gather for the RE-Net shape (d_in = d_out = 200, 100 blocks of 2x2).
//
// One CTA owns kNodesPerCta consecutive destination rows of a CSR and the contiguous edge range that
// feeds them.  The edge range is split EVENLY over the CTA's warps (degree skew -- ICEWS18 in-degrees:
// median 3, p99 53, max 148 -- no longer idles warps); each warp walks its slice, keeps the running
// destination's sum in registers (a warp-level segmented reduction: edges are destination-sorted) and
// flushes it into a shared-memory tile when the destination changes.  The epilogue applies
// norm / self-loop / activation from the tile with fully coalesced 8-byte accesses.
//
// Lane mapping (fully coalesced): lane l < 25 owns blocks {l, l+25, l+50, l+75}.  Per edge it issues
// 4 x LDG.64 on the source row (each instruction covers 200 contiguous bytes across the warp,
// L1::no_allocate: streamed) and 4 x LDG.128 on the relation's block table row (400 contiguous bytes
// per instruction, L1-allocating: hot relations stay in L1).
//
// The same body serves forward (Hout = act(norm*agg + loop)) and backward-dH (reverse CSR, transposed
// 2x2 blocks, per-edge scale norm[dst], no activation).
#pragma once
#include "common.cuh"

namespace renet {

constexpr int kTileNodes = 16;   // default tile; the forward kernel is also instantiated with 32
constexpr int kTileWarps = 8;

__device__ __forceinline__ float2 ldg_f2_stream(const float* p) {
  float2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0,%1}, [%2];" : "=f"(r.x), "=f"(r.y) : "l"(p));
  return r;
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)),
               "l"(gmem_src)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// Prefetch what the epilogue needs (the tile's self-loop rows and norms) into shared memory with cp.async
// BEFORE the edge loop, so the epilogue has no exposed global latency.  nthreads threads, local id t.
__device__ __forceinline__ void tile_prefetch_epilogue(float (*loopbuf)[200], float* normbuf,
                                                       const float* __restrict__ loop_rows /* Hout + v0*200 */,
                                                       const float* __restrict__ norm_v0, int nv, bool has_loop,
                                                       int t, int nthreads) {
  if (has_loop)
    for (int i = t; i < nv * 50; i += nthreads) cp_async16(&loopbuf[0][0] + i * 4, loop_rows + i * 4);
  if (t < nv) normbuf[t] = __ldg(norm_v0 + t);
  cp_async_commit();
}

struct EdgeData {
  float2 h[4];
  float4 w[4];
};

template <bool STREAM_X = true>
__device__ __forceinline__ void load_edge(EdgeData& d, const float* __restrict__ X, const float* __restrict__ W,
                                          int s, int t, int lane) {
  const float* xp = X + (int64_t)s * 200 + 2 * lane;
  const float* wp = W + (int64_t)t * 400 + 4 * lane;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    d.h[k] = STREAM_X ? ldg_f2_stream(xp + 50 * k) : __ldg(reinterpret_cast<const float2*>(xp + 50 * k));
    d.w[k] = ldg_f4(wp + 100 * k);
  }
}

template <bool TRANSPOSE>
__device__ __forceinline__ void fma_edge(float (&acc)[8], const EdgeData& d, float sc) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float x = d.h[k].x * sc, y = d.h[k].y * sc;
    const float4 w = d.w[k];   // block (w.x w.y; w.z w.w) = W[b][i][j] row-major
    if (!TRANSPOSE) {          // out[j] += sum_i in[i] * W[i][j]
      acc[2 * k] = fmaf(x, w.x, fmaf(y, w.z, acc[2 * k]));
      acc[2 * k + 1] = fmaf(x, w.y, fmaf(y, w.w, acc[2 * k + 1]));
    } else {                   // din[i] += sum_j W[i][j] * g[j]
      acc[2 * k] = fmaf(x, w.x, fmaf(y, w.y, acc[2 * k]));
      acc[2 * k + 1] = fmaf(x, w.z, fmaf(y, w.w, acc[2 * k + 1]));
    }
  }
}

// Deterministic hand-over of partial sums between the warps of a tile (DET = true).  A destination's edges are
// contiguous, so a warp's slice consists of: possibly the TAIL of a destination an earlier warp started (its first
// segment, when e0 > row start), then destinations it starts itself.  A started destination is written to agg[nd] by
// plain stores -- exactly one warp starts any destination, so there is no atomic and no zero-initialisation -- and a
// continued one into the warp's private head[warp] slot, announced in head_mask[nd] (bit = warp).  The epilogue adds
// agg[nd] (if the row has edges) and the announced heads in ascending warp order = edge order: the sum is
// reproducible run to run.  Without DET the partial sums are added into a zeroed agg with shared-memory atomics
// (compiled to ATOMS.CAST.SPIN loops: ~20 % of the LSU wavefronts of the kernel, and run-to-run rounding noise).
struct TileHeads {
  float (*head)[200];   // [kTileWarps][200]
  int* head_mask;       // [nodes per tile], zeroed by the caller before the barrier that precedes tile_accumulate
};

// Sum for row r, columns c, c+1 after the barrier that follows tile_accumulate (DET mode).
__device__ __forceinline__ float2 tile_row_sum(const float (*agg)[200], const TileHeads& th, const int* s_rp, int r,
                                               int c) {
  float2 a = make_float2(0.f, 0.f);
  if (s_rp[r + 1] > s_rp[r]) {
    int m = th.head_mask[r];
    // the starter's partial is in agg unless the row's first edge belongs to a continuation, which cannot happen:
    // the warp holding a row's first edge is by definition its starter
    a = *reinterpret_cast<const float2*>(&agg[r][c]);
    while (m) {
      const int w = __ffs(m) - 1;
      m &= m - 1;
      const float2 hv = *reinterpret_cast<const float2*>(&th.head[w][c]);
      a.x += hv.x; a.y += hv.y;
    }
  }
  return a;
}

// Accumulate the tile's messages into `agg` (shared, [kTileNodes][200]; zeroed by the caller unless DET).
// s_rp: shared copy of row_ptr[v0 .. v0+nv].  EDGE_SCALE: multiply each message by scale[col_a[e]]
// (backward: norm of the edge's destination).
template <bool TRANSPOSE, bool INDEXED, bool EDGE_SCALE, bool STREAM_X = true, bool DET = false>
__device__ __forceinline__ void tile_accumulate(float (*agg)[200], const int* s_rp, int nv,
                                                const float* __restrict__ X, const int32_t* __restrict__ x_index,
                                                const float* __restrict__ W, const int32_t* __restrict__ col_a,
                                                const int32_t* __restrict__ col_type,
                                                const float* __restrict__ scale, TileHeads th = TileHeads{nullptr, nullptr}) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool active = lane < 25;
  const int ebeg = s_rp[0], eend = s_rp[nv];
  const int chunk = (eend - ebeg + kTileWarps - 1) / kTileWarps;
  const int e0 = ebeg + warp * chunk;
  const int e1 = min(eend, e0 + chunk);
  if (e0 >= e1) return;
  int node = 0;
  while (s_rp[node + 1] <= e0) ++node;
  int node_end = s_rp[node + 1];
  bool continued = DET && e0 > s_rp[node];    // the first segment finishes a destination an earlier warp started
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;

  auto flush = [&](int nd) {
    if (DET) {
      float* dst = continued ? th.head[warp] : agg[nd];
      if (continued && lane == 0) atomicOr(th.head_mask + nd, 1 << warp);
      continued = false;
      if (active) {
#pragma unroll
        for (int k = 0; k < 4; ++k)
          *reinterpret_cast<float2*>(dst + 2 * (lane + 25 * k)) = make_float2(acc[2 * k], acc[2 * k + 1]);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    } else if (active) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        atomicAdd(&agg[nd][2 * (lane + 25 * k)], acc[2 * k]);
        atomicAdd(&agg[nd][2 * (lane + 25 * k) + 1], acc[2 * k + 1]);
        acc[2 * k] = acc[2 * k + 1] = 0.f;
      }
    }
  };
  auto advance = [&](int e) {   // warp-uniform
    if (e >= node_end) {
      flush(node);
      do { ++node; node_end = s_rp[node + 1]; } while (e >= node_end);
    }
  };

  for (int base = e0; base < e1; base += 32) {
    const int e = base + lane;
    int my_s = 0, my_t = 0;
    float my_sc = 1.f;
    if (e < e1) {
      my_s = __ldg(col_a + e);
      my_t = __ldg(col_type + e);
      if (EDGE_SCALE) my_sc = __ldg(scale + my_s);
      if (INDEXED) my_s = __ldg(x_index + my_s);
    }
    const int cnt = min(32, e1 - base);
    for (int j = 0; j < cnt; j += 2) {
      const int sa = __shfl_sync(0xffffffffu, my_s, j), ta = __shfl_sync(0xffffffffu, my_t, j);
      const int jb = min(j + 1, cnt - 1);
      const int sb = __shfl_sync(0xffffffffu, my_s, jb), tb = __shfl_sync(0xffffffffu, my_t, jb);
      const float ca = EDGE_SCALE ? __shfl_sync(0xffffffffu, my_sc, j) : 1.f;
      const float cb = EDGE_SCALE ? __shfl_sync(0xffffffffu, my_sc, jb) : 1.f;
      // (letting lanes 25..31 shadow lanes 0..6 to drop the predication was measured slower)
      EdgeData da, db;
      if (active) {             // both edges' 16 loads are issued before any use
        load_edge<STREAM_X>(da, X, W, sa, ta, lane);
        load_edge<STREAM_X>(db, X, W, sb, tb, lane);
      }
      advance(base + j);
      if (active) fma_edge<TRANSPOSE>(acc, da, ca);
      if (j + 1 < cnt) {
        advance(base + j + 1);
        if (active) fma_edge<TRANSPOSE>(acc, db, cb);
      }
    }
  }
  flush(node);
}

}  // namespace renet
