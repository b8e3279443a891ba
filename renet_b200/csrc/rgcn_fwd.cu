// Fused RGCN block-diagonal message passing, forward (reference RGCN.py:79-94 + 42-48):
//
//   Hout[v] = act( norm[v] * sum_{e: dst(e)=v} blockdiag(W[type_e]) . Hin[src_e]  +  loop[v] )
//
// replaces the reference's index_select (E x 400 weight materialisation, RGCN.py:81-85), the
// E*100 tiny bmm (RGCN.py:86-87), DGL's atomic copy-reduce (fn.sum, RGCN.py:91), the norm multiply
// (RGCN.py:93-94), the self-loop add and the activation (RGCN.py:45-48) with ONE pass over a
// destination-sorted CSR: no per-edge message ever reaches memory and no atomics are needed.
//
// Fast path (d_in = d_out = 200, num_bases = 100, 2x2 blocks -- the only shape RE-Net uses,
// model.py:36): see rgcn_tile.cuh.  One CTA = 16 destination rows, edges split evenly over 8 warps,
// warp-level segmented reduction into a shared tile, fused norm / self-loop / activation epilogue.
#include <stdlib.h>

#include "common.cuh"
#include "rgcn_tile.cuh"
#include "rgcn_stream.cuh"

namespace renet {
namespace {

// Tile kernel (round 1; rgcn_tile.cuh): one CTA per 16 destinations.  The path for small graphs (inference on a handful of
// sub-graphs: a persistent one-CTA-per-SM launch would cost more than the work) and for DGL's edge-less pass-through; at
// batch scale, and on layer 2's read-out sub-graph of a batch, the persistent kernel of rgcn_stream.cuh takes over
// (gather_use_stream).
template <bool RELU, bool HAS_LOOP, bool INDEXED, int NODES = kTileNodes>
__global__ void __launch_bounds__(kTileWarps * 32, 768 / (kTileWarps * 32))
rgcn_gather_d200_kernel(const float* __restrict__ H, const int32_t* __restrict__ h_index,
                        const float* __restrict__ W, const int32_t* __restrict__ row_ptr,
                        const int32_t* __restrict__ col_src, const int32_t* __restrict__ col_type,
                        const float* __restrict__ norm, float* __restrict__ Hout, int N, int passthrough) {
  __shared__ __align__(16) float agg[NODES][200];
  __shared__ __align__(16) float loopbuf[HAS_LOOP ? NODES : 1][200];
  __shared__ __align__(16) float head[kTileWarps][200];
  __shared__ int head_mask[NODES];
  __shared__ float normbuf[NODES];
  __shared__ int s_rp[NODES + 1];
  const int tid = threadIdx.x;
  const int v0 = blockIdx.x * NODES;
  const int nv = min(NODES, N - v0);
  tile_prefetch_epilogue(loopbuf, normbuf, Hout + (int64_t)v0 * 200, norm + v0, nv, HAS_LOOP, tid, kTileWarps * 32);
  if (tid < NODES) head_mask[tid] = 0;
  if (tid <= nv) s_rp[tid] = __ldg(row_ptr + v0 + tid);
  __syncthreads();
  const TileHeads th{head, head_mask};
  tile_accumulate<false, INDEXED, false, true, true>(agg, s_rp, nv, H, h_index, W, col_src, col_type, nullptr, th);
  cp_async_wait_all();
  __syncthreads();
  // epilogue: nv rows x 100 float2, coalesced; self-loop rows and norms were prefetched into shared memory
  for (int i = tid; i < nv * 100; i += kTileWarps * 32) {
    const int r = i / 100, c = (i % 100) * 2;
    const int v = v0 + r;
    float2 a = tile_row_sum(agg, th, s_rp, r, c);
    if (passthrough) {  // graph without edges: DGL 0.4 skips the reduce, h is left as is
      const int64_t hr = INDEXED ? (int64_t)__ldg(h_index + v) : v;
      a = *reinterpret_cast<const float2*>(H + hr * 200 + c);
    }
    const float nvv = normbuf[r];
    float* op = Hout + (int64_t)v * 200 + c;
    float2 o = make_float2(a.x * nvv, a.y * nvv);
    if (HAS_LOOP) {
      const float2 l = *reinterpret_cast<const float2*>(&loopbuf[r][c]);
      o.x += l.x; o.y += l.y;
    }
    if (RELU) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); }
    *reinterpret_cast<float2*>(op) = o;
  }
}

// Generic shapes (any d_in, d_out, num_bases): one thread per (node, output feature).  Only the
// small known-answer cases use it; RE-Net itself always runs the d200 path.
__global__ void rgcn_gather_generic_kernel(const float* __restrict__ H, const int32_t* __restrict__ h_index,
                                           const float* __restrict__ W, const int32_t* __restrict__ row_ptr,
                                           const int32_t* __restrict__ col_src,
                                           const int32_t* __restrict__ col_type, const float* __restrict__ norm,
                                           float* __restrict__ Hout, int64_t N, int d_in, int d_out, int nb,
                                           int relu, int has_loop, int passthrough) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * d_out) return;
  const int64_t v = i / d_out;
  const int c = (int)(i % d_out);
  const int si = d_in / nb, so = d_out / nb;
  const int b = c / so, j = c % so;
  float acc = 0.f;
  for (int e = row_ptr[v]; e < row_ptr[v + 1]; ++e) {
    int64_t s = col_src[e];
    if (h_index) s = h_index[s];
    const float* w = W + (int64_t)col_type[e] * nb * si * so + (int64_t)b * si * so + j;
    const float* h = H + s * d_in + b * si;
    for (int k = 0; k < si; ++k) acc = fmaf(h[k], w[k * so], acc);
  }
  if (passthrough) {
    const int64_t r = h_index ? (int64_t)h_index[v] : v;
    acc = H[r * d_in + c];
  }
  float o = acc * norm[v];
  if (has_loop) o += Hout[i];
  if (relu) o = fmaxf(o, 0.f);
  Hout[i] = o;
}

}  // namespace

// Which kernel serves the d=200 shape: 0 = automatic (the stream kernel at batch scale, the tile kernel for small graphs),
// 1 = tile, 3 = stream.  RENET_GATHER_KERNEL=tile|stream picks one per process for A/B measurements
// (tools/bench_gather.py); results agree to fp32 summation order.
int gather_kernel_choice() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("RENET_GATHER_KERNEL");
    v = 0;
    if (e && e[0] == 't') v = 1;
    else if (e && e[0] == 's') v = 3;
  }
  return v;
}
bool gather_use_stream(int64_t E, int64_t N, bool indexed_input) {
  // E may be an upper bound (device-assembled batches and read-out sub-graphs pass their capacity), so the destination
  // count decides with it: the persistent kernel pays a prologue of about 7 us per launch.  Graphs whose input rows come
  // through an index (layer 1: the embedding table through node_ent) amortise it from kStreamMinNodes on (the tile kernel
  // is faster on 12 k- and 21 k-node layer-1 graphs, DESIGN §5: that threshold was not moved here).  Plain input rows
  // (layer 2's read-out sub-graph: about 12 edges per destination, rows of H1) amortise it from kStreamMinPlainNodes on
  // (measured on read-out sub-graphs of 2 k to 10 k destinations, DESIGN §5).  And the kernel is built for feature
  // matrices that live in L2 (ICEWS18: 27 MB of the H100's 50 MB): with two rows in flight per warp it cannot cover HBM
  // latency, so when the destinations' own feature rows exceed L2 (kStreamMaxNodes; the synthetic 1 M-entity shard, 800 MB)
  // the tile kernel stays
  const int c = gather_kernel_choice();
  const int64_t min_nodes = indexed_input ? kStreamMinNodes : kStreamMinPlainNodes;
  return c == 3 || (c == 0 && E >= kStreamMinEdges && N >= min_nodes && N <= kStreamMaxNodes);
}

// debug hook (tools/stream_timeline.py): per-warp time stamps of the next stream-kernel launches; never set in production
static long long* g_stream_dbg = nullptr;
void set_stream_debug_buffer(long long* p) { g_stream_dbg = p; }

int stream_cfg_choice() {             // read per launch: a test compares hubs on and off in one process
  const char* e = getenv("RENET_STREAM_CFG");
  return e ? atoi(e) : 0;
}

template <bool RELU, bool HAS_LOOP, bool INDEXED, class Cfg>
static int launch_stream_cfg(const float* H, const int32_t* h_index, const float* W, const int32_t* row_ptr,
                             const int32_t* col_src, const int32_t* col_type, const float* norm, float* Hout, int N, int R2,
                             const int32_t* hot_rel, int n_hot, int E_hint, cudaStream_t stream) {
  static bool attr_done = false;        // one device per process (one process per GPU)
  if (!attr_done) {
    RENET_CHECK_CUDA(cudaFuncSetAttribute(rgcn_gather_stream_kernel<RELU, HAS_LOOP, INDEXED, false, Cfg>,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    attr_done = true;
  }
  // Programmatic dependent launch (launch.cuh, DESIGN §4): the prologue before the kernel's griddepcontrol.wait (partition
  // search, row_ptr slice, relation ranking, resident relation rows, first index blocks) runs under the previous kernel's
  // tail when that kernel writes none of these pre-wait inputs.  norm is read after the wait; it is listed all the same,
  // so a norm the previous kernel writes keeps the plain order.
  const int64_t e4 = (int64_t)E_hint * 4, n4 = ((int64_t)N + 1) * 4;
  return launch_pdl("rgcn_gather_stream_kernel",
                    {{row_ptr, n4}, {col_src, e4}, {col_type, e4}, {h_index, INDEXED ? (int64_t)N * 4 : 0},
                     {norm, (int64_t)N * 4}, {W, (int64_t)R2 * 1600}, {hot_rel, hot_rel ? (int64_t)n_hot * 4 : 0}},
                    {{Hout, (int64_t)N * 800}}, rgcn_gather_stream_kernel<RELU, HAS_LOOP, INDEXED, false, Cfg>,
                    dim3(kNumSMs), dim3(Cfg::kThreads), Cfg::kSmemBytes, stream, H, h_index, W, row_ptr, col_src, col_type,
                    norm, Hout, N, R2, hot_rel, n_hot, E_hint, g_stream_dbg);
}

template <bool RELU, bool HAS_LOOP, bool INDEXED>
static int launch_stream(const float* H, const int32_t* h_index, const float* W, const int32_t* row_ptr,
                         const int32_t* col_src, const int32_t* col_type, const float* norm, float* Hout, int N, int R2,
                         const int32_t* hot_rel, int n_hot, int E_hint, cudaStream_t stream) {
#define RENET_ST(...) return launch_stream_cfg<RELU, HAS_LOOP, INDEXED, __VA_ARGS__>(H, h_index, W, row_ptr, col_src, col_type, norm, Hout, N, R2, hot_rel, n_hot, E_hint, stream)
  if (RELU && HAS_LOOP) {               // experiment configurations exist for the layer-1 shape only (RENET_STREAM_CFG)
    switch (stream_cfg_choice()) {
      case 1: RENET_ST(StCfg<28, 2, 31, false>);
      case 2: RENET_ST(StCfg<24, 2, 44, false>);
      default: break;
    }
  }
  // layer 1 (input rows through an index: a CTA's sources are a few hundred consecutive node ids, half of its edges
  // come from 64 of them) keeps hub source rows resident; RENET_STREAM_CFG=3 turns them off (A/B measurements, tests:
  // the results are bitwise the same).  Plain input rows (layer 2's read-out sub-graph) keep 82 relation rows and no hubs:
  // tools/stream_reuse_model.py counts 27 % fewer L2 bytes per edge there with 49 / 64, which has not been measured
  if constexpr (INDEXED)
    if (stream_cfg_choice() != 3) RENET_ST(StHubs);
  RENET_ST(StDefault<false>);
#undef RENET_ST
}

int launch_rgcn_gather(const float* H, const int32_t* h_index, const float* W, const int32_t* row_ptr,
                       const int32_t* col_src, const int32_t* col_type, const float* norm, float* Hout,
                       int64_t N, int64_t E, int d_in, int d_out, int nb, int relu, int has_loop,
                       cudaStream_t stream, int R2, const int32_t* hot_rel, int n_hot) {
  if (N == 0) return RENET_OK;
  const int passthrough = (E == 0) ? 1 : 0;
  const bool fast = d_in == 200 && d_out == 200 && nb == 100 &&
                    ((reinterpret_cast<uintptr_t>(H) | reinterpret_cast<uintptr_t>(W) |
                      reinterpret_cast<uintptr_t>(Hout)) & 15) == 0;
  if (fast) {
    const int key = (relu ? 4 : 0) | (has_loop ? 2 : 0) | (h_index ? 1 : 0);
    if (!passthrough && gather_use_stream(E, N, h_index != nullptr)) {
#define RENET_LAUNCH_STREAM(R, L, I) return launch_stream<R, L, I>(H, h_index, W, row_ptr, col_src, col_type, norm, Hout, (int)N, R2, hot_rel, n_hot, (int)E, stream)
      switch (key) {
        case 0: RENET_LAUNCH_STREAM(false, false, false);
        case 1: RENET_LAUNCH_STREAM(false, false, true);
        case 2: RENET_LAUNCH_STREAM(false, true, false);
        case 3: RENET_LAUNCH_STREAM(false, true, true);
        case 4: RENET_LAUNCH_STREAM(true, false, false);
        case 5: RENET_LAUNCH_STREAM(true, false, true);
        case 6: RENET_LAUNCH_STREAM(true, true, false);
        default: RENET_LAUNCH_STREAM(true, true, true);
      }
#undef RENET_LAUNCH_STREAM
    }
    const unsigned block = kTileWarps * 32;
    const unsigned n_tiles = (unsigned)((N + kTileNodes - 1) / kTileNodes);
#define RENET_LAUNCH_GATHER(R, L, I)                                                                            \
    rgcn_gather_d200_kernel<R, L, I><<<n_tiles, block, 0, stream>>>(H, h_index, W, row_ptr, col_src, col_type, norm, Hout, (int)N, passthrough)
    switch (key) {
      case 0: RENET_LAUNCH_GATHER(false, false, false); break;
      case 1: RENET_LAUNCH_GATHER(false, false, true); break;
      case 2: RENET_LAUNCH_GATHER(false, true, false); break;
      case 3: RENET_LAUNCH_GATHER(false, true, true); break;
      case 4: RENET_LAUNCH_GATHER(true, false, false); break;
      case 5: RENET_LAUNCH_GATHER(true, false, true); break;
      case 6: RENET_LAUNCH_GATHER(true, true, false); break;
      default: RENET_LAUNCH_GATHER(true, true, true); break;
    }
#undef RENET_LAUNCH_GATHER
    RENET_CHECK_LAUNCH("rgcn_gather_d200_kernel");
  } else {
    const int64_t total = N * d_out;
    rgcn_gather_generic_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(
        H, h_index, W, row_ptr, col_src, col_type, norm, Hout, N, d_in, d_out, nb, relu, has_loop, passthrough);
    RENET_CHECK_LAUNCH("rgcn_gather_generic_kernel");
  }
  return RENET_OK;
}

}  // namespace renet
