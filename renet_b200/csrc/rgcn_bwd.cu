// Backward of the fused RGCN block layer (autograd of reference RGCN.py:33-51, 79-94; the reference
// gets it from torch.autograd through index_select / bmm / DGL's reduce, train.py:139).
//
//   P      = dHout * act'(Hout)                                        (relu mask)
//   dHin[u] = sum_{e: src(e)=u} blockdiag(W[type_e])^T . (norm[dst_e] P[dst_e])  +  P[u] @ Wloop^T
//   dW[r]  += sum_{e: type_e=r} Hin[src_e] (x) norm[dst_e] P[dst_e]    (outer product per 2x2 block)
//   dWloop += Hin^T @ P
//
// dHin is the forward gather run on the reversed graph (CSR by source, transposed 2x2 blocks): again
// atomics-free.  dW is a reduction keyed by relation with heavy skew (top-10 relations carry 60% of
// ICEWS18 edges): edges are grouped by relation, each warp reduces a run of edges in registers and
// flushes once per relation change with 128-bit vector REDs.
#include "common.cuh"
#include "rgcn_tile.cuh"
#include "rgcn_stream.cuh"

namespace renet {
namespace {

constexpr int kWarpsPerCta = 8;

__global__ void relu_mask_kernel(const float* __restrict__ dHout, const float* __restrict__ Hout,
                                 float* __restrict__ P, int64_t n4, int relu) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 g = ldg_f4(dHout + i * 4);
  if (relu) {
    const float4 o = ldg_f4(Hout + i * 4);
    g.x = o.x > 0.f ? g.x : 0.f; g.y = o.y > 0.f ? g.y : 0.f;
    g.z = o.z > 0.f ? g.z : 0.f; g.w = o.w > 0.f ? g.w : 0.f;
  }
  st_f4(P + i * 4, g);
}
__global__ void relu_mask_scalar_kernel(const float* __restrict__ dHout, const float* __restrict__ Hout,
                                        float* __restrict__ P, int64_t n, int relu) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  P[i] = (relu && !(Hout[i] > 0.f)) ? 0.f : dHout[i];
}

__global__ void transpose_kernel(const float* __restrict__ src, float* __restrict__ dst, int rows, int cols) {
  __shared__ float tile[32][33];
  const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    int r = r0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < rows && c < cols) ? src[(int64_t)r * cols + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    int c = c0 + i, r = r0 + threadIdx.x;
    if (r < rows && c < cols) dst[(int64_t)c * rows + r] = tile[threadIdx.x][i];
  }
}

// dH[u] = dH[u] (loop part, already there when HAS_LOOP) + sum over out-edges of W^T (norm[dst] P[dst]).
// Tile kernel (rgcn_tile.cuh): 16 source rows per CTA, the out-edge range split evenly
// over the warps; transposed 2x2 blocks, per-edge scale norm[dst].  DET: the warps hand partial rows over through
// TileHeads (rgcn_tile.cuh) instead of shared-memory atomics, as in the forward tile kernel.
template <bool HAS_LOOP, bool DET = false>
__global__ void __launch_bounds__(kTileWarps * 32)
rgcn_dh_tile_kernel(const float* __restrict__ P, const float* __restrict__ W, const int32_t* __restrict__ t_row_ptr,
                    const int32_t* __restrict__ t_col_dst, const int32_t* __restrict__ t_col_type,
                    const float* __restrict__ norm, float* __restrict__ dH, int N) {
  __shared__ __align__(16) float agg[kTileNodes][200];
  __shared__ __align__(16) float head[DET ? kTileWarps : 1][200];
  __shared__ int head_mask[kTileNodes];
  __shared__ int s_rp[kTileNodes + 1];
  const int tid = threadIdx.x;
  const int v0 = blockIdx.x * kTileNodes;
  const int nv = min(kTileNodes, N - v0);
  if (DET) {
    if (tid < kTileNodes) head_mask[tid] = 0;
  } else {
    for (int i = tid; i < kTileNodes * 200; i += kTileWarps * 32) (&agg[0][0])[i] = 0.f;
  }
  if (tid <= nv) s_rp[tid] = __ldg(t_row_ptr + v0 + tid);
  __syncthreads();
  const TileHeads th = DET ? TileHeads{head, head_mask} : TileHeads{nullptr, nullptr};
  tile_accumulate<true, false, true, true, DET>(agg, s_rp, nv, P, nullptr, W, t_col_dst, t_col_type, norm, th);
  __syncthreads();
  for (int i = tid; i < nv * 100; i += kTileWarps * 32) {
    const int r = i / 100, c = (i % 100) * 2;
    float2 o = DET ? tile_row_sum(agg, th, s_rp, r, c) : *reinterpret_cast<const float2*>(&agg[r][c]);
    float* op = dH + (int64_t)(v0 + r) * 200 + c;
    if (HAS_LOOP) {
      const float2 l = *reinterpret_cast<const float2*>(op);
      o.x += l.x; o.y += l.y;
    }
    *reinterpret_cast<float2*>(op) = o;
  }
}

__global__ void rgcn_dh_generic_kernel(const float* __restrict__ P, const float* __restrict__ W,
                                       const int32_t* __restrict__ t_row_ptr, const int32_t* __restrict__ t_col_dst,
                                       const int32_t* __restrict__ t_col_type, const float* __restrict__ norm,
                                       float* __restrict__ dH, int64_t N, int d_in, int d_out, int nb, int has_loop) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * d_in) return;
  const int64_t u = idx / d_in;
  const int c = (int)(idx % d_in);
  const int si = d_in / nb, so = d_out / nb;
  const int b = c / si, i = c % si;
  float acc = 0.f;
  for (int e = t_row_ptr[u]; e < t_row_ptr[u + 1]; ++e) {
    const int64_t d = t_col_dst[e];
    const float* w = W + (int64_t)t_col_type[e] * nb * si * so + (int64_t)b * si * so + (int64_t)i * so;
    const float* g = P + d * d_out + b * so;
    float s = 0.f;
    for (int j = 0; j < so; ++j) s = fmaf(w[j], g[j], s);
    acc = fmaf(s, norm[d], acc);
  }
  dH[idx] = (has_loop ? dH[idx] : 0.f) + acc;
}

// dW: warp per run of kEdgesPerWarp consecutive edges of the relation-grouped list.  DET: instead of adding its partial
// row for relation r into dW, run w stores it to dW = partials[w + r] (unique: along the relation-grouped list the
// (run, relation) pairs form a staircase on which w + r strictly increases; at most runs + R2 rows), and
// rgcn_dw_reduce_kernel adds them up in run order.
constexpr int kEdgesPerWarp = 64;
template <bool INDEXED, bool DET = false>
__global__ void __launch_bounds__(kWarpsPerCta * 32)
rgcn_dw_d200_kernel(const float* __restrict__ H, const int32_t* __restrict__ h_index, const float* __restrict__ P,
                    const int32_t* __restrict__ rel_ptr, const int32_t* __restrict__ rel_src,
                    const int32_t* __restrict__ rel_dst, const float* __restrict__ norm, float* __restrict__ dW,
                    int E, int R2) {
  const int lane = threadIdx.x & 31;
  const int warp = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
  const int e0 = warp * kEdgesPerWarp;
  if (e0 >= E) return;
  const int e1 = min(E, e0 + kEdgesPerWarp);
  const bool active = lane < 25;
  const int foff = lane * 8, woff = lane * 16;
  // relation of the first edge: largest r with rel_ptr[r] <= e0 (binary search, warp-uniform)
  int lo = 0, hi = R2;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(rel_ptr + mid) <= e0) lo = mid; else hi = mid;
  }
  int r = lo;
  int r_end = __ldg(rel_ptr + r + 1);
  float acc[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = 0.f;
  float* const wbase = dW + (DET ? (int64_t)warp * 400 : 0) + woff;
  auto flush = [&](int rr) {
    if (active) {
      float* wp = wbase + (int64_t)rr * 400;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float4 v = make_float4(acc[4 * k], acc[4 * k + 1], acc[4 * k + 2], acc[4 * k + 3]);
        if (DET) st_f4(wp + 4 * k, v);
        else red_add_f4(wp + 4 * k, v);
        acc[4 * k] = acc[4 * k + 1] = acc[4 * k + 2] = acc[4 * k + 3] = 0.f;
      }
    }
  };
  for (int base = e0; base < e1; base += 32) {
    const int e = base + lane;
    int my_s = 0, my_d = 0;
    float my_n = 0.f;
    if (e < e1) {
      my_s = __ldg(rel_src + e);
      my_d = __ldg(rel_dst + e);
      my_n = __ldg(norm + my_d);
      if (INDEXED) my_s = __ldg(h_index + my_s);
    }
    const int cnt = min(32, e1 - base);
#pragma unroll 2
    for (int j = 0; j < cnt; ++j) {
      while (base + j >= r_end) {  // relation boundary (possibly skipping empty relations)
        flush(r);
        ++r;
        r_end = __ldg(rel_ptr + r + 1);
      }
      const int s = __shfl_sync(0xffffffffu, my_s, j);
      const int d = __shfl_sync(0xffffffffu, my_d, j);
      const float sc = __shfl_sync(0xffffffffu, my_n, j);
      if (active) {
        const float* hp = H + (int64_t)s * 200 + foff;
        const float* gp = P + (int64_t)d * 200 + foff;
        const float4 h0 = ldg_f4_stream(hp), h1 = ldg_f4_stream(hp + 4);
        float4 g0 = ldg_f4_stream(gp), g1 = ldg_f4_stream(gp + 4);
        g0.x *= sc; g0.y *= sc; g0.z *= sc; g0.w *= sc;
        g1.x *= sc; g1.y *= sc; g1.z *= sc; g1.w *= sc;
        // dW[b][i][j] += h[b*2+i] * g[b*2+j]
        acc[0] = fmaf(h0.x, g0.x, acc[0]);  acc[1] = fmaf(h0.x, g0.y, acc[1]);
        acc[2] = fmaf(h0.y, g0.x, acc[2]);  acc[3] = fmaf(h0.y, g0.y, acc[3]);
        acc[4] = fmaf(h0.z, g0.z, acc[4]);  acc[5] = fmaf(h0.z, g0.w, acc[5]);
        acc[6] = fmaf(h0.w, g0.z, acc[6]);  acc[7] = fmaf(h0.w, g0.w, acc[7]);
        acc[8] = fmaf(h1.x, g1.x, acc[8]);  acc[9] = fmaf(h1.x, g1.y, acc[9]);
        acc[10] = fmaf(h1.y, g1.x, acc[10]); acc[11] = fmaf(h1.y, g1.y, acc[11]);
        acc[12] = fmaf(h1.z, g1.z, acc[12]); acc[13] = fmaf(h1.z, g1.w, acc[13]);
        acc[14] = fmaf(h1.w, g1.z, acc[14]); acc[15] = fmaf(h1.w, g1.w, acc[15]);
      }
    }
  }
  flush(r);
}

// DET dW: dW[r] += the partial rows of the runs holding relation r's edges, in run order (thread = 4 of the 400 columns)
__global__ void __launch_bounds__(100)
rgcn_dw_reduce_kernel(const float* __restrict__ parts, const int32_t* __restrict__ rel_ptr, float* __restrict__ dW) {
  const int r = blockIdx.x, c = threadIdx.x * 4;
  const int e0 = __ldg(rel_ptr + r), e1 = __ldg(rel_ptr + r + 1);
  if (e0 >= e1) return;
  float* op = dW + (int64_t)r * 400 + c;
  float4 s = *reinterpret_cast<const float4*>(op);
  const int w1 = (e1 - 1) / kEdgesPerWarp;
#pragma unroll 8
  for (int w = e0 / kEdgesPerWarp; w <= w1; ++w) {
    const float4 p = ldg_f4(parts + (int64_t)(w + r) * 400 + c);
    s.x += p.x; s.y += p.y; s.z += p.z; s.w += p.w;
  }
  st_f4(op, s);
}

__global__ void rgcn_dw_generic_kernel(const float* __restrict__ H, const int32_t* __restrict__ h_index,
                                       const float* __restrict__ P, const int32_t* __restrict__ rel_ptr,
                                       const int32_t* __restrict__ rel_src, const int32_t* __restrict__ rel_dst,
                                       const float* __restrict__ norm, float* __restrict__ dW, int R2, int d_in,
                                       int d_out, int nb) {
  const int si = d_in / nb, so = d_out / nb;
  const int per_r = nb * si * so;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)R2 * per_r) return;
  const int r = (int)(idx / per_r), w = (int)(idx % per_r);
  const int b = w / (si * so), i = (w / so) % si, j = w % so;
  float acc = 0.f;
  for (int e = rel_ptr[r]; e < rel_ptr[r + 1]; ++e) {
    int64_t s = rel_src[e];
    if (h_index) s = h_index[s];
    const int64_t d = rel_dst[e];
    acc = fmaf(H[s * d_in + b * si + i], norm[d] * P[d * d_out + b * so + j], acc);
  }
  dW[idx] += acc;
}

__global__ void scatter_add_rows_kernel(const float* __restrict__ src, const int32_t* __restrict__ index,
                                        float* __restrict__ dst, int64_t n_rows, int d4) {
  const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n_rows) return;
  const int64_t t = __ldg(index + w);
  for (int i = lane; i < d4; i += 32) red_add_f4(dst + t * d4 * 4 + i * 4, ldg_f4(src + w * d4 * 4 + i * 4));
}
__global__ void scatter_add_rows_scalar_kernel(const float* __restrict__ src, const int32_t* __restrict__ index,
                                               float* __restrict__ dst, int64_t n_rows, int d) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rows * d) return;
  atomicAdd(dst + (int64_t)index[i / d] * d + (i % d), src[i]);
}

}  // namespace

int launch_scatter_add_rows(const float* src, const int32_t* index, float* dst, int64_t n_rows, int d,
                            cudaStream_t stream) {
  if (deterministic()) return scatter_add_rows_det(src, d, index, nullptr, dst, n_rows, d, stream);
  const bool vec = d % 4 == 0 && ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0;
  if (vec) {
    const int64_t threads = n_rows * 32;
    scatter_add_rows_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(src, index, dst, n_rows, d / 4);
    RENET_CHECK_LAUNCH("scatter_add_rows_kernel");
  } else {
    const int64_t total = n_rows * d;
    scatter_add_rows_scalar_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(src, index, dst, n_rows, d);
    RENET_CHECK_LAUNCH("scatter_add_rows_scalar_kernel");
  }
  return RENET_OK;
}

// dH = dLoop @ Wloop^T (written), dWloop += Hin^T @ dLoop.  WloopT_ws: d_in*d_out floats.
int launch_selfloop_bwd(const float* H, const int32_t* h_index, const float* Wloop, const float* dLoop, float* dH,
                        float* dWloop, float* WloopT_ws, int64_t N, int d_in, int d_out, cudaStream_t stream) {
  dim3 tg((d_in + 31) / 32, (d_out + 31) / 32);
  transpose_kernel<<<tg, dim3(32, 8), 0, stream>>>(Wloop, WloopT_ws, d_in, d_out);
  RENET_CHECK_LAUNCH("transpose_kernel");
  int rc;
  if ((rc = sgemm_nn(dLoop, nullptr, d_out, WloopT_ws, d_in, dH, d_in, nullptr, N, d_in, d_out, false, stream, false)))
    return rc;
  return sgemm_tn(H, h_index, d_in, dLoop, d_out, dWloop, d_out, d_in, d_out, N, true, stream);
}

// G_ws: [N*d_out] floats for P, followed by [d_in*d_out] floats for Wloop^T.
int launch_rgcn_bwd(const float* H, const int32_t* h_index, const float* W, const float* Wloop,
                    const int32_t* t_row_ptr, const int32_t* t_col_dst, const int32_t* t_col_type,
                    const int32_t* rel_ptr, const int32_t* rel_src, const int32_t* rel_dst, const float* norm,
                    const float* Hout, const float* dHout, float* dH, float* dW, float* dWloop, float* G_ws,
                    int64_t N, int64_t E, int d_in, int d_out, int nb, int R2, int relu, cudaStream_t stream,
                    int64_t N_dst) {
  // N = rows of H / dH (sources); N_dst = rows of Hout / dHout / norm (destinations): equal except for the read-out
  // sub-graph (readout_subgraph.cu), whose destinations are a compacted subset
  if (N_dst < 0) N_dst = N;
  float* P = G_ws;
  float* WloopT = G_ws + ((N_dst * d_out + 3) & ~int64_t(3));
  const int64_t n = N_dst * d_out;
  const bool al = ((reinterpret_cast<uintptr_t>(dHout) | reinterpret_cast<uintptr_t>(Hout) |
                    reinterpret_cast<uintptr_t>(P)) & 15) == 0;
  if (n % 4 == 0 && al) {
    relu_mask_kernel<<<(unsigned)((n / 4 + 255) / 256), 256, 0, stream>>>(dHout, Hout, P, n / 4, relu);
    RENET_CHECK_LAUNCH("relu_mask_kernel");
  } else {
    relu_mask_scalar_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(dHout, Hout, P, n, relu);
    RENET_CHECK_LAUNCH("relu_mask_scalar_kernel");
  }
  int rc;
  if (Wloop != nullptr) {
    if ((rc = launch_selfloop_bwd(H, h_index, Wloop, P, dH, dWloop, WloopT, N, d_in, d_out, stream))) return rc;
  }
  const bool fast = d_in == 200 && d_out == 200 && nb == 100 &&
                    ((reinterpret_cast<uintptr_t>(H) | reinterpret_cast<uintptr_t>(W) | reinterpret_cast<uintptr_t>(dH) |
                      reinterpret_cast<uintptr_t>(dW) | reinterpret_cast<uintptr_t>(P)) & 15) == 0;
  if (fast) {
    if (E > 0 && gather_use_stream(E, N, true)) {       // kStreamMinNodes, as before the forward read-out threshold
      // batch scale: the persistent bulk-copy kernel on the reversed graph -- no atomics, bitwise reproducible dH
      static bool attr_done = false;
      if (!attr_done) {
        RENET_CHECK_CUDA(cudaFuncSetAttribute(rgcn_gather_stream_kernel<false, true, false, true>,
                                              cudaFuncAttributeMaxDynamicSharedMemorySize, StDefault<true>::kSmemBytes));
        RENET_CHECK_CUDA(cudaFuncSetAttribute(rgcn_gather_stream_kernel<false, false, false, true>,
                                              cudaFuncAttributeMaxDynamicSharedMemorySize, StDefault<true>::kSmemBytes));
        attr_done = true;
      }
      if (Wloop != nullptr)
        rgcn_gather_stream_kernel<false, true, false, true><<<kNumSMs, StDefault<true>::kThreads, StDefault<true>::kSmemBytes, stream>>>(
            P, nullptr, W, t_row_ptr, t_col_dst, t_col_type, norm, dH, (int)N, R2, nullptr, 0, (int)E, nullptr);
      else
        rgcn_gather_stream_kernel<false, false, false, true><<<kNumSMs, StDefault<true>::kThreads, StDefault<true>::kSmemBytes, stream>>>(
            P, nullptr, W, t_row_ptr, t_col_dst, t_col_type, norm, dH, (int)N, R2, nullptr, 0, (int)E, nullptr);
      RENET_CHECK_LAUNCH("rgcn_gather_stream_kernel(bwd)");
    } else if (deterministic()) {
      const unsigned grid = (unsigned)((N + kTileNodes - 1) / kTileNodes);
      if (Wloop != nullptr)
        rgcn_dh_tile_kernel<true, true><<<grid, kTileWarps * 32, 0, stream>>>(P, W, t_row_ptr, t_col_dst, t_col_type, norm, dH, (int)N);
      else
        rgcn_dh_tile_kernel<false, true><<<grid, kTileWarps * 32, 0, stream>>>(P, W, t_row_ptr, t_col_dst, t_col_type, norm, dH, (int)N);
      RENET_CHECK_LAUNCH("rgcn_dh_tile_kernel");
    } else {
      const unsigned grid = (unsigned)((N + kTileNodes - 1) / kTileNodes);
      if (Wloop != nullptr)
        rgcn_dh_tile_kernel<true><<<grid, kTileWarps * 32, 0, stream>>>(P, W, t_row_ptr, t_col_dst, t_col_type, norm, dH, (int)N);
      else
        rgcn_dh_tile_kernel<false><<<grid, kTileWarps * 32, 0, stream>>>(P, W, t_row_ptr, t_col_dst, t_col_type, norm, dH, (int)N);
      RENET_CHECK_LAUNCH("rgcn_dh_tile_kernel");
    }
    const int64_t warps = (E + kEdgesPerWarp - 1) / kEdgesPerWarp;
    const unsigned g2 = (unsigned)((warps + kWarpsPerCta - 1) / kWarpsPerCta);
    if (deterministic()) {
      void* parts = nullptr;
      if ((rc = det_scratch((warps + R2) * 400 * (int64_t)sizeof(float), stream, &parts))) return rc;
      float* Wp = static_cast<float*>(parts);
      if (h_index)
        rgcn_dw_d200_kernel<true, true><<<g2, kWarpsPerCta * 32, 0, stream>>>(H, h_index, P, rel_ptr, rel_src, rel_dst, norm, Wp, (int)E, R2);
      else
        rgcn_dw_d200_kernel<false, true><<<g2, kWarpsPerCta * 32, 0, stream>>>(H, h_index, P, rel_ptr, rel_src, rel_dst, norm, Wp, (int)E, R2);
      RENET_CHECK_LAUNCH("rgcn_dw_d200_kernel");
      rgcn_dw_reduce_kernel<<<R2, 100, 0, stream>>>(Wp, rel_ptr, dW);
      RENET_CHECK_LAUNCH("rgcn_dw_reduce_kernel");
      return RENET_OK;
    }
    if (h_index)
      rgcn_dw_d200_kernel<true><<<g2, kWarpsPerCta * 32, 0, stream>>>(H, h_index, P, rel_ptr, rel_src, rel_dst, norm, dW, (int)E, R2);
    else
      rgcn_dw_d200_kernel<false><<<g2, kWarpsPerCta * 32, 0, stream>>>(H, h_index, P, rel_ptr, rel_src, rel_dst, norm, dW, (int)E, R2);
    RENET_CHECK_LAUNCH("rgcn_dw_d200_kernel");
  } else {
    const int64_t t1 = N * d_in;
    rgcn_dh_generic_kernel<<<(unsigned)((t1 + 255) / 256), 256, 0, stream>>>(P, W, t_row_ptr, t_col_dst, t_col_type,
                                                                            norm, dH, N, d_in, d_out, nb, Wloop != nullptr);
    RENET_CHECK_LAUNCH("rgcn_dh_generic_kernel");
    const int64_t t2 = (int64_t)R2 * nb * (d_in / nb) * (d_out / nb);
    rgcn_dw_generic_kernel<<<(unsigned)((t2 + 255) / 256), 256, 0, stream>>>(H, h_index, P, rel_ptr, rel_src, rel_dst,
                                                                            norm, dW, R2, d_in, d_out, nb);
    RENET_CHECK_LAUNCH("rgcn_dw_generic_kernel");
  }
  return RENET_OK;
}

}  // namespace renet
