// Host-side history-graph batching in C++ (no CUDA): the contract of reference utils.py:149-181,209-244
// (get_neighs_by_t, get_g_list_id, make_subgraph, get_node_ids_to_g_id, dgl.batch) on flat arrays.
//
// The reference spends 0.4-2.3 s per batch here in Python (sets, 239 DGL subgraph calls, S tiny .cpu()
// copies); the numpy version in renet_b200/utils.py needs 50-100 ms.  This version works on two flat
// stores built once per dataset --
//   graph store  : every timestamp's graph, nodes ascending by entity id, edges sorted by destination
//   history store: every sample's history entries (timestamp, neighbour local rows, subject local row)
// -- and emits the batched graph directly in CSR form plus the read-out / sequence bookkeeping into ONE
// caller-provided staging buffer (pinned by the caller), so a step is one H2D copy.
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <unordered_map>
#include <vector>

#include "../../include/renet_b200.h"

#include <atomic>
#include <thread>

namespace renet {
void set_error(const char* fmt, ...);
}

namespace {
std::atomic<int> g_host_threads{8};
// components are independent: a handful of short-lived threads pull component indices from a counter
template <class F>
void parallel_for(int64_t n, F f) {
  unsigned hw = std::thread::hardware_concurrency();
  const int cap = std::max(1, g_host_threads.load());
  const int nt = (int)std::min<int64_t>(std::min<unsigned>(hw ? hw : 1, (unsigned)cap), (n + 15) / 16);
  if (nt <= 1) { for (int64_t i = 0; i < n; ++i) f(i); return; }
  std::atomic<int64_t> next{0};
  auto work = [&]() { for (int64_t i = next.fetch_add(4); i < n; i = next.fetch_add(4)) for (int64_t j = i; j < std::min(n, i + 4); ++j) f(j); };
  std::vector<std::thread> th;
  for (int t = 1; t < nt; ++t) th.emplace_back(work);
  work();
  for (auto& t : th) t.join();
}
}  // namespace

extern "C" int renet_set_host_threads(int n) {
  const int prev = g_host_threads.load();
  g_host_threads.store(n < 1 ? 1 : n);
  return prev;
}

namespace {
// Steps 1-3 of the batching, shared by the all-host batcher and the host half of the device batcher.
struct Plan {
  std::vector<int32_t> len, comp_graph, row_comp, row_srow, row_seq, newid, node_ent;
  std::vector<int64_t> mark_off, comp_start;
  int max_len = 0;
  int64_t Q = 0, S = 0, G = 0, N = 0;
  int32_t* nid = nullptr;       // where the node marks / ids live: newid, or the caller's output buffer
};

// returns RENET_OK / error; S == 0 leaves the plan empty
int build_plan(Plan& P, const char* fn, int64_t T, const int64_t* g_node_off, const int32_t* g_node_ent, const int64_t* h_samp_off,
               const int64_t* h_samp_entry, const int32_t* h_ent_graph, const int32_t* h_ent_srow, const int64_t* h_ent_off,
               const int32_t* h_nbr_row, const int64_t* sample_idx, int64_t B, int32_t sort, int64_t* s_idx_out,
               int32_t max_len_capacity, int32_t* newid_out = nullptr, int64_t newid_capacity = 0,
               const int64_t* sample_group = nullptr) {
  // ---- 1. order samples by history length, descending, stable (model.py:80-81, utils.py:212-215) ----
  P.len.resize(B);
  int max_len = 0;
  for (int64_t i = 0; i < B; ++i) {
    P.len[i] = (int32_t)(h_samp_off[sample_idx[i] + 1] - h_samp_off[sample_idx[i]]);
    max_len = std::max(max_len, (int)P.len[i]);
  }
  if (max_len > max_len_capacity) { renet::set_error("%s: history longer than %d", fn, max_len_capacity); return RENET_ERR_INVALID_ARG; }
  P.max_len = max_len;
  int64_t Q = 0, S = 0;
  if (sort) {
    std::vector<int64_t> start(max_len + 2, 0);
    for (int64_t i = 0; i < B; ++i) start[max_len - P.len[i] + 1]++;       // bucket by (max_len - len)
    for (int k = 0; k <= max_len; ++k) start[k + 1] += start[k];
    for (int64_t i = 0; i < B; ++i) s_idx_out[start[max_len - P.len[i]]++] = i;
  } else {
    for (int64_t i = 0; i < B; ++i) s_idx_out[i] = i;
  }
  for (int64_t i = 0; i < B; ++i) if (P.len[i] > 0) { ++Q; S += P.len[i]; }
  if (!sort) {   // unsorted twin (utils.py:251-255) takes the FIRST Q samples: they must be the non-empty ones
    for (int64_t i = 0; i < Q; ++i)
      if (P.len[i] == 0) { renet::set_error("%s: unsorted batches must list their non-empty histories first", fn); return RENET_ERR_INVALID_ARG; }
  }
  P.Q = Q; P.S = S;
  if (S == 0) return RENET_OK;
  // ---- 2. components = distinct timestamps in first-appearance order (utils.py:149-170); with isolation groups, the
  // distinct (group, timestamp) pairs in first-appearance order ------------------------------------------------------
  std::vector<int32_t> comp_of_graph(T, -1);
  P.row_comp.resize(S); P.row_srow.resize(S); P.row_seq.resize(S);
  std::vector<int64_t> row_entry(S);
  std::vector<int64_t> row_group(sample_group ? S : 0);
  int64_t r = 0;
  for (int64_t q = 0; q < Q; ++q) {           // pass A: the samples' entry lists (contiguous per sample)
    const int64_t smp = sample_idx[s_idx_out[q]];
    if (q + 4 < Q) __builtin_prefetch(h_samp_entry + h_samp_off[sample_idx[s_idx_out[q + 4]]]);
    for (int64_t ei = h_samp_off[smp]; ei < h_samp_off[smp + 1]; ++ei, ++r) {
      row_entry[r] = h_samp_entry[ei];
      P.row_seq[r] = (int32_t)q;
      if (sample_group) row_group[r] = sample_group[s_idx_out[q]];
    }
  }
  std::unordered_map<int64_t, std::unordered_map<int32_t, int32_t>> comp_of_pair;   // group -> graph -> component
  constexpr int64_t kAheadB = 16;
  for (int64_t i = 0; i < S; ++i) {           // pass B: per-entry fields (random reads: prefetched ahead)
    if (i + kAheadB < S) {
      __builtin_prefetch(h_ent_graph + row_entry[i + kAheadB]);
      __builtin_prefetch(h_ent_srow + row_entry[i + kAheadB]);
    }
    const int64_t e = row_entry[i];
    const int32_t g = h_ent_graph[e];
    if (sample_group) {
      auto ins = comp_of_pair[row_group[i]].emplace(g, (int32_t)P.comp_graph.size());
      if (ins.second) P.comp_graph.push_back(g);
      P.row_comp[i] = ins.first->second;
    } else {
      if (comp_of_graph[g] < 0) { comp_of_graph[g] = (int32_t)P.comp_graph.size(); P.comp_graph.push_back(g); }
      P.row_comp[i] = comp_of_graph[g];
    }
    P.row_srow[i] = h_ent_srow[e];
  }
  const int64_t G = P.G = (int64_t)P.comp_graph.size();
  // ---- 3. node sets: mark local rows of every component's graph, then number them ----------------------------
  P.mark_off.assign(G + 1, 0);
  for (int64_t c = 0; c < G; ++c) P.mark_off[c + 1] = P.mark_off[c] + (g_node_off[P.comp_graph[c] + 1] - g_node_off[P.comp_graph[c]]);
  // marks go into a bitmap (M bits: 25 KB for ICEWS18, L1-resident) -- the marking loop is a chain of dependent random
  // reads into the history store, so the entries a few rows ahead are prefetched -- and numbering walks the set bits
  // only: in global bit order = (component, local row) order, which is the batched node order.
  const int64_t M = P.mark_off[G];
  std::vector<uint64_t> bits((M + 63) / 64 + 1, 0);
  constexpr int64_t kAhead = 12;
  for (int64_t i = 0; i < S; ++i) {
    if (i + kAhead < S) {
      const int64_t ea = row_entry[i + kAhead];
      __builtin_prefetch(h_ent_off + ea);
      if (i + kAhead / 2 < S) __builtin_prefetch(h_nbr_row + h_ent_off[row_entry[i + kAhead / 2]]);
    }
    const int64_t base = P.mark_off[P.row_comp[i]];
    int64_t b = base + P.row_srow[i];
    bits[b >> 6] |= uint64_t(1) << (b & 63);
    const int64_t e = row_entry[i];
    for (int64_t k = h_ent_off[e]; k < h_ent_off[e + 1]; ++k) {
      b = base + h_nbr_row[k];
      bits[b >> 6] |= uint64_t(1) << (b & 63);
    }
  }
  if (newid_out != nullptr && M <= newid_capacity) {      // build the ids in place in the caller's buffer
    P.nid = newid_out;
    memset(P.nid, 0xff, (size_t)M * 4);
  } else {
    P.newid.assign(M, -1);       // -1 = not selected; else the batched node id
    P.nid = P.newid.data();
  }
  P.comp_start.assign(G + 1, 0);
  P.node_ent.clear();
  P.node_ent.reserve(S * 4);
  int64_t N = 0, c = 0;
  const int32_t* ent = G > 0 ? g_node_ent + g_node_off[P.comp_graph[0]] : nullptr;
  for (int64_t w = 0; w < (int64_t)bits.size(); ++w) {
    uint64_t x = bits[w];
    while (x) {
      const int64_t gidx = (w << 6) + __builtin_ctzll(x);
      x &= x - 1;
      while (gidx >= P.mark_off[c + 1]) {        // entered the next component (also skips components without marks)
        ++c;
        P.comp_start[c] = N;
        ent = g_node_ent + g_node_off[P.comp_graph[c]];
      }
      P.nid[gidx] = (int32_t)N++;
      P.node_ent.push_back(ent[gidx - P.mark_off[c]]);
    }
  }
  while (c < G) P.comp_start[++c] = N;
  P.comp_start[G] = N;
  P.N = N;
  return RENET_OK;
}

// read-out rows + sequence bookkeeping (utils.py:172-181, Aggregator.py:160-165)
void emit_sequences(const Plan& P, const int64_t* s_idx_out, int32_t* o_readout, int32_t* o_rowcomp, int32_t* o_rowseq,
                    int32_t* o_seqstart, int32_t* o_seqlen, int32_t* o_packed, int32_t* batch_sizes_out) {
  for (int64_t i = 0; i < P.S; ++i) {
    o_readout[i] = P.nid[P.mark_off[P.row_comp[i]] + P.row_srow[i]];
    o_rowcomp[i] = P.row_comp[i];
    o_rowseq[i] = P.row_seq[i];
  }
  int64_t acc = 0;
  for (int64_t q = 0; q < P.Q; ++q) {
    o_seqstart[q] = (int32_t)acc;
    o_seqlen[q] = P.len[s_idx_out[q]];
    acc += o_seqlen[q];
  }
  int64_t p = 0;
  for (int t = 0; t < P.max_len; ++t) {
    int32_t n_act = 0;
    for (int64_t q = 0; q < P.Q; ++q) if (o_seqlen[q] > t) { o_packed[p++] = o_seqstart[q] + t; ++n_act; }
    batch_sizes_out[t] = n_act;
  }
}
}  // namespace

extern "C" int renet_host_assemble_batch(
    // ---- graph store ------------------------------------------------------------------------------
    int64_t T, const int64_t* g_node_off, const int32_t* g_node_ent, const int64_t* g_edge_off,
    const int32_t* g_src, const int32_t* g_dst, const int32_t* g_type_s, const int32_t* g_type_o,
    // ---- history store ----------------------------------------------------------------------------
    const int64_t* h_samp_off, const int64_t* h_samp_entry, const int32_t* h_ent_graph, const int32_t* h_ent_srow, const int64_t* h_ent_off,
    const int32_t* h_nbr_row,
    // ---- batch --------------------------------------------------------------------------------------
    const int64_t* sample_idx, int64_t B, int32_t sort,
    // ---- outputs --------------------------------------------------------------------------------------
    int64_t* s_idx_out, int32_t* out, int64_t out_capacity, int32_t* batch_sizes_out, int32_t max_len_capacity,
    int64_t* sizes /* [10]: N, E, S, Q, G, max_len, words_used, 0, 0, 0 */) {
  if (B < 0 || !sizes) { renet::set_error("renet_host_assemble_batch: bad arguments"); return RENET_ERR_INVALID_ARG; }
  Plan P;
  int prc = build_plan(P, "renet_host_assemble_batch", T, g_node_off, g_node_ent, h_samp_off, h_samp_entry, h_ent_graph, h_ent_srow,
                       h_ent_off, h_nbr_row, sample_idx, B, sort, s_idx_out, max_len_capacity);
  if (prc != RENET_OK) return prc;
  const int64_t Q = P.Q, S = P.S, G = P.G, N = P.N;
  for (int i = 0; i < 10; ++i) sizes[i] = 0;
  sizes[2] = S; sizes[3] = Q; sizes[5] = P.max_len;
  if (S == 0) return RENET_OK;
  const std::vector<int32_t>& comp_graph = P.comp_graph;
  const int32_t* newid = P.nid;
  const std::vector<int64_t>& mark_off = P.mark_off;
  const std::vector<int64_t>& comp_start = P.comp_start;
  // ---- 4. count induced edges per component (utils.make_subgraph, utils.py:115-131), in parallel -------------
  std::vector<int64_t> comp_estart(G + 1, 0);
  parallel_for(G, [&](int64_t c) {
    const int32_t g = comp_graph[c];
    const int32_t* m = newid + mark_off[c];
    int64_t cnt = 0;
    for (int64_t k = g_edge_off[g]; k < g_edge_off[g + 1]; ++k) cnt += (m[g_src[k]] >= 0) & (m[g_dst[k]] >= 0);
    comp_estart[c + 1] = cnt;
  });
  for (int64_t c = 0; c < G; ++c) comp_estart[c + 1] += comp_estart[c];
  const int64_t E = comp_estart[G];
  // layout of `out` (int32 words):
  //  node_ent[N] row_ptr[N+1] col_src[E] col_type_s[E] col_type_o[E] norm[N](f32 bits)
  //  readout[S] row_comp[S] row_seq[S] seq_start[Q] seq_len[Q] packed_row[S]
  //  s_idx[B] comp_graph[G]      (s_idx: device copy of s_idx_out, so no separate H2D is needed)
  const int64_t words = N + (N + 1) + 3 * E + N + 3 * S + 2 * Q + S + B + G;
  sizes[0] = N; sizes[1] = E; sizes[4] = G; sizes[6] = words;
  if (words > out_capacity) return 1;   // caller grows the staging buffer and retries
  int32_t* o_node = out;
  int32_t* o_rp = o_node + N;
  int32_t* o_src = o_rp + N + 1;
  int32_t* o_ts = o_src + E;
  int32_t* o_to = o_ts + E;
  float* o_norm = reinterpret_cast<float*>(o_to + E);
  int32_t* o_readout = o_to + E + N;
  int32_t* o_rowcomp = o_readout + S;
  int32_t* o_rowseq = o_rowcomp + S;
  int32_t* o_seqstart = o_rowseq + S;
  int32_t* o_seqlen = o_seqstart + Q;
  int32_t* o_packed = o_seqlen + Q;
  // ---- 5. emit nodes + edges (per-timestamp edge lists are destination-sorted => CSR for free) ----------------
  o_rp[0] = 0;
  memcpy(o_node, P.node_ent.data(), (size_t)N * 4);
  parallel_for(G, [&](int64_t c) {
    const int32_t g = comp_graph[c];
    const int32_t* m = newid + mark_off[c];
    int64_t ecur = comp_estart[c];
    int64_t node = comp_start[c];            // next node whose row_ptr end is not yet written
    for (int64_t k = g_edge_off[g]; k < g_edge_off[g + 1]; ++k) {
      const int32_t s = m[g_src[k]], d = m[g_dst[k]];
      if ((s | d) < 0) continue;
      while (node < d) o_rp[++node] = (int32_t)ecur;
      o_src[ecur] = s; o_ts[ecur] = g_type_s[k]; o_to[ecur] = g_type_o[k];
      ++ecur;
    }
    while (node < comp_start[c + 1]) o_rp[++node] = (int32_t)ecur;
  });
  for (int64_t v = 0; v < N; ++v) {
    const int32_t d = o_rp[v + 1] - o_rp[v];
    o_norm[v] = 1.0f / (float)(d > 0 ? d : 1);       // recomputed per sub-graph (utils.py:126-127)
  }
  // ---- 6. read-out rows + sequence bookkeeping ------------------------------------------------------------------
  emit_sequences(P, s_idx_out, o_readout, o_rowcomp, o_rowseq, o_seqstart, o_seqlen, o_packed, batch_sizes_out);
  int32_t* o_sidx = o_packed + S;
  for (int64_t i = 0; i < B; ++i) o_sidx[i] = (int32_t)s_idx_out[i];
  int32_t* o_cg = o_sidx + B;
  for (int64_t c = 0; c < G; ++c) o_cg[c] = comp_graph[c];
  return RENET_OK;
}

// Host half of the DEVICE batcher: steps 1-3 + 6 only (everything whose cost is O(S + nodes)); the O(edges) part --
// filtering every candidate edge of the touched timestamps against the node marks and emitting the CSR -- is
// renet_induce_edges (device_batch.cu) on the GPU against a graph store resident in HBM.
//
// layout of `out` (int32 words):
//   newid[M] node_ent[N] readout[S] row_comp[S] row_seq[S] seq_start[Q] seq_len[Q] packed_row[S] s_idx[B] comp_graph[G]
//   mark_off[G+1] cand_off[G+1]
// newid: per component c, one word per local row of its timestamp's graph (offset mark_off[c]): batched node id or -1;
// cand_off: prefix sum of the components' (un-induced) edge counts, i.e. the candidate edges the device filters.
// sample_group (optional, one entry per selected sample): isolation groups -- the components are the distinct (group,
// timestamp) pairs, so the node sets of different groups never mix.  comp_graph, mark_off, cand_off and renet_induce_edges
// already work per component and let any component point at any graph, so the device half is the same.
extern "C" int renet_host_plan_batch_grouped(
    int64_t T, const int64_t* g_node_off, const int32_t* g_node_ent, const int64_t* g_edge_off,
    const int64_t* h_samp_off, const int64_t* h_samp_entry, const int32_t* h_ent_graph, const int32_t* h_ent_srow,
    const int64_t* h_ent_off, const int32_t* h_nbr_row, const int64_t* sample_idx, const int64_t* sample_group, int64_t B,
    int32_t sort, int64_t* s_idx_out, int32_t* out, int64_t out_capacity, int32_t* batch_sizes_out, int32_t max_len_capacity,
    int64_t* sizes /* [10]: N, E_cand, S, Q, G, max_len, words_used, M, 0, 0 */) {
  if (B < 0 || !sizes) { renet::set_error("renet_host_plan_batch: bad arguments"); return RENET_ERR_INVALID_ARG; }
  Plan P;
  int prc = build_plan(P, "renet_host_plan_batch", T, g_node_off, g_node_ent, h_samp_off, h_samp_entry, h_ent_graph, h_ent_srow, h_ent_off,
                       h_nbr_row, sample_idx, B, sort, s_idx_out, max_len_capacity, out, out_capacity, sample_group);
  if (prc != RENET_OK) return prc;
  const int64_t Q = P.Q, S = P.S, G = P.G, N = P.N;
  for (int i = 0; i < 10; ++i) sizes[i] = 0;
  sizes[2] = S; sizes[3] = Q; sizes[5] = P.max_len;
  if (S == 0) return RENET_OK;
  const int64_t M = P.mark_off[G];
  int64_t e_cand = 0;
  for (int64_t c = 0; c < G; ++c) e_cand += g_edge_off[P.comp_graph[c] + 1] - g_edge_off[P.comp_graph[c]];
  if (M >= (int64_t(1) << 31) || e_cand >= (int64_t(1) << 31)) { renet::set_error("renet_host_plan_batch: batch too large for 32-bit offsets"); return RENET_ERR_INVALID_ARG; }
  const int64_t words = M + N + 3 * S + 2 * Q + S + B + G + 2 * (G + 1);
  sizes[0] = N; sizes[1] = e_cand; sizes[4] = G; sizes[6] = words; sizes[7] = M;
  if (words > out_capacity) return 1;   // caller grows the staging buffer and retries
  int32_t* o_newid = out;
  int32_t* o_node = o_newid + M;
  int32_t* o_readout = o_node + N;
  int32_t* o_rowcomp = o_readout + S;
  int32_t* o_rowseq = o_rowcomp + S;
  int32_t* o_seqstart = o_rowseq + S;
  int32_t* o_seqlen = o_seqstart + Q;
  int32_t* o_packed = o_seqlen + Q;
  int32_t* o_sidx = o_packed + S;
  int32_t* o_cg = o_sidx + B;
  int32_t* o_moff = o_cg + G;
  int32_t* o_coff = o_moff + G + 1;
  if (P.nid != o_newid) memcpy(o_newid, P.nid, (size_t)M * 4);
  memcpy(o_node, P.node_ent.data(), (size_t)N * 4);
  emit_sequences(P, s_idx_out, o_readout, o_rowcomp, o_rowseq, o_seqstart, o_seqlen, o_packed, batch_sizes_out);
  for (int64_t i = 0; i < B; ++i) o_sidx[i] = (int32_t)s_idx_out[i];
  int64_t acc = 0;
  for (int64_t c = 0; c < G; ++c) {
    o_cg[c] = P.comp_graph[c];
    o_moff[c] = (int32_t)P.mark_off[c];
    o_coff[c] = (int32_t)acc;
    acc += g_edge_off[P.comp_graph[c] + 1] - g_edge_off[P.comp_graph[c]];
  }
  o_moff[G] = (int32_t)M;
  o_coff[G] = (int32_t)acc;
  return RENET_OK;
}

extern "C" int renet_host_plan_batch(
    int64_t T, const int64_t* g_node_off, const int32_t* g_node_ent, const int64_t* g_edge_off,
    const int64_t* h_samp_off, const int64_t* h_samp_entry, const int32_t* h_ent_graph, const int32_t* h_ent_srow,
    const int64_t* h_ent_off, const int32_t* h_nbr_row, const int64_t* sample_idx, int64_t B, int32_t sort,
    int64_t* s_idx_out, int32_t* out, int64_t out_capacity, int32_t* batch_sizes_out, int32_t max_len_capacity,
    int64_t* sizes) {
  return renet_host_plan_batch_grouped(T, g_node_off, g_node_ent, g_edge_off, h_samp_off, h_samp_entry, h_ent_graph, h_ent_srow,
                                       h_ent_off, h_nbr_row, sample_idx, nullptr, B, sort, s_idx_out, out, out_capacity,
                                       batch_sizes_out, max_len_capacity, sizes);
}

// ---- native loader: a pool of C++ worker threads that run batch jobs ahead of the consumer ------------------------------
// The Python prefetcher used a ThreadPoolExecutor; its workers fought the consumer thread for the GIL around every
// ctypes call.  Here the workers are plain C++ threads: submit() enqueues a job (the arguments of
// renet_host_plan_batch / renet_host_assemble_batch; every pointer must stay valid until wait() returns for the
// ticket), wait() blocks -- without the GIL, being a ctypes call -- until that job has run and returns its code.
#include <condition_variable>
#include <deque>
#include <functional>
#include <mutex>
#include <unordered_map>

namespace {
struct Loader {
  std::mutex mu;
  std::condition_variable cv_job, cv_done;
  std::deque<std::pair<int64_t, std::function<int()>>> queue;
  std::unordered_map<int64_t, int> done;
  std::vector<std::thread> threads;
  int64_t next_ticket = 0;
  bool stop = false;

  explicit Loader(int n) {
    for (int i = 0; i < n; ++i) threads.emplace_back([this] { run(); });
  }
  ~Loader() {
    { std::lock_guard<std::mutex> lk(mu); stop = true; }
    cv_job.notify_all();
    for (auto& t : threads) t.join();
  }
  void run() {
    for (;;) {
      std::pair<int64_t, std::function<int()>> job;
      {
        std::unique_lock<std::mutex> lk(mu);
        cv_job.wait(lk, [this] { return stop || !queue.empty(); });
        if (queue.empty()) return;      // stop requested and nothing left
        job = std::move(queue.front());
        queue.pop_front();
      }
      const int rc = job.second();
      { std::lock_guard<std::mutex> lk(mu); done[job.first] = rc; }
      cv_done.notify_all();
    }
  }
  int64_t submit(std::function<int()> f) {
    int64_t t;
    { std::lock_guard<std::mutex> lk(mu); t = next_ticket++; queue.emplace_back(t, std::move(f)); }
    cv_job.notify_one();
    return t;
  }
  int wait(int64_t ticket) {
    std::unique_lock<std::mutex> lk(mu);
    cv_done.wait(lk, [&] { return done.count(ticket) != 0; });
    const int rc = done[ticket];
    done.erase(ticket);
    return rc;
  }
};
}  // namespace

extern "C" void* renet_loader_create(int32_t n_threads) {
  if (n_threads < 1) n_threads = 1;
  if (n_threads > 64) n_threads = 64;
  return new Loader(n_threads);
}

extern "C" void renet_loader_destroy(void* loader) { delete static_cast<Loader*>(loader); }

extern "C" int64_t renet_loader_submit_plan(
    void* loader, int64_t T, const int64_t* g_node_off, const int32_t* g_node_ent, const int64_t* g_edge_off,
    const int64_t* h_samp_off, const int64_t* h_samp_entry, const int32_t* h_ent_graph, const int32_t* h_ent_srow,
    const int64_t* h_ent_off, const int32_t* h_nbr_row, const int64_t* sample_idx, int64_t B, int32_t sort,
    int64_t* s_idx_out, int32_t* out, int64_t out_capacity, int32_t* batch_sizes_out, int32_t max_len_capacity,
    int64_t* sizes) {
  if (!loader) return -1;
  return static_cast<Loader*>(loader)->submit([=]() {
    return renet_host_plan_batch(T, g_node_off, g_node_ent, g_edge_off, h_samp_off, h_samp_entry, h_ent_graph, h_ent_srow,
                                 h_ent_off, h_nbr_row, sample_idx, B, sort, s_idx_out, out, out_capacity, batch_sizes_out,
                                 max_len_capacity, sizes);
  });
}

extern "C" int64_t renet_loader_submit_assemble(
    void* loader, int64_t T, const int64_t* g_node_off, const int32_t* g_node_ent, const int64_t* g_edge_off,
    const int32_t* g_src, const int32_t* g_dst, const int32_t* g_type_s, const int32_t* g_type_o,
    const int64_t* h_samp_off, const int64_t* h_samp_entry, const int32_t* h_ent_graph, const int32_t* h_ent_srow,
    const int64_t* h_ent_off, const int32_t* h_nbr_row, const int64_t* sample_idx, int64_t B, int32_t sort,
    int64_t* s_idx_out, int32_t* out, int64_t out_capacity, int32_t* batch_sizes_out, int32_t max_len_capacity,
    int64_t* sizes) {
  if (!loader) return -1;
  return static_cast<Loader*>(loader)->submit([=]() {
    return renet_host_assemble_batch(T, g_node_off, g_node_ent, g_edge_off, g_src, g_dst, g_type_s, g_type_o, h_samp_off,
                                     h_samp_entry, h_ent_graph, h_ent_srow, h_ent_off, h_nbr_row, sample_idx, B, sort,
                                     s_idx_out, out, out_capacity, batch_sizes_out, max_len_capacity, sizes);
  });
}

extern "C" int renet_loader_wait(void* loader, int64_t ticket) {
  if (!loader || ticket < 0) { renet::set_error("renet_loader_wait: bad loader / ticket"); return RENET_ERR_INVALID_ARG; }
  return static_cast<Loader*>(loader)->wait(ticket);
}
