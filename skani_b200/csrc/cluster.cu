// cluster.cu -- sk_cluster: ANI clustering of a triangle's results (greedy representatives or single linkage) on the GPU.
//
// Edge build: the results are uploaded in chunks through the context's pinned staging; a filter kernel validates every row and
// appends the edges (ani > 0.1 and ani >= min_ani) as (min id << 32 | max id, ani, row).  Both directions of every edge are
// radix-sorted on their 64-bit (a << 32 | b) keys: the sorted keys are the adjacency of a symmetric CSR (neighbour = low
// word), the values index the edge, and equal neighbouring keys are duplicate pairs.
// Greedy: rounds of cl_greedy_decide over a compacted, rank-ordered frontier of undecided vertices, reading live states
// (cluster_core.cuh says why that is safe); the frontier is compacted and its size read back every GREEDY_ROUNDS rounds.
// Then cl_assign gives every member its representative.  A path in rank order decides about one vertex per round: n rounds.
// Single linkage: hook (cl_hook, atomicMin in rank space) and pointer jumping until a hook pass changes nothing; every
// component then has one root, its smallest rank.
// sk_cluster_linkage (average / complete linkage): the same edge build with every printed row an edge, then rounds over a
// sorted list of directed cluster pairs (linkage_core.cuh): a warp per cluster finds its best partner, mutual best pairs
// merge (an exclusive scan places their records), and the relabelled list is radix-sorted and combined by key.  Flat
// clusters reuse single linkage's jump / component / numbering kernels; the dendrogram is the merge records sorted on the
// device and numbered the scipy way on the host.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <chrono>
#include <cmath>
#include <string>
#include <vector>

#include "cluster_core.cuh"
#include "linkage_core.cuh"
#include "sk_internal.h"

using namespace sk;

namespace {

constexpr uint64_t CHUNK_ROWS = 1ull << 20;   // results per upload chunk (72 MiB)
constexpr int GREEDY_ROUNDS = 8;              // greedy rounds between two read-backs of the frontier size
constexpr int TPB = 256;

inline unsigned blocks_for(uint64_t n) { return (unsigned)std::max<uint64_t>(1, (n + TPB - 1) / TPB); }

// rows [0, m) of a chunk that starts at result row0: range and self-pair checks (first offending row per kind), then the
// edges appended at *n_edges (one atomic per warp)
__global__ void cl_filter_kernel(const sk_ani_result* __restrict__ res, uint64_t m, uint64_t row0, uint32_t n, float min_ani,
                                 unsigned long long* __restrict__ n_edges, uint64_t* __restrict__ ekey, float* __restrict__ eani,
                                 uint64_t* __restrict__ erow, unsigned long long* __restrict__ bad /* [2]: id range, self pair */) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool edge = false;
  uint32_t a = 0, b = 0;
  float ani = 0.f;
  if (i < m) {
    const sk_ani_result& r = res[i];
    a = r.ref_id; b = r.query_id; ani = r.ani;
    if (a >= n || b >= n) atomicMin(&bad[0], (unsigned long long)(row0 + i));
    else if (a == b) atomicMin(&bad[1], (unsigned long long)(row0 + i));
    else edge = cl_is_edge(ani, min_ani);
  }
  const unsigned mask = __ballot_sync(0xffffffffu, edge);
  if (!mask) return;
  const int lane = threadIdx.x & 31, leader = __ffs(mask) - 1;
  unsigned long long base = 0;
  if (lane == leader) base = atomicAdd(n_edges, (unsigned long long)__popc(mask));
  base = __shfl_sync(0xffffffffu, base, leader);
  if (!edge) return;
  const uint64_t at = base + __popc(mask & ((1u << lane) - 1));
  ekey[at] = (uint64_t)min(a, b) << 32 | max(a, b);
  eani[at] = ani;
  erow[at] = row0 + i;
}

// edge e -> its two directed adjacency keys, both carrying e
__global__ void cl_directed_kernel(const uint64_t* __restrict__ ekey, uint64_t E, uint64_t* __restrict__ key, uint32_t* __restrict__ val) {
  const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const uint64_t k = ekey[e];
  key[2 * e] = k; val[2 * e] = (uint32_t)e;
  key[2 * e + 1] = (k << 32) | (k >> 32); val[2 * e + 1] = (uint32_t)e;
}

// first adjacency index whose key repeats the one before it
__global__ void cl_dup_kernel(const uint64_t* __restrict__ key, uint64_t n, unsigned long long* __restrict__ dup) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x + 1;
  if (i < n && key[i] == key[i - 1]) atomicMin(dup, (unsigned long long)i);
}

// CSR offsets: off[v] = first adjacency index of vertex v, v <= n
__global__ void cl_offsets_kernel(const uint64_t* __restrict__ key, uint64_t n_adj, uint32_t n, uint64_t* __restrict__ off) {
  const uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v > n) return;
  const uint64_t want = v << 32;
  uint64_t lo = 0, hi = n_adj;
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if (key[mid] < want) lo = mid + 1; else hi = mid;
  }
  off[v] = lo;
}

// order[rank[v]] = v
__global__ void cl_order_kernel(const uint32_t* __restrict__ rank, uint32_t n, uint32_t* __restrict__ order) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < n) order[rank[v]] = v;
}

// one greedy round over the frontier
__global__ void cl_greedy_kernel(const uint32_t* __restrict__ frontier, uint32_t m, const uint64_t* __restrict__ off,
                                 const uint64_t* __restrict__ adj, const uint32_t* __restrict__ rank, uint8_t* state) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const uint32_t v = frontier[i];
  volatile uint8_t* vs = state;
  if (vs[v] != CL_UNDECIDED) return;
  const uint8_t s = cl_greedy_decide(v, off, adj, rank, vs);
  if (s != CL_UNDECIDED) vs[v] = s;
}

struct Undecided {
  const uint8_t* state;
  __device__ bool operator()(uint32_t v) const { return state[v] == CL_UNDECIDED; }
};

// greedy: representative and result row of every vertex; flag[rank[v]] = v is a representative
__global__ void cl_assign_kernel(uint32_t n, const uint64_t* __restrict__ off, const uint64_t* __restrict__ adj,
                                 const uint32_t* __restrict__ adj_e, const float* __restrict__ eani, const uint64_t* __restrict__ erow,
                                 const uint32_t* __restrict__ rank, const uint8_t* __restrict__ state, uint32_t* __restrict__ rep,
                                 uint64_t* __restrict__ edge, uint32_t* __restrict__ flag) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  uint32_t r = v;
  uint64_t e = UINT64_MAX, at = 0;
  if (state[v] == CL_MEMBER && cl_assign(v, off, adj, adj_e, eani, rank, state, &r, &at)) e = erow[adj_e[at]];
  rep[v] = r; edge[v] = e;
  flag[rank[v]] = state[v] == CL_REP;
}

__global__ void cl_iota_kernel(uint32_t* __restrict__ p, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = i;
}

// one hook pass over the edges in rank space; *changed = 1 when a parent was lowered
__global__ void cl_hook_kernel(const uint64_t* __restrict__ ekey, uint64_t E, const uint32_t* __restrict__ rank, uint32_t* parent,
                               uint32_t* __restrict__ changed) {
  const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  volatile uint32_t* vp = parent;
  const uint64_t k = ekey[e];
  uint32_t slot, val;
  if (cl_hook(vp[rank[(uint32_t)(k >> 32)]], vp[rank[(uint32_t)k]], &slot, &val) && atomicMin(&parent[slot], val) > val) *changed = 1;
}

__global__ void cl_jump_kernel(uint32_t* parent, uint32_t n) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  volatile uint32_t* vp = parent;
  vp[r] = cl_find(vp, r);
}

// single linkage: representative = the component's root, result row of the edge to it when there is one
__global__ void cl_component_kernel(uint32_t n, const uint64_t* __restrict__ off, const uint64_t* __restrict__ adj,
                                    const uint32_t* __restrict__ adj_e, const uint64_t* __restrict__ erow, const uint32_t* __restrict__ rank,
                                    const uint32_t* __restrict__ order, const uint32_t* __restrict__ parent, uint32_t* __restrict__ rep,
                                    uint64_t* __restrict__ edge, uint32_t* __restrict__ flag) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  const uint32_t rv = rank[v], r = order[parent[rv]];
  uint64_t e = UINT64_MAX;
  if (r != v) {
    const uint64_t want = (uint64_t)v << 32 | r;
    uint64_t lo = off[v], hi = off[v + 1];
    while (lo < hi) {
      const uint64_t mid = (lo + hi) >> 1;
      if (adj[mid] < want) lo = mid + 1; else hi = mid;
    }
    if (lo < off[v + 1] && adj[lo] == want) e = erow[adj_e[lo]];
  }
  rep[v] = r; edge[v] = e;
  flag[rv] = parent[rv] == rv;
}

// cluster[v] = number of representatives ranked before rep[v] (incl = inclusive scan of the flags in rank order)
__global__ void cl_number_kernel(uint32_t n, const uint32_t* __restrict__ rep, const uint32_t* __restrict__ rank,
                                 const uint32_t* __restrict__ incl, uint32_t* __restrict__ cluster) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < n) cluster[v] = incl[rank[rep[v]]] - 1;
}

// ---- average / complete linkage (linkage_core.cuh).  The pair list holds directed cluster pairs, keys A << 32 | B in rank
// space, sorted, one entry per pair; sentinel keys (hi word = n) mark entries to drop and sort to the end.

// edge e -> its two directed pairs in rank space with value {q, 1, q}; the first row with ani >= 2 in *bad
__global__ void lk_init_kernel(const uint64_t* __restrict__ ekey, const float* __restrict__ eani, const uint64_t* __restrict__ erow,
                               uint64_t E, const uint32_t* __restrict__ rank, uint64_t* __restrict__ key, LkVal* __restrict__ val,
                               unsigned long long* __restrict__ bad) {
  const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const uint64_t k = ekey[e];
  const uint64_t a = rank[(uint32_t)(k >> 32)], b = rank[(uint32_t)k];
  const float ani = eani[e];
  if (!(ani < LK_MAX_ANI)) atomicMin(bad, (unsigned long long)erow[e]);
  const uint32_t q = ani < LK_MAX_ANI ? lk_q(ani) : 0;
  key[2 * e] = a << 32 | b; key[2 * e + 1] = b << 32 | a;
  val[2 * e] = val[2 * e + 1] = LkVal{q, 1, q};
}

struct LkCombine {
  __device__ LkVal operator()(const LkVal& a, const LkVal& b) const { return lk_combine(a, b); }
};

// index i starts a cluster's segment (or the sentinel run) among the *nruns live entries
struct LkHead {
  const uint64_t* key;
  const int* nruns;
  __device__ bool operator()(uint32_t i) const { return (int)i < *nruns && (i == 0 || (key[i] >> 32) != (key[i - 1] >> 32)); }
};

// a warp per segment: the cluster's best partner (best[A] = LK_NONE when it does not qualify) and the index of that pair;
// pairs that can never qualify again become sentinels.  seg_id[w] = A, LK_NONE for the sentinel run.
__global__ void lk_best_kernel(uint64_t* key, const LkVal* __restrict__ val, const uint32_t* __restrict__ seg, const int* __restrict__ nseg,
                               const int* __restrict__ nruns, uint32_t n, int method, uint32_t qcut, bool dendrogram,
                               const uint32_t* __restrict__ size, uint32_t* __restrict__ best, uint32_t* __restrict__ best_at,
                               uint32_t* __restrict__ seg_id) {
  const uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= (uint64_t)*nseg) return;
  const uint32_t i0 = seg[w], i1 = w + 1 < (uint64_t)*nseg ? seg[w + 1] : (uint32_t)*nruns;
  const uint64_t sent = (uint64_t)n << 32 | n;
  const uint32_t A = (uint32_t)(key[i0] >> 32);
  __syncwarp();
  if (A >= n) { if (lane == 0) seg_id[w] = LK_NONE; return; }
  const uint64_t na = size[A];
  bool found = false;
  uint64_t bs = 0, bp = 1;
  uint32_t bid = 0, bat = 0;
  for (uint32_t i = i0 + lane; i < i1; i += 32) {
    const uint32_t B = (uint32_t)key[i];
    uint64_t s, p;
    lk_value(method, val[i], na, size[B], &s, &p);
    if (lk_droppable(method, s, p, qcut, dendrogram)) { key[i] = sent; continue; }
    if (!found || lk_better(s, p, B, bs, bp, bid)) { found = true; bs = s; bp = p; bid = B; bat = i; }
  }
  for (int d = 16; d; d >>= 1) {
    const bool of = __shfl_xor_sync(0xffffffffu, found, d);
    const uint64_t os = __shfl_xor_sync(0xffffffffu, bs, d), op = __shfl_xor_sync(0xffffffffu, bp, d);
    const uint32_t oid = __shfl_xor_sync(0xffffffffu, bid, d), oat = __shfl_xor_sync(0xffffffffu, bat, d);
    if (of && (!found || lk_better(os, op, oid, bs, bp, bid))) { found = true; bs = os; bp = op; bid = oid; bat = oat; }
  }
  if (lane) return;
  seg_id[w] = A;
  best[A] = found && lk_qualifies(bs, bp, qcut, dendrogram) ? bid : LK_NONE;
  best_at[A] = bat;
}

// per segment: flag[w] = 1 when A merges and keeps its id; a deactivated A gets lab[A] = LK_NONE, a merging larger id the
// smaller one.  Flags past *nseg are cleared for the scan.
__global__ void lk_merge_kernel(const uint32_t* __restrict__ seg_id, const int* __restrict__ nseg, uint32_t nseg_ub,
                                const uint32_t* __restrict__ best, uint32_t* __restrict__ lab, uint32_t* __restrict__ flag) {
  const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= nseg_ub) return;
  flag[w] = 0;
  if (w >= (uint32_t)*nseg || seg_id[w] == LK_NONE) return;
  const uint32_t A = seg_id[w];
  const int d = lk_decide(A, best);
  if (d == LK_DEACTIVATE) lab[A] = LK_NONE;
  else if (d == LK_MERGE_HIGH) lab[A] = best[A];
  else if (d == LK_MERGE_LOW) flag[w] = 1;
}

// the merges of the round at merges[*nm + pos[w]] (pos = exclusive scan of the flags), sizes, and parent[B] = A for merges
// at or above the cut
__global__ void lk_commit_kernel(const uint32_t* __restrict__ seg_id, const int* __restrict__ nseg, const uint32_t* __restrict__ flag,
                                 const uint32_t* __restrict__ pos, const uint32_t* __restrict__ best, const uint32_t* __restrict__ best_at,
                                 const LkVal* __restrict__ val, int method, uint32_t qcut, uint32_t round, const uint32_t* __restrict__ nm,
                                 uint32_t* size, uint32_t* __restrict__ parent, LkMerge* __restrict__ merges) {
  const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= (uint32_t)*nseg || !flag[w]) return;
  const uint32_t A = seg_id[w], B = best[A], na = size[A], nb = size[B];
  uint64_t s, p;
  lk_value(method, val[best_at[A]], na, nb, &s, &p);
  merges[*nm + pos[w]] = LkMerge{s, p, round, A, B, na + nb};
  if (lk_qualifies(s, p, qcut, false)) parent[B] = A;
  size[A] = na + nb;
}

// *nm += the round's merges; *rounds = round + 1 when there were any
__global__ void lk_count_kernel(const int* __restrict__ nseg, const uint32_t* __restrict__ flag, const uint32_t* __restrict__ pos,
                                uint32_t round, uint32_t* __restrict__ nm, uint32_t* __restrict__ rounds) {
  const int k = *nseg;
  const uint32_t t = k ? pos[k - 1] + flag[k - 1] : 0;
  if (t) { *nm += t; *rounds = round + 1; }
}

// pairs renamed to their clusters' new ids; self pairs, pairs of deactivated clusters and entries past *nruns -> sentinel
__global__ void lk_relabel_kernel(uint64_t* __restrict__ key, uint32_t m, const int* __restrict__ nruns, uint32_t n,
                                  const uint32_t* __restrict__ lab) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const uint64_t sent = (uint64_t)n << 32 | n, k = key[i];
  if ((int)i >= *nruns || (k >> 32) >= n) { key[i] = sent; return; }
  const uint32_t a = lab[(uint32_t)(k >> 32)], b = lab[(uint32_t)k];
  key[i] = a == LK_NONE || b == LK_NONE || a == b ? sent : (uint64_t)a << 32 | b;
}

}  // namespace

int sk::build_graph(sk_ctx* ctx, const char* who, uint32_t n, const sk_ani_result* results, uint64_t n_results, float min_ani, Graph& g) {
  cudaStream_t st = ctx->stream;
  const auto launched = [&](unsigned k = 1) { count_launch(ctx, k); return cudaGetLastError(); };
  DTmp<uint8_t> chunk;
  DTmp<unsigned long long> cnt;   // [0] edges, [1] bad id, [2] self pair, [3] duplicate
  SK_TRY(cl_alloc(ctx, cnt, 4, "counters", who));
  SK_TRY(cl_alloc(ctx, g.ekey, n_results, "edge keys", who));
  SK_TRY(cl_alloc(ctx, g.eani, n_results, "edge ANIs", who));
  SK_TRY(cl_alloc(ctx, g.erow, n_results, "edge rows", who));
  SK_TRY(cl_alloc(ctx, chunk, std::min(n_results, CHUNK_ROWS) * sizeof(sk_ani_result), "result chunk", who));
  SK_CUDA(cudaMemsetAsync(cnt.p, 0, 8, st));
  SK_CUDA(cudaMemsetAsync(cnt.p + 1, 0xff, 24, st));
  const bool pinned = host_pinned(results);
  for (uint64_t r0 = 0; r0 < n_results; r0 += CHUNK_ROWS) {
    const uint64_t m = std::min(CHUNK_ROWS, n_results - r0);
    SK_TRY(upload_runs(ctx, chunk.p, {{(const uint8_t*)(results + r0), m * sizeof(sk_ani_result)}}, pinned));
    cl_filter_kernel<<<blocks_for(m), TPB, 0, st>>>((const sk_ani_result*)chunk.p, m, r0, n, min_ani, cnt.p, g.ekey.p, g.eani.p, g.erow.p, cnt.p + 1);
    SK_CUDA(launched());
  }
  unsigned long long h_cnt[4];
  SK_CUDA(cudaMemcpyAsync(h_cnt, cnt.p, sizeof(h_cnt), cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaStreamSynchronize(st));
  chunk.release();
  const std::string w = who;
  if (h_cnt[1] != UINT64_MAX) { ctx->err = w + ": genome id >= n_genomes = " + std::to_string(n) + " in " + row_text(results, h_cnt[1]); return SK_ERR_PARAM; }
  if (h_cnt[2] != UINT64_MAX) { ctx->err = w + ": self pair in " + row_text(results, h_cnt[2]); return SK_ERR_PARAM; }
  const uint64_t E = h_cnt[0], A = 2 * E;
  g.E = E;
  if (A > (uint64_t)INT32_MAX) { ctx->err = w + ": " + std::to_string(E) + " edges, more than one radix sort takes (2^30)"; return SK_ERR_NOMEM; }
  // ---- symmetric CSR: both directions sorted by (a << 32 | b)
  for (int b = 0; b < 2; b++) {
    SK_TRY(cl_alloc(ctx, g.key[b], A, "adjacency keys", who));
    SK_TRY(cl_alloc(ctx, g.val[b], A, "adjacency edges", who));
  }
  SK_TRY(cl_alloc(ctx, g.off, (uint64_t)n + 1, "CSR offsets", who));
  cub::DoubleBuffer<uint64_t> dk(g.key[0].p, g.key[1].p);
  cub::DoubleBuffer<uint32_t> dv(g.val[0].p, g.val[1].p);
  if (E) {
    cl_directed_kernel<<<blocks_for(E), TPB, 0, st>>>(g.ekey.p, E, g.key[0].p, g.val[0].p);
    SK_CUDA(launched());
    int bits = 33;
    while (bits < 64 && (1ull << (bits - 32)) < n) bits++;
    size_t tb = 0;
    SK_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, dk, dv, (int)A, 0, bits, st));
    DTmp<uint8_t> tmp;
    SK_TRY(cl_alloc(ctx, tmp, tb, "sort temporaries", who));
    SK_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, dk, dv, (int)A, 0, bits, st));
    SK_CUDA(launched());
    cl_dup_kernel<<<blocks_for(A), TPB, 0, st>>>(dk.Current(), A, cnt.p + 3);
    SK_CUDA(launched());
  }
  g.adj = dk.Current();
  g.adj_e = dv.Current();
  (dk.Current() == g.key[0].p ? g.key[1] : g.key[0]).release();
  (dv.Current() == g.val[0].p ? g.val[1] : g.val[0]).release();
  cl_offsets_kernel<<<blocks_for((uint64_t)n + 1), TPB, 0, st>>>(g.adj, A, n, g.off.p);
  SK_CUDA(launched());
  SK_CUDA(cudaMemcpyAsync(&h_cnt[3], cnt.p + 3, 8, cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaStreamSynchronize(st));
  if (h_cnt[3] != UINT64_MAX) {
    uint64_t k = 0;
    SK_CUDA(cudaMemcpy(&k, g.adj + h_cnt[3], 8, cudaMemcpyDeviceToHost));
    const uint64_t a = k >> 32, b = (uint32_t)k;
    ctx->err = w + ": pair (" + std::to_string(std::min(a, b)) + ", " + std::to_string(std::max(a, b)) + ") is listed twice among the edges";
    return SK_ERR_PARAM;
  }
  return SK_OK;
}

int sk::greedy_rounds(sk_ctx* ctx, const char* who, const uint32_t* frontier, uint32_t m, const Graph& g, const uint32_t* d_rank,
                      uint8_t* state, uint32_t* rounds) {
  cudaStream_t st = ctx->stream;
  const auto launched = [&](unsigned k = 1) { count_launch(ctx, k); return cudaGetLastError(); };
  DTmp<uint32_t> front[2], d_m;
  SK_TRY(cl_alloc(ctx, front[0], m, "frontier", who));
  SK_TRY(cl_alloc(ctx, front[1], m, "frontier", who));
  SK_TRY(cl_alloc(ctx, d_m, 1, "frontier size", who));
  SK_CUDA(cudaMemcpyAsync(front[0].p, frontier, (size_t)m * 4, cudaMemcpyDeviceToDevice, st));
  size_t tb = 0;
  SK_CUDA(cub::DeviceSelect::If(nullptr, tb, front[0].p, front[1].p, d_m.p, (int)m, Undecided{state}, st));
  DTmp<uint8_t> tmp;
  SK_TRY(cl_alloc(ctx, tmp, tb, "frontier compaction", who));
  const uint32_t m0 = m;
  uint32_t r = 0;
  int cur = 0;
  // each round decides at least the undecided vertex of smallest rank, so m rounds always finish
  while (m) {
    for (int k = 0; k < GREEDY_ROUNDS; k++) {
      cl_greedy_kernel<<<blocks_for(m), TPB, 0, st>>>(front[cur].p, m, g.off.p, g.adj, d_rank, state);
      r++;
    }
    SK_CUDA(launched(GREEDY_ROUNDS));
    SK_CUDA(cub::DeviceSelect::If(tmp.p, tb, front[cur].p, front[cur ^ 1].p, d_m.p, (int)m, Undecided{state}, st));
    SK_CUDA(launched());
    SK_CUDA(cudaMemcpyAsync(&m, d_m.p, 4, cudaMemcpyDeviceToHost, st));
    SK_CUDA(cudaStreamSynchronize(st));
    cur ^= 1;
    if (r > m0 + GREEDY_ROUNDS) { ctx->err = std::string(who) + ": greedy rounds did not converge"; return SK_ERR_STATE; }
  }
  *rounds += r;
  return SK_OK;
}

int sk::greedy_assign(sk_ctx* ctx, uint32_t n, const Graph& g, const uint32_t* d_rank, const uint8_t* state, uint32_t* d_rep,
                      uint64_t* d_edge, uint32_t* flag) {
  cl_assign_kernel<<<blocks_for(n), TPB, 0, ctx->stream>>>(n, g.off.p, g.adj, g.adj_e, g.eani.p, g.erow.p, d_rank, state, d_rep, d_edge, flag);
  count_launch(ctx, 1);
  SK_CUDA(cudaGetLastError());
  return SK_OK;
}

// representatives (flag[rank[v]] = 1) numbered in rank order, then rep / cluster / edge read back
int sk::number_and_read_back(sk_ctx* ctx, const char* who, uint32_t n, const uint32_t* d_rank, const uint32_t* d_rep, const uint64_t* d_edge,
                         uint32_t* flag, uint32_t* d_cluster, uint32_t* rep, uint32_t* cluster, uint64_t* edge, uint32_t* n_clusters) {
  cudaStream_t st = ctx->stream;
  *n_clusters = 0;
  if (!n) return SK_OK;
  size_t tb = 0;
  SK_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tb, flag, flag, (int)n, st));
  DTmp<uint8_t> tmp;
  SK_TRY(cl_alloc(ctx, tmp, tb, "scan temporaries", who));
  SK_CUDA(cub::DeviceScan::InclusiveSum(tmp.p, tb, flag, flag, (int)n, st));
  count_launch(ctx, 1);
  cl_number_kernel<<<blocks_for(n), TPB, 0, st>>>(n, d_rep, d_rank, flag, d_cluster);
  count_launch(ctx, 1);
  SK_CUDA(cudaGetLastError());
  SK_CUDA(cudaMemcpyAsync(rep, d_rep, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaMemcpyAsync(cluster, d_cluster, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaMemcpyAsync(edge, d_edge, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaMemcpyAsync(n_clusters, flag + n - 1, 4, cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaStreamSynchronize(st));
  return SK_OK;
}

namespace {

int cluster_impl(sk_ctx* ctx, uint32_t n, const sk_ani_result* results, uint64_t n_results, const uint32_t* rank,
                 const sk_cluster_params* cp, uint32_t* rep, uint32_t* cluster, uint64_t* edge, sk_cluster_stats* stats) {
  cudaStream_t st = ctx->stream;
  const auto launched = [&](unsigned k = 1) { count_launch(ctx, k); return cudaGetLastError(); };
  Graph g;
  SK_TRY(build_graph(ctx, "sk_cluster", n, results, n_results, cp->min_ani, g));
  const uint64_t E = g.E;
  const uint64_t* adj = g.adj;
  const uint32_t* adj_e = g.adj_e;
  // ---- per vertex
  DTmp<uint32_t> d_rank, order, d_rep, d_cluster, flag;
  DTmp<uint64_t> d_edge;
  SK_TRY(cl_alloc(ctx, d_rank, n, "ranks"));
  SK_TRY(cl_alloc(ctx, order, n, "rank order"));
  SK_TRY(cl_alloc(ctx, d_rep, n, "representatives"));
  SK_TRY(cl_alloc(ctx, d_cluster, n, "clusters"));
  SK_TRY(cl_alloc(ctx, flag, n, "flags"));
  SK_TRY(cl_alloc(ctx, d_edge, n, "edges per genome"));
  SK_CUDA(h2d_small(ctx, d_rank.p, rank, (size_t)n * 4));
  cl_order_kernel<<<blocks_for(n), TPB, 0, st>>>(d_rank.p, n, order.p);
  SK_CUDA(launched());
  uint32_t rounds = 0;
  if (!cp->single_linkage) {
    DTmp<uint8_t> state;
    SK_TRY(cl_alloc(ctx, state, n, "states"));
    SK_CUDA(cudaMemsetAsync(state.p, 0, n, st));
    SK_TRY(greedy_rounds(ctx, "sk_cluster", order.p, n, g, d_rank.p, state.p, &rounds));
    SK_TRY(greedy_assign(ctx, n, g, d_rank.p, state.p, d_rep.p, d_edge.p, flag.p));
  } else {
    DTmp<uint32_t> parent, changed;
    SK_TRY(cl_alloc(ctx, parent, n, "parents"));
    SK_TRY(cl_alloc(ctx, changed, 1, "change flag"));
    cl_iota_kernel<<<blocks_for(n), TPB, 0, st>>>(parent.p, n);
    SK_CUDA(launched());
    // every pass that leaves two parents of an edge apart lowers one of them, so at most n passes change something
    for (uint32_t h_changed = 1; h_changed && E;) {
      SK_CUDA(cudaMemsetAsync(changed.p, 0, 4, st));
      cl_hook_kernel<<<blocks_for(E), TPB, 0, st>>>(g.ekey.p, E, d_rank.p, parent.p, changed.p);
      SK_CUDA(launched());
      rounds++;
      SK_CUDA(cudaMemcpyAsync(&h_changed, changed.p, 4, cudaMemcpyDeviceToHost, st));
      SK_CUDA(cudaStreamSynchronize(st));
      if (!h_changed) break;
      cl_jump_kernel<<<blocks_for(n), TPB, 0, st>>>(parent.p, n);
      SK_CUDA(launched());
      if (rounds > n + 1) { ctx->err = "sk_cluster: single linkage did not converge"; return SK_ERR_STATE; }
    }
    cl_component_kernel<<<blocks_for(n), TPB, 0, st>>>(n, g.off.p, adj, adj_e, g.erow.p, d_rank.p, order.p, parent.p, d_rep.p, d_edge.p, flag.p);
    SK_CUDA(launched());
  }
  uint32_t n_clusters = 0;
  SK_TRY(number_and_read_back(ctx, "sk_cluster", n, d_rank.p, d_rep.p, d_edge.p, flag.p, d_cluster.p, rep, cluster, edge, &n_clusters));
  if (stats) { stats->n_edges = E; stats->n_clusters = n_clusters; stats->rounds = rounds; }
  return SK_OK;
}

}  // namespace

// rank must be a permutation of 0 .. n - 1: the reason it is not, empty when it is
std::string sk::rank_error(uint32_t n, const uint32_t* rank) {
  std::vector<uint8_t> seen(n, 0);
  for (uint32_t g = 0; g < n; g++) {
    if (rank[g] >= n || seen[rank[g]]) return "rank is not a permutation of 0.." + std::to_string(n) + " - 1 (genome " + std::to_string(g) + ")";
    seen[rank[g]] = 1;
  }
  return "";
}

namespace {

constexpr int LK_ROUNDS = 8;   // linkage rounds between two read-backs of the pair count

int linkage_impl(sk_ctx* ctx, uint32_t n, const sk_ani_result* results, uint64_t n_results, const uint32_t* rank,
                 const sk_linkage_params* lp, uint32_t* rep, uint32_t* cluster, uint64_t* edge, sk_merge* merges, sk_cluster_stats* stats) {
  const char* who = "sk_cluster_linkage";
  cudaStream_t st = ctx->stream;
  const auto launched = [&](unsigned k = 1) { count_launch(ctx, k); return cudaGetLastError(); };
  Graph g;
  SK_TRY(build_graph(ctx, who, n, results, n_results, 0.f, g));
  const uint64_t E = g.E;
  const uint32_t M0 = (uint32_t)(2 * E), qcut = lk_q(lp->min_ani);
  const int method = lp->method;
  const bool dendro = lp->dendrogram != 0;
  DTmp<uint32_t> d_rank, order, d_rep, d_cluster, flag, parent, lab, size, best, best_at;
  DTmp<uint64_t> d_edge;
  SK_TRY(cl_alloc(ctx, d_rank, n, "ranks", who));
  SK_TRY(cl_alloc(ctx, order, n, "rank order", who));
  SK_TRY(cl_alloc(ctx, d_rep, n, "representatives", who));
  SK_TRY(cl_alloc(ctx, d_cluster, n, "clusters", who));
  SK_TRY(cl_alloc(ctx, flag, n, "flags", who));
  SK_TRY(cl_alloc(ctx, d_edge, n, "edges per genome", who));
  SK_TRY(cl_alloc(ctx, parent, n, "parents", who));
  SK_TRY(cl_alloc(ctx, lab, n, "labels", who));
  SK_TRY(cl_alloc(ctx, size, n, "cluster sizes", who));
  SK_TRY(cl_alloc(ctx, best, n, "best partners", who));
  SK_TRY(cl_alloc(ctx, best_at, n, "best pairs", who));
  SK_CUDA(h2d_small(ctx, d_rank.p, rank, (size_t)n * 4));
  cl_order_kernel<<<blocks_for(n), TPB, 0, st>>>(d_rank.p, n, order.p);
  cl_iota_kernel<<<blocks_for(n), TPB, 0, st>>>(parent.p, n);
  cl_iota_kernel<<<blocks_for(n), TPB, 0, st>>>(lab.p, n);
  SK_CUDA(launched(3));
  {
    std::vector<uint32_t> ones(n, 1);
    SK_CUDA(h2d_small(ctx, size.p, ones.data(), (size_t)n * 4));
  }
  // ---- pair list: keys and values double-buffered for the sort, the reduce writing back into the free half
  DTmp<uint64_t> key[2];
  DTmp<LkVal> val[2];
  DTmp<uint32_t> seg, seg_id, pos, flags;
  DTmp<int> counts;                 // [0] runs, [1] segments
  DTmp<uint32_t> tally;             // [0] merges, [1] rounds
  DTmp<LkMerge> recs;
  DTmp<unsigned long long> bad;
  const uint32_t seg_cap = std::min<uint64_t>(M0, (uint64_t)n + 1);
  for (int b = 0; b < 2; b++) {
    SK_TRY(cl_alloc(ctx, key[b], M0, "pair keys", who));
    SK_TRY(cl_alloc(ctx, val[b], M0, "pair values", who));
  }
  SK_TRY(cl_alloc(ctx, seg, seg_cap, "segments", who));
  SK_TRY(cl_alloc(ctx, seg_id, seg_cap, "segment clusters", who));
  SK_TRY(cl_alloc(ctx, pos, seg_cap, "merge positions", who));
  SK_TRY(cl_alloc(ctx, flags, seg_cap, "merge flags", who));
  SK_TRY(cl_alloc(ctx, counts, 2, "counts", who));
  SK_TRY(cl_alloc(ctx, tally, 2, "merge tally", who));
  SK_TRY(cl_alloc(ctx, recs, n ? n - 1 : 0, "merge records", who));
  SK_TRY(cl_alloc(ctx, bad, 1, "bad row", who));
  SK_CUDA(cudaMemsetAsync(tally.p, 0, 8, st));
  SK_CUDA(cudaMemsetAsync(bad.p, 0xff, 8, st));
  SK_CUDA(cudaMemsetAsync(counts.p, 0, 8, st));
  if (E) {
    lk_init_kernel<<<blocks_for(E), TPB, 0, st>>>(g.ekey.p, g.eani.p, g.erow.p, E, d_rank.p, key[0].p, val[0].p, bad.p);
    SK_CUDA(launched());
  }
  unsigned long long h_bad = 0;
  SK_CUDA(cudaMemcpyAsync(&h_bad, bad.p, 8, cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaStreamSynchronize(st));
  if (h_bad != UINT64_MAX) { ctx->err = std::string(who) + ": ani >= 2 in " + row_text(results, h_bad); return SK_ERR_PARAM; }
  g.ekey.release(); g.eani.release();
  // cub temporaries sized for the first (largest) round
  int bits = 33;
  while (bits < 64 && (1ull << (bits - 32)) < (uint64_t)n + 1) bits++;
  cub::DoubleBuffer<uint64_t> dk(key[0].p, key[1].p);
  cub::DoubleBuffer<LkVal> dv(val[0].p, val[1].p);
  size_t tb = 0, t1 = 0;
  const thrust::counting_iterator<uint32_t> idx(0);
  SK_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t1, dk, dv, (int)M0, 0, bits, st)); tb = std::max(tb, t1);
  SK_CUDA(cub::DeviceReduce::ReduceByKey(nullptr, t1, key[0].p, key[1].p, val[0].p, val[1].p, counts.p, LkCombine{}, (int)M0, st)); tb = std::max(tb, t1);
  SK_CUDA(cub::DeviceSelect::If(nullptr, t1, idx, seg.p, counts.p + 1, (int)M0, LkHead{key[0].p, counts.p}, st)); tb = std::max(tb, t1);
  SK_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, t1, flags.p, pos.p, (int)seg_cap, st)); tb = std::max(tb, t1);
  DTmp<uint8_t> tmp;
  SK_TRY(cl_alloc(ctx, tmp, tb, "sort / reduce temporaries", who));
  int cur = 0;   // the sorted, reduced list is in key[cur], val[cur]
  // sort the m entries of key[cur], then combine equal keys into the other half: *counts = runs
  const auto sort_reduce = [&](uint32_t m) -> int {
    dk = cub::DoubleBuffer<uint64_t>(key[cur].p, key[cur ^ 1].p);
    dv = cub::DoubleBuffer<LkVal>(val[cur].p, val[cur ^ 1].p);
    SK_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, dk, dv, (int)m, 0, bits, st));
    const int s = dk.Current() == key[0].p ? 0 : 1;
    SK_CUDA(cub::DeviceReduce::ReduceByKey(tmp.p, tb, key[s].p, key[s ^ 1].p, val[s].p, val[s ^ 1].p, counts.p, LkCombine{}, (int)m, st));
    SK_CUDA(launched(2));
    cur = s ^ 1;
    return SK_OK;
  };
  uint32_t m = M0, round = 0;
  if (m) SK_TRY(sort_reduce(m));
  // every round with a pair left merges the pair of largest value or deactivates every cluster, so n rounds always finish
  while (m) {
    for (int k = 0; k < LK_ROUNDS; k++, round++) {
      const uint32_t nseg_ub = std::min<uint64_t>(m, (uint64_t)n + 1);
      SK_CUDA(cub::DeviceSelect::If(tmp.p, tb, idx, seg.p, counts.p + 1, (int)m, LkHead{key[cur].p, counts.p}, st));
      lk_best_kernel<<<blocks_for((uint64_t)nseg_ub * 32), TPB, 0, st>>>(key[cur].p, val[cur].p, seg.p, counts.p + 1, counts.p, n, method,
                                                                       qcut, dendro, size.p, best.p, best_at.p, seg_id.p);
      lk_merge_kernel<<<blocks_for(nseg_ub), TPB, 0, st>>>(seg_id.p, counts.p + 1, nseg_ub, best.p, lab.p, flags.p);
      SK_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tb, flags.p, pos.p, (int)nseg_ub, st));
      lk_commit_kernel<<<blocks_for(nseg_ub), TPB, 0, st>>>(seg_id.p, counts.p + 1, flags.p, pos.p, best.p, best_at.p, val[cur].p, method,
                                                          qcut, round, tally.p, size.p, parent.p, recs.p);
      lk_count_kernel<<<1, 1, 0, st>>>(counts.p + 1, flags.p, pos.p, round, tally.p, tally.p + 1);
      lk_relabel_kernel<<<blocks_for(m), TPB, 0, st>>>(key[cur].p, m, counts.p, n, lab.p);
      SK_CUDA(launched(7));
      SK_TRY(sort_reduce(m));
    }
    // the list shrinks to its runs; it is empty when no run is left but the sentinels
    int runs = 0;
    uint64_t first = 0;
    SK_CUDA(cudaMemcpyAsync(&runs, counts.p, 4, cudaMemcpyDeviceToHost, st));
    SK_CUDA(cudaMemcpyAsync(&first, key[cur].p, 8, cudaMemcpyDeviceToHost, st));
    SK_CUDA(cudaStreamSynchronize(st));
    m = runs && (first >> 32) < n ? (uint32_t)runs : 0;
    if (round > n + LK_ROUNDS) { ctx->err = std::string(who) + ": linkage rounds did not converge"; return SK_ERR_STATE; }
  }
  // ---- flat clusters from parent[]: roots are the smallest ranks
  cl_jump_kernel<<<blocks_for(n), TPB, 0, st>>>(parent.p, n);
  cl_component_kernel<<<blocks_for(n), TPB, 0, st>>>(n, g.off.p, g.adj, g.adj_e, g.erow.p, d_rank.p, order.p, parent.p, d_rep.p, d_edge.p, flag.p);
  SK_CUDA(launched(2));
  uint32_t n_clusters = 0, h_tally[2] = {0, 0};
  SK_TRY(number_and_read_back(ctx, who, n, d_rank.p, d_rep.p, d_edge.p, flag.p, d_cluster.p, rep, cluster, edge, &n_clusters));
  SK_CUDA(cudaMemcpyAsync(h_tally, tally.p, 8, cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaStreamSynchronize(st));
  const uint32_t nm = h_tally[0];
  if (dendro && n) {
    // ---- merges in dendrogram order on the device, then scipy's cluster numbers (n + row) on the host
    std::vector<LkMerge> h(nm);
    if (nm) {
      size_t mb = 0;
      SK_CUDA(cub::DeviceMergeSort::SortKeys(nullptr, mb, recs.p, (int)nm, LkMergeOrder{}, st));
      DTmp<uint8_t> mtmp;
      SK_TRY(cl_alloc(ctx, mtmp, mb, "merge sort temporaries", who));
      SK_CUDA(cub::DeviceMergeSort::SortKeys(mtmp.p, mb, recs.p, (int)nm, LkMergeOrder{}, st));
      SK_CUDA(launched());
      SK_CUDA(cudaMemcpyAsync(h.data(), recs.p, (size_t)nm * sizeof(LkMerge), cudaMemcpyDeviceToHost, st));
      SK_CUDA(cudaStreamSynchronize(st));
    }
    std::vector<uint32_t> node(n);           // by id (rank): its cluster's current scipy number
    std::vector<uint64_t> members(n, 1);
    std::vector<uint8_t> gone(n, 0);
    for (uint32_t g0 = 0; g0 < n; g0++) node[rank[g0]] = g0;
    const auto join = [&](uint32_t j, uint32_t a, uint32_t b, double h, uint64_t sz) {
      merges[j] = sk_merge{std::min(node[a], node[b]), std::max(node[a], node[b]), h, sz};
      node[a] = n + j; members[a] = sz; gone[b] = 1;
    };
    for (uint32_t j = 0; j < nm; j++) join(j, h[j].a, h[j].b, lk_height(h[j]), h[j].size);
    // the clusters left are joined at height 1 in id order
    uint32_t j = nm, first = UINT32_MAX;
    for (uint32_t r = 0; r < n; r++) {
      if (gone[r]) continue;
      if (first == UINT32_MAX) first = r;
      else join(j++, first, r, 1.0, members[first] + members[r]);
    }
  }
  if (stats) { stats->n_edges = E; stats->n_clusters = n_clusters; stats->rounds = h_tally[1]; }
  return SK_OK;
}

}  // namespace

int sk_cluster(sk_ctx* ctx, uint32_t n_genomes, const sk_ani_result* results, uint64_t n_results, const uint32_t* rank,
               const sk_cluster_params* cp, uint32_t* rep, uint32_t* cluster, uint64_t* edge, sk_cluster_stats* stats) {
  if (!ctx) return SK_ERR_PARAM;
  if (!cp || !rep || !cluster || !edge || (n_results && !results) || (n_genomes && !rank)) {
    ctx->err = "sk_cluster: NULL argument"; return SK_ERR_PARAM;
  }
  if (std::isnan(cp->min_ani)) { ctx->err = "sk_cluster: min_ani is NaN"; return SK_ERR_PARAM; }
  const std::string bad = rank_error(n_genomes, rank);
  if (!bad.empty()) { ctx->err = "sk_cluster: " + bad; return SK_ERR_PARAM; }
  SK_CUDA(cudaSetDevice(ctx->device));
  const auto t0 = std::chrono::steady_clock::now();
  const int rc = cluster_impl(ctx, n_genomes, results, n_results, rank, cp, rep, cluster, edge, stats);
  if (rc == SK_OK && stats) stats->t_device = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return rc;
}

int sk_cluster_linkage(sk_ctx* ctx, uint32_t n_genomes, const sk_ani_result* results, uint64_t n_results, const uint32_t* rank,
                       const sk_linkage_params* lp, uint32_t* rep, uint32_t* cluster, uint64_t* edge, sk_merge* merges,
                       sk_cluster_stats* stats) {
  if (!ctx) return SK_ERR_PARAM;
  if (!lp || !rep || !cluster || !edge || (n_results && !results) || (n_genomes && !rank) || (lp->dendrogram && n_genomes > 1 && !merges)) {
    ctx->err = "sk_cluster_linkage: NULL argument"; return SK_ERR_PARAM;
  }
  if (!(lp->min_ani > CL_MIN_PRINTED_ANI && lp->min_ani <= 1.f)) {
    ctx->err = "sk_cluster_linkage: min_ani " + std::to_string(lp->min_ani) + " is not in (0.1, 1]"; return SK_ERR_PARAM;
  }
  if (lp->method != SK_LINKAGE_AVERAGE && lp->method != SK_LINKAGE_COMPLETE) {
    ctx->err = "sk_cluster_linkage: unknown method " + std::to_string(lp->method) + " (0 average, 1 complete)"; return SK_ERR_PARAM;
  }
  const std::string bad = rank_error(n_genomes, rank);
  if (!bad.empty()) { ctx->err = "sk_cluster_linkage: " + bad; return SK_ERR_PARAM; }
  SK_CUDA(cudaSetDevice(ctx->device));
  const auto t0 = std::chrono::steady_clock::now();
  const int rc = linkage_impl(ctx, n_genomes, results, n_results, rank, lp, rep, cluster, edge, merges, stats);
  if (rc == SK_OK && stats) stats->t_device = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return rc;
}
