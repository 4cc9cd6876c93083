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
#include <cub/cub.cuh>

#include <chrono>
#include <cmath>
#include <string>
#include <vector>

#include "cluster_core.cuh"
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

// device temporaries of sk_cluster: a failed allocation is SK_ERR_NOMEM
template <typename T>
int cl_alloc(sk_ctx* ctx, DTmp<T>& t, uint64_t count, const char* what) {
  if (t.alloc(count, ctx) != cudaSuccess) {
    cudaGetLastError();
    ctx->err = std::string("sk_cluster: out of device memory (") + what + ", " + std::to_string(count * sizeof(T)) + " bytes)";
    return SK_ERR_NOMEM;
  }
  return SK_OK;
}

std::string row_text(const sk_ani_result* results, uint64_t row) {
  return "row " + std::to_string(row) + " (" + std::to_string(results[row].ref_id) + ", " + std::to_string(results[row].query_id) + ")";
}

int cluster_impl(sk_ctx* ctx, uint32_t n, const sk_ani_result* results, uint64_t n_results, const uint32_t* rank,
                 const sk_cluster_params* cp, uint32_t* rep, uint32_t* cluster, uint64_t* edge, sk_cluster_stats* stats) {
  cudaStream_t st = ctx->stream;
  const auto launched = [&](unsigned k = 1) { count_launch(ctx, k); return cudaGetLastError(); };
  // ---- edges
  DTmp<uint8_t> chunk;
  DTmp<uint64_t> ekey, erow;
  DTmp<float> eani;
  DTmp<unsigned long long> cnt;   // [0] edges, [1] bad id, [2] self pair, [3] duplicate
  SK_TRY(cl_alloc(ctx, cnt, 4, "counters"));
  SK_TRY(cl_alloc(ctx, ekey, n_results, "edge keys"));
  SK_TRY(cl_alloc(ctx, eani, n_results, "edge ANIs"));
  SK_TRY(cl_alloc(ctx, erow, n_results, "edge rows"));
  SK_TRY(cl_alloc(ctx, chunk, std::min(n_results, CHUNK_ROWS) * sizeof(sk_ani_result), "result chunk"));
  SK_CUDA(cudaMemsetAsync(cnt.p, 0, 8, st));
  SK_CUDA(cudaMemsetAsync(cnt.p + 1, 0xff, 24, st));
  const bool pinned = host_pinned(results);
  for (uint64_t r0 = 0; r0 < n_results; r0 += CHUNK_ROWS) {
    const uint64_t m = std::min(CHUNK_ROWS, n_results - r0);
    SK_TRY(upload_runs(ctx, chunk.p, {{(const uint8_t*)(results + r0), m * sizeof(sk_ani_result)}}, pinned));
    cl_filter_kernel<<<blocks_for(m), TPB, 0, st>>>((const sk_ani_result*)chunk.p, m, r0, n, cp->min_ani, cnt.p, ekey.p, eani.p, erow.p, cnt.p + 1);
    SK_CUDA(launched());
  }
  unsigned long long h_cnt[4];
  SK_CUDA(cudaMemcpyAsync(h_cnt, cnt.p, sizeof(h_cnt), cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaStreamSynchronize(st));
  chunk.release();
  if (h_cnt[1] != UINT64_MAX) { ctx->err = "sk_cluster: genome id >= n_genomes = " + std::to_string(n) + " in " + row_text(results, h_cnt[1]); return SK_ERR_PARAM; }
  if (h_cnt[2] != UINT64_MAX) { ctx->err = "sk_cluster: self pair in " + row_text(results, h_cnt[2]); return SK_ERR_PARAM; }
  const uint64_t E = h_cnt[0], A = 2 * E;
  if (A > (uint64_t)INT32_MAX) { ctx->err = "sk_cluster: " + std::to_string(E) + " edges, more than one radix sort takes (2^30)"; return SK_ERR_NOMEM; }
  // ---- symmetric CSR: both directions sorted by (a << 32 | b)
  DTmp<uint64_t> key[2], off;
  DTmp<uint32_t> val[2];
  for (int b = 0; b < 2; b++) {
    SK_TRY(cl_alloc(ctx, key[b], A, "adjacency keys"));
    SK_TRY(cl_alloc(ctx, val[b], A, "adjacency edges"));
  }
  SK_TRY(cl_alloc(ctx, off, (uint64_t)n + 1, "CSR offsets"));
  cub::DoubleBuffer<uint64_t> dk(key[0].p, key[1].p);
  cub::DoubleBuffer<uint32_t> dv(val[0].p, val[1].p);
  if (E) {
    cl_directed_kernel<<<blocks_for(E), TPB, 0, st>>>(ekey.p, E, key[0].p, val[0].p);
    SK_CUDA(launched());
    int bits = 33;
    while (bits < 64 && (1ull << (bits - 32)) < n) bits++;
    size_t tb = 0;
    SK_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, dk, dv, (int)A, 0, bits, st));
    DTmp<uint8_t> tmp;
    SK_TRY(cl_alloc(ctx, tmp, tb, "sort temporaries"));
    SK_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, dk, dv, (int)A, 0, bits, st));
    SK_CUDA(launched());
    cl_dup_kernel<<<blocks_for(A), TPB, 0, st>>>(dk.Current(), A, cnt.p + 3);
    SK_CUDA(launched());
  }
  const uint64_t* adj = dk.Current();
  const uint32_t* adj_e = dv.Current();
  DTmp<uint64_t>& spare_key = dk.Current() == key[0].p ? key[1] : key[0];
  DTmp<uint32_t>& spare_val = dv.Current() == val[0].p ? val[1] : val[0];
  spare_key.release(); spare_val.release();
  cl_offsets_kernel<<<blocks_for((uint64_t)n + 1), TPB, 0, st>>>(adj, A, n, off.p);
  SK_CUDA(launched());
  SK_CUDA(cudaMemcpyAsync(&h_cnt[3], cnt.p + 3, 8, cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaStreamSynchronize(st));
  if (h_cnt[3] != UINT64_MAX) {
    uint64_t k = 0;
    SK_CUDA(cudaMemcpy(&k, adj + h_cnt[3], 8, cudaMemcpyDeviceToHost));
    const uint64_t a = k >> 32, b = (uint32_t)k;
    ctx->err = "sk_cluster: pair (" + std::to_string(std::min(a, b)) + ", " + std::to_string(std::max(a, b)) + ") is listed twice among the edges";
    return SK_ERR_PARAM;
  }
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
    DTmp<uint32_t> front[2], d_m;
    SK_TRY(cl_alloc(ctx, state, n, "states"));
    SK_TRY(cl_alloc(ctx, front[0], n, "frontier"));
    SK_TRY(cl_alloc(ctx, front[1], n, "frontier"));
    SK_TRY(cl_alloc(ctx, d_m, 1, "frontier size"));
    SK_CUDA(cudaMemsetAsync(state.p, 0, n, st));
    SK_CUDA(cudaMemcpyAsync(front[0].p, order.p, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
    size_t tb = 0;
    SK_CUDA(cub::DeviceSelect::If(nullptr, tb, front[0].p, front[1].p, d_m.p, (int)n, Undecided{state.p}, st));
    DTmp<uint8_t> tmp;
    SK_TRY(cl_alloc(ctx, tmp, tb, "frontier compaction"));
    uint32_t m = n;
    int cur = 0;
    // each round decides at least the undecided vertex of smallest rank, so n rounds always finish
    while (m) {
      for (int k = 0; k < GREEDY_ROUNDS; k++) {
        cl_greedy_kernel<<<blocks_for(m), TPB, 0, st>>>(front[cur].p, m, off.p, adj, d_rank.p, state.p);
        rounds++;
      }
      SK_CUDA(launched(GREEDY_ROUNDS));
      SK_CUDA(cub::DeviceSelect::If(tmp.p, tb, front[cur].p, front[cur ^ 1].p, d_m.p, (int)m, Undecided{state.p}, st));
      SK_CUDA(launched());
      SK_CUDA(cudaMemcpyAsync(&m, d_m.p, 4, cudaMemcpyDeviceToHost, st));
      SK_CUDA(cudaStreamSynchronize(st));
      cur ^= 1;
      if (rounds > n + GREEDY_ROUNDS) { ctx->err = "sk_cluster: greedy rounds did not converge"; return SK_ERR_STATE; }
    }
    cl_assign_kernel<<<blocks_for(n), TPB, 0, st>>>(n, off.p, adj, adj_e, eani.p, erow.p, d_rank.p, state.p, d_rep.p, d_edge.p, flag.p);
    SK_CUDA(launched());
  } else {
    DTmp<uint32_t> parent, changed;
    SK_TRY(cl_alloc(ctx, parent, n, "parents"));
    SK_TRY(cl_alloc(ctx, changed, 1, "change flag"));
    cl_iota_kernel<<<blocks_for(n), TPB, 0, st>>>(parent.p, n);
    SK_CUDA(launched());
    // every pass that leaves two parents of an edge apart lowers one of them, so at most n passes change something
    for (uint32_t h_changed = 1; h_changed && E;) {
      SK_CUDA(cudaMemsetAsync(changed.p, 0, 4, st));
      cl_hook_kernel<<<blocks_for(E), TPB, 0, st>>>(ekey.p, E, d_rank.p, parent.p, changed.p);
      SK_CUDA(launched());
      rounds++;
      SK_CUDA(cudaMemcpyAsync(&h_changed, changed.p, 4, cudaMemcpyDeviceToHost, st));
      SK_CUDA(cudaStreamSynchronize(st));
      if (!h_changed) break;
      cl_jump_kernel<<<blocks_for(n), TPB, 0, st>>>(parent.p, n);
      SK_CUDA(launched());
      if (rounds > n + 1) { ctx->err = "sk_cluster: single linkage did not converge"; return SK_ERR_STATE; }
    }
    cl_component_kernel<<<blocks_for(n), TPB, 0, st>>>(n, off.p, adj, adj_e, erow.p, d_rank.p, order.p, parent.p, d_rep.p, d_edge.p, flag.p);
    SK_CUDA(launched());
  }
  // ---- representatives numbered in rank order
  if (n) {
    size_t tb = 0;
    SK_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tb, flag.p, flag.p, (int)n, st));
    DTmp<uint8_t> tmp;
    SK_TRY(cl_alloc(ctx, tmp, tb, "scan temporaries"));
    SK_CUDA(cub::DeviceScan::InclusiveSum(tmp.p, tb, flag.p, flag.p, (int)n, st));
    SK_CUDA(launched());
    cl_number_kernel<<<blocks_for(n), TPB, 0, st>>>(n, d_rep.p, d_rank.p, flag.p, d_cluster.p);
    SK_CUDA(launched());
    SK_CUDA(cudaMemcpyAsync(rep, d_rep.p, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    SK_CUDA(cudaMemcpyAsync(cluster, d_cluster.p, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    SK_CUDA(cudaMemcpyAsync(edge, d_edge.p, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
  }
  uint32_t n_clusters = 0;
  if (n) SK_CUDA(cudaMemcpyAsync(&n_clusters, flag.p + n - 1, 4, cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaStreamSynchronize(st));
  if (stats) { stats->n_edges = E; stats->n_clusters = n_clusters; stats->rounds = rounds; }
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
  {   // rank must be a permutation of 0 .. n_genomes - 1
    std::vector<uint8_t> seen(n_genomes, 0);
    for (uint32_t g = 0; g < n_genomes; g++) {
      if (rank[g] >= n_genomes || seen[rank[g]]) {
        ctx->err = "sk_cluster: rank is not a permutation of 0.." + std::to_string(n_genomes) + " - 1 (genome " + std::to_string(g) + ")";
        return SK_ERR_PARAM;
      }
      seen[rank[g]] = 1;
    }
  }
  SK_CUDA(cudaSetDevice(ctx->device));
  const auto t0 = std::chrono::steady_clock::now();
  const int rc = cluster_impl(ctx, n_genomes, results, n_results, rank, cp, rep, cluster, edge, stats);
  if (rc == SK_OK && stats) stats->t_device = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return rc;
}
