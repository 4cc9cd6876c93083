// cluster_core.cuh -- per-vertex logic of sk_cluster (cluster.cu) as __host__ __device__ functions, so that the same code
// runs inside the CUDA kernels and inside tests/emu/emu_cluster.cpp on the host (see sk_core.cuh).
//
// The graph is a symmetric CSR over genome ids: vertex v's neighbours are the low 32 bits of adj[off[v] .. off[v + 1])
// (keys v << 32 | u, ascending), and adj_e[i] indexes the edge's ANI.  rank[v] is the caller's priority (0 = first choice
// as a representative).
//
// Greedy representatives: a vertex is a representative unless it has an edge to an earlier-ranked representative.  The
// state of v depends only on the final states of its earlier-ranked neighbours, so rounds may read live states: a state
// only moves from CL_UNDECIDED to a final value, and a final value is always the sequential loop's value.  Whatever the
// visit order within a round, the result is the one of the sequential loop in rank order.
#pragma once
#include <stdint.h>

#include "sk_core.cuh"

namespace sk {

constexpr uint8_t CL_UNDECIDED = 0, CL_REP = 1, CL_MEMBER = 2;
constexpr float CL_MIN_PRINTED_ANI = 0.1f;   // rows with ani <= 0.1 are never written nor clustered (src/triangle.rs:101)

// is a result row an edge at threshold min_ani?  NaN and the -1 sentinel never are.
SK_HD bool cl_is_edge(float ani, float min_ani) { return ani > CL_MIN_PRINTED_ANI && ani >= min_ani; }

// one greedy step of an undecided vertex v, reading its neighbours' states as they are now
SK_HD uint8_t cl_greedy_decide(uint32_t v, const uint64_t* off, const uint64_t* adj, const uint32_t* rank, const volatile uint8_t* state) {
  const uint32_t rv = rank[v];
  bool all_member = true;
  for (uint64_t i = off[v]; i < off[v + 1]; i++) {
    const uint32_t u = (uint32_t)adj[i];
    if (rank[u] > rv) continue;
    const uint8_t s = state[u];
    if (s == CL_REP) return CL_MEMBER;
    all_member &= s == CL_MEMBER;
  }
  return all_member ? CL_REP : CL_UNDECIDED;
}

// does candidate (ani_a, rank_a) beat (ani_b, rank_b) as a member's representative: higher ANI, then smaller rank
SK_HD bool cl_better(float ani_a, uint32_t rank_a, float ani_b, uint32_t rank_b) {
  return ani_a > ani_b || (ani_a == ani_b && rank_a < rank_b);
}

// the representative neighbour of member v with the highest ANI (ties: smaller rank) and the adjacency index of its edge;
// false when v has no representative neighbour
SK_HD bool cl_assign(uint32_t v, const uint64_t* off, const uint64_t* adj, const uint32_t* adj_e, const float* edge_ani,
                     const uint32_t* rank, const uint8_t* state, uint32_t* rep, uint64_t* at) {
  bool found = false;
  float best_ani = 0.f;
  uint32_t best_rank = 0;
  for (uint64_t i = off[v]; i < off[v + 1]; i++) {
    const uint32_t u = (uint32_t)adj[i];
    if (state[u] != CL_REP) continue;
    const float a = edge_ani[adj_e[i]];
    if (!found || cl_better(a, rank[u], best_ani, best_rank)) { found = true; best_ani = a; best_rank = rank[u]; *rep = u; *at = i; }
  }
  return found;
}

// Single linkage in rank space: parent[r] <= r is a vertex of r's component, and a root is parent[r] == r.
// The root of r after following parents (no writes).
SK_HD uint32_t cl_find(const volatile uint32_t* parent, uint32_t r) {
  uint32_t p = parent[r];
  while (true) {
    const uint32_t q = parent[p];
    if (q == p) return p;
    p = q;
  }
}
// The hook of an edge whose endpoints' current parents are pa and pb: the larger parent is lowered to the smaller one
// (*slot = which parent entry to lower, *val = the value, applied as a min).  False when both parents already agree.
SK_HD bool cl_hook(uint32_t pa, uint32_t pb, uint32_t* slot, uint32_t* val) {
  if (pa == pb) return false;
  *slot = pa > pb ? pa : pb;
  *val = pa < pb ? pa : pb;
  return true;
}

}  // namespace sk
