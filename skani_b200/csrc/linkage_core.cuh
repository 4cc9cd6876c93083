// linkage_core.cuh -- per-cluster logic of sk_cluster_linkage (cluster.cu) as __host__ __device__ functions, so that the same
// code runs inside the CUDA kernels and inside tests/emu/emu_linkage.cpp on the host (see sk_core.cuh).
//
// Average (UPGMA) and complete linkage over the edges of a triangle (rows with ani > 0.1); a pair of genomes without an edge
// has similarity 0.  Every float32 in (0.1, 2) is an integer multiple of 2^-27, so q = ani * 2^27 is an exact integer
// < 2^28 and sums over < 2^30 edges fit a uint64.  Clusters are named by their smallest member rank (the id).  The pair
// list holds both directions (A << 32 | B) of every cluster pair with at least one edge and an LkVal:
//   s    = the sum of q over the edges between A and B (average linkage),
//   cnt  = the number of those edges, minq = their smallest q (complete linkage).
// The value of a pair is the rational s' / p': average s / (|A| |B|); complete minq / 1 when cnt == |A| |B| (every member
// pair is an edge), otherwise 0 / 1.  Values are compared exactly by cross-multiplying in 128 bits.  A cluster's best
// partner has the largest value, ties to the smaller partner id: a strict total order, so a fold over a segment gives the
// same partner in any visit order.
// Rounds: every active cluster finds its best partner; pairs that are each other's best partner and qualify (value >= the
// cut q(min_ani), or value > 0 when the whole dendrogram is wanted) merge into the smaller id; a cluster whose best partner
// does not qualify can never merge again (a merged pair's value lies between, or for complete linkage at most, its parts'
// values) and is deactivated with its pairs.  Merged pairs combine by s sum / cnt sum / minq min: integer and associative,
// so nothing depends on thread timing.  For inputs without ties this gives exactly the merges of sequential HAC.
#pragma once
#include <stdint.h>

#include "sk_core.cuh"

namespace sk {

constexpr int LK_AVERAGE = 0, LK_COMPLETE = 1;
constexpr uint32_t LK_NONE = 0xFFFFFFFFu;   // best[]: no qualifying partner; lab[]: a deactivated cluster
constexpr float LK_MAX_ANI = 2.f;           // q = ani * 2^27 is exact below 2 (and < 2^28)

struct LkVal {
  uint64_t s;
  uint32_t cnt, minq;
};

// q of an edge's ANI (exact for 0.1 < ani < 2)
SK_HD uint32_t lk_q(float ani) { return (uint32_t)((double)ani * 134217728.0); }

SK_HD LkVal lk_combine(const LkVal& a, const LkVal& b) { return {a.s + b.s, a.cnt + b.cnt, a.minq < b.minq ? a.minq : b.minq}; }

// 128-bit product x * y as (hi, lo)
SK_HD void lk_mul128(uint64_t x, uint64_t y, uint64_t* hi, uint64_t* lo) {
#ifdef __CUDA_ARCH__
  *hi = __umul64hi(x, y);
  *lo = x * y;
#else
  const unsigned __int128 m = (unsigned __int128)x * y;
  *hi = (uint64_t)(m >> 64);
  *lo = (uint64_t)m;
#endif
}

// s1 / p1 < s2 / p2 (p > 0), exactly
SK_HD bool lk_less(uint64_t s1, uint64_t p1, uint64_t s2, uint64_t p2) {
  uint64_t h1, l1, h2, l2;
  lk_mul128(s1, p2, &h1, &l1);
  lk_mul128(s2, p1, &h2, &l2);
  return h1 < h2 || (h1 == h2 && l1 < l2);
}

// the value of a pair between clusters of sizes na and nb, as the rational *s / *p
SK_HD void lk_value(int method, const LkVal& v, uint64_t na, uint64_t nb, uint64_t* s, uint64_t* p) {
  const uint64_t pairs = na * nb;
  if (method == LK_AVERAGE) { *s = v.s; *p = pairs; }
  else { *s = v.cnt == pairs ? v.minq : 0; *p = 1; }
}

// does partner (s1 / p1, id1) beat (s2 / p2, id2): larger value, ties to the smaller id
SK_HD bool lk_better(uint64_t s1, uint64_t p1, uint32_t id1, uint64_t s2, uint64_t p2, uint32_t id2) {
  if (lk_less(s2, p2, s1, p1)) return true;
  if (lk_less(s1, p1, s2, p2)) return false;
  return id1 < id2;
}

// may a pair of value s / p merge: at or above the cut qcut / 1, or in dendrogram mode any value above 0
SK_HD bool lk_qualifies(uint64_t s, uint64_t p, uint32_t qcut, bool dendrogram) {
  return dendrogram ? s > 0 : !lk_less(s, p, qcut, 1);
}

// can a pair be dropped from the list for good: a complete-linkage pair that does not qualify never will (its value only
// falls when either side grows, to 0 once it is partial); average-linkage pairs still feed later averages
SK_HD bool lk_droppable(int method, uint64_t s, uint64_t p, uint32_t qcut, bool dendrogram) {
  return method == LK_COMPLETE && !lk_qualifies(s, p, qcut, dendrogram);
}

// a cluster's decision once every best partner of the round is known (best[x] = LK_NONE: x has no qualifying partner)
constexpr int LK_KEEP = 0, LK_DEACTIVATE = 1, LK_MERGE_LOW = 2, LK_MERGE_HIGH = 3;
SK_HD int lk_decide(uint32_t a, const uint32_t* best) {
  const uint32_t b = best[a];
  if (b == LK_NONE) return LK_DEACTIVATE;
  if (best[b] != a) return LK_KEEP;
  return a < b ? LK_MERGE_LOW : LK_MERGE_HIGH;   // the smaller id keeps its name; the larger one is relabelled to it
}

// one merge of a dendrogram: clusters a < b (ids) joined in `round` at value s / p into a cluster of `size` genomes
struct LkMerge {
  uint64_t s, p;
  uint32_t round, a, b, size;
};

// dendrogram order: value descending, then round, then id.  Heights are monotone, so children come before parents.
struct LkMergeOrder {
  SK_HD bool operator()(const LkMerge& x, const LkMerge& y) const {
    if (lk_less(y.s, y.p, x.s, x.p)) return true;
    if (lk_less(x.s, x.p, y.s, y.p)) return false;
    return x.round != y.round ? x.round < y.round : x.a < y.a;
  }
};

// scipy height 1 - value, rounded to nearest
SK_HD double lk_height(const LkMerge& m) { return 1.0 - (double)m.s / ((double)m.p * 134217728.0); }

}  // namespace sk
