// chain_core.cuh -- per-item logic of the chaining path as __host__ __device__ functions (see sk_core.cuh for
// why: the same code runs inside the CUDA kernels and inside tests/emu on the host for logic validation).
// Reference: src/chain.rs (bluenote-1577/skani v0.3.0).  All scoring is done in integers: every f64 the reference
// computes in score_anchors / chain_anchors_ani is an integer < 2^32, hence exact (SURVEY App. A.7).
#pragma once
#include <math.h>
#include <stdint.h>

#include "sk_core.cuh"

namespace sk {

constexpr uint32_t FRAGMENT_LENGTH = 20000;   // CHUNK_SIZE_DNA, src/params.rs:40 (fragment_length_formula :125-134)
constexpr uint32_t BP_CHAIN_BAND = 2500;      // src/params.rs:45 ; past_chain_length = min(F/2, 2500) = 2500 (src/chain.rs:842)
constexpr int32_t MAX_GAP = 300;              // D_MAX_GAP_LENGTH src/params.rs:19
constexpr int64_t MAX_LIN = 5000;             // D_MAX_LIN_LENGTH src/params.rs:21
constexpr int32_t ANCHOR_SCORE = 20;          // D_ANCHOR_SCORE_ANI src/params.rs:22
constexpr uint32_t MIN_ANCHORS = 3;           // D_MIN_ANCHORS_ANI src/params.rs:24
constexpr int32_t MIN_SCORE = 45;             // 3 * 20 * 0.75 (src/chain.rs:113)
constexpr uint32_t MIN_LENGTH_COVER = 500;    // src/params.rs:44
constexpr uint32_t REGRESS_CUTOFF = 150000;   // TOTAL_BASES_REGRESS_CUTOFF src/params.rs:53

struct AnchorRec {      // one anchor; the query contig is a property of its chunk
  uint32_t qpos, rpos;
  uint32_t rc;          // ref_contig << 1 | reverse_match
};

// ---- chunk assignment (src/chain.rs:738-836) as two segmented scans over the compact list of hit records ----
// closed form (SURVEY App. A.6): inside one query contig, anchor number x (0-based) with need(x) =
// max(0, ceil((pos - P0)/F) - 1) lands in chunk x + min_{s<=x}(need(s) - s).
struct FirstState {     // segmented "first element of the contig" scan
  uint32_t ctg;
  uint32_t p0;          // query position of the contig's first hit record
  uint32_t a0;          // pair-local anchor index of that record's first anchor
  uint32_t valid;       // 0 = identity
};
// The operators are written with selects instead of early returns: inside the block scans they run in every shuffle step,
// and branches there cost divergence and reconvergence instructions.
struct FirstOp {
  SK_HD FirstState operator()(const FirstState& a, const FirstState& b) const {
    // b wins unless it is the identity or continues a's contig (then the earlier element's values win)
    const bool take_b = b.valid && (!a.valid || a.ctg != b.ctg);
    FirstState r;
    r.ctg = take_b ? b.ctg : a.ctg;
    r.p0 = take_b ? b.p0 : a.p0;
    r.a0 = take_b ? b.a0 : a.a0;
    r.valid = take_b ? b.valid : a.valid;
    return r;
  }
};
struct MinState {       // segmented prefix-min of v = need - (index of the record's last anchor); 16 bytes, no padding
  int64_t v;
  uint32_t ctg;
  uint32_t valid;
};
struct MinOp {
  SK_HD MinState operator()(const MinState& a, const MinState& b) const {
    // b invalid: a; a invalid or another contig: b; same contig: b with the smaller v
    const bool same = a.valid && a.ctg == b.ctg;
    MinState r;
    r.ctg = b.valid ? b.ctg : a.ctg;
    r.valid = a.valid | b.valid;
    r.v = !b.valid ? a.v : (same && a.v < b.v) ? a.v : b.v;
    return r;
  }
};
SK_HD uint32_t chunk_need(uint32_t pos, uint32_t p0) {
  uint32_t d = pos - p0;
  if (d == 0) return 0;
  uint32_t c = (d + FRAGMENT_LENGTH - 1) / FRAGMENT_LENGTH;  // ceil
  return c - 1;
}
// chunk (contig-local) of the anchor with contig-local index al, given the prefix min over earlier records
SK_HD uint32_t chunk_local_of(uint64_t al, bool has_prev, int64_t m_prev, uint32_t need) {
  if (!has_prev) return need;  // first record of the contig: need = 0
  int64_t c = (int64_t)al + m_prev;
  return (uint32_t)(c < (int64_t)need ? c : (int64_t)need);
}
// the hit record's term of the segmented prefix min: need - (contig-local index of its last anchor)
SK_HD int64_t record_min_key(uint32_t need, uint32_t al, uint32_t nh) {
  return (int64_t)need - (int64_t)al - (int64_t)(nh - 1);
}
// Per hit record (al = contig-local index of its first anchor, nh anchors), given the prefix min m_prev over the earlier
// hit records of its contig (has_prev = there are any): clf / cll = chunk_local_of(al / al + nh - 1, ...) are the
// contig-local chunks of its first and last anchor.  The previous hit record's last anchor (index al - 1) sits in chunk
// al - 1 + m_prev: the record's first anchor starts a chunk iff it is the contig's first hit or lands in a later chunk,
// and the record starts that chunk (if any) plus one chunk per step from clf to cll.
SK_HD uint32_t record_starts_chunk(uint32_t al, bool has_prev, int64_t m_prev, uint32_t clf) {
  return (!has_prev || (int64_t)al - 1 + m_prev != (int64_t)clf) ? 1u : 0u;
}
SK_HD uint32_t record_chunk_starts(uint32_t st, uint32_t clf, uint32_t cll) {
  return st + (cll - clf);
}
// Anchor u of a hit record whose first anchor is in contig-local chunk clf: its chunk (chunks only move forward until they
// reach need), and whether it starts a chunk (the first anchor iff the record starts one, a later anchor iff anchor u - 1
// had not yet reached need).
SK_HD uint32_t anchor_chunk_local(uint32_t clf, uint32_t u, uint32_t need) {
  return clf + u < need ? clf + u : need;
}
SK_HD bool anchor_starts_chunk(uint32_t clf, uint32_t u, uint32_t need, bool record_starts) {
  return (u == 0) ? record_starts : clf + u - 1 < need;
}
// window of contig-local chunk cl of a contig whose first hit is at p0: it holds the seeds with lo < pos <= hi.  The pair's
// last chunk is patched afterwards to end at its last anchor (src/chain.rs:796-824).
SK_HD int64_t chunk_window_lo(uint32_t p0, uint32_t cl) {
  return (cl == 0) ? -1ll : (int64_t)p0 + (int64_t)cl * FRAGMENT_LENGTH;
}
SK_HD int64_t chunk_window_hi(uint32_t p0, uint32_t cl) {
  return (int64_t)p0 + (int64_t)(cl + 1) * FRAGMENT_LENGTH;
}

// ---- chain intervals: 5 x u64 keys whose lexicographic order is the derived PartialOrd of ChainInterval
// (score, num_anchors, interval_on_query, interval_on_ref, ref_contig, query_contig, chunk_id, reverse_chain, overlap=0)
// src/types.rs:508-519.  Scores are small non-negative integers so the integer order equals the f64 order.
struct IntervalKey {
  uint64_t k[5];
};
SK_HD IntervalKey make_interval(int32_t score, uint32_t num_anchors, uint32_t q0, uint32_t q1, uint32_t r0, uint32_t r1,
                                uint32_t ref_contig, uint32_t query_contig, uint32_t chunk_id, uint32_t reverse) {
  IntervalKey x;
  x.k[0] = ((uint64_t)(uint32_t)score << 32) | num_anchors;
  x.k[1] = ((uint64_t)q0 << 32) | q1;
  x.k[2] = ((uint64_t)r0 << 32) | r1;
  x.k[3] = ((uint64_t)ref_contig << 32) | query_contig;
  x.k[4] = ((uint64_t)chunk_id << 1) | (reverse & 1u);
  return x;
}
SK_HD uint32_t iv_score(const IntervalKey& x) { return (uint32_t)(x.k[0] >> 32); }
SK_HD uint32_t iv_num_anchors(const IntervalKey& x) { return (uint32_t)x.k[0]; }
SK_HD uint32_t iv_q0(const IntervalKey& x) { return (uint32_t)(x.k[1] >> 32); }
SK_HD uint32_t iv_q1(const IntervalKey& x) { return (uint32_t)x.k[1]; }
SK_HD uint32_t iv_r0(const IntervalKey& x) { return (uint32_t)(x.k[2] >> 32); }
SK_HD uint32_t iv_r1(const IntervalKey& x) { return (uint32_t)x.k[2]; }
SK_HD uint32_t iv_rctg(const IntervalKey& x) { return (uint32_t)(x.k[3] >> 32); }
SK_HD uint32_t iv_qctg(const IntervalKey& x) { return (uint32_t)x.k[3]; }
SK_HD uint32_t iv_chunk(const IntervalKey& x) { return (uint32_t)(x.k[4] >> 1); }
SK_HD uint32_t iv_rev(const IntervalKey& x) { return (uint32_t)(x.k[4] & 1u); }
// true iff x sorts BEFORE y in the descending order of src/chain.rs:1012
SK_HD bool interval_before(const IntervalKey& x, const IntervalKey& y) {
  for (int i = 0; i < 5; i++) {
    if (x.k[i] != y.k[i]) return x.k[i] > y.k[i];
  }
  return false;
}

// greedy non-overlap test pieces (src/chain.rs:1023-1086): contribution of one accepted interval `a` to candidate `c`
SK_HD void overlap_contrib(const IntervalKey& c, const IntervalKey& a, uint32_t* sum_r, uint32_t* hit_r, uint32_t* sum_q,
                           uint32_t* hit_q) {
  if (iv_rctg(a) == iv_rctg(c) && iv_r0(a) < iv_r1(c) && iv_r0(c) < iv_r1(a)) {  // half-open overlap (bio IntervalTree::find)
    uint32_t x = iv_r1(c) - iv_r0(a), y = iv_r1(a) - iv_r0(c);
    *sum_r += x < y ? x : y;
    *hit_r += 1;
  }
  if (iv_qctg(a) == iv_qctg(c) && iv_q0(a) < iv_q1(c) && iv_q0(c) < iv_q1(a)) {
    uint32_t x = iv_q1(c) - iv_q0(a), y = iv_q1(a) - iv_q0(c);
    *sum_q += x < y ? x : y;
    *hit_q += 1;
  }
}
SK_HD bool overlap_accept(const IntervalKey& c, uint32_t sum_r, uint32_t hit_r, uint32_t sum_q, uint32_t hit_q) {
  bool ok_r = (hit_r == 0) || ((float)sum_r < (float)(iv_r1(c) - iv_r0(c)) * 0.5f);  // OVERLAP_ORTHOLOGOUS_FRACTION (:1042)
  bool ok_q = (hit_q == 0) || ((float)sum_q < (float)(iv_q1(c) - iv_q0(c)) * 0.5f);  // (:1072)
  return ok_r && ok_q;
}

// ---- per-chunk identity (src/chain.rs:253-396), given the chunk's accumulated interval statistics ----
struct ChunkAcc {
  uint32_t total_anchors;  // sum num_anchors
  uint32_t rq0, rq1;       // min q0 / max q1
  uint32_t tbcq;           // total_bases_contained_query (wrapping u32)
  uint32_t n_int;
};
// returns false if the chunk yields no estimate; else est / weight
SK_HD bool chunk_estimate(const ChunkAcc& acc, uint32_t c, uint32_t k, uint32_t n_seeds, uint32_t num_in, uint32_t upper_lower,
                          double* est, uint32_t* weight) {
  if (acc.n_int == 0 || acc.total_anchors == 0) return false;        // :253-255
  if (acc.rq1 - acc.rq0 < MIN_LENGTH_COVER) return false;            // :257-259
  uint32_t considered = n_seeds;
  double putative = pow((double)acc.total_anchors / (double)num_in, 1.0 / (double)k);  // :331-335
  if (putative > 0.950 && acc.tbcq > c * 4u && acc.rq1 - acc.rq0 < (FRAGMENT_LENGTH * 9u / 10u) &&
      (double)considered > 1.05 * (double)upper_lower) {             // :336-347
    considered = upper_lower;
  }
  double ml = (double)acc.total_anchors / (double)considered;
  if (ml > 1.0) ml = 1.0;                                            // f64::min(1., x) (:368-372)
  *est = pow(ml, 1.0 / (double)k);                                   // :373-377
  *weight = considered;
  return true;
}

// ---- fastrand 1.9.0 WyRand (SURVEY App. D.4): the state after n draws is seed + n * INC, so draw #n is random access
SK_HD uint64_t wyrand_at(uint64_t seed, uint64_t n_prev_draws) {
  uint64_t s = seed + (n_prev_draws + 1) * 0xA0761D6478BD642Full;
  uint64_t b = s ^ 0xE7037ED1A0B428DBull;
#if defined(__CUDA_ARCH__)
  uint64_t hi = __umul64hi(s, b), lo = s * b;
#else
  __uint128_t t = (__uint128_t)s * b;
  uint64_t hi = (uint64_t)(t >> 64), lo = (uint64_t)t;
#endif
  return lo ^ hi;
}
// Lemire bounded draw without the (astronomically rare) rejection loop; *needs_reject reports when the loop would run
SK_HD uint64_t lemire_below(uint64_t r, uint64_t n, bool* needs_reject) {
#if defined(__CUDA_ARCH__)
  uint64_t hi = __umul64hi(r, n), lo = r * n;
#else
  __uint128_t t = (__uint128_t)r * n;
  uint64_t hi = (uint64_t)(t >> 64), lo = (uint64_t)t;
#endif
  *needs_reject = false;
  if (lo < n) {
    uint64_t thr = (0 - n) % n;
    if (lo < thr) *needs_reject = true;
  }
  return hi;
}

// ---- gbdt 0.1.1 predict (LAD), SURVEY App. D.5; tables from gbdt_tables.inc (complete depth-3 trees, heap order)
SK_HD float gbdt_eval(const unsigned char* feat, const float* thr, const float* leaf, int ntrees, float shrink, float bias,
                      const float x[5]) {
  float v = bias;
  for (int t = 0; t < ntrees; t++) {
    const unsigned char* f = feat + 7 * t;
    const float* th = thr + 7 * t;
    int node = 0;
    for (int d = 0; d < 3; d++) node = 2 * node + ((x[f[node]] < th[node]) ? 1 : 2);
#if defined(__CUDA_ARCH__)
    v = __fadd_rn(v, __fmul_rn(shrink, leaf[8 * t + (node - 7)]));  // f32 multiply then add, never fused
#else
    volatile float prod = shrink * leaf[8 * t + (node - 7)];
    v = v + prod;
#endif
  }
  return v;
}

}  // namespace sk
