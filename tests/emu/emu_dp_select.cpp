// Host emulation of the chain back end's banded DP (dp_group_kernel<GL, NE, FULLBAND> and dp_warp_kernel<NB> in
// skani_b200/csrc/chain.cu) and of select_kernel's two greedy passes, in the kernels' own arrangement, checked against the
// oracle (chain_chunks, get_nonoverlapping_chains, chunk_stats, chain_len_sums) on the constructed lists of
// tests/dp_select_cases.py.  Development/test harness only, not a product path.
//
// DP, per instantiation: lanes own anchors i = GL * block + lane, register set s holds block (current - s); the group kernel
// evaluates the candidate of set s at distance d = m - gl + GL * s for s = 1 .. NE - 1 and ONE edge candidate from set 0
// (gl < m) or set NE, keeps the lane's best as the key (score - 1) << 5 | (31 - d), takes the group maximum and decodes it to
// (score, j); unfilled sets carry the contig sentinel 0xFFFFFFFC, slots past the chunk end 0xFFFFFFFE, and reverse-strand ref
// positions are held negated.  The warp kernel picks set t or t + 1 by lo_set = lane < m and lets j = i - d wrap.  Chunks of
// a group-kernel warp share the longest chunk's loop (chunks sorted by size as the radix sort leaves them).  Root and depth
// propagate through the winner; the chain end of a root is the atomicMax of score << 32 | index.
// Selection: sort into the descending derived order, then
//   shared-memory path: dependency lists of the first SEL_DEPS earlier candidates overlapping on either axis, the kept flags
//     of those, a full scan of the accepted list past SEL_DEPS, the inline sum / 0.5f test of select_kernel (line for line);
//   global path: the 16 kb-cell occupancy bitmaps with sel_cell_hash, consulted for spans of at most 32 cells, then
//     overlap_contrib / overlap_accept over the accepted list.
// Both run on every list; kept flags, the per-axis hit counts (kept intervals overlapping the candidate: the reference's
// IntervalTree::find counts), the per-chunk sums and the pair's chain length sums are compared with the oracle.
//
// Input (stdin, whitespace separated):  D GL NE FULLBAND NB band c n_chunks { n { qctg qpos rctg rpos rev } }   (GL = 0: warp)
//                                       S name n_chunks n { score num_anchors q0 q1 r0 r1 rctg qctg chunk rev }
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../skani_b200/csrc/chain_core.cuh"
#include "../../oracle/skani_oracle.hpp"

using namespace sk;

// select_kernel's constants (chain.cu); the test compares them with the kernel source
constexpr uint32_t SEL_DEPS = 4;
constexpr uint32_t SEL_SMEM_MAX = 1024;
constexpr uint32_t SEL_CELL_SHIFT = 14;
constexpr uint32_t SEL_MAP_BITS = 4096;
static uint32_t sel_cell_hash(uint32_t ctg, uint32_t cell) { return (cell + ctg * 0x9E37u) & (SEL_MAP_BITS - 1); }

static int failures = 0;
static std::string g_tag;
#define FAIL(...) do { failures++; if (failures <= 20) { fprintf(stdout, "FAIL %s: ", g_tag.c_str()); fprintf(stdout, __VA_ARGS__); fprintf(stdout, "\n"); } } while (0)

static long n_dp_configs, n_chunks_all, n_anchors_all, n_iv_all, n_lists, n_dep_path, n_scan_path, n_bitmap_skip, n_bitmap_scan,
    n_wide_forced, n_edge_cand_wins, n_sentinel_rejects;

struct Chunk { uint32_t qctg; std::vector<AnchorRec> a; };

// ---- the per-candidate tests the two DP kernels share -------------------------------------------------------------------
static bool in_band(uint32_t d, uint32_t band) { return d <= band; }
static bool dq_ok(uint32_t dq) { return dq - 1u < BP_CHAIN_BAND; }
static bool dr_ok(uint32_t dr) { return dr - 1u < (uint32_t)MAX_LIN; }
static bool gap_ok(uint32_t g) { return g + (uint32_t)MAX_GAP <= 2u * (uint32_t)MAX_GAP; }

struct DpOut { std::vector<int32_t> score; std::vector<uint32_t> ptr, depth; std::vector<unsigned long long> key; };

static void atomic_max(unsigned long long& x, unsigned long long v) { if (v > x) x = v; }

// dp_group_kernel<GL, NE, FULLBAND>: one warp = 32 / GL chunks (indices into `cs`), nmax = the longest of them
static void dp_group_warp(const std::vector<const Chunk*>& cs, int GL, int NE, bool FULLBAND, uint32_t band, std::vector<DpOut*>& outs) {
  const int NB = NE + 1, LG = GL == 8 ? 3 : 2;
  uint32_t nmax = 0;
  for (auto* c : cs) nmax = std::max<uint32_t>(nmax, (uint32_t)c->a.size());
  for (size_t w = 0; w < cs.size(); w++) {
    const Chunk& C = *cs[w];
    DpOut& O = *outs[w];
    const uint32_t n = (uint32_t)C.a.size();
    O.score.assign(n, 0); O.ptr.assign(n, 0); O.depth.assign(n, 0); O.key.assign(n, 0);
    // registers per lane and set
    std::vector<std::vector<uint32_t>> q(GL, std::vector<uint32_t>(NB, 0)), r = q, rc = q, rt = q, dp = q;
    std::vector<std::vector<int32_t>> sc(GL, std::vector<int32_t>(NB, 0));
    std::vector<uint32_t> my_ptr(GL, 0);
    for (int l = 0; l < GL; l++) for (int s = 0; s < NB; s++) rc[l][s] = 0xFFFFFFFCu;
    for (uint32_t b0 = 0; b0 < nmax; b0 += GL) {
      for (int l = 0; l < GL; l++) {
        for (int s = NB - 1; s > 0; s--) { q[l][s] = q[l][s - 1]; r[l][s] = r[l][s - 1]; rc[l][s] = rc[l][s - 1]; rt[l][s] = rt[l][s - 1]; dp[l][s] = dp[l][s - 1]; sc[l][s] = sc[l][s - 1]; }
        const uint32_t idx = b0 + l;
        AnchorRec x; x.qpos = 0; x.rpos = 0; x.rc = 0xFFFFFFFEu;
        if (idx < n) { x = C.a[idx]; O.key[idx] = idx; }
        q[l][0] = x.qpos; r[l][0] = (x.rc & 1u) ? (0u - x.rpos) : x.rpos; rc[l][0] = x.rc; sc[l][0] = 0; rt[l][0] = idx; dp[l][0] = 1;
        my_ptr[l] = idx;
      }
      for (uint32_t m = 0; m < (uint32_t)GL; m++) {
        const uint32_t i = b0 + m;
        const uint32_t cq = q[m][0], cr = r[m][0], crc = rc[m][0];
        int32_t kmax = 0;
        int edge_lane_best = -1;
        for (int gl = 0; gl < GL; gl++) {
          int32_t best = 0;
          bool best_edge = false;
          auto eval = [&](uint32_t qs, uint32_t rs, uint32_t rcs, int32_t scs, uint32_t d, bool edge) {
            const uint32_t dq = cq - qs;
            const uint32_t dr = cr - rs;
            const uint32_t g = dr - dq;
            const bool ok = (FULLBAND || in_band(d, band)) & (rcs == crc) & dq_ok(dq) & dr_ok(dr) & gap_ok(g);
            if (rcs != crc && (rcs == 0xFFFFFFFCu || rcs == 0xFFFFFFFEu)) n_sentinel_rejects++;
            const int32_t gi = (int32_t)g;
            const int32_t nsm1 = scs + (ANCHOR_SCORE - 1) - (gi < 0 ? -gi : gi);
            const int32_t key = (int32_t)(((uint32_t)nsm1 << 5) | (31u - d));
            const int32_t v = ok ? key : 0;
            if (v > best) { best = v; best_edge = edge; }
          };
          for (int s2 = 1; s2 < NE; s2++) eval(q[gl][s2], r[gl][s2], rc[gl][s2], sc[gl][s2], m + (uint32_t)(GL * s2) - gl, false);
          const bool lo_set = (uint32_t)gl < m;
          const int se = lo_set ? 0 : NE;
          eval(q[gl][se], r[gl][se], rc[gl][se], sc[gl][se], m - gl + (lo_set ? 0u : (uint32_t)(GL * NE)), true);
          if (best > kmax) { kmax = best; edge_lane_best = best_edge ? gl : -1; }
        }
        const bool has = kmax > 0;
        if (has && edge_lane_best >= 0) n_edge_cand_wins++;
        const int32_t smax = (kmax >> 5) + 1;
        const uint32_t dwin = 31u - ((uint32_t)kmax & 31u);
        const uint32_t jw = i - dwin;
        const int sidx = (int)(b0 >> LG) - (int)(jw >> LG);
        const uint32_t wl = jw & (uint32_t)(GL - 1);
        uint32_t rsel = rt[wl][0], dsel = dp[wl][0];
        for (int s = 1; s < NB; s++) if (sidx == s) { rsel = rt[wl][s]; dsel = dp[wl][s]; }
        if (has) { sc[m][0] = smax; rt[m][0] = rsel; dp[m][0] = dsel + 1; my_ptr[m] = jw; }
      }
      for (int l = 0; l < GL; l++) {
        const uint32_t idx = b0 + l;
        if (idx < n) {
          O.depth[idx] = dp[l][0];
          if (rt[l][0] >= n) { FAIL("anchor %u, field root: %u is outside the chunk of %u", idx, rt[l][0], n); continue; }
          if (rt[l][0] != idx) atomic_max(O.key[rt[l][0]], ((unsigned long long)(uint32_t)sc[l][0] << 32) | idx);
          O.score[idx] = sc[l][0]; O.ptr[idx] = my_ptr[l];
        }
      }
    }
  }
}

// dp_warp_kernel<NB>: one chunk per warp
static void dp_warp(const Chunk& C, int NB, uint32_t band, DpOut& O) {
  const uint32_t n = (uint32_t)C.a.size();
  O.score.assign(n, 0); O.ptr.assign(n, 0); O.depth.assign(n, 0); O.key.assign(n, 0);
  std::vector<std::vector<uint32_t>> q(32, std::vector<uint32_t>(NB, 0)), r = q, rc = q, rt = q, dp = q;
  std::vector<std::vector<int32_t>> sc(32, std::vector<int32_t>(NB, 0));
  std::vector<uint32_t> my_ptr(32, 0);
  for (uint32_t b0 = 0; b0 < n; b0 += 32) {
    for (int l = 0; l < 32; l++) {
      for (int s = NB - 1; s > 0; s--) { q[l][s] = q[l][s - 1]; r[l][s] = r[l][s - 1]; rc[l][s] = rc[l][s - 1]; rt[l][s] = rt[l][s - 1]; dp[l][s] = dp[l][s - 1]; sc[l][s] = sc[l][s - 1]; }
      const uint32_t idx = b0 + l;
      AnchorRec x; x.qpos = 0; x.rpos = 0; x.rc = 0;
      if (idx < n) { x = C.a[idx]; O.key[idx] = idx; }
      q[l][0] = x.qpos; r[l][0] = x.rpos; rc[l][0] = x.rc; sc[l][0] = 0; rt[l][0] = idx; dp[l][0] = 1;
      my_ptr[l] = idx;
    }
    const uint32_t mend = std::min(32u, n - b0);
    for (uint32_t m = 0; m < mend; m++) {
      const uint32_t i = b0 + m;
      const uint32_t cq = q[m][0], cr = r[m][0], crc = rc[m][0];
      std::vector<int32_t> best_ns(32, 0);
      std::vector<uint32_t> best_j1(32, 0);
      for (uint32_t lane = 0; lane < 32; lane++) {
        const bool lo_set = lane < m;
        for (int t = 0; t < NB - 1; t++) {
          const int s = lo_set ? t : t + 1;
          const uint32_t d = m + 32u * (uint32_t)t + (lo_set ? 0u : 32u) - lane;
          const uint32_t j = i - d;
          const uint32_t dq = cq - q[lane][s];
          const uint32_t tr = cr - r[lane][s];
          const uint32_t dr = (crc & 1u) ? (0u - tr) : tr;
          const uint32_t g = dr - dq;
          const bool ok = in_band(d, band) & (d <= i) & (rc[lane][s] == crc) & dq_ok(dq) & dr_ok(dr) & gap_ok(g);
          const int32_t gi = (int32_t)g;
          const int32_t ns = sc[lane][s] + ANCHOR_SCORE - (gi < 0 ? -gi : gi);
          if (ok && ns > best_ns[lane]) { best_ns[lane] = ns; best_j1[lane] = j + 1; }
        }
      }
      int32_t smax = 0;
      for (int l = 0; l < 32; l++) smax = std::max(smax, best_ns[l]);
      if (smax > 0) {
        uint32_t jm = 0;
        for (int l = 0; l < 32; l++) jm = std::max(jm, best_ns[l] == smax ? best_j1[l] : 0u);
        const uint32_t jw = jm - 1;
        const int sidx = (int)(b0 >> 5) - (int)(jw >> 5);
        const uint32_t wl = jw & 31u;
        uint32_t rsel = rt[wl][0], dsel = dp[wl][0];
        for (int s = 1; s < NB; s++) if (sidx == s) { rsel = rt[wl][s]; dsel = dp[wl][s]; }
        sc[m][0] = smax; rt[m][0] = rsel; dp[m][0] = dsel + 1; my_ptr[m] = jw;
      }
    }
    for (int l = 0; l < 32; l++) {
      const uint32_t idx = b0 + l;
      if (idx < n) {
        O.depth[idx] = dp[l][0];
        if (rt[l][0] >= n) { FAIL("anchor %u, field root: %u is outside the chunk of %u", idx, rt[l][0], n); continue; }
        if (rt[l][0] != idx) atomic_max(O.key[rt[l][0]], ((unsigned long long)(uint32_t)sc[l][0] << 32) | idx);
        O.score[idx] = sc[l][0]; O.ptr[idx] = my_ptr[l];
      }
    }
  }
}

// the kernels' interval emission (one per surviving root)
static void emit_intervals(const Chunk& C, const DpOut& O, uint32_t chunk_id, std::vector<IntervalKey>& iv) {
  const uint32_t n = (uint32_t)C.a.size();
  for (uint32_t i = 0; i < n; i++) {
    if (O.depth[i] != 1) continue;
    const unsigned long long key = O.key[i];
    const uint32_t b = (uint32_t)key, score = (uint32_t)(key >> 32);
    if (b == i || b >= n) continue;
    const uint32_t num_anchors = O.depth[b];
    if (num_anchors < MIN_ANCHORS || (int32_t)score < MIN_SCORE) continue;
    const AnchorRec f = C.a[i], l = C.a[b];
    const uint32_t r0 = f.rpos < l.rpos ? f.rpos : l.rpos, r1 = f.rpos < l.rpos ? l.rpos : f.rpos;
    iv.push_back(make_interval((int32_t)score, num_anchors, f.qpos, l.qpos, r0, r1, f.rc >> 1, C.qctg, chunk_id, f.rc & 1u));
  }
}

// ---- selection ------------------------------------------------------------------------------------------------------------
struct SelOut { std::vector<uint8_t> kept; std::vector<uint32_t> hits; std::vector<bool> dep_path; std::vector<uint32_t> cnt; };
struct AccRec { uint32_t q0, q1, r0, r1, qctg, rctg; };

// select_kernel's shared-memory path on the sorted candidates (line for line; hits counted alongside the sums)
static SelOut select_smem(const std::vector<IntervalKey>& s) {
  const uint32_t n = (uint32_t)s.size();
  SelOut o; o.kept.assign(n, 0); o.hits.assign(2 * n, 0); o.dep_path.assign(n, false); o.cnt.assign(n, 0);
  std::vector<AccRec> s_cand(n);
  for (uint32_t i = 0; i < n; i++) {
    const IntervalKey& c = s[i];
    AccRec x; x.q0 = iv_q0(c); x.q1 = iv_q1(c); x.r0 = iv_r0(c); x.r1 = iv_r1(c); x.qctg = iv_qctg(c); x.rctg = iv_rctg(c);
    s_cand[i] = x;
  }
  std::vector<uint16_t> s_dep((size_t)n * SEL_DEPS);
  std::vector<uint32_t> s_cnt(n);
  for (uint32_t i = 0; i < n; i++) {
    const AccRec c = s_cand[i];
    uint32_t cnt = 0;
    for (uint32_t j = 0; j < i; j++) {
      const AccRec x = s_cand[j];
      const bool ov = (x.rctg == c.rctg && x.r0 < c.r1 && c.r0 < x.r1) || (x.qctg == c.qctg && x.q0 < c.q1 && c.q0 < x.q1);
      if (ov) { if (cnt < SEL_DEPS) s_dep[i * SEL_DEPS + cnt] = (uint16_t)j; cnt++; }
    }
    s_cnt[i] = std::min(cnt, 0xFFFFu);
  }
  std::vector<uint32_t> s_accpos;
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t cnt = s_cnt[i];
    o.cnt[i] = cnt;
    bool ok = true;
    if (cnt != 0) {
      const AccRec c = s_cand[i];
      uint32_t sum_r = 0, sum_q = 0, hit_r = 0, hit_q = 0;
      if (cnt <= SEL_DEPS) {
        o.dep_path[i] = true;
        for (uint32_t lane = 0; lane < cnt; lane++) {
          const uint32_t j = s_dep[i * SEL_DEPS + lane];
          if (o.kept[j]) {
            const AccRec x = s_cand[j];
            if (x.rctg == c.rctg && x.r0 < c.r1 && c.r0 < x.r1) { const uint32_t u = c.r1 - x.r0, v = x.r1 - c.r0; sum_r += u < v ? u : v; hit_r++; }
            if (x.qctg == c.qctg && x.q0 < c.q1 && c.q0 < x.q1) { const uint32_t u = c.q1 - x.q0, v = x.q1 - c.q0; sum_q += u < v ? u : v; hit_q++; }
          }
        }
      } else {
        for (uint32_t a = 0; a < s_accpos.size(); a++) {
          const AccRec x = s_cand[s_accpos[a]];
          if (x.rctg == c.rctg && x.r0 < c.r1 && c.r0 < x.r1) { const uint32_t u = c.r1 - x.r0, v = x.r1 - c.r0; sum_r += u < v ? u : v; hit_r++; }
          if (x.qctg == c.qctg && x.q0 < c.q1 && c.q0 < x.q1) { const uint32_t u = c.q1 - x.q0, v = x.q1 - c.q0; sum_q += u < v ? u : v; hit_q++; }
        }
      }
      const bool ok_r = (sum_r == 0) || ((float)sum_r < (float)(c.r1 - c.r0) * 0.5f);
      const bool ok_q = (sum_q == 0) || ((float)sum_q < (float)(c.q1 - c.q0) * 0.5f);
      ok = ok_r && ok_q;
      o.hits[2 * i] = hit_r; o.hits[2 * i + 1] = hit_q;
    }
    o.kept[i] = ok ? 1 : 0;
    if (ok) s_accpos.push_back(i);
  }
  return o;
}

// select_kernel's global-memory path (bitmap pre-check, then chain_core.cuh's overlap_contrib / overlap_accept)
static SelOut select_global(const std::vector<IntervalKey>& s) {
  const uint32_t n = (uint32_t)s.size();
  SelOut o; o.kept.assign(n, 0); o.hits.assign(2 * n, 0); o.dep_path.assign(n, false); o.cnt.assign(n, 0);
  std::vector<uint32_t> s_qmap(SEL_MAP_BITS / 32, 0), s_rmap(SEL_MAP_BITS / 32, 0), acc;
  for (uint32_t i = 0; i < n; i++) {
    const IntervalKey c = s[i];
    const uint32_t q0 = iv_q0(c), q1 = iv_q1(c), r0 = iv_r0(c), r1 = iv_r1(c), qc = iv_qctg(c), rcg = iv_rctg(c);
    const uint32_t cq0 = q0 >> SEL_CELL_SHIFT, ncq = ((q1 - 1) >> SEL_CELL_SHIFT) - cq0 + 1;
    const uint32_t cr0 = r0 >> SEL_CELL_SHIFT, ncr = ((r1 - 1) >> SEL_CELL_SHIFT) - cr0 + 1;
    bool need_scan = true;
    if (ncq <= 32 && ncr <= 32) {
      bool occ = false;
      for (uint32_t lane = 0; lane < 32; lane++) {
        if (lane < ncq) { uint32_t h = sel_cell_hash(qc, cq0 + lane); occ |= (s_qmap[h >> 5] >> (h & 31)) & 1u; }
        if (lane < ncr) { uint32_t h = sel_cell_hash(rcg, cr0 + lane); occ |= (s_rmap[h >> 5] >> (h & 31)) & 1u; }
      }
      need_scan = occ;
      if (occ) n_bitmap_scan++; else n_bitmap_skip++;
    } else if (!acc.empty()) {
      n_wide_forced++;
    }
    bool ok = true;
    if (need_scan) {
      uint32_t sum_r = 0, hit_r = 0, sum_q = 0, hit_q = 0;
      for (uint32_t a : acc) overlap_contrib(c, s[a], &sum_r, &hit_r, &sum_q, &hit_q);
      ok = overlap_accept(c, sum_r, hit_r, sum_q, hit_q);
      o.hits[2 * i] = hit_r; o.hits[2 * i + 1] = hit_q;
    }
    o.dep_path[i] = need_scan;   // here: the candidate was scanned
    if (ok) {
      acc.push_back(i);
      for (uint32_t t = 0; t < ncq; t++) { uint32_t h = sel_cell_hash(qc, cq0 + t); s_qmap[h >> 5] |= 1u << (h & 31); }
      for (uint32_t t = 0; t < ncr; t++) { uint32_t h = sel_cell_hash(rcg, cr0 + t); s_rmap[h >> 5] |= 1u << (h & 31); }
    }
    o.kept[i] = ok ? 1 : 0;
  }
  return o;
}

static orc::ChainInterval to_orc(const IntervalKey& x) {
  orc::ChainInterval v;
  v.score = iv_score(x); v.num_anchors = iv_num_anchors(x); v.q0 = iv_q0(x); v.q1 = iv_q1(x); v.r0 = iv_r0(x); v.r1 = iv_r1(x);
  v.ref_contig = iv_rctg(x); v.query_contig = iv_qctg(x); v.chunk_id = iv_chunk(x); v.reverse_chain = iv_rev(x); v.overlap = 0;
  return v;
}
static const char* IVF[] = {"score", "num_anchors", "q0", "q1", "r0", "r1", "ref_contig", "query_contig", "chunk", "reverse"};
static int64_t ivf(const orc::ChainInterval& v, int f) {
  switch (f) {
    case 0: return (int64_t)v.score; case 1: return (int64_t)v.num_anchors; case 2: return v.q0; case 3: return v.q1;
    case 4: return v.r0; case 5: return v.r1; case 6: return (int64_t)v.ref_contig; case 7: return (int64_t)v.query_contig;
    case 8: return (int64_t)v.chunk_id; default: return v.reverse_chain;
  }
}

// both selection paths on the emulated list `iv` against the oracle's selection of `expect` (the same intervals)
static void check_selection(std::vector<IntervalKey> iv, std::vector<orc::ChainInterval> expect, uint32_t n_chunks, uint32_t c,
                            uint32_t k, bool switched, const std::string& name) {
  n_lists++;
  std::sort(iv.begin(), iv.end(), [](const IntervalKey& a, const IntervalKey& b) { return interval_before(a, b); });
  std::vector<uint8_t> okept;
  std::vector<uint32_t> ohits;
  auto per_chunk = orc::get_nonoverlapping_chains(expect, n_chunks, &okept, &ohits);
  if (expect.size() != iv.size()) { FAIL("%s: %zu intervals emulated, %zu in the oracle", name.c_str(), iv.size(), expect.size()); return; }
  for (size_t i = 0; i < iv.size(); i++) {
    const orc::ChainInterval e = to_orc(iv[i]);
    for (int f = 0; f < 10; f++)
      if (ivf(e, f) != ivf(expect[i], f)) { FAIL("%s: interval %zu, field %s: emulated %lld, oracle %lld", name.c_str(), i, IVF[f], (long long)ivf(e, f), (long long)ivf(expect[i], f)); return; }
  }
  const SelOut paths[2] = {select_smem(iv), select_global(iv)};
  const char* pname[2] = {"shared-memory path", "global path"};
  for (int p = 0; p < 2; p++) {
    const SelOut& o = paths[p];
    for (size_t i = 0; i < iv.size(); i++) {
      if (o.kept[i] != okept[i]) { FAIL("%s, %s: interval %zu, field kept: emulated %d, oracle %d", name.c_str(), pname[p], i, o.kept[i], okept[i]); return; }
      // the shared-memory path sees every kept overlap; the global path only when the bitmap sends it to the scan, and a
      // skipped candidate must have no kept overlap at all
      const bool seen = p == 0 ? o.cnt[i] != 0 : o.dep_path[i];
      for (int ax = 0; ax < 2; ax++) {
        const uint32_t h = seen ? o.hits[2 * i + ax] : 0u;
        if (h != ohits[2 * i + ax]) { FAIL("%s, %s: interval %zu, field %s: emulated %u, oracle %u", name.c_str(), pname[p], i, ax ? "hits_query" : "hits_ref", h, ohits[2 * i + ax]); return; }
      }
    }
  }
  const SelOut& o = paths[0];
  for (size_t i = 0; i < iv.size(); i++) { if (o.cnt[i] && o.dep_path[i]) n_dep_path++; else if (o.cnt[i]) n_scan_path++; }
  // the dependency-list edge: the lowest-scoring candidate of deps_4 / deps_kept_4 has exactly 4 earlier overlapping
  // candidates and takes the list, that of the _5 cases has 5 and takes the full scan
  if (name.rfind("deps_", 0) == 0) {
    size_t last = 0;
    for (size_t i = 0; i < iv.size(); i++) if (iv_score(iv[i]) == 10) last = i;
    const uint32_t want = name.find("_4") != std::string::npos ? 4u : 5u;
    if (o.cnt[last] != want || o.dep_path[last] != (want == 4)) FAIL("%s: the last candidate has %u earlier overlaps and took the %s (SEL_DEPS = %u)", name.c_str(), o.cnt[last], o.dep_path[last] ? "dependency list" : "full scan", SEL_DEPS);
  }
  // per-chunk sums and the pair's chain length sums, as select_kernel accumulates them, from the shared-memory decisions
  std::vector<ChunkAcc> acc(n_chunks);
  for (auto& a : acc) { a.total_anchors = 0; a.rq0 = 0xFFFFFFFFu; a.rq1 = 0; a.tbcq = 0; a.n_int = 0; }
  uint32_t sumlen = 0, nch = 0;
  for (size_t i = 0; i < iv.size(); i++) {
    if (!o.kept[i]) continue;
    const IntervalKey& x = iv[i];
    ChunkAcc& a = acc[iv_chunk(x)];
    a.total_anchors += iv_num_anchors(x); a.rq0 = std::min(a.rq0, iv_q0(x)); a.rq1 = std::max(a.rq1, iv_q1(x));
    a.tbcq += (switched ? (iv_r1(x) - iv_r0(x)) : (iv_q1(x) - iv_q0(x))) + k + 2 * c;
    a.n_int++;
    sumlen += (iv_q1(x) - iv_q0(x)) + 2 * c + k; nch++;
  }
  for (uint32_t ch = 0; ch < n_chunks; ch++) {
    const orc::ChunkStats s = orc::chunk_stats(per_chunk[ch], {}, c, k, orc::MIN_LENGTH_COVER, switched);
    const uint32_t e[5] = {acc[ch].total_anchors, acc[ch].rq0, acc[ch].rq1, acc[ch].tbcq, acc[ch].n_int};
    const uint32_t x[5] = {(uint32_t)s.total_anchors, s.rq0, s.rq1, s.tbcq, s.n_int};
    const char* nm[5] = {"total_anchors", "rq0", "rq1", "tbcq", "n_int"};
    for (int f = 0; f < 5; f++) if (e[f] != x[f]) { FAIL("%s: chunk %u, field %s: emulated %u, oracle %u", name.c_str(), ch, nm[f], e[f], x[f]); return; }
  }
  uint32_t osum, on;
  orc::chain_len_sums(per_chunk, c, k, &osum, &on);
  if (sumlen != osum || nch != on) FAIL("%s: pair_sumlen / pair_nchains: emulated %u / %u, oracle %u / %u", name.c_str(), sumlen, nch, osum, on);
}

static orc::MapParams map_params(uint32_t c, uint32_t k) {
  orc::Sketch unit;
  unit.c = c; unit.k = k;
  return orc::map_params_from_sketch(unit, orc::CommandParams(), -1);
}

static void run_dp(int GL, int NE, bool FULLBAND, int NB, uint32_t band, uint32_t c, const std::vector<Chunk>& chunks) {
  n_dp_configs++;
  char tag[128];
  if (GL) snprintf(tag, sizeof(tag), "dp_group_kernel<GL=%d, NE=%d, FULLBAND=%d> band %u", GL, NE, (int)FULLBAND, band);
  else snprintf(tag, sizeof(tag), "dp_warp_kernel<NB=%d> band %u", NB, band);
  g_tag = tag;
  const uint32_t k = 15;
  std::vector<DpOut> outs(chunks.size());
  if (GL) {
    // the radix sort by descending size is stable: equal sizes keep their chunk order
    std::vector<uint32_t> perm(chunks.size());
    for (uint32_t i = 0; i < perm.size(); i++) perm[i] = i;
    std::stable_sort(perm.begin(), perm.end(), [&](uint32_t a, uint32_t b) { return chunks[a].a.size() > chunks[b].a.size(); });
    const size_t GW = 32 / GL;
    for (size_t w0 = 0; w0 < perm.size(); w0 += GW) {
      std::vector<const Chunk*> cs;
      std::vector<DpOut*> os;
      for (size_t t = w0; t < std::min(perm.size(), w0 + GW); t++) { cs.push_back(&chunks[perm[t]]); os.push_back(&outs[perm[t]]); }
      dp_group_warp(cs, GL, NE, FULLBAND, band, os);
    }
  } else {
    for (size_t i = 0; i < chunks.size(); i++) dp_warp(chunks[i], NB, band, outs[i]);
  }
  // oracle
  std::vector<std::vector<orc::Anchor>> oc(chunks.size());
  for (size_t i = 0; i < chunks.size(); i++)
    for (const AnchorRec& a : chunks[i].a) oc[i].push_back(orc::Anchor{chunks[i].qctg, a.qpos, a.rc >> 1, a.rpos, (a.rc & 1u) != 0});
  std::vector<double> osc;
  std::vector<uint32_t> optr;
  std::vector<orc::ChainInterval> oiv = orc::chain_chunks(oc, map_params(c, k), &osc, &optr);
  size_t off = 0;
  std::vector<IntervalKey> iv;
  for (size_t i = 0; i < chunks.size(); i++) {
    for (size_t x = 0; x < chunks[i].a.size(); x++) {
      if (outs[i].score[x] != (int32_t)osc[off + x]) { FAIL("chunk %zu anchor %zu, field score: emulated %d, oracle %d", i, x, outs[i].score[x], (int32_t)osc[off + x]); return; }
      if (outs[i].ptr[x] != optr[off + x]) { FAIL("chunk %zu anchor %zu, field pointer: emulated %u, oracle %u", i, x, outs[i].ptr[x], optr[off + x]); return; }
    }
    off += chunks[i].a.size();
    n_anchors_all += chunks[i].a.size();
    emit_intervals(chunks[i], outs[i], (uint32_t)i, iv);
  }
  n_chunks_all += chunks.size();
  n_iv_all += iv.size();
  check_selection(iv, oiv, (uint32_t)chunks.size(), c, k, false, "intervals of the DP");
}

int main(int argc, char** argv) {
  if (argc > 1 && !strcmp(argv[1], "--constants")) {
    printf("SEL_DEPS=%u SEL_SMEM_MAX=%u SEL_CELL_SHIFT=%u SEL_MAP_BITS=%u\n", SEL_DEPS, SEL_SMEM_MAX, SEL_CELL_SHIFT, SEL_MAP_BITS);
    return 0;
  }
  char kind[8];
  while (scanf("%7s", kind) == 1) {
    if (kind[0] == 'D') {
      int GL, NE, FB, NB;
      unsigned band, c, nc;
      if (scanf("%d %d %d %d %u %u %u", &GL, &NE, &FB, &NB, &band, &c, &nc) != 7) return 2;
      std::vector<Chunk> chunks(nc);
      for (auto& C : chunks) {
        unsigned n;
        if (scanf("%u", &n) != 1) return 2;
        C.a.resize(n);
        for (unsigned t = 0; t < n; t++) {
          unsigned qc, qp, rcg, rp, rev;
          if (scanf("%u %u %u %u %u", &qc, &qp, &rcg, &rp, &rev) != 5) return 2;
          C.qctg = qc; C.a[t].qpos = qp; C.a[t].rpos = rp; C.a[t].rc = (rcg << 1) | rev;
        }
      }
      run_dp(GL, NE, FB != 0, NB, band, c, chunks);
    } else {
      char name[256];
      unsigned nc, n, sw;
      if (scanf("%255s %u %u %u", name, &nc, &n, &sw) != 4) return 2;
      std::vector<IntervalKey> iv(n);
      std::vector<orc::ChainInterval> ex(n);
      for (unsigned i = 0; i < n; i++) {
        long long x[10];
        for (int f = 0; f < 10; f++) if (scanf("%lld", &x[f]) != 1) return 2;
        iv[i] = make_interval((int32_t)x[0], (uint32_t)x[1], (uint32_t)x[2], (uint32_t)x[3], (uint32_t)x[4], (uint32_t)x[5],
                              (uint32_t)x[6], (uint32_t)x[7], (uint32_t)x[8], (uint32_t)x[9]);
        ex[i] = to_orc(iv[i]);
      }
      g_tag = "select";
      check_selection(iv, ex, nc, 125, 15, sw != 0, name);
    }
  }
  printf("dp configs %ld, chunks %ld, anchors %ld, intervals %ld, lists %ld, dependency-list candidates %ld, full-scan candidates "
         "%ld, bitmap skips %ld, bitmap scans %ld, wide spans scanned %ld, edge-candidate wins %ld, sentinel rejects %ld, %d failures\n",
         n_dp_configs, n_chunks_all, n_anchors_all, n_iv_all, n_lists, n_dep_path, n_scan_path, n_bitmap_skip, n_bitmap_scan,
         n_wide_forced, n_edge_cand_wins, n_sentinel_rejects, failures);
  return failures ? 1 : 0;
}
