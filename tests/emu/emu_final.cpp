// Host emulation of final_kernel (skani_b200/csrc/chain.cu) over the __host__ __device__ functions of chain_core.cuh it
// calls, checked against the oracle's final_estimate (calculate_ani's tail + predict_from_ani_res) on constructed sorted
// (est, weight) lists, f32 result fields bit for bit.  Development/test harness only, not a product path.
//   1. lists of n = 1, 2, 9, 10, 11, 2^m - 1, 2^m, 2^m + 1, 1024, 1025 and 70,000 estimates under the plain, --robust and
//      --median trims, with the running weight exactly on floor(total * lower) / floor(total * upper) and one off either
//      side; tied estimates with different weights; all estimates 1.0; pools below, at and above 1,024 buckets;
//   2. the bootstrap's sequential redo: pools where some draw is rejected by Lemire's loop (found by search), and every
//      list again with the redo forced, against a plain sequential WyRand + Lemire loop with a cumulative-weight search
//      (pools too large to expand as the oracle does: 2^40 and more);
//   3. the GBDT of both models with a feature on every node threshold and its neighbours, and predictions of 100 and more;
//   4. the AF / both-AF cutoffs exactly on the cutoff, ani at 0.9f and its neighbours, total_bases_covered at 150,000 and
//      150,001.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <random>
#include <vector>

#include "../../skani_b200/csrc/chain_core.cuh"
#include "../../oracle/skani_oracle.hpp"

namespace tables {
#include "../../skani_b200/csrc/gbdt_tables.inc"
}

static int failures = 0;
#define CHECK(cond, ...) do { if (!(cond)) { failures++; if (failures < 30) { fprintf(stderr, "FAIL %s:%d: ", __FILE__, __LINE__); fprintf(stderr, __VA_ARGS__); fprintf(stderr, "\n"); } } } while (0)

using Ests = std::vector<std::pair<double, size_t>>;

// edges reached (the test asserts every one is non-zero)
static long n_cases, n_small_n, n_boot, n_pow2, n_not_pow2, n_lower_exact, n_upper_exact, n_lower_off, n_upper_off, n_ties,
    n_all_one, n_pool_lt, n_pool_eq, n_pool_gt, n_search_path, n_rejections, n_redo_cmp, n_big_pool, n_gbdt_eq, n_gbdt_nb,
    n_pred_ge100, n_af_edge, n_both_edge, n_gate_ani, n_gate_tbc, n_reg_applied, n_kept;

struct Model {
  std::vector<float> thr, leaf;
  const unsigned char* feat;
  float shrink, bias;
  int ntrees;
};
static Model models[2];
static float b2f(uint32_t b) { float f; memcpy(&f, &b, 4); return f; }
static void load_models() {
  for (int i = 0; i < 1365; i++) { models[0].thr.push_back(b2f(tables::SK_GBDT_C125_THR[i])); models[1].thr.push_back(b2f(tables::SK_GBDT_C200_THR[i])); }
  for (int i = 0; i < 1560; i++) { models[0].leaf.push_back(b2f(tables::SK_GBDT_C125_LEAF[i])); models[1].leaf.push_back(b2f(tables::SK_GBDT_C200_LEAF[i])); }
  models[0].feat = tables::SK_GBDT_C125_FEAT; models[1].feat = tables::SK_GBDT_C200_FEAT;
  models[0].shrink = b2f(SK_GBDT_C125_SHRINK_BITS); models[1].shrink = b2f(SK_GBDT_C200_SHRINK_BITS);
  models[0].bias = b2f(SK_GBDT_C125_BIAS_BITS); models[1].bias = b2f(SK_GBDT_C200_BIAS_BITS);
  models[0].ntrees = SK_GBDT_C125_NTREES; models[1].ntrees = SK_GBDT_C200_NTREES;
}
static float predict(int m, const float x[5]) {
  const Model& M = models[m];
  return sk::gbdt_eval(M.feat, M.thr.data(), M.leaf.data(), M.ntrees, M.shrink, M.bias, x);
}

struct SeqWyRand {   // fastrand 1.9.0, sequential form (SURVEY App. D.4)
  uint64_t state;
  uint64_t next() {
    state += 0xA0761D6478BD642Full;
    __uint128_t t = (__uint128_t)state * (__uint128_t)(state ^ 0xE7037ED1A0B428DBull);
    return (uint64_t)t ^ (uint64_t)(t >> 64);
  }
  uint64_t below(uint64_t n) {   // Lemire with the rejection loop
    uint64_t r = next();
    __uint128_t m = (__uint128_t)r * n;
    if ((uint64_t)m < n) {
      const uint64_t t = (0 - n) % n;
      while ((uint64_t)m < t) { r = next(); m = (__uint128_t)r * n; }
    }
    return (uint64_t)(m >> 64);
  }
};
// the reference's bootstrap replicate means, drawn sequentially; the pool is not expanded: a draw picks the first estimate
// whose running weight exceeds it (a linear scan, independent of cum_search)
static std::vector<double> seq_bootstrap(const Ests& e) {
  std::vector<uint64_t> cum;
  uint64_t run = 0;
  for (auto& x : e) cum.push_back(run += x.second);
  SeqWyRand rng{sk::BOOT_SEED};
  std::vector<double> res;
  std::vector<uint64_t> idx(e.size());
  for (uint32_t it = 0; it < sk::BOOT_ITERS; it++) {
    for (auto& v : idx) v = rng.below(run);
    double s = 0;
    for (uint64_t v : idx) {
      size_t a = std::upper_bound(cum.begin(), cum.end(), v) - cum.begin();
      s += e[a].first;
    }
    res.push_back(s / (double)e.size());
  }
  return res;
}

struct Emu {
  orc::AniEstResult r;
  std::vector<double> boot;    // replicate means as final_kernel leaves them (after a redo if any)
  bool rejected = false;
};
// final_kernel's flow, thread by thread in order, on one sorted list
static Emu emu_final(const Ests& ests, uint32_t tqb, uint32_t avg, uint64_t qlen, uint64_t rlen, const float qq[3], const float qr[3],
                     const orc::MapParams& mp, bool force_redo) {
  Emu out;
  const uint32_t n = (uint32_t)ests.size();
  std::vector<double> e(n);
  std::vector<uint32_t> w(n);
  for (uint32_t i = 0; i < n; i++) { e[i] = ests[i].first; w[i] = (uint32_t)ests[i].second; }
  uint64_t total = 0;
  for (uint32_t i = 0; i < n; i++) total += w[i];
  double lower, upper;
  sk::trim_fractions(mp.median, mp.robust, &lower, &upper);
  uint32_t lo, hi;
  sk::trim_bounds(w.data(), n, total, lower, upper, &lo, &hi);
  {  // edges of the trim: the running weight exactly on / one off a bound at the index the bound picked
    uint64_t curr = 0;
    const uint64_t tl = (uint64_t)((double)total * lower), tu = (uint64_t)((double)total * upper);
    for (uint32_t i = 0; i < n; i++) {
      curr += w[i];
      if (i == lo && lower > 0.) { if (curr == tl) n_lower_exact++; else if (curr == tl + 1 || curr + w[i] == tl + 1) n_lower_off++; }
      if (i + 1 == hi && upper < 1.) { if (curr == tu) n_upper_exact++; else if (curr == tu + 1 || curr - w[i] + 1 == tu) n_upper_off++; }
    }
  }
  const double final_mean = sk::trimmed_mean(e.data(), w.data(), lo, hi);
  const double sd = sk::pop_std(e.data(), n);
  double ci_lo = 0., ci_hi = 1.;
  if (sk::boot_enabled(n)) {
    std::vector<uint64_t> cum(n);
    uint64_t run = 0;
    for (uint32_t i = 0; i < n; i++) cum[i] = run += w[i];
    const uint32_t gshift = sk::guide_shift(total), nbuck = sk::guide_buckets(total, gshift);
    CHECK(nbuck <= sk::GUIDE_BUCKETS, "guide table of %u buckets", nbuck);
    std::vector<uint16_t> guide(nbuck);
    for (uint32_t b = 0; b < nbuck; b++) guide[b] = sk::guide_entry(cum.data(), n, b, gshift);
    out.boot.resize(sk::BOOT_ITERS);
    bool rej = false;
    for (uint32_t rep = 0; rep < sk::BOOT_ITERS; rep++) {
      bool rj, rj2;
      const double ms = sk::boot_replicate<false>(cum.data(), e.data(), n, total, nullptr, 0, rep, &rj);
      if (n < sk::GUIDE_MAX_N) {
        out.boot[rep] = sk::boot_replicate<true>(cum.data(), e.data(), n, total, guide.data(), gshift, rep, &rj2);
        CHECK(memcmp(&ms, &out.boot[rep], 8) == 0 && rj == rj2, "guide and search lookups differ (n %u replicate %u)", n, rep);
      } else {
        out.boot[rep] = ms;
      }
      rej |= rj;
    }
    out.rejected = rej;
    if (rej || force_redo) {
      std::vector<double> redo(sk::BOOT_ITERS);
      sk::boot_redo(cum.data(), e.data(), n, total, redo.data());
      if (!rej) {   // no draw rejected: the redo must give every replicate back unchanged
        CHECK(memcmp(redo.data(), out.boot.data(), 8 * sk::BOOT_ITERS) == 0, "forced redo differs from the replicates (n %u)", n);
        n_redo_cmp++;
      }
      out.boot = redo;
    }
    std::vector<int> seen(sk::BOOT_ITERS, 0);
    for (uint32_t i = 0; i < sk::BOOT_ITERS; i++) {
      const uint32_t rank = sk::boot_rank(out.boot.data(), i);
      CHECK(rank < sk::BOOT_ITERS && !seen[rank], "ranks are not a permutation");
      if (rank < sk::BOOT_ITERS) seen[rank] = 1;
      if (rank == sk::CI_LO_RANK) ci_lo = out.boot[i];
      if (rank == sk::CI_HI_RANK) ci_hi = out.boot[i];
    }
  }
  double final_ani = final_mean;
  const double cq = sk::covered_frac(tqb, qlen), cr = sk::covered_frac(tqb, rlen);
  if (sk::af_cut(cq, cr, mp.frac_cover_cutoff, mp.both_frac_cover_cutoff)) final_ani = -1.;
  orc::AniEstResult& r = out.r;
  r.ani = (float)final_ani;
  r.align_fraction_query = (float)cq; r.align_fraction_ref = (float)cr;
  r.ci_lower = (float)ci_lo; r.ci_upper = (float)ci_hi; r.std = (float)sd;
  r.quant_10_contig_len_q = qq[0]; r.quant_50_contig_len_q = qq[1]; r.quant_90_contig_len_q = qq[2];
  r.quant_10_contig_len_r = qr[0]; r.quant_50_contig_len_r = qr[1]; r.quant_90_contig_len_r = qr[2];
  r.avg_chain_int_len = avg; r.total_bases_covered = tqb;
  if (mp.model >= 0 && sk::regress_gate(r.ani, r.total_bases_covered)) {
    float x[5];
    sk::regress_features(r.ani, r.std, qq[1], qq[2], qr[1], qr[2], avg, x);
    const Model& M = models[mp.model];
    std::vector<float> term(M.ntrees);   // final_kernel: one tree per thread, then the terms summed in tree order
    for (int t = 0; t < M.ntrees; t++) term[t] = sk::gbdt_tree_term(M.feat, M.thr.data(), M.leaf.data(), t, M.shrink, x);
    float pred = M.bias;
    for (int t = 0; t < M.ntrees; t++) pred = sk::fadd_rn(pred, term[t]);
    const float ev = predict(mp.model, x);
    CHECK(memcmp(&pred, &ev, 4) == 0, "per-tree terms and gbdt_eval differ");
    if (pred >= 100.f) n_pred_ge100++;
    else n_reg_applied++;
    sk::regress_apply(pred, &r.ani, &r.ci_lower, &r.ci_upper);
  }
  return out;
}

static bool same_f(float a, float b) { return memcmp(&a, &b, 4) == 0; }
static orc::MapParams params(int trim, double min_af, double both_min_af, int model) {
  orc::Sketch unit;
  unit.c = 125; unit.k = 15;
  orc::CommandParams cp;
  cp.robust = trim == 1; cp.median = trim == 2;
  cp.min_aligned_frac = min_af; cp.both_min_aligned_frac = both_min_af;
  return orc::map_params_from_sketch(unit, cp, model);
}

// one case: the emulation against the oracle (pools the oracle can expand) or against the sequential loop
static void check_case(const Ests& ests, uint32_t tqb, uint32_t avg, uint64_t qlen, uint64_t rlen, const orc::MapParams& mp,
                       const char* what) {
  const float qq[3] = {1200.f, 45000.f, 310000.f}, qr[3] = {900.f, 60000.f, 280000.f};
  n_cases++;
  const uint32_t n = (uint32_t)ests.size();
  uint64_t pool = 0;
  for (auto& x : ests) pool += x.second;
  if (n < sk::BOOT_MIN_N) n_small_n++;
  else {
    n_boot++;
    if ((n & (n - 1)) == 0) n_pow2++; else n_not_pow2++;
    if (pool < sk::GUIDE_BUCKETS) n_pool_lt++;
    else if (pool == sk::GUIDE_BUCKETS) n_pool_eq++;
    else n_pool_gt++;
    if (n >= sk::GUIDE_MAX_N) n_search_path++;
  }
  for (size_t i = 1; i < n; i++) if (ests[i].first == ests[i - 1].first && ests[i].second != ests[i - 1].second) { n_ties++; break; }
  if (n && std::all_of(ests.begin(), ests.end(), [](const std::pair<double, size_t>& x) { return x.first == 1.0; })) n_all_one++;
  const Emu em = emu_final(ests, tqb, avg, qlen, rlen, qq, qr, mp, false);
  const Emu forced = emu_final(ests, tqb, avg, qlen, rlen, qq, qr, mp, true);
  CHECK(memcmp(&em.r, &forced.r, sizeof(em.r)) == 0, "%s: the forced redo changes the result", what);
  if (em.rejected) n_rejections++;
  if (n >= sk::BOOT_MIN_N && (pool > (1ull << 24) || em.rejected)) {
    n_big_pool++;
    const std::vector<double> ref = seq_bootstrap(ests);
    CHECK(memcmp(ref.data(), em.boot.data(), 8 * sk::BOOT_ITERS) == 0, "%s: replicate means differ from the sequential loop (n %u, pool %llu)",
          what, n, (unsigned long long)pool);
    return;
  }
  const orc::AniEstResult o = orc::final_estimate(ests, tqb, avg, qlen, rlen, qq, qr, mp);
  const orc::AniEstResult& g = em.r;
  if (o.ani > 0.f) n_kept++;
  CHECK(same_f(g.ani, o.ani) && same_f(g.std, o.std) && same_f(g.ci_lower, o.ci_lower) && same_f(g.ci_upper, o.ci_upper) &&
            same_f(g.align_fraction_query, o.align_fraction_query) && same_f(g.align_fraction_ref, o.align_fraction_ref) &&
            g.avg_chain_int_len == o.avg_chain_int_len && g.total_bases_covered == o.total_bases_covered,
        "%s (n %u, pool %llu): ani %.9g/%.9g std %.9g/%.9g ci %.9g/%.9g %.9g/%.9g af %.9g/%.9g", what, n, (unsigned long long)pool,
        (double)g.ani, (double)o.ani, (double)g.std, (double)o.std, (double)g.ci_lower, (double)o.ci_lower, (double)g.ci_upper,
        (double)o.ci_upper, (double)g.align_fraction_query, (double)o.align_fraction_query);
}

// n weights summing to T, with the running weight passing through each of `marks` (distinct, in (0, T)) exactly
static std::vector<uint64_t> partition(std::mt19937_64& rng, uint32_t n, uint64_t T, std::vector<uint64_t> marks) {
  std::vector<uint64_t> pts;
  for (uint64_t m : marks) if (m > 0 && m < T) pts.push_back(m);
  std::sort(pts.begin(), pts.end());
  pts.erase(std::unique(pts.begin(), pts.end()), pts.end());
  while (pts.size() + 1 < n) {
    pts.push_back(1 + rng() % (T - 1));
    std::sort(pts.begin(), pts.end());
    pts.erase(std::unique(pts.begin(), pts.end()), pts.end());
  }
  while (pts.size() + 1 > n) pts.erase(pts.begin() + (rng() % pts.size()));   // may drop a mark: rare, counted by the edges
  std::vector<uint64_t> w;
  uint64_t prev = 0;
  for (uint64_t p : pts) { w.push_back(p - prev); prev = p; }
  w.push_back(T - prev);
  return w;
}
static Ests sorted_list(std::mt19937_64& rng, const std::vector<uint64_t>& w, int est_kind) {
  std::uniform_real_distribution<double> u(0.78, 1.0);
  std::vector<double> e(w.size());
  for (auto& x : e) x = est_kind == 1 ? 1.0 : u(rng);
  std::sort(e.begin(), e.end());
  if (est_kind == 2)   // ties: runs of equal estimates
    for (size_t i = 1; i < e.size(); i++) if (rng() % 3 == 0) e[i] = e[i - 1];
  Ests out;
  for (size_t i = 0; i < w.size(); i++) out.push_back({e[i], (size_t)w[i]});
  if (est_kind == 2) std::sort(out.begin(), out.end());   // the (f64, usize) order reorders the weights of a tie
  return out;
}

int main() {
  load_models();
  std::mt19937_64 rng(20261015);
  const uint64_t QLEN = 3000000, RLEN = 2500000;
  // ---- 1. list shapes x trims x trim edges x pools
  const uint32_t ns[] = {1, 2, 9, 10, 11, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025};
  for (uint32_t n : ns)
    for (int trim = 0; trim < 3; trim++)
      for (int kind = 0; kind < 3; kind++)
        for (int rep = 0; rep < 4; rep++) {
          const double lower = trim == 0 ? 0. : trim == 1 ? 0.10 : 0.499, upper = trim == 0 ? 1. : trim == 1 ? 0.90 : 0.501;
          uint64_t T;
          switch (rep) {
            case 0: T = n + rng() % (std::max<uint32_t>(n, 8) * 3); break;     // small weights
            case 1: T = std::max<uint64_t>(n, 1024); break;                    // pool at the guide table's size (or n)
            case 2: T = std::max<uint64_t>(n, 1025); break;
            default: T = std::max<uint64_t>(n, (1ull << 20) - rng() % 1000);  // large pool (2^20)
          }
          if (rep == 3 && kind != 0) continue;
          const uint64_t tl = (uint64_t)((double)T * lower), tu = (uint64_t)((double)T * upper);
          for (int off = -1; off <= 1; off++) {
            const std::vector<uint64_t> w = partition(rng, n, T, {tl + off, tu + off});
            const Ests l = sorted_list(rng, w, kind);
            for (int model = -1; model < 2; model++) {
              if (model >= 0 && (n % 3 != 0 && n > 2)) continue;             // learned ANI on a subset of the shapes
              char what[96];
              snprintf(what, sizeof(what), "n %u trim %d kind %d pool %llu off %d model %d", n, trim, kind, (unsigned long long)T, off, model);
              check_case(l, 600000, 4100, QLEN, RLEN, params(trim, 0.15, -0.01, model), what);
            }
          }
        }
  {  // 70,000 estimates: the search lookups (no guide table), pool small enough for the oracle
    std::vector<uint64_t> w(70000);
    for (auto& x : w) x = 1 + rng() % 3;
    check_case(sorted_list(rng, w, 0), 5000000, 2500, QLEN * 4, RLEN * 4, params(1, 0.15, -0.01, 0), "n 70000");
  }
  // ---- 2. Lemire rejections: pools near n * 2^32 where one of the first 100 n draws is rejected
  {
    int found = 0;
    for (int tries = 0; tries < 20000 && found < 4; tries++) {
      const uint32_t n = tries % 2 ? 1024 : 512 + (uint32_t)(rng() % 512);
      std::vector<uint64_t> w(n);
      for (auto& x : w) x = (1ull << 31) + rng() % (1ull << 31);
      uint64_t pool = 0;
      for (auto x : w) pool += x;
      bool rej = false;
      for (uint64_t d = 0; d < (uint64_t)sk::BOOT_ITERS * n && !rej; d++) sk::lemire_below(sk::wyrand_at(sk::BOOT_SEED, d), pool, &rej);
      if (!rej) continue;
      found++;
      check_case(sorted_list(rng, w, found & 1 ? 0 : 2), 300000, 4000, QLEN, RLEN, params(0, 0.15, -0.01, 0), "rejection");
    }
    CHECK(found > 0, "no pool with a Lemire rejection found");
    for (int i = 0; i < 3; i++) {   // 2^40 and larger pools without a rejection
      std::vector<uint64_t> w(256 + 256 * i);
      for (auto& x : w) x = (1ull << 32) - 1 - rng() % 1000;
      check_case(sorted_list(rng, w, 0), 300000, 4000, QLEN, RLEN, params(1, 0.15, -0.01, 0), "pool 2^40");
    }
  }
  // ---- 3. GBDT: every node threshold of both models, the feature at t and its neighbours; predictions >= 100
  {
    std::uniform_real_distribution<float> ani(90.f, 100.f), sd(0.f, 3.f), ql(500.f, 3e6f), cl(200.f, 20000.f);
    for (int m = 0; m < 2; m++) {
      const Model& M = models[m];
      for (int node = 0; node < 7 * M.ntrees; node++) {
        const float t = M.thr[node];
        for (const float v : {t, std::nextafter(t, INFINITY), std::nextafter(t, -INFINITY)}) {
          float x[5] = {ani(rng), sd(rng), ql(rng), ql(rng), cl(rng)};
          x[M.feat[node]] = v;
          const float a = predict(m, x), b = orc::gbdt_predict(m, x);
          CHECK(same_f(a, b), "gbdt model %d node %d: %.9g vs %.9g", m, node, (double)a, (double)b);
          if (a >= 100.f) n_pred_ge100++;
          // was the equality (or neighbour) comparison evaluated on the walk of the tree?
          const int tr = node / 7;
          int nd = 0;
          for (int d = 0; d < 3; d++) {
            const float xv = x[M.feat[7 * tr + nd]], th = M.thr[7 * tr + nd];
            if (7 * tr + nd == node) { if (xv == th) n_gbdt_eq++; else n_gbdt_nb++; }
            nd = 2 * nd + (xv < th ? 1 : 2);
          }
        }
      }
      // learned ANI through the whole final estimate: estimates all 0.99-1.0 give predictions at and above 100
      for (int i = 0; i < 400; i++) {
        std::vector<uint64_t> w(12 + i % 40);
        for (auto& x : w) x = 50 + rng() % 200;
        Ests l = sorted_list(rng, w, i % 4 == 0 ? 1 : 0);
        if (i % 4) for (auto& x : l) x.first = 0.99 + 0.01 * std::pow(x.first, 40.0);
        std::sort(l.begin(), l.end());
        check_case(l, 400000 + 997 * i, 3000 + 37 * i, QLEN, RLEN, params(i % 3, 0.15, -0.01, m), "gbdt");
      }
    }
  }
  // ---- 4. AF cutoffs exactly on min_af / both_min_af, the regression gate's edges
  {
    std::vector<uint64_t> w(12, 100);
    const Ests base = sorted_list(rng, w, 0);
    for (uint64_t m : {1ull, 7ull, 1000ull, 123457ull}) {
      // tqb / len == 0.15 exactly (3 m / 20 m rounds to the double nearest 0.15, the cutoff itself)
      const uint32_t tqb = (uint32_t)(3 * m);
      check_case(base, tqb, 4000, 20 * m, 20 * m, params(0, 0.15, -0.01, 0), "af on the cutoff");
      check_case(base, tqb, 4000, 20 * m, 20 * m - 1, params(0, 0.15, -0.01, 0), "af: one side on the cutoff");
      n_af_edge++;
      check_case(base, tqb, 4000, 20 * m, 20 * m, params(0, 0.15, 0.15, 0), "both-af on the cutoff");
      check_case(base, tqb, 4000, 20 * m + 1, 20 * m, params(0, 0.15, 0.15, 0), "both-af: one side below");
      n_both_edge++;
    }
    for (int model = 0; model < 2; model++) {
      for (const float a : {0.9f, std::nextafter(0.9f, 1.f), std::nextafter(0.9f, 0.f)}) {
        Ests l;   // every estimate equal to a: the trimmed mean is a exactly
        for (int i = 0; i < 12; i++) l.push_back({(double)a, (size_t)(100 + i)});
        check_case(l, 400000, 4000, QLEN, RLEN, params(0, 0.15, -0.01, model), "ani at 0.9f");
        n_gate_ani++;
      }
      for (const uint32_t tbc : {sk::REGRESS_CUTOFF - 1, sk::REGRESS_CUTOFF, sk::REGRESS_CUTOFF + 1}) {
        std::vector<uint64_t> w2(14, 77);
        Ests l = sorted_list(rng, w2, 0);
        for (auto& x : l) x.first = 0.95 + 0.04 * x.first;
        std::sort(l.begin(), l.end());
        check_case(l, tbc, 4000, 400000, 400000, params(0, 0.15, -0.01, model), "total_bases_covered at the gate");
        n_gate_tbc++;
      }
    }
  }
  printf("cases %ld: estimate kept %ld, n < 10 %ld, bootstrap %ld (n a power of two %ld, not %ld), search lookups %ld\n", n_cases,
         n_kept, n_small_n, n_boot, n_pow2, n_not_pow2, n_search_path);
  printf("trim: lower exact %ld, lower off by one %ld, upper exact %ld, upper off by one %ld; ties %ld, all 1.0 %ld\n", n_lower_exact,
         n_lower_off, n_upper_exact, n_upper_off, n_ties, n_all_one);
  printf("pool: below 1024 %ld, at 1024 %ld, above %ld; rejections %ld, forced redo %ld, sequential-loop pools %ld\n", n_pool_lt,
         n_pool_eq, n_pool_gt, n_rejections, n_redo_cmp, n_big_pool);
  printf("gbdt: on a threshold %ld, next to one %ld, learned applied %ld, prediction >= 100 %ld\n", n_gbdt_eq, n_gbdt_nb, n_reg_applied,
         n_pred_ge100);
  printf("cutoffs: af %ld, both-af %ld, ani gate %ld, bases gate %ld\n", n_af_edge, n_both_edge, n_gate_ani, n_gate_tbc);
  printf("%d failures\n", failures);
  return failures ? 1 : 0;
}
