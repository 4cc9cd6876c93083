// Host emulation of the chaining path's per-item logic (skani_b200/csrc/chain_core.cuh: the __host__ __device__ functions
// the CUDA kernels call) checked against the CPU oracle's parity taps.  Development/test harness only: it validates the
// closed forms without a GPU; it is not a product path.
//   1. chunk assignment: FirstOp / MinOp segmented scans + chunk_need + chunk_local_of, driven sequentially, and the
//      per-record / per-anchor closed forms chunk_anchor_kernel (chain.cu) applies (record_starts_chunk,
//      record_chunk_starts, anchor_chunk_local, anchor_starts_chunk), against the oracle's chunk boundaries (sequential
//      loop of src/chain.rs:738-836), including anchor-free stretches > 20 kb ("catch-up" singleton chunks) and
//      multi-contig queries;
//   2. interval order (IntervalKey / interval_before) and the greedy non-overlap decisions (overlap_contrib /
//      overlap_accept) against the oracle's sorted interval list and kept flags (src/chain.rs:1008-1099);
//   3. wyrand_at / lemire_below (random access) against a sequential WyRand + Lemire (SURVEY App. D.4);
//   4. gbdt_eval on the flattened tables against the oracle's tree walk (SURVEY App. D.5), bit-exact f32.
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
static long catchup_anchors = 0;   // anchors whose chunk is held back below `need` by the catch-up rule
#define CHECK(cond, ...) do { if (!(cond)) { failures++; fprintf(stderr, "FAIL %s:%d: ", __FILE__, __LINE__); fprintf(stderr, __VA_ARGS__); fprintf(stderr, "\n"); } } while (0)

static std::vector<uint8_t> random_seq(std::mt19937_64& rng, size_t n) {
  std::vector<uint8_t> s(n);
  for (auto& b : s) b = "ACGT"[rng() & 3];
  return s;
}
static std::vector<uint8_t> mutate(std::mt19937_64& rng, const std::vector<uint8_t>& a, double rate) {
  std::vector<uint8_t> s = a;
  std::uniform_real_distribution<double> u(0, 1);
  for (auto& b : s) if (u(rng) < rate) b = "ACGT"[rng() & 3];
  return s;
}
static orc::Sketch sketch_of(const char* name, const std::vector<std::vector<uint8_t>>& ctgs, const orc::SketchParams& sp) {
  std::vector<std::pair<const uint8_t*, size_t>> v;
  for (auto& c : ctgs) v.push_back({c.data(), c.size()});
  return orc::sketch_from_contigs(name, v, nullptr, sp, true);
}

// ---- 1. chunk ids from the sorted anchor list, with the device functions in chunk_kernel's order of application
static std::vector<uint32_t> emu_chunk_first(const std::vector<orc::Anchor>& an) {
  std::vector<uint32_t> first;
  sk::FirstState carryF; carryF.valid = 0; carryF.ctg = 0; carryF.p0 = 0; carryF.a0 = 0;
  sk::MinState carryM; carryM.valid = 0; carryM.ctg = 0; carryM.v = 0;
  uint32_t prev_ctg = 0xFFFFFFFFu, prev_cl = 0;
  for (size_t a = 0; a < an.size();) {
    size_t e = a + 1;      // one hit record = the anchors of one query seed position
    while (e < an.size() && an[e].query_contig == an[a].query_contig && an[e].query_pos == an[a].query_pos) e++;
    const uint32_t nh = (uint32_t)(e - a);
    sk::FirstState f; f.valid = 1; f.ctg = an[a].query_contig; f.p0 = an[a].query_pos; f.a0 = (uint32_t)a;
    carryF = sk::FirstOp()(carryF, f);                       // inclusive scan
    const uint32_t need = sk::chunk_need(an[a].query_pos, carryF.p0);
    const uint32_t al = (uint32_t)a - carryF.a0;
    const bool has_prev = carryM.valid && carryM.ctg == an[a].query_contig;   // exclusive scan state
    // the kernel's per-record and per-anchor closed forms (chunk_anchor_kernel), checked against the plain rule "an anchor
    // starts a chunk iff its chunk differs from the previous anchor's"
    const uint32_t clf = sk::chunk_local_of(al, has_prev, carryM.v, need);
    const uint32_t cll = sk::chunk_local_of((uint64_t)al + nh - 1, has_prev, carryM.v, need);
    const uint32_t st = sk::record_starts_chunk(al, has_prev, carryM.v, clf);
    uint32_t starts = 0;
    for (uint32_t t = 0; t < nh; t++) {
      const uint32_t cl = sk::chunk_local_of((uint64_t)al + t, has_prev, carryM.v, need);
      CHECK(cl == sk::anchor_chunk_local(clf, t, need), "anchor_chunk_local of anchor %zu", a + t);
      if (cl != need) catchup_anchors++;
      const bool plain = a + t == 0 || prev_ctg != an[a].query_contig || prev_cl != cl;
      const bool start = sk::anchor_starts_chunk(clf, t, need, st != 0);
      CHECK(start == plain, "anchor_starts_chunk of anchor %zu", a + t);
      if (start) { first.push_back((uint32_t)(a + t)); starts++; }
      prev_ctg = an[a].query_contig; prev_cl = cl;
    }
    CHECK(starts == sk::record_chunk_starts(st, clf, cll), "record_chunk_starts of the record at anchor %zu", a);
    sk::MinState m; m.valid = 1; m.ctg = an[a].query_contig; m.v = sk::record_min_key(need, al, nh);
    carryM = sk::MinOp()(carryM, m);
    a = e;
  }
  first.push_back((uint32_t)an.size());
  return first;
}

// ---- 1b. chunk_anchor_kernel's own arrangement: the query-role records in TILE-record tiles with carries, every tile's
// scans combined as the kernel's block scans combine them (256 threads x 4 blocked items, shuffle-up warp scans, warp
// aggregates folded in order, the MinOp scan exclusive and seeded with identM), and again left to right and under random
// bracketings.  The three must agree on everything the kernel reads, so an operator that stops being associative on the
// inputs the kernel feeds it fails here.
constexpr uint32_t TILE = 1024, THREADS = 256, ITEMS = 4;
static long tiles_run = 0, rounds_run = 0, bracketings_run = 0, multi_round_tiles = 0, straddling_records = 0, empty_tiles = 0;

static bool same(const sk::FirstState& a, const sk::FirstState& b) {
  return a.valid == b.valid && (!a.valid || (a.ctg == b.ctg && a.p0 == b.p0 && a.a0 == b.a0));
}
static bool same(const sk::MinState& a, const sk::MinState& b) {
  return a.valid == b.valid && (!a.valid || (a.ctg == b.ctg && a.v == b.v));
}

// inclusive (has_init = false) or exclusive-with-initial-value scan of TILE items as cub::BlockScan<..., 256,
// BLOCK_SCAN_WARP_SCANS> arranges the operator applications; returns the aggregate (without the initial value)
template <typename T, typename Op>
static T block_scan(const std::vector<T>& x, std::vector<T>& out, Op op, bool has_init, const T& init) {
  std::vector<T> part(THREADS);
  for (uint32_t t = 0; t < THREADS; t++) {                  // thread-local reduction of 4 blocked items
    T p = x[t * ITEMS];
    for (uint32_t i = 1; i < ITEMS; i++) p = op(p, x[t * ITEMS + i]);
    part[t] = p;
  }
  std::vector<T> inc(part);                                 // shuffle-up inclusive warp scans
  for (uint32_t w = 0; w < THREADS / 32; w++)
    for (uint32_t off = 1; off < 32; off <<= 1) {
      std::vector<T> prev(inc.begin() + w * 32, inc.begin() + w * 32 + 32);
      for (uint32_t l = off; l < 32; l++) inc[w * 32 + l] = op(prev[l - off], prev[l]);
    }
  std::vector<T> wpre(THREADS / 32);                        // warp prefixes: aggregates folded in warp order
  T agg = inc[31];
  for (uint32_t w = 1; w < THREADS / 32; w++) { wpre[w] = agg; agg = op(agg, inc[w * 32 + 31]); }
  for (uint32_t t = 0; t < THREADS; t++) {
    const uint32_t w = t / 32, l = t % 32;
    bool has_pre = true;
    T pre;                                                  // everything before thread t
    if (w == 0) {
      if (l == 0) { has_pre = has_init; pre = init; }
      else pre = has_init ? op(init, inc[t - 1]) : inc[t - 1];
    } else {
      const T wp = has_init ? op(init, wpre[w]) : wpre[w];
      pre = (l == 0) ? wp : op(wp, inc[t - 1]);
    }
    for (uint32_t i = 0; i < ITEMS; i++) {
      const T& v = x[t * ITEMS + i];
      if (has_init) { out[t * ITEMS + i] = pre; pre = op(pre, v); }
      else { pre = has_pre ? op(pre, v) : v; has_pre = true; out[t * ITEMS + i] = pre; }
    }
  }
  return agg;
}
// the same scan, left to right
template <typename T, typename Op>
static void seq_scan(const std::vector<T>& x, std::vector<T>& out, Op op, bool has_init, const T& init) {
  T run = init;
  for (size_t i = 0; i < x.size(); i++) {
    if (has_init) { out[i] = run; run = op(run, x[i]); }
    else { run = i ? op(run, x[i]) : x[i]; out[i] = run; }
  }
}
// inclusive prefixes of x[l, r) under a random bracketing (random split points, left part combined into the right part)
template <typename T, typename Op>
static void rand_scan(const std::vector<T>& x, std::vector<T>& inc, Op op, size_t l, size_t r, std::mt19937_64& rng) {
  if (r - l == 1) { inc[l] = x[l]; return; }
  const size_t m = l + 1 + rng() % (r - l - 1);
  rand_scan(x, inc, op, l, m, rng);
  rand_scan(x, inc, op, m, r, rng);
  for (size_t i = m; i < r; i++) inc[i] = op(inc[m - 1], inc[i]);
}

struct QRec { uint32_t ctg, pos; };
// records of the query-role sketch in (contig, pos) order
static std::vector<QRec> query_records(const orc::Sketch& s) {
  std::vector<QRec> v;
  const orc::KmerSeeds& m = s.kmer_seeds_k;
  orc::SeedPosition tmp;
  for (size_t i = 0; i < m.capacity(); i++) {
    if (!m.slot_used(i)) continue;
    const orc::SeedPosition* p;
    const size_t n = s.get_seed_positions(m.slot_key(i), &p, &tmp);
    for (size_t a = 0; a < n; a++) v.push_back({p[a].contig_index_canonical >> 1, p[a].pos});
  }
  std::sort(v.begin(), v.end(), [](const QRec& a, const QRec& b) { return a.ctg != b.ctg ? a.ctg < b.ctg : a.pos < b.pos; });
  v.erase(std::unique(v.begin(), v.end(), [](const QRec& a, const QRec& b) { return a.ctg == b.ctg && a.pos == b.pos; }), v.end());
  return v;
}

// chunk_first of the pair as chunk_anchor_kernel computes it, tile by tile (stg_first, pair-local anchor indices)
static std::vector<uint32_t> emu_chunk_tiles(const std::vector<orc::Anchor>& an, const std::vector<QRec>& rec,
                                             std::mt19937_64& rng, const char* what) {
  const sk::FirstOp fop;
  const sk::MinOp mop;
  std::vector<uint32_t> nh_all(rec.size(), 0);
  for (size_t a = 0, r = 0; a < an.size(); a++) {           // anchors of a record are consecutive, records in order
    while (r < rec.size() && (rec[r].ctg != an[a].query_contig || rec[r].pos != an[a].query_pos)) r++;
    if (r == rec.size()) { CHECK(false, "%s: anchor %zu has no query record", what, a); return {}; }
    nh_all[r]++;
  }
  sk::FirstState carryF; carryF.valid = 0; carryF.ctg = 0; carryF.p0 = 0; carryF.a0 = 0;
  sk::MinState carryM; carryM.valid = 0; carryM.ctg = 0; carryM.v = 0;
  sk::MinState identM; identM.valid = 0; identM.ctg = 0; identM.v = 0;
  uint32_t carryA = 0, carryC = 0;
  std::vector<uint32_t> first;
  for (size_t t0 = 0; t0 < rec.size(); t0 += TILE) {
    tiles_run++;
    std::vector<uint32_t> nh(TILE, 0), pos(TILE, 0), ctg(TILE, 0), aoff(TILE);
    for (uint32_t i = 0; i < TILE && t0 + i < rec.size(); i++)
      if ((nh[i] = nh_all[t0 + i])) { pos[i] = rec[t0 + i].pos; ctg[i] = rec[t0 + i].ctg; }
    uint32_t aggA = 0;
    for (uint32_t i = 0; i < TILE; i++) { aoff[i] = carryA + aggA; aggA += nh[i]; }
    std::vector<sk::FirstState> fs(TILE), fk(TILE), f2(TILE);
    std::vector<sk::MinState> ms(TILE), mk(TILE), m2(TILE);
    for (uint32_t i = 0; i < TILE; i++) { fs[i].valid = nh[i] ? 1u : 0u; fs[i].ctg = ctg[i]; fs[i].p0 = pos[i]; fs[i].a0 = aoff[i]; }
    const sk::FirstState aggF = block_scan(fs, fk, fop, false, carryF);
    seq_scan(fs, f2, fop, false, carryF);
    for (uint32_t i = 0; i < TILE; i++) CHECK(same(fk[i], f2[i]), "%s: FirstOp block scan != sequential at item %u", what, i);
    for (int b = 0; b < 2; b++, bracketings_run++) {
      rand_scan(fs, f2, fop, 0, TILE, rng);
      for (uint32_t i = 0; i < TILE; i++) CHECK(same(fk[i], f2[i]), "%s: FirstOp bracketing differs at item %u", what, i);
    }
    std::vector<uint32_t> need(TILE, 0), al(TILE, 0);
    for (uint32_t i = 0; i < TILE; i++) {
      ms[i] = identM;
      if (!nh[i]) continue;
      const sk::FirstState f = fop(carryF, fk[i]);
      need[i] = sk::chunk_need(pos[i], f.p0);
      al[i] = aoff[i] - f.a0;
      ms[i].valid = 1; ms[i].ctg = ctg[i]; ms[i].v = sk::record_min_key(need[i], al[i], nh[i]);
      fs[i] = f;                                            // p0 of the record's contig
    }
    carryF = fop(carryF, aggF);
    const sk::MinState aggM = block_scan(ms, mk, mop, true, identM);
    seq_scan(ms, m2, mop, true, identM);
    for (uint32_t i = 0; i < TILE; i++) CHECK(same(mk[i], m2[i]), "%s: MinOp block scan != sequential at item %u", what, i);
    for (int b = 0; b < 2; b++, bracketings_run++) {
      rand_scan(ms, m2, mop, 0, TILE, rng);                 // inclusive; the exclusive value of item i is the inclusive of i - 1
      for (uint32_t i = 1; i < TILE; i++) CHECK(same(mk[i], mop(identM, m2[i - 1])), "%s: MinOp bracketing differs at item %u", what, i);
    }
    std::vector<uint32_t> clf(TILE, 0), cll(TILE, 0), st(TILE, 0), inc(TILE, 0), cid(TILE, 0);
    for (uint32_t i = 0; i < TILE; i++) {
      if (!nh[i]) continue;
      const sk::MinState e = mop(carryM, mk[i]);
      const bool has_prev = e.valid && e.ctg == ctg[i];
      clf[i] = sk::chunk_local_of(al[i], has_prev, e.v, need[i]);
      cll[i] = sk::chunk_local_of((uint64_t)al[i] + nh[i] - 1, has_prev, e.v, need[i]);
      st[i] = sk::record_starts_chunk(al[i], has_prev, e.v, clf[i]);
      inc[i] = sk::record_chunk_starts(st[i], clf[i], cll[i]);
    }
    carryM = mop(carryM, aggM);
    uint32_t aggC = 0;
    for (uint32_t i = 0; i < TILE; i++) { cid[i] = carryC + aggC + st[i] - 1; aggC += inc[i]; }
    // emission in rounds of TILE anchors: anchor j of the tile belongs to the record whose range holds it
    if (aggA == 0) empty_tiles++;
    if (aggA > TILE) multi_round_tiles++;
    for (uint32_t i = 0; i < TILE; i++)
      if (nh[i] && (aoff[i] - carryA) / TILE != (aoff[i] - carryA + nh[i] - 1) / TILE) straddling_records++;
    for (uint32_t base = 0; base < aggA; base += TILE) rounds_run++;
    for (uint32_t i = 0; i < TILE; i++)
      for (uint32_t u = 0; u < nh[i]; u++) {
        const uint32_t cl = sk::anchor_chunk_local(clf[i], u, need[i]);
        if (!sk::anchor_starts_chunk(clf[i], u, need[i], st[i] != 0)) continue;
        const uint32_t mycid = cid[i] + (cl - clf[i]);
        CHECK(mycid == first.size(), "%s: chunk id %u out of order (%zu chunks so far)", what, mycid, first.size());
        first.push_back(aoff[i] + u);
        // an anchor that reached need lies in its chunk's window; catch-up anchors (cl < need) lie beyond it
        const int64_t lo = sk::chunk_window_lo(fs[i].p0, cl), hi = sk::chunk_window_hi(fs[i].p0, cl);
        CHECK(cl < need[i] || (lo < (int64_t)pos[i] && (int64_t)pos[i] <= hi), "%s: anchor %u outside its chunk window", what, aoff[i] + u);
      }
    carryA += aggA;
    carryC += aggC;
  }
  CHECK(carryA == an.size(), "%s: %u anchors emitted, %zu expected", what, carryA, an.size());
  CHECK(carryC == first.size(), "%s: chunk count %u vs %zu chunk starts", what, carryC, first.size());
  first.push_back((uint32_t)an.size());
  return first;
}

// ---- 2. interval order + greedy filter
static void check_intervals(const orc::ChainDebug& d, const char* what) {
  std::vector<sk::IntervalKey> keys;
  for (auto& iv : d.intervals_all)
    keys.push_back(sk::make_interval((int32_t)iv.score, (uint32_t)iv.num_anchors, iv.q0, iv.q1, iv.r0, iv.r1, (uint32_t)iv.ref_contig,
                                     (uint32_t)iv.query_contig, (uint32_t)iv.chunk_id, iv.reverse_chain ? 1u : 0u));
  for (size_t i = 0; i + 1 < keys.size(); i++) {
    CHECK(!sk::interval_before(keys[i + 1], keys[i]), "%s: interval %zu sorts after %zu", what, i, i + 1);
    CHECK((double)sk::iv_score(keys[i]) == d.intervals_all[i].score, "%s: score not an integer", what);
  }
  // the device sorts with interval_before: a std::sort of shuffled keys must give the oracle's order back
  std::vector<size_t> perm(keys.size());
  for (size_t i = 0; i < perm.size(); i++) perm[i] = i;
  std::mt19937_64 rng(11);
  std::shuffle(perm.begin(), perm.end(), rng);
  std::sort(perm.begin(), perm.end(), [&](size_t x, size_t y) { return sk::interval_before(keys[x], keys[y]); });
  for (size_t i = 0; i < perm.size(); i++)
    CHECK(memcmp(&keys[perm[i]], &keys[i], sizeof(sk::IntervalKey)) == 0, "%s: sorted position %zu differs", what, i);
  std::vector<size_t> acc;
  for (size_t i = 0; i < keys.size(); i++) {
    uint32_t sr = 0, hr = 0, sq = 0, hq = 0;
    for (size_t j : acc) sk::overlap_contrib(keys[i], keys[j], &sr, &hr, &sq, &hq);
    const bool keep = sk::overlap_accept(keys[i], sr, hr, sq, hq);
    CHECK(keep == (d.interval_kept[i] != 0), "%s: greedy decision of interval %zu", what, i);
    if (keep) acc.push_back(i);
  }
}

struct SeqWyRand {   // fastrand 1.9.0, sequential form (SURVEY App. D.4)
  uint64_t state;
  uint64_t next() {
    state += 0xA0761D6478BD642Full;
    __uint128_t t = (__uint128_t)state * (__uint128_t)(state ^ 0xE7037ED1A0B428DBull);
    return (uint64_t)t ^ (uint64_t)(t >> 64);
  }
};

int main() {
  std::mt19937_64 rng(20260924);
  int pairs_checked = 0, chunks_checked = 0, intervals_checked = 0, pairs_at_bound = 0;
  for (uint64_t c : {125ull, 30ull}) {
    orc::SketchParams sp; sp.c = c; sp.k = 15; sp.marker_c = c == 30 ? 200 : 1000;
    orc::CommandParams cp;
    const size_t L = 400000;
    std::vector<uint8_t> base = random_seq(rng, L);
    std::vector<std::pair<std::string, orc::Sketch>> sk;
    sk.push_back({"plain", sketch_of("a_plain", {mutate(rng, base, 0.01)}, sp)});
    sk.push_back({"divergent", sketch_of("b_div", {mutate(rng, base, 0.06)}, sp)});
    {  // 90 / 65 / 24 kb replaced by unrelated sequence: anchor-free stretches in BOTH roles -> the catch-up rule (src/chain.rs:744-793)
      std::vector<uint8_t> g = mutate(rng, base, 0.02);
      const size_t from[3] = {60000, 220000, 330000}, to[3] = {150000, 285000, 354000};
      for (int i = 0; i < 3; i++) {
        std::vector<uint8_t> junk = random_seq(rng, to[i] - from[i]);
        std::copy(junk.begin(), junk.end(), g.begin() + from[i]);
      }
      sk.push_back({"gappy", sketch_of("c_gappy", {g}, sp)});
    }
    {  // 12 contigs of uneven length, two of them reverse-complemented, one with a duplicated 40 kb block (repeats)
      std::vector<uint8_t> g = mutate(rng, base, 0.03);
      std::vector<std::vector<uint8_t>> ctgs;
      size_t p = 0;
      for (int i = 0; i < 12 && p < L; i++) {
        size_t len = std::min<size_t>(L - p, 5000 + (rng() % 70000));
        std::vector<uint8_t> ctg(g.begin() + p, g.begin() + p + len);
        if (i % 5 == 1) {
          std::reverse(ctg.begin(), ctg.end());
          for (auto& b : ctg) b = b == 'A' ? 'T' : b == 'C' ? 'G' : b == 'G' ? 'C' : 'A';
        }
        if (i == 3) ctg.insert(ctg.end(), g.begin() + 20000, g.begin() + 60000);
        ctgs.push_back(std::move(ctg));
        p += len;
      }
      sk.push_back({"contigs", sketch_of("d_contigs", ctgs, sp)});
    }
    {  // two repeat-rich genomes: 16 copies of a 2.5 kb unit, each with its own point mutations, between unique spacers
      // (records carry many anchors in both roles: tiles of more than TILE anchors, records straddling emission rounds)
      const std::vector<uint8_t> unit = random_seq(rng, 2500);
      for (const char* name : {"e_repeats", "f_repeats"}) {
        std::vector<uint8_t> g = mutate(rng, base, 0.01);
        std::vector<uint8_t> block;
        for (int i = 0; i < 16; i++) {
          const std::vector<uint8_t> u = mutate(rng, unit, 0.01), sp300 = random_seq(rng, 300);
          block.insert(block.end(), u.begin(), u.end());
          block.insert(block.end(), sp300.begin(), sp300.end());
        }
        g.insert(g.begin() + 100000, block.begin(), block.end());
        sk.push_back({name, sketch_of(name, {g}, sp)});
      }
    }
    {  // an anchor-free stretch of 200 kb, longer than one tile of records at both c (about 128 kb at c = 125)
      std::vector<uint8_t> g = mutate(rng, base, 0.01);
      const std::vector<uint8_t> junk = random_seq(rng, 200000);
      std::copy(junk.begin(), junk.end(), g.begin() + 50000);
      sk.push_back({"g_longgap", sketch_of("g_longgap", {g}, sp)});
    }
    for (size_t i = 0; i < sk.size(); i++)
      for (size_t j = 0; j < sk.size(); j++) {
        if (i == j) continue;
        orc::ChainDebug d;
        orc::MapParams mp = orc::map_params_from_sketch(sk[i].second, cp, orc::get_model_id(c, true));
        orc::chain_seeds(sk[i].second, sk[j].second, mp, &d);
        std::string what = "c=" + std::to_string(c) + " " + sk[i].first + " x " + sk[j].first;
        CHECK(d.anchors.size() > 500, "%s: only %zu anchors", what.c_str(), d.anchors.size());
        std::vector<uint32_t> first = emu_chunk_first(d.anchors);
        CHECK(first == d.chunk_first, "%s: chunk boundaries differ (%zu vs %zu chunks)", what.c_str(), first.size(), d.chunk_first.size());
        const orc::Sketch& qrole = d.switched ? sk[i].second : sk[j].second;   // the iterated, chunked genome
        std::vector<uint32_t> tiled = emu_chunk_tiles(d.anchors, query_records(qrole), rng, what.c_str());
        CHECK(tiled == d.chunk_first, "%s: tiled chunk boundaries differ (%zu vs %zu chunks)", what.c_str(), tiled.size(), d.chunk_first.size());
        uint64_t bound = 0;                                   // the staging slice of the pair: sum of ceil(len / 20 kb)
        for (uint32_t len : qrole.contig_lengths) bound += (len + sk::FRAGMENT_LENGTH - 1) / sk::FRAGMENT_LENGTH;
        CHECK(d.chunk_first.size() - 1 <= bound, "%s: %zu chunks above the bound %llu", what.c_str(), d.chunk_first.size() - 1,
              (unsigned long long)bound);
        if (d.chunk_first.size() - 1 == bound) pairs_at_bound++;
        CHECK(!d.intervals_all.empty(), "%s: no intervals", what.c_str());
        check_intervals(d, what.c_str());
        pairs_checked++; chunks_checked += (int)d.chunk_first.size() - 1; intervals_checked += (int)d.intervals_all.size();
      }
  }
  // ---- 3. random-access WyRand == sequential stream; Lemire without the rejection loop
  {
    SeqWyRand s{7};
    for (uint64_t n = 0; n < 200000; n++) {
      uint64_t r = s.next();
      CHECK(r == sk::wyrand_at(7, n), "wyrand draw %llu", (unsigned long long)n);
      uint64_t bound = 1 + (rng() % 100000);
      bool rej = false;
      uint64_t v = sk::lemire_below(r, bound, &rej);
      __uint128_t m = (__uint128_t)r * bound;
      CHECK(v == (uint64_t)(m >> 64) && v < bound, "lemire value");
      bool would = (uint64_t)m < bound && (uint64_t)m < (0 - bound) % bound;
      CHECK(rej == would, "lemire rejection flag");
    }
  }
  // ---- 4. GBDT: flattened complete depth-3 trees == the oracle's predict, both models
  {
    auto b2f = [](uint32_t b) { float f; memcpy(&f, &b, 4); return f; };
    std::vector<float> thr[2], leaf[2];
    for (int i = 0; i < 1365; i++) { thr[0].push_back(b2f(tables::SK_GBDT_C125_THR[i])); thr[1].push_back(b2f(tables::SK_GBDT_C200_THR[i])); }
    for (int i = 0; i < 1560; i++) { leaf[0].push_back(b2f(tables::SK_GBDT_C125_LEAF[i])); leaf[1].push_back(b2f(tables::SK_GBDT_C200_LEAF[i])); }
    const unsigned char* feat[2] = {tables::SK_GBDT_C125_FEAT, tables::SK_GBDT_C200_FEAT};
    const float shrink[2] = {b2f(SK_GBDT_C125_SHRINK_BITS), b2f(SK_GBDT_C200_SHRINK_BITS)};
    const float bias[2] = {b2f(SK_GBDT_C125_BIAS_BITS), b2f(SK_GBDT_C200_BIAS_BITS)};
    const int ntrees[2] = {SK_GBDT_C125_NTREES, SK_GBDT_C200_NTREES};
    std::uniform_real_distribution<float> ani(88.f, 100.f), sd(0.f, 6.f), ql(500.f, 3e6f), cl(200.f, 20000.f);
    for (int it = 0; it < 200000; it++) {
      float x[5] = {ani(rng), sd(rng), ql(rng), ql(rng), cl(rng)};
      if (it % 7 == 0) x[2] = std::floor(x[2]);
      for (int m = 0; m < 2; m++) {
        float a = sk::gbdt_eval(feat[m], thr[m].data(), leaf[m].data(), ntrees[m], shrink[m], bias[m], x);
        float b = orc::gbdt_predict(m, x);
        CHECK(memcmp(&a, &b, 4) == 0, "gbdt model %d: %.9g vs %.9g", m, (double)a, (double)b);
      }
    }
  }
  CHECK(catchup_anchors > 0, "no input exercised the catch-up rule");
  CHECK(multi_round_tiles > 0, "no tile emitted its anchors in more than one round");
  CHECK(straddling_records > 0, "no record's anchors straddled two emission rounds");
  CHECK(empty_tiles > 0, "no tile without anchors");
  printf("tiles %ld (%ld without anchors, %ld with several rounds), rounds %ld, straddling records %ld, bracketings %ld, "
         "pairs at the chunk bound %d\n", tiles_run, empty_tiles, multi_round_tiles, rounds_run, straddling_records, bracketings_run,
         pairs_at_bound);
  printf("%d pairs, %d chunks, %d intervals, %ld catch-up anchors, %d failures\n", pairs_checked, chunks_checked, intervals_checked,
         catchup_anchors, failures);
  return failures ? 1 : 0;
}
