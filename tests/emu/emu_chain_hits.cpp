// Host emulation of the chain front end's compacted hit stream (skani_b200/csrc/chain.cu), checked against the CPU oracle
// and against a plain record-order pass.  Development/test harness only: it validates the arrangement without a GPU.
//   1. probe_kernel's per-tile compaction: every (item, warp) group of 32 consecutive records is one ballot; the groups'
//      counts are offset in record order, so a tile's hit entries (ref group start, record index in the tile | nh << 10)
//      land in slots [tile * TILE, tile * TILE + tile_hits) in record order; the "counted" bits go to rec_cnt, one word per
//      group;
//   2. the pair-local exclusive offsets of the tiles' hit counts;
//   3. chunk_anchor_kernel stepping over TILE hits at a time: each slot finds its source tile with the kernel's lock-step
//      search, reads its entry and gathers its record's position and contig; the chunk closed forms of chain_core.cuh run
//      with carries across steps and anchors are emitted in rounds of TILE;
//   4. chunkstat_kernel's lookup of the counted bit.
// Inputs: the query-role records of oracle pairs (plain, gappy, multi-contig, repeat-rich genomes; c = 125 and 30), and
// constructed hit patterns: a step whose hits span many tiles with runs of hit-free tiles, a tile in which every record
// hits, a pair whose only hit is its last record, hit counts that are and are not multiples of TILE, a contig boundary
// on a step boundary, a record with `band` anchors straddling a step boundary and an emission round.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <random>
#include <string>
#include <vector>

#include "../../skani_b200/csrc/chain_core.cuh"
#include "../../oracle/skani_oracle.hpp"

static int failures = 0;
#define CHECK(cond, ...) do { if (!(cond)) { failures++; fprintf(stderr, "FAIL %s:%d: ", __FILE__, __LINE__); fprintf(stderr, __VA_ARGS__); fprintf(stderr, "\n"); } } while (0)

constexpr uint32_t TILE = 1024, CT = 256, ITEMS = 4;
static long steps_run = 0, steps_multi_tile = 0, empty_tiles_skipped = 0, full_tiles = 0, straddle_step = 0,
            straddle_round = 0, ctg_on_step = 0, exact_multiple = 0, partial_last = 0;

struct Rec { uint32_t ctg, pos, nh, rs, counted; };
struct Out {                      // what chunk_anchor_kernel writes for a pair
  std::vector<uint32_t> anc_rec;  // per anchor: its record | its index in the record << 16 (test-local packing)
  std::vector<uint32_t> first;    // chunk starts (pair-local anchor index)
  std::vector<int64_t> lo, hi;    // chunk windows (the last chunk patched to the last hit's position)
};

// the chunk closed forms over hit records in record order, one record at a time (no tiles, no steps)
static Out plain_pass(const std::vector<Rec>& rec) {
  Out o;
  sk::FirstState cF; cF.valid = 0; cF.ctg = 0; cF.p0 = 0; cF.a0 = 0;
  sk::MinState cM; cM.valid = 0; cM.ctg = 0; cM.v = 0;
  uint32_t A = 0, last_q = 0, last_c = 0;
  for (uint32_t r = 0; r < rec.size(); r++) {
    const Rec& x = rec[r];
    if (!x.nh) continue;
    sk::FirstState f; f.valid = 1; f.ctg = x.ctg; f.p0 = x.pos; f.a0 = A;
    cF = sk::FirstOp()(cF, f);
    const uint32_t need = sk::chunk_need(x.pos, cF.p0), al = A - cF.a0;
    const bool has_prev = cM.valid && cM.ctg == x.ctg;
    const uint32_t clf = sk::chunk_local_of(al, has_prev, cM.v, need);
    const uint32_t st = sk::record_starts_chunk(al, has_prev, cM.v, clf);
    for (uint32_t u = 0; u < x.nh; u++) {
      o.anc_rec.push_back(r | (u << 16));
      const uint32_t cl = sk::anchor_chunk_local(clf, u, need);
      if (sk::anchor_starts_chunk(clf, u, need, st != 0)) {
        o.first.push_back(A + u);
        o.lo.push_back(sk::chunk_window_lo(cF.p0, cl)); o.hi.push_back(sk::chunk_window_hi(cF.p0, cl));
      }
      last_c = (uint32_t)o.first.size() - 1;
    }
    last_q = x.pos;
    sk::MinState m; m.valid = 1; m.ctg = x.ctg; m.v = sk::record_min_key(need, al, x.nh);
    cM = sk::MinOp()(cM, m);
    A += x.nh;
  }
  if (!o.first.empty()) o.hi[last_c] = last_q;
  return o;
}

// probe_kernel's output for one pair: hit slots (n_rec of them), tile_hits, rec_cnt (TILE / 32 words per tile)
static void probe_emu(const std::vector<Rec>& rec, std::vector<uint64_t>& hit, std::vector<uint32_t>& tile_hits,
                      std::vector<uint32_t>& rec_cnt) {
  const uint32_t n = (uint32_t)rec.size(), n_t = (n + TILE - 1) / TILE;
  hit.assign(n, ~0ull); tile_hits.assign(n_t, 0); rec_cnt.assign((size_t)n_t * (TILE / 32), 0);
  for (uint32_t j = 0; j < n_t; j++) {
    uint32_t hm[ITEMS * CT / 32], gcnt[ITEMS * CT / 32], goff[ITEMS * CT / 32];
    for (uint32_t it = 0; it < ITEMS; it++)
      for (uint32_t w = 0; w < CT / 32; w++) {
        const uint32_t g = it * (CT / 32) + w;
        uint32_t m = 0, c = 0;
        for (uint32_t lane = 0; lane < 32; lane++) {      // thread w * 32 + lane, item it: record it * CT + threadIdx.x
          const uint32_t t = j * TILE + it * CT + w * 32 + lane;
          if (t < n && rec[t].nh) m |= 1u << lane;
          if (t < n && rec[t].counted) c |= 1u << lane;
        }
        hm[g] = m; gcnt[g] = __builtin_popcount(m);
        rec_cnt[(size_t)j * (TILE / 32) + g] = c;
      }
    uint32_t run = 0;
    for (uint32_t g = 0; g < ITEMS * CT / 32; g++) { goff[g] = run; run += gcnt[g]; }
    tile_hits[j] = run;
    if (run == TILE) full_tiles++;
    for (uint32_t g = 0; g < ITEMS * CT / 32; g++)
      for (uint32_t lane = 0; lane < 32; lane++) {
        if (!((hm[g] >> lane) & 1u)) continue;
        const uint32_t idx = g * 32 + lane;                 // = it * CT + threadIdx.x
        const uint32_t slot = goff[g] + __builtin_popcount(hm[g] & ((1u << lane) - 1u));
        const Rec& x = rec[j * TILE + idx];
        hit[(size_t)j * TILE + slot] = (uint64_t)x.rs | (uint64_t)(idx | (x.nh << 10)) << 32;
      }
  }
}

// chunk_anchor_kernel over the probe's output
static Out step_pass(const std::vector<Rec>& rec, const std::vector<uint64_t>& hit, std::vector<uint32_t> hoff) {
  const uint32_t n_t = (uint32_t)hoff.size();
  uint32_t H = 0;
  for (uint32_t j = 0; j < n_t; j++) { const uint32_t c = hoff[j]; hoff[j] = H; H += c; }   // in place, as the kernel
  Out o;
  sk::FirstState cF; cF.valid = 0; cF.ctg = 0; cF.p0 = 0; cF.a0 = 0;
  sk::MinState cM; cM.valid = 0; cM.ctg = 0; cM.v = 0;
  uint32_t carryA = 0, last_q = 0, last_c = 0, prev_ctg = ~0u;
  uint64_t A_total = 0;
  for (const Rec& x : rec) A_total += x.nh;
  for (uint32_t h0 = 0; h0 < H; h0 += TILE) {
    steps_run++;
    std::vector<uint32_t> srec(TILE, 0), nh(TILE, 0), aoff(TILE, 0);
    uint32_t jmin = ~0u, jmax = 0;
    for (uint32_t i = 0; i < TILE; i++) {
      const uint32_t h = h0 + i;
      if (h >= H) continue;                                 // padding slot: nh = 0
      uint32_t j = 0;
      for (uint32_t len = n_t; len > 1;) {                  // the kernel's search: the last tile with hoff[j] <= h
        const uint32_t half = len >> 1;
        if (hoff[j + half] <= h) j += half;
        len -= half;
      }
      jmin = std::min(jmin, j); jmax = std::max(jmax, j);
      const uint64_t e = hit[(size_t)j * TILE + (h - hoff[j])];
      CHECK(e != ~0ull, "step %u slot %u reads an unwritten hit slot", h0 / TILE, i);
      const uint32_t ey = (uint32_t)(e >> 32);
      srec[i] = j * TILE + (ey & (TILE - 1));
      nh[i] = ey >> 10;
      CHECK(srec[i] < rec.size() && nh[i] == rec[srec[i]].nh && (uint32_t)e == rec[srec[i]].rs, "hit %u: entry differs from its record", h);
    }
    if (jmax > jmin + 1) steps_multi_tile++;
    for (uint32_t j = jmin + 1; j < jmax; j++) if (hoff[j] == hoff[j + 1]) empty_tiles_skipped++;
    if (h0 > 0 && rec[srec[0]].ctg != prev_ctg) ctg_on_step++;
    uint32_t aggA = 0;
    for (uint32_t i = 0; i < TILE; i++) { aoff[i] = carryA + aggA; aggA += nh[i]; }
    for (uint32_t i = 0; i < TILE; i++) {
      if (!nh[i]) continue;
      const Rec& x = rec[srec[i]];
      sk::FirstState f; f.valid = 1; f.ctg = x.ctg; f.p0 = x.pos; f.a0 = aoff[i];
      cF = sk::FirstOp()(cF, f);
      const uint32_t need = sk::chunk_need(x.pos, cF.p0), al = aoff[i] - cF.a0;
      const bool has_prev = cM.valid && cM.ctg == x.ctg;
      const uint32_t clf = sk::chunk_local_of(al, has_prev, cM.v, need);
      const uint32_t st = sk::record_starts_chunk(al, has_prev, cM.v, clf);
      const uint32_t lo = aoff[i] - carryA;
      if (lo / TILE != (lo + nh[i] - 1) / TILE) straddle_round++;
      for (uint32_t u = 0; u < nh[i]; u++) {
        o.anc_rec.push_back(srec[i] | (u << 16));
        const uint32_t cl = sk::anchor_chunk_local(clf, u, need);
        if (sk::anchor_starts_chunk(clf, u, need, st != 0)) {
          o.first.push_back(aoff[i] + u);
          o.lo.push_back(sk::chunk_window_lo(cF.p0, cl)); o.hi.push_back(sk::chunk_window_hi(cF.p0, cl));
        }
        if (aoff[i] + u + 1 == A_total) { last_q = x.pos; last_c = (uint32_t)o.first.size() - 1; }
      }
      sk::MinState m; m.valid = 1; m.ctg = x.ctg; m.v = sk::record_min_key(need, al, nh[i]);
      cM = sk::MinOp()(cM, m);
      prev_ctg = x.ctg;
    }
    if (h0 + TILE < H && nh[TILE - 1] > 1 && rec[srec[TILE - 1]].nh > 1) straddle_step++;   // last hit of a full step
    carryA += aggA;
  }
  if (H % TILE == 0 && H) exact_multiple++;
  else if (H) partial_last++;
  if (!o.first.empty()) o.hi[last_c] = last_q;
  return o;
}

static void check_pair(const std::vector<Rec>& rec, const char* what, const std::vector<uint32_t>* oracle_first) {
  std::vector<uint64_t> hit;
  std::vector<uint32_t> tile_hits, rec_cnt;
  probe_emu(rec, hit, tile_hits, rec_cnt);
  // chunkstat_kernel's lookup (the pair's words start at tile_off * TILE / 32; here the pair is alone: 0)
  for (uint32_t t = 0; t < rec.size(); t++)
    CHECK(((rec_cnt[t >> 5] >> (t & 31u)) & 1u) == rec[t].counted, "%s: counted bit of record %u", what, t);
  // each tile's slots hold its hit records in record order
  for (uint32_t j = 0, k = 0; j < tile_hits.size(); j++)
    for (uint32_t s = 0; s < tile_hits[j]; s++) {
      while (!rec[k].nh) k++;
      CHECK((uint32_t)(hit[(size_t)j * TILE + s] >> 32 & (TILE - 1)) + j * TILE == k, "%s: tile %u slot %u out of record order", what, j, s);
      k++;
    }
  const Out a = plain_pass(rec), b = step_pass(rec, hit, tile_hits);
  CHECK(a.anc_rec == b.anc_rec, "%s: anchors differ (%zu vs %zu)", what, a.anc_rec.size(), b.anc_rec.size());
  CHECK(a.first == b.first && a.lo == b.lo && a.hi == b.hi, "%s: chunks differ (%zu vs %zu)", what, a.first.size(), b.first.size());
  if (oracle_first) {
    std::vector<uint32_t> f = b.first;
    f.push_back((uint32_t)b.anc_rec.size());
    CHECK(f == *oracle_first, "%s: chunk boundaries differ from the oracle (%zu vs %zu)", what, f.size(), oracle_first->size());
  }
}

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
// the query-role records in (contig, pos) order with the anchors the oracle found for each
static std::vector<Rec> records_of(const orc::Sketch& s, const std::vector<orc::Anchor>& an) {
  std::vector<Rec> v;
  const orc::KmerSeeds& m = s.kmer_seeds_k;
  orc::SeedPosition tmp;
  for (size_t i = 0; i < m.capacity(); i++) {
    if (!m.slot_used(i)) continue;
    const orc::SeedPosition* p;
    const size_t n = s.get_seed_positions(m.slot_key(i), &p, &tmp);
    for (size_t a = 0; a < n; a++) v.push_back({p[a].contig_index_canonical >> 1, p[a].pos, 0, 0, 1});
  }
  std::sort(v.begin(), v.end(), [](const Rec& a, const Rec& b) { return a.ctg != b.ctg ? a.ctg < b.ctg : a.pos < b.pos; });
  v.erase(std::unique(v.begin(), v.end(), [](const Rec& a, const Rec& b) { return a.ctg == b.ctg && a.pos == b.pos; }), v.end());
  for (size_t a = 0, r = 0; a < an.size(); a++) {
    while (r < v.size() && (v[r].ctg != an[a].query_contig || v[r].pos != an[a].query_pos)) r++;
    if (r == v.size()) { CHECK(false, "anchor %zu has no query record", a); break; }
    v[r].nh++;
    v[r].rs = (uint32_t)(r * 7 + 3);                        // a stand-in group start: only its round trip is checked
  }
  return v;
}

// constructed pairs: records every 125 bp; nh from a pattern, contig breaks where asked
static std::vector<Rec> constructed(uint32_t n, const std::vector<uint32_t>& nh_of, const std::vector<uint32_t>& ctg_starts,
                                    std::mt19937_64& rng) {
  std::vector<Rec> v(n);
  uint32_t ctg = 0, pos = 0;
  for (uint32_t t = 0; t < n; t++) {
    if (std::find(ctg_starts.begin(), ctg_starts.end(), t) != ctg_starts.end()) { ctg++; pos = 0; }
    pos += 60 + (uint32_t)(rng() % 130);
    v[t] = {ctg, pos, nh_of[t], t ^ 0x5a5a5u, (uint32_t)(nh_of[t] > 0 || rng() % 3 != 0)};
  }
  return v;
}

int main() {
  std::mt19937_64 rng(20261017);
  int oracle_pairs = 0, constructed_pairs = 0;
  // ---- oracle pairs (the shapes of emu_chain.cpp at both c)
  for (uint64_t c : {125ull, 30ull}) {
    orc::SketchParams sp; sp.c = c; sp.k = 15; sp.marker_c = c == 30 ? 200 : 1000;
    orc::CommandParams cp;
    const size_t L = 400000;
    std::vector<uint8_t> base = random_seq(rng, L);
    std::vector<std::pair<std::string, orc::Sketch>> sk;
    sk.push_back({"plain", sketch_of("a_plain", {mutate(rng, base, 0.01)}, sp)});
    sk.push_back({"divergent", sketch_of("b_div", {mutate(rng, base, 0.06)}, sp)});
    {
      std::vector<uint8_t> g = mutate(rng, base, 0.02);
      const std::vector<uint8_t> junk = random_seq(rng, 200000);
      std::copy(junk.begin(), junk.end(), g.begin() + 50000);
      sk.push_back({"longgap", sketch_of("c_longgap", {g}, sp)});
    }
    {
      std::vector<uint8_t> g = mutate(rng, base, 0.03);
      std::vector<std::vector<uint8_t>> ctgs;
      for (size_t p = 0; p < L;) {
        const size_t len = std::min<size_t>(L - p, 5000 + (rng() % 70000));
        ctgs.emplace_back(g.begin() + p, g.begin() + p + len);
        p += len;
      }
      sk.push_back({"contigs", sketch_of("d_contigs", ctgs, sp)});
    }
    {
      const std::vector<uint8_t> unit = random_seq(rng, 2500);
      std::vector<uint8_t> g = mutate(rng, base, 0.01), block;
      for (int i = 0; i < 16; i++) {
        const std::vector<uint8_t> u = mutate(rng, unit, 0.01), s300 = random_seq(rng, 300);
        block.insert(block.end(), u.begin(), u.end());
        block.insert(block.end(), s300.begin(), s300.end());
      }
      g.insert(g.begin() + 100000, block.begin(), block.end());
      sk.push_back({"repeats", sketch_of("e_repeats", {g}, sp)});
    }
    for (size_t i = 0; i < sk.size(); i++)
      for (size_t j = 0; j < sk.size(); j++) {
        if (i == j) continue;
        orc::ChainDebug d;
        orc::MapParams mp = orc::map_params_from_sketch(sk[i].second, cp, orc::get_model_id(c, true));
        orc::chain_seeds(sk[i].second, sk[j].second, mp, &d);
        const orc::Sketch& qrole = d.switched ? sk[i].second : sk[j].second;
        const std::string what = "c=" + std::to_string(c) + " " + sk[i].first + " x " + sk[j].first;
        check_pair(records_of(qrole, d.anchors), what.c_str(), &d.chunk_first);
        oracle_pairs++;
      }
  }
  // ---- constructed hit patterns (band 16 = the chain band at c = 125)
  const uint32_t band = 16;
  {  // one step's 1 024 hits spread over ~40 tiles, tiles 3..9 without hits; then a tile where every record hits
    const uint32_t n = 48 * TILE;
    std::vector<uint32_t> nh(n, 0);
    for (uint32_t t = 0; t < 40 * TILE; t++) if ((t / TILE < 3 || t / TILE > 9) && rng() % 30 == 0) nh[t] = 1 + (uint32_t)(rng() % 3);
    for (uint32_t t = 41 * TILE; t < 42 * TILE; t++) nh[t] = 1;
    check_pair(constructed(n, nh, {5000, 30000}, rng), "sparse steps + full tile", nullptr);
    constructed_pairs++;
  }
  {  // the only hit is the pair's last record
    const uint32_t n = 3 * TILE + 17;
    std::vector<uint32_t> nh(n, 0);
    nh[n - 1] = 2;
    check_pair(constructed(n, nh, {}, rng), "last record only", nullptr);
    constructed_pairs++;
  }
  for (uint32_t H : {3 * TILE, 3 * TILE + 1, 2 * TILE - 1}) {   // hit counts on and off a multiple of TILE
    const uint32_t n = 5 * TILE + 100;
    std::vector<uint32_t> nh(n, 0), idx(n);
    for (uint32_t t = 0; t < n; t++) idx[t] = t;
    std::shuffle(idx.begin(), idx.end(), rng);
    for (uint32_t k = 0; k < H; k++) nh[idx[k]] = 1 + (uint32_t)(rng() % 2);
    check_pair(constructed(n, nh, {2 * TILE}, rng), ("H=" + std::to_string(H)).c_str(), nullptr);
    constructed_pairs++;
  }
  {  // a contig starts at the first hit of step 1; the last hit of step 0 carries `band` anchors and straddles a round
    const uint32_t n = 6 * TILE;
    std::vector<uint32_t> nh(n, 0);
    uint32_t k = 0, first_of_step1 = 0;
    for (uint32_t t = 0; t < n; t++) {
      if (rng() % 2) continue;
      nh[t] = (k == TILE - 1) ? band : 1 + (uint32_t)(rng() % 4);
      if (k == TILE) first_of_step1 = t;
      k++;
    }
    check_pair(constructed(n, nh, {first_of_step1}, rng), "contig on step boundary", nullptr);
    constructed_pairs++;
  }
  CHECK(steps_multi_tile > 0 && empty_tiles_skipped > 0, "no step spanned several tiles across hit-free tiles");
  CHECK(full_tiles > 0, "no tile in which every record hits");
  CHECK(exact_multiple > 0 && partial_last > 0, "hit counts on and off a multiple of TILE not both reached");
  CHECK(ctg_on_step > 0, "no contig boundary on a step boundary");
  CHECK(straddle_step > 0 && straddle_round > 0, "no record straddling a step boundary and an emission round");
  printf("steps %ld (%ld over several tiles, %ld hit-free tiles passed), full tiles %ld, contig on step boundary %ld, "
         "straddling: step %ld round %ld, H multiple of TILE %ld / not %ld\n", steps_run, steps_multi_tile, empty_tiles_skipped,
         full_tiles, ctg_on_step, straddle_step, straddle_round, exact_multiple, partial_last);
  printf("%d oracle pairs, %d constructed pairs, %d failures\n", oracle_pairs, constructed_pairs, failures);
  return failures ? 1 : 0;
}
