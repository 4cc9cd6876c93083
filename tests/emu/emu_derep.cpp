// Host emulation of sk_dereplicate's oriented screen predicate (skani_b200/csrc/derep_core.cuh: dr_screen_pass, the
// __host__ __device__ function dr_rows_kernel calls for every (row genome, slot genome) pair) checked against the CPU
// oracle's screen_refs as sk_screen_triangle applies it: the pair (i, j), i < j, is decided with row i as screen_refs' query.
// Development/test harness only; not a product path.
//
// For genome indices in both orders (the wave genome below or above the representative), the predicate is asked with either
// genome first (the representative-indexed screen asks with the row genome first; the order must not matter).  Marker
// counts 0, 19, 20, 21, 30, 107 and 1000 on either side, shared counts 0, 1, thr - 1, thr, thr + 1 and the full overlap
// (thr = max(floor(cutoff * min), 1)), screen_val 0 (-> 0.80) and 0.95, rescue on and off.  Also the index key and pair key.
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <vector>

#include "../../skani_b200/csrc/derep_core.cuh"
#include "../../oracle/skani_oracle.hpp"

static int failures = 0;
#define CHECK(cond, ...) do { if (!(cond)) { if (failures++ < 20) { fprintf(stderr, "FAIL %s:%d: ", __FILE__, __LINE__); fprintf(stderr, __VA_ARGS__); fprintf(stderr, "\n"); } } } while (0)

static double powi21(double x) {   // f64::powi(x, 21) as __powidf2 evaluates it (src/screen.rs:60,124,176)
  double r = 1.0, a = x;
  int b = sk::MARKER_K;
  while (true) {
    if (b & 1) r *= a;
    b /= 2;
    if (b == 0) break;
    a *= a;
  }
  return r;
}

// two sketches with card_a / card_b markers sharing exactly `shared` of them
static void make_pair(uint64_t card_a, uint64_t card_b, uint64_t shared, orc::Sketch& a, orc::Sketch& b) {
  a = orc::Sketch(); b = orc::Sketch();
  for (uint64_t i = 0; i < shared; i++) { a.marker_seeds.insert(i * 7919 + 1); b.marker_seeds.insert(i * 7919 + 1); }
  for (uint64_t i = shared; i < card_a; i++) a.marker_seeds.insert((1ull << 40) + i);
  for (uint64_t i = shared; i < card_b; i++) b.marker_seeds.insert((2ull << 40) + i);
}

int main() {
  const uint64_t cards[] = {0, 19, 20, 21, 30, 107, 1000};
  const double svs[] = {0., 0.95};
  long cases = 0, rescued_low = 0, not_rescued_high = 0, on_thr = 0;
  for (double sv0 : svs) {
    const double sv = sv0 == 0. ? orc::SEARCH_ANI_CUTOFF_DEFAULT : sv0;
    const double cutoff = powi21(sv);
    for (uint64_t cg : cards) {        // the wave (row) genome's markers
      for (uint64_t cr : cards) {      // the representative's markers
        const uint64_t mn = std::min(cg, cr);
        uint64_t thr = (uint64_t)(cutoff * (double)mn);
        if (thr < 1) thr = 1;
        std::vector<uint64_t> counts{0, 1, thr - 1, thr, thr + 1, mn};
        std::sort(counts.begin(), counts.end());
        counts.erase(std::unique(counts.begin(), counts.end()), counts.end());
        for (uint64_t cnt : counts) {
          if (cnt > mn) continue;
          orc::Sketch g, r;
          make_pair(cg, cr, cnt, g, r);
          orc::KmerToSketch* idx_g = orc::kmer_to_sketch_from_refs({&g});
          orc::KmerToSketch* idx_r = orc::kmer_to_sketch_from_refs({&r});
          for (int rescue = 0; rescue < 2; rescue++) {
            for (int g_low = 0; g_low < 2; g_low++) {   // genome indices: wave genome 3, representative 9 or the reverse
              const uint32_t gi = g_low ? 3 : 9, ri = g_low ? 9 : 3;
              // sk_screen_triangle's decision: screen_refs with the smaller index as the query, the larger as the one ref
              const orc::Sketch& q = g_low ? g : r;
              const orc::Sketch& ref = g_low ? r : g;
              std::vector<const orc::Sketch*> refs{&ref};
              const bool want = !orc::screen_refs(sv, g_low ? *idx_r : *idx_g, q, refs, rescue != 0).empty();
              const bool got = sk::dr_screen_pass(gi, cg, ri, cr, cnt, rescue != 0, cutoff);
              const bool got2 = sk::dr_screen_pass(ri, cr, gi, cg, cnt, rescue != 0, cutoff);
              CHECK(got == want && got2 == want, "sv %.2f genome %u (%lu markers) rep %u (%lu) count %lu rescue %d: got %d/%d want %d", sv, gi, cg,
                    ri, cr, cnt, rescue, got, got2, want);
              cases++;
              const uint64_t low_card = g_low ? cg : cr, high_card = g_low ? cr : cg;
              if (rescue && low_card < 20 && cnt == 0 && got) rescued_low++;
              if (rescue && high_card < 20 && low_card >= 20 && cnt == 0 && !got) not_rescued_high++;
              if (cnt == thr && mn > 0) on_thr++;
              CHECK(sk::dr_pair_key(gi, ri) == ((uint64_t)std::min(gi, ri) << 32 | std::max(gi, ri)), "pair key");
            }
          }
          orc::kmer_to_sketch_free(idx_g);
          orc::kmer_to_sketch_free(idx_r);
        }
      }
    }
  }
  for (uint64_t m : {0ull, 1ull, (1ull << 42) - 1})
    for (uint32_t s : {0u, 1u, sk::DR_MAX_SLOTS}) {
      const uint64_t k = sk::dr_key(m, s);
      CHECK(sk::dr_key_marker(k) == m && sk::dr_key_slot(k) == s && (k >> sk::DR_PREFIX_SHIFT) == (m >> (2 * sk::MARKER_K - sk::DR_PREFIX_BITS)),
            "key of marker %llu slot %u", (unsigned long long)m, s);
    }
  printf("%ld cases, %ld on a threshold, %ld rescued by the smaller index, %ld small larger indices not rescued, %d failures\n", cases, on_thr,
         rescued_low, not_rescued_high, failures);
  return failures ? 1 : 0;
}
