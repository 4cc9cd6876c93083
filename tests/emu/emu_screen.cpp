// Host emulation of the marker screen's predicate (skani_b200/csrc/sk_core.cuh: screen_pass / screen_row_rescued, the
// __host__ __device__ functions screen_rows_kernel and ts_rows_kernel call) checked against the CPU oracle's
// check_markers_quickly, screen_refs and screen_refs_indices.  Development/test harness only; not a product path.
//
// For every pair of marker counts (cards) of a grid that straddles each step of thr = max(floor(0.8^21 * mn), 1), every
// shared count of {0, 1, thr - 1, thr, thr + 1, full overlap}, screen_val in {0, 0.5, 0.8, 0.95, 0.99, 1.0} (0 replaced
// by 0.80 first, as every caller does), both rescue_small values and both argument orders, two oracle sketches with
// exactly those markers are built and every mode of the device predicate must give the oracle's answer:
//   mode 0 / 1  : check_markers_quickly(a, b, sv, rescue_small) / (.., false)      (symmetric: called in both orders)
//   mode 2 / tri: screen_refs(sv, idx{col}, row, {col}, rescue_small)               (the row is screen_refs' query)
//   mode 3      : screen_refs_indices(sv, idx{col}, row, {col})
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <vector>

#include "../../skani_b200/csrc/sk_core.cuh"
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

// two sketches with card_a / card_b markers sharing exactly `shared` of them (markers are distinct and < 2^42)
static void make_pair(uint64_t card_a, uint64_t card_b, uint64_t shared, orc::Sketch& a, orc::Sketch& b) {
  a = orc::Sketch(); b = orc::Sketch();
  for (uint64_t i = 0; i < shared; i++) { a.marker_seeds.insert(i * 7919 + 1); b.marker_seeds.insert(i * 7919 + 1); }
  for (uint64_t i = shared; i < card_a; i++) a.marker_seeds.insert((1ull << 40) + i);
  for (uint64_t i = shared; i < card_b; i++) b.marker_seeds.insert((2ull << 40) + i);
}

// screen_refs / screen_refs_indices of `row` against the one-sketch ref list {col} (idx = its inverted index)
static bool oracle_index(const orc::Sketch& row, const orc::Sketch& col, const orc::KmerToSketch& idx, double sv, int mode, bool rescue) {
  std::vector<const orc::Sketch*> refs{&col};
  auto pass = mode == sk::MODE_INDEX_NORESCUE ? orc::screen_refs_indices(sv, idx, row, refs) : orc::screen_refs(sv, idx, row, refs, rescue);
  return !pass.empty();
}

int main() {
  std::vector<uint64_t> cards;
  for (uint64_t c = 0; c <= 25; c++) cards.push_back(c);
  for (uint64_t c = 105; c <= 112; c++) cards.push_back(c);
  for (uint64_t c = 214; c <= 220; c++) cards.push_back(c);
  for (uint64_t c = 323; c <= 330; c++) cards.push_back(c);
  cards.push_back(1000); cards.push_back(5000);
  const double svs[] = {0., 0.5, 0.8, 0.95, 0.99, 1.0};
  long cases = 0, on_thr = 0, thr_quick_only = 0, rescued_row = 0, small_col_not_rescued = 0;
  for (double sv0 : svs) {
    const double sv = sv0 == 0. ? orc::SEARCH_ANI_CUTOFF_DEFAULT : sv0;
    const double cutoff = powi21(sv);
    for (uint64_t ca : cards) {
      for (uint64_t cb : cards) {
        const uint64_t mn = ca < cb ? ca : cb;
        uint64_t thr = (uint64_t)(cutoff * (double)mn);
        if (thr < 1) thr = 1;
        std::vector<uint64_t> counts{0, 1, thr - 1, thr, thr + 1, mn};
        std::sort(counts.begin(), counts.end());
        counts.erase(std::unique(counts.begin(), counts.end()), counts.end());
        for (uint64_t cnt : counts) {
          if (cnt > mn) continue;
          orc::Sketch a, b;
          make_pair(ca, cb, cnt, a, b);
          orc::KmerToSketch* idx_a = orc::kmer_to_sketch_from_refs({&a});
          orc::KmerToSketch* idx_b = orc::kmer_to_sketch_from_refs({&b});
          for (int rescue = 0; rescue < 2; rescue++) {
            for (int order = 0; order < 2; order++) {   // (row, col) = (a, b) and (b, a)
              const orc::Sketch& row = order ? b : a;
              const orc::Sketch& col = order ? a : b;
              const uint64_t cr = order ? cb : ca, cc = order ? ca : cb;
              const orc::KmerToSketch& idx_col = order ? *idx_a : *idx_b;
              // modes 0 / 1: both argument orders of check_markers_quickly must agree with the device predicate
              for (int mode = 0; mode < 2; mode++) {
                const bool rs = mode == 0 && rescue;
                const bool want = orc::check_markers_quickly(row, col, sv, rs);
                const bool want2 = orc::check_markers_quickly(col, row, sv, rs);
                const bool got = sk::screen_pass(mode, rescue != 0, cr, cc, cnt, cutoff);
                CHECK(got == want && want == want2, "mode %d sv %.2f cards %lu/%lu count %lu rescue %d: got %d want %d/%d", mode, sv, cr, cc, cnt,
                      rescue, got, want, want2);
                cases++;
              }
              bool tri_got = false, tri_want = false;
              for (int mode : {(int)sk::MODE_INDEX, (int)sk::MODE_INDEX_NORESCUE, (int)sk::MODE_TRIANGLE}) {
                const int omode = mode == sk::MODE_TRIANGLE ? sk::MODE_INDEX : mode;   // the triangle screens with screen_refs
                const bool want = oracle_index(row, col, idx_col, sv, omode, rescue != 0);
                const bool got = sk::screen_pass(mode, rescue != 0, cr, cc, cnt, cutoff);
                CHECK(got == want, "mode %d sv %.2f cards row %lu col %lu count %lu rescue %d: got %d want %d", mode, sv, cr, cc, cnt, rescue,
                      got, want);
                if (mode == sk::MODE_TRIANGLE) { tri_got = got; tri_want = want; }
                cases++;
              }
              CHECK(sk::screen_row_rescued(sk::MODE_TRIANGLE, rescue != 0, cr) == (rescue && cr < 20), "row rescue, card %lu", cr);
              if (rescue && cr < 20 && cnt == 0 && tri_got && tri_want) rescued_row++;
              if (rescue && cc < 20 && cr >= 20 && cnt == 0 && !tri_got && !tri_want) small_col_not_rescued++;
              if (cnt == thr && mn > 0) {
                on_thr++;
                const bool q = sk::screen_pass(sk::MODE_QUICK_NORESCUE, false, cr, cc, cnt, cutoff);
                const bool t = sk::screen_pass(sk::MODE_INDEX_NORESCUE, false, cr, cc, cnt, cutoff);
                if (q && !t) thr_quick_only++;
              }
            }
          }
          orc::kmer_to_sketch_free(idx_a);
          orc::kmer_to_sketch_free(idx_b);
        }
      }
    }
  }
  printf("%ld cases, %ld on a threshold (%ld pass the quick screen and fail screen_refs), %ld rescued rows without a shared marker, "
         "%ld small columns that do not rescue their row, %d failures\n",
         cases, on_thr, thr_quick_only, rescued_row, small_col_not_rescued, failures);
  return failures ? 1 : 0;
}
