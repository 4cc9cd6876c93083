// Pair components and the multi-context pair split (skani_b200/csrc/ws_plan.hpp: pair_components, partition_pairs) on random
// pair graphs: clustered genomes, one giant component, isolated pairs and an empty list, split over 1 to 12 contexts (also more
// contexts than pairs).  Checks that the groups of pair_components are the components of the pair graph (an independent
// union-find) in order of their smallest genome with sorted pairs, and that partition_pairs puts every pair in exactly one
// sorted list, keeps a component of at most cap pairs on one context, gives the same split across runs, and leaves no
// context's load more than cap above the smallest load.
// Development/test harness only.
#include <cstdio>
#include <random>
#include <set>
#include <string>
#include <vector>

#include "../../skani_b200/csrc/ws_plan.hpp"

namespace {

int failures = 0;
#define CHECK(cond, ...) do { if (!(cond)) { failures++; if (failures < 20) { fprintf(stderr, "case %d: ", cs); fprintf(stderr, __VA_ARGS__); fputc('\n', stderr); } } } while (0)

void add_pair(std::set<uint64_t>& s, uint32_t a, uint32_t b) {
  if (a == b) return;
  if (a > b) std::swap(a, b);
  s.insert(((uint64_t)a << 32) | b);
}

// kind 0: clusters of consecutive or scattered ids; 1: one giant component; 2: isolated pairs; 3: no pairs
std::vector<uint64_t> make_pairs(std::mt19937_64& rng, int kind, uint32_t n) {
  std::set<uint64_t> ps;
  if (kind == 0) {
    const uint32_t k = 1 + rng() % 40;
    std::vector<uint32_t> cl(n);
    for (uint32_t g = 0; g < n; g++) cl[g] = (rng() % 2) ? g * k / n : (uint32_t)(rng() % k);
    for (uint32_t a = 0; a < n; a++)
      for (uint32_t b = a + 1; b < n; b++)
        if (cl[a] == cl[b] && rng() % 3 == 0) add_pair(ps, a, b);
  } else if (kind == 1) {
    for (uint32_t g = 1; g < n; g++) add_pair(ps, g, (uint32_t)(rng() % g));
    for (uint32_t i = 0; i < n; i++) add_pair(ps, (uint32_t)(rng() % n), (uint32_t)(rng() % n));
  } else if (kind == 2) {
    std::vector<uint32_t> perm(n);
    for (uint32_t g = 0; g < n; g++) perm[g] = g;
    std::shuffle(perm.begin(), perm.end(), rng);
    for (uint32_t i = 0; i + 1 < n; i += 2) if (rng() % 2) add_pair(ps, perm[i], perm[i + 1]);
  }
  return std::vector<uint64_t>(ps.begin(), ps.end());
}

}  // namespace

int main() {
  std::mt19937_64 rng(20261018);
  int cs = 0;
  long n_pairs = 0, n_components = 0, n_whole = 0, n_cut = 0, n_more_contexts = 0;
  for (cs = 0; cs < 3000; cs++) {
    const uint32_t n = 2 + rng() % 300;
    const std::vector<uint64_t> pairs = make_pairs(rng, cs % 4, n);
    const uint32_t W = cs % 5 == 0 ? 1 : 2 + rng() % 11;
    // reference components (independent union-find)
    std::vector<uint32_t> par(n);
    for (uint32_t g = 0; g < n; g++) par[g] = g;
    auto f = [&](uint32_t x) { while (par[x] != x) x = par[x] = par[par[x]]; return x; };
    for (uint64_t q : pairs) { uint32_t a = f((uint32_t)(q >> 32)), b = f((uint32_t)q); if (a != b) par[a] = b; }
    // ---- pair_components: the groups are the components, in order of their smallest genome, pairs sorted inside
    const skws::PairComponents pc = skws::pair_components(pairs, n);
    CHECK(!pc.first.empty() && pc.first.front() == 0 && pc.first.back() == pairs.size(), "group bounds do not cover the pairs");
    std::vector<uint64_t> cat(pc.pairs);
    std::sort(cat.begin(), cat.end());
    CHECK(cat == pairs, "grouped pairs are not the input pairs");
    std::set<uint32_t> seen_comps;
    uint32_t prev_root = 0;
    for (size_t k = 0; k + 1 < pc.first.size(); k++) {
      const size_t p0 = pc.first[k], p1 = pc.first[k + 1];
      CHECK(p0 < p1, "empty group %zu", k);
      if (p0 >= p1) continue;
      const uint32_t comp = f((uint32_t)(pc.pairs[p0] >> 32));
      uint32_t root = UINT32_MAX;
      for (size_t i = p0; i < p1; i++) {
        CHECK(f((uint32_t)(pc.pairs[i] >> 32)) == comp, "group %zu mixes components", k);
        CHECK(i == p0 || pc.pairs[i - 1] < pc.pairs[i], "group %zu not sorted", k);
        root = std::min(root, (uint32_t)(pc.pairs[i] >> 32));
      }
      CHECK(seen_comps.insert(comp).second, "component split over two groups");
      CHECK(k == 0 || root > prev_root, "groups not in order of their smallest genome");
      prev_root = root;
    }
    n_components += (long)seen_comps.size();
    // ---- partition_pairs
    std::vector<std::vector<uint64_t>> s1, s2;
    skws::partition_pairs(pairs, W, n, s1);
    skws::partition_pairs(pairs, W, n, s2);
    CHECK(s1 == s2, "split differs between runs");
    CHECK(s1.size() == W, "%zu lists for %u contexts", s1.size(), W);
    const size_t cap = std::max<size_t>(1, (pairs.size() + 2 * (size_t)W - 1) / (2 * (size_t)W));
    std::vector<uint64_t> all;
    std::vector<uint32_t> ctx_of(n, UINT32_MAX);   // context of a genome's component when it is not cut (by component root)
    std::vector<size_t> comp_pairs(n, 0);
    for (uint64_t q : pairs) comp_pairs[f((uint32_t)q)]++;
    size_t lo = SIZE_MAX, hi = 0;
    for (uint32_t d = 0; d < W && d < s1.size(); d++) {
      const std::vector<uint64_t>& v = s1[d];
      for (size_t i = 1; i < v.size(); i++) CHECK(v[i - 1] < v[i], "context %u's list not sorted", d);
      all.insert(all.end(), v.begin(), v.end());
      for (uint64_t q : v) {
        const uint32_t c = f((uint32_t)q);
        if (comp_pairs[c] > cap) continue;
        CHECK(ctx_of[c] == UINT32_MAX || ctx_of[c] == d, "a component of %zu <= %zu pairs is on two contexts", comp_pairs[c], cap);
        ctx_of[c] = d;
      }
      lo = std::min(lo, v.size());
      hi = std::max(hi, v.size());
    }
    std::sort(all.begin(), all.end());
    CHECK(all == pairs, "pairs: %zu in the lists, %zu given", all.size(), pairs.size());
    CHECK(hi - lo <= cap, "loads %zu .. %zu differ by more than the cap %zu", lo, hi, cap);
    for (uint32_t g = 0; g < n; g++) if (f(g) == g && comp_pairs[g]) (comp_pairs[g] <= cap ? n_whole : n_cut)++;
    n_more_contexts += W > pairs.size();
    n_pairs += (long)pairs.size();
  }
  printf("%d cases, %ld pairs, %ld components (%ld kept whole, %ld cut), %ld with more contexts than pairs, %d failures\n", cs, n_pairs,
         n_components, n_whole, n_cut, n_more_contexts, failures);
  return failures ? 1 : 0;
}
