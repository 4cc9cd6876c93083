// Working-set planner of sk_triangle_store (skani_b200/csrc/ws_plan.hpp) on random pair graphs: clustered genomes, one giant
// component, mostly isolated genomes, skewed genome sizes.  Checks that every pair lands in exactly one working set, that a
// working set holds exactly the genomes its pairs touch and stays within the budget, that the plan is identical across
// runs, that chunk pairs appear exactly for the components over budget, and that a genome over budget / 2 is refused.
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

struct Case { std::vector<uint64_t> pairs; std::vector<uint64_t> bytes; uint64_t budget; };

std::vector<uint64_t> sizes(std::mt19937_64& rng, uint32_t n, bool skewed) {
  std::vector<uint64_t> b(n);
  for (auto& x : b) x = skewed ? (rng() % 8 == 0 ? 200000 + rng() % 800000 : 1000 + rng() % 20000) : 40000 + rng() % 20000;
  return b;
}

void add_pair(std::set<uint64_t>& s, uint32_t a, uint32_t b) {
  if (a == b) return;
  if (a > b) std::swap(a, b);
  s.insert(((uint64_t)a << 32) | b);
}

Case make_case(std::mt19937_64& rng, int kind) {
  Case c;
  std::set<uint64_t> ps;
  const uint32_t n = 50 + rng() % 400;
  c.bytes = sizes(rng, n, kind == 3);
  if (kind == 0 || kind == 3) {            // clusters of consecutive or scattered ids, dense inside
    const uint32_t k = 1 + rng() % 30;
    std::vector<uint32_t> cl(n);
    for (uint32_t g = 0; g < n; g++) cl[g] = (rng() % 2) ? g * k / n : (uint32_t)(rng() % k);
    for (uint32_t a = 0; a < n; a++)
      for (uint32_t b = a + 1; b < n; b++)
        if (cl[a] == cl[b] && rng() % 3 == 0) add_pair(ps, a, b);
  } else if (kind == 1) {                  // one giant component
    for (uint32_t g = 1; g < n; g++) add_pair(ps, g, (uint32_t)(rng() % g));
    for (uint32_t i = 0; i < n; i++) add_pair(ps, (uint32_t)(rng() % n), (uint32_t)(rng() % n));
  } else {                                 // mostly isolated genomes, a few pairs
    for (uint32_t i = 0; i < n / 20; i++) add_pair(ps, (uint32_t)(rng() % n), (uint32_t)(rng() % n));
  }
  c.pairs.assign(ps.begin(), ps.end());
  uint64_t mx = 0, total = 0;
  for (uint64_t b : c.bytes) { mx = std::max(mx, b); total += b; }
  // budgets from "everything fits" down to just above twice the largest genome
  const int r = (int)(rng() % 4);
  c.budget = r == 0 ? total + 1 : r == 1 ? std::max(2 * mx, total / 4) : r == 2 ? std::max(2 * mx, total / 16) : 2 * mx + rng() % 1000;
  return c;
}

}  // namespace

int main() {
  std::mt19937_64 rng(20260924);
  int cs = 0;
  long n_sets = 0, n_chunk_sets = 0, n_split = 0, n_refused = 0, n_pairs = 0, n_ffd_multi = 0;
  for (cs = 0; cs < 2000; cs++) {
    Case c = make_case(rng, cs % 4);
    const uint32_t n = (uint32_t)c.bytes.size();
    skws::Plan p1, p2;
    std::string e1, e2;
    const bool ok1 = skws::plan_working_sets(c.pairs, c.bytes, c.budget, p1, e1);
    const bool ok2 = skws::plan_working_sets(c.pairs, c.bytes, c.budget, p2, e2);
    CHECK(ok1 && ok2, "refused: %s", e1.c_str());
    if (!ok1) continue;
    // identical across runs
    bool same = p1.sets.size() == p2.sets.size() && p1.n_split_components == p2.n_split_components;
    for (size_t w = 0; same && w < p1.sets.size(); w++)
      same = p1.sets[w].genomes == p2.sets[w].genomes && p1.sets[w].pairs == p2.sets[w].pairs && p1.sets[w].bytes == p2.sets[w].bytes &&
             p1.sets[w].chunk_pair == p2.sets[w].chunk_pair;
    CHECK(same, "plan differs between runs");
    // reference components (independent union-find) and their bytes
    std::vector<uint32_t> par(n);
    for (uint32_t g = 0; g < n; g++) par[g] = g;
    auto f = [&](uint32_t x) { while (par[x] != x) x = par[x] = par[par[x]]; return x; };
    for (uint64_t q : c.pairs) { uint32_t a = f((uint32_t)(q >> 32)), b = f((uint32_t)q); if (a != b) par[a] = b; }
    std::vector<uint64_t> cbytes(n, 0);
    std::vector<char> in_pair(n, 0);
    for (uint64_t q : c.pairs) in_pair[q >> 32] = in_pair[(uint32_t)q] = 1;
    for (uint32_t g = 0; g < n; g++) if (in_pair[g]) cbytes[f(g)] += c.bytes[g];
    uint32_t split = 0;
    for (uint32_t g = 0; g < n; g++) if (in_pair[g] && f(g) == g && cbytes[g] > c.budget) split++;
    CHECK(split == p1.n_split_components, "split components %u, plan says %u", split, p1.n_split_components);
    // every pair exactly once; working sets within budget and holding exactly their pairs' genomes
    std::vector<uint64_t> all;
    for (const auto& ws : p1.sets) {
      CHECK(!ws.pairs.empty(), "empty working set");
      CHECK(ws.bytes <= c.budget, "working set of %llu bytes over the budget %llu", (unsigned long long)ws.bytes, (unsigned long long)c.budget);
      std::set<uint32_t> touched;
      for (uint64_t q : ws.pairs) { touched.insert((uint32_t)(q >> 32)); touched.insert((uint32_t)q); }
      CHECK(std::vector<uint32_t>(touched.begin(), touched.end()) == ws.genomes, "genome list is not the pairs' genomes");
      uint64_t b = 0;
      for (uint32_t g : ws.genomes) b += c.bytes[g];
      CHECK(b == ws.bytes, "byte count");
      // chunk pairs exactly for components over budget
      for (uint64_t q : ws.pairs) {
        const bool over = cbytes[f((uint32_t)q)] > c.budget;
        CHECK(over == ws.chunk_pair, "pair in a %s working set of a component %s budget", ws.chunk_pair ? "chunk-pair" : "packed", over ? "over" : "within");
      }
      all.insert(all.end(), ws.pairs.begin(), ws.pairs.end());
      n_sets++;
      n_chunk_sets += ws.chunk_pair;
      if (!ws.chunk_pair) {
        std::set<uint32_t> comps;
        for (uint32_t g : ws.genomes) comps.insert(f(g));
        n_ffd_multi += comps.size() > 1;
      }
    }
    std::sort(all.begin(), all.end());
    CHECK(all == c.pairs, "pairs: %zu in the plan, %zu screened", all.size(), c.pairs.size());
    n_pairs += (long)c.pairs.size();
    n_split += p1.n_split_components;
    // a genome over budget / 2 is refused (and only then)
    if (n) {
      std::vector<uint64_t> big = c.bytes;
      const uint32_t g = (uint32_t)(rng() % n);
      big[g] = c.budget / 2 + 1;
      skws::Plan p3;
      std::string e3;
      CHECK(!skws::plan_working_sets(c.pairs, big, c.budget, p3, e3) && e3.find("genome " + std::to_string(g)) != std::string::npos, "oversized genome accepted");
      big[g] = c.budget / 2;
      CHECK(skws::plan_working_sets(c.pairs, big, c.budget, p3, e3), "genome of exactly budget / 2 refused");
      n_refused++;
    }
  }
  printf("%d cases, %ld pairs, %ld working sets (%ld chunk pairs, %ld packing several components), %ld split components, %ld refusals, %d failures\n",
         cs, n_pairs, n_sets, n_chunk_sets, n_ffd_multi, n_split, n_refused, failures);
  return failures ? 1 : 0;
}
