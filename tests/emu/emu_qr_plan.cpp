// Query x reference working-set planner of sk_query_ref_store (plan_query_ref_working_sets, skani_b200/csrc/ws_plan.hpp) on
// random bipartite pair graphs: clustered, one query hitting every reference, every query hitting one reference, skewed genome
// sizes, and few queries against many references.  Checks that every pair lands in exactly one working set, that a working
// set's reference and query lists are ascending, in range and exactly the genomes its pairs touch, that it stays within the
// budget, that the plan is identical across runs, that a genome over budget / 2 on either side is refused, and that with one
// query against many references every reference is gathered exactly once (with two or three, at most once per query).
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

struct Case { std::vector<uint64_t> pairs, rbytes, qbytes; uint64_t budget; int kind; };

std::vector<uint64_t> sizes(std::mt19937_64& rng, uint32_t n, bool skewed) {
  std::vector<uint64_t> b(n);
  for (auto& x : b) x = skewed ? (rng() % 8 == 0 ? 200000 + rng() % 800000 : 1000 + rng() % 20000) : 40000 + rng() % 20000;
  return b;
}

constexpr int KINDS = 5;   // 0 clustered, 1 one query hits every reference, 2 every query hits one reference, 3 skewed, 4 few queries

Case make_case(std::mt19937_64& rng, int kind) {
  Case c;
  c.kind = kind;
  std::set<uint64_t> ps;
  const uint32_t NR = 20 + rng() % 300, NQ = kind == 4 ? (rng() % 2 ? 1 : 2 + rng() % 2) : 1 + rng() % 200;
  c.rbytes = sizes(rng, NR, kind == 3);
  c.qbytes = sizes(rng, NQ, kind == 3);
  auto add = [&](uint32_t r, uint32_t q) { ps.insert(((uint64_t)r << 32) | q); };
  if (kind == 0 || kind == 3) {            // clusters of consecutive or scattered ids on both sides
    const uint32_t k = 1 + rng() % 30;
    auto cl = [&](uint32_t g, uint32_t n) { return (rng() % 2) ? g * k / n : (uint32_t)(rng() % k); };
    std::vector<uint32_t> cr(NR), cq(NQ);
    for (uint32_t r = 0; r < NR; r++) cr[r] = cl(r, NR);
    for (uint32_t q = 0; q < NQ; q++) cq[q] = cl(q, NQ);
    for (uint32_t r = 0; r < NR; r++)
      for (uint32_t q = 0; q < NQ; q++)
        if (cr[r] == cq[q] && rng() % 3 == 0) add(r, q);
  } else if (kind == 1) {                  // one query hits every reference, a few other pairs
    const uint32_t q0 = (uint32_t)(rng() % NQ);
    for (uint32_t r = 0; r < NR; r++) add(r, q0);
    for (uint32_t i = 0; i < NQ / 4; i++) add((uint32_t)(rng() % NR), (uint32_t)(rng() % NQ));
  } else if (kind == 2) {                  // every query hits one reference
    const uint32_t r0 = (uint32_t)(rng() % NR);
    for (uint32_t q = 0; q < NQ; q++) add(r0, q);
  } else {                                 // few queries, each against most references
    for (uint32_t q = 0; q < NQ; q++)
      for (uint32_t r = 0; r < NR; r++)
        if (rng() % 4) add(r, q);
  }
  c.pairs.assign(ps.begin(), ps.end());
  uint64_t mx = 0, total = 0;
  for (auto* v : {&c.rbytes, &c.qbytes})
    for (uint64_t b : *v) { mx = std::max(mx, b); total += b; }
  // budgets from "everything fits" down to just above twice the largest genome
  const int r = (int)(rng() % 4);
  c.budget = r == 0 ? std::max(total + 1, 2 * mx) : r == 1 ? std::max(2 * mx, total / 4) : r == 2 ? std::max(2 * mx, total / 16) : 2 * mx + rng() % 1000;
  return c;
}

bool ascending(const std::vector<uint32_t>& v, uint32_t n) {
  for (size_t i = 0; i < v.size(); i++)
    if (v[i] >= n || (i && v[i] <= v[i - 1])) return false;
  return true;
}

}  // namespace

int main() {
  std::mt19937_64 rng(20261015);
  int cs = 0;
  long n_sets = 0, n_chunk_sets = 0, n_split = 0, n_refused = 0, n_pairs = 0, n_once = 0;
  for (cs = 0; cs < 2500; cs++) {
    Case c = make_case(rng, cs % KINDS);
    const uint32_t NR = (uint32_t)c.rbytes.size(), NQ = (uint32_t)c.qbytes.size();
    skws::QrPlan p1, p2;
    std::string e1, e2;
    const bool ok1 = skws::plan_query_ref_working_sets(c.pairs, c.rbytes, c.qbytes, c.budget, p1, e1);
    const bool ok2 = skws::plan_query_ref_working_sets(c.pairs, c.rbytes, c.qbytes, c.budget, p2, e2);
    CHECK(ok1 && ok2, "refused: %s", e1.c_str());
    if (!ok1) continue;
    bool same = p1.sets.size() == p2.sets.size() && p1.n_split_components == p2.n_split_components;
    for (size_t w = 0; same && w < p1.sets.size(); w++)
      same = p1.sets[w].refs == p2.sets[w].refs && p1.sets[w].queries == p2.sets[w].queries && p1.sets[w].pairs == p2.sets[w].pairs &&
             p1.sets[w].bytes == p2.sets[w].bytes && p1.sets[w].chunk_pair == p2.sets[w].chunk_pair;
    CHECK(same, "plan differs between runs");
    std::vector<uint64_t> all;
    std::vector<uint32_t> ref_gathers(NR, 0);
    for (const auto& ws : p1.sets) {
      CHECK(!ws.pairs.empty(), "empty working set");
      CHECK(ws.bytes <= c.budget, "working set of %llu bytes over the budget %llu", (unsigned long long)ws.bytes, (unsigned long long)c.budget);
      CHECK(ascending(ws.refs, NR), "reference list not ascending in [0, %u)", NR);
      CHECK(ascending(ws.queries, NQ), "query list not ascending in [0, %u)", NQ);
      std::set<uint32_t> tr, tq;
      for (uint64_t q : ws.pairs) { tr.insert((uint32_t)(q >> 32)); tq.insert((uint32_t)q); }
      CHECK(std::vector<uint32_t>(tr.begin(), tr.end()) == ws.refs, "reference list is not the pairs' references");
      CHECK(std::vector<uint32_t>(tq.begin(), tq.end()) == ws.queries, "query list is not the pairs' queries");
      uint64_t b = 0;
      for (uint32_t r : ws.refs) { b += c.rbytes[r]; ref_gathers[r]++; }
      for (uint32_t q : ws.queries) b += c.qbytes[q];
      CHECK(b == ws.bytes, "byte count");
      CHECK(std::is_sorted(ws.pairs.begin(), ws.pairs.end()), "pairs not sorted");
      all.insert(all.end(), ws.pairs.begin(), ws.pairs.end());
      n_sets++;
      n_chunk_sets += ws.chunk_pair;
    }
    std::sort(all.begin(), all.end());
    CHECK(all == c.pairs, "pairs: %zu in the plan, %zu screened", all.size(), c.pairs.size());
    if (c.kind == 4) {   // few queries, many references: a single query sits in one chunk, so every reference is gathered once;
                         // queries spread over several chunks bring a reference back at most once per query
      bool ok = true;
      for (uint64_t p : c.pairs) ok = ok && ref_gathers[p >> 32] >= 1 && ref_gathers[p >> 32] <= (NQ == 1 ? 1 : NQ);
      CHECK(ok, "a reference is gathered more often than expected (%u queries)", NQ);
      n_once += NQ == 1 && p1.n_split_components > 0;
    }
    n_pairs += (long)c.pairs.size();
    n_split += p1.n_split_components;
    // a genome over budget / 2 on either side is refused (and only then)
    for (int side = 0; side < 2; side++) {
      std::vector<uint64_t> rb = c.rbytes, qb = c.qbytes;
      std::vector<uint64_t>& v = side ? qb : rb;
      const uint32_t g = (uint32_t)(rng() % v.size());
      v[g] = c.budget / 2 + 1;
      skws::QrPlan p3;
      std::string e3;
      CHECK(!skws::plan_query_ref_working_sets(c.pairs, rb, qb, c.budget, p3, e3) &&
                e3.find(std::string(side ? "query " : "reference ") + std::to_string(g) + " ") == 0, "oversized genome accepted: %s", e3.c_str());
      v[g] = c.budget / 2;
      CHECK(skws::plan_query_ref_working_sets(c.pairs, rb, qb, c.budget, p3, e3), "genome of exactly budget / 2 refused");
      n_refused++;
    }
  }
  printf("%d cases, %ld pairs, %ld working sets (%ld chunk pairs), %ld split components, %ld single-gather checks, %ld refusals, %d failures\n",
         cs, n_pairs, n_sets, n_chunk_sets, n_split, n_once, n_refused, failures);
  return failures ? 1 : 0;
}
