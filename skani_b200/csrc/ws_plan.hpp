// ws_plan.hpp -- working-set planner of sk_triangle_store and sk_query_ref_store (host only, no CUDA: tests/emu/emu_ws_plan.cpp
// and tests/emu/emu_qr_plan.cpp run it on the CPU).
//
// The triangle's screened pairs are cut into working sets: groups of pairs whose genomes, gathered from the host sketch
// store, fit a device budget.  A pair's chain result depends only on its two sketches, so every pair is chained in exactly
// one working set and the union of the working sets' results is the triangle's.
//   1. Pairs are grouped by connected component of the pair graph (a cluster of related genomes), as partition_pairs in
//      multi.cu does: a component's genomes are gathered once.
//   2. A component whose genome bytes fit the budget is one item; items are packed into working sets by first-fit
//      decreasing (largest first, ties by smallest genome id).
//   3. A component over budget is cut, in genome-id order, into chunks of at most budget / 2 bytes.  Its working sets are the
//      chunk pairs (x <= y) that hold at least one pair, with the genomes those pairs touch: at most budget / 2 + budget / 2.
//   4. A genome over budget / 2 cannot be placed in every chunk pair: the plan is refused.
// Deterministic: the plan depends only on the pair list, the genome sizes and the budget.
#pragma once
#include <algorithm>
#include <cstdint>
#include <string>
#include <vector>

namespace skws {

struct WorkingSet {
  std::vector<uint32_t> genomes;   // ascending global genome ids
  std::vector<uint64_t> pairs;     // global (i << 32 | j), i < j, sorted
  uint64_t bytes = 0;              // sum of the genomes' bytes
  bool chunk_pair = false;         // one chunk pair of a component over budget
};

struct Plan {
  std::vector<WorkingSet> sets;
  uint32_t n_split_components = 0;
};

// false (and a message in err) if a genome is larger than budget / 2; otherwise every pair of sorted_pairs is in exactly one
// working set of plan.sets and every working set holds at most budget bytes
inline bool plan_working_sets(const std::vector<uint64_t>& sorted_pairs, const std::vector<uint64_t>& genome_bytes, uint64_t budget,
                              Plan& plan, std::string& err) {
  plan = Plan();
  const uint32_t n = (uint32_t)genome_bytes.size();
  for (uint32_t g = 0; g < n; g++)
    if (genome_bytes[g] > budget / 2) {
      err = "genome " + std::to_string(g) + " needs " + std::to_string(genome_bytes[g]) + " device bytes, more than half the working-set budget of " +
            std::to_string(budget) + " bytes";
      return false;
    }
  if (sorted_pairs.empty()) return true;
  // connected components, root = smallest genome of the component
  std::vector<uint32_t> parent(n);
  for (uint32_t g = 0; g < n; g++) parent[g] = g;
  auto find = [&](uint32_t x) { while (parent[x] != x) { parent[x] = parent[parent[x]]; x = parent[x]; } return x; };
  for (uint64_t p : sorted_pairs) {
    const uint32_t a = find((uint32_t)(p >> 32)), b = find((uint32_t)p);
    if (a != b) parent[std::max(a, b)] = std::min(a, b);
  }
  // pairs grouped by component (stable: sorted inside a group)
  std::vector<std::pair<uint32_t, uint64_t>> keyed(sorted_pairs.size());
  for (size_t i = 0; i < sorted_pairs.size(); i++) keyed[i] = {find((uint32_t)(sorted_pairs[i] >> 32)), sorted_pairs[i]};
  std::stable_sort(keyed.begin(), keyed.end(), [](const std::pair<uint32_t, uint64_t>& a, const std::pair<uint32_t, uint64_t>& b) { return a.first < b.first; });
  struct Comp { uint32_t root; size_t p0, p1; std::vector<uint32_t> genomes; uint64_t bytes = 0; };
  std::vector<Comp> comps;
  for (size_t i = 0; i < keyed.size();) {
    size_t j = i;
    while (j < keyed.size() && keyed[j].first == keyed[i].first) j++;
    Comp c; c.root = keyed[i].first; c.p0 = i; c.p1 = j;
    for (size_t k = i; k < j; k++) { c.genomes.push_back((uint32_t)(keyed[k].second >> 32)); c.genomes.push_back((uint32_t)keyed[k].second); }
    std::sort(c.genomes.begin(), c.genomes.end());
    c.genomes.erase(std::unique(c.genomes.begin(), c.genomes.end()), c.genomes.end());
    for (uint32_t g : c.genomes) c.bytes += genome_bytes[g];
    comps.push_back(std::move(c));
    i = j;
  }
  // components that fit: first-fit decreasing
  std::vector<size_t> fit;
  for (size_t c = 0; c < comps.size(); c++) if (comps[c].bytes <= budget) fit.push_back(c);
  std::stable_sort(fit.begin(), fit.end(), [&](size_t a, size_t b) { return comps[a].bytes > comps[b].bytes; });   // ties: root order
  std::vector<std::vector<size_t>> bins;
  std::vector<uint64_t> load;
  for (size_t c : fit) {
    size_t b = 0;
    while (b < bins.size() && load[b] + comps[c].bytes > budget) b++;
    if (b == bins.size()) { bins.emplace_back(); load.push_back(0); }
    bins[b].push_back(c);
    load[b] += comps[c].bytes;
  }
  for (size_t b = 0; b < bins.size(); b++) {
    WorkingSet ws;
    for (size_t c : bins[b]) {
      ws.genomes.insert(ws.genomes.end(), comps[c].genomes.begin(), comps[c].genomes.end());
      for (size_t k = comps[c].p0; k < comps[c].p1; k++) ws.pairs.push_back(keyed[k].second);
    }
    std::sort(ws.genomes.begin(), ws.genomes.end());
    std::sort(ws.pairs.begin(), ws.pairs.end());
    ws.bytes = load[b];
    plan.sets.push_back(std::move(ws));
  }
  // components over budget: chunks of at most budget / 2 in genome-id order, one working set per chunk pair holding pairs
  std::vector<uint32_t> chunk_of(n, 0);
  for (const Comp& c : comps) {
    if (c.bytes <= budget) continue;
    plan.n_split_components++;
    uint32_t n_chunks = 0;
    uint64_t acc = 0;
    for (size_t k = 0; k < c.genomes.size(); k++) {
      const uint64_t b = genome_bytes[c.genomes[k]];
      if (k == 0 || acc + b > budget / 2) { n_chunks++; acc = 0; }
      acc += b;
      chunk_of[c.genomes[k]] = n_chunks - 1;
    }
    // pairs by chunk pair (x, y), x <= y because i < j and chunks follow genome order
    std::vector<std::pair<uint64_t, uint64_t>> byc;
    for (size_t k = c.p0; k < c.p1; k++) {
      const uint64_t p = keyed[k].second;
      byc.push_back({((uint64_t)chunk_of[(uint32_t)(p >> 32)] << 32) | chunk_of[(uint32_t)p], p});
    }
    std::sort(byc.begin(), byc.end());
    for (size_t i = 0; i < byc.size();) {
      size_t j = i;
      WorkingSet ws;
      ws.chunk_pair = true;
      while (j < byc.size() && byc[j].first == byc[i].first) {
        ws.pairs.push_back(byc[j].second);
        ws.genomes.push_back((uint32_t)(byc[j].second >> 32)); ws.genomes.push_back((uint32_t)byc[j].second);
        j++;
      }
      std::sort(ws.genomes.begin(), ws.genomes.end());
      ws.genomes.erase(std::unique(ws.genomes.begin(), ws.genomes.end()), ws.genomes.end());
      for (uint32_t g : ws.genomes) ws.bytes += genome_bytes[g];
      plan.sets.push_back(std::move(ws));
      i = j;
    }
  }
  return true;
}

// ---- query x reference (sk_query_ref_store) ----------------------------------------------------------------------------
struct QrWorkingSet {
  std::vector<uint32_t> refs;      // ascending reference ids
  std::vector<uint32_t> queries;   // ascending query ids
  std::vector<uint64_t> pairs;     // global (r << 32 | q), sorted
  uint64_t bytes = 0;              // sum of the genomes' bytes
  bool chunk_pair = false;
};

struct QrPlan {
  std::vector<QrWorkingSet> sets;
  uint32_t n_split_components = 0;
};

// The bipartite pair graph as one genome graph: reference r is genome r, query q is genome NR + q, so pairs sorted by (r, q)
// stay sorted and keep i < j.  plan_working_sets cuts it; each working set's genome list splits at NR.  References come first
// in id order, so a component over budget with few queries and many references is cut into reference chunks plus a last chunk
// holding the queries: every reference is gathered once.
inline bool plan_query_ref_working_sets(const std::vector<uint64_t>& sorted_pairs_rq, const std::vector<uint64_t>& ref_bytes,
                                        const std::vector<uint64_t>& query_bytes, uint64_t budget, QrPlan& plan, std::string& err) {
  plan = QrPlan();
  const uint64_t NR = ref_bytes.size();
  if (NR + query_bytes.size() >= (1ull << 32)) { err = "more than 2^32 references and queries together"; return false; }
  std::vector<uint64_t> bytes(ref_bytes);
  bytes.insert(bytes.end(), query_bytes.begin(), query_bytes.end());
  for (uint64_t g = 0; g < bytes.size(); g++)
    if (bytes[g] > budget / 2) {
      err = (g < NR ? "reference " + std::to_string(g) : "query " + std::to_string(g - NR)) + " needs " + std::to_string(bytes[g]) +
            " device bytes, more than half the working-set budget of " + std::to_string(budget) + " bytes";
      return false;
    }
  std::vector<uint64_t> pairs(sorted_pairs_rq.size());
  for (size_t i = 0; i < pairs.size(); i++) pairs[i] = sorted_pairs_rq[i] + NR;   // (r << 32) | (NR + q)
  Plan p;
  if (!plan_working_sets(pairs, bytes, budget, p, err)) return false;
  plan.n_split_components = p.n_split_components;
  for (WorkingSet& ws : p.sets) {
    QrWorkingSet q;
    const size_t cut = std::lower_bound(ws.genomes.begin(), ws.genomes.end(), (uint32_t)NR) - ws.genomes.begin();
    q.refs.assign(ws.genomes.begin(), ws.genomes.begin() + cut);
    for (size_t i = cut; i < ws.genomes.size(); i++) q.queries.push_back(ws.genomes[i] - (uint32_t)NR);
    q.pairs.resize(ws.pairs.size());
    for (size_t i = 0; i < ws.pairs.size(); i++) q.pairs[i] = ws.pairs[i] - NR;
    q.bytes = ws.bytes;
    q.chunk_pair = ws.chunk_pair;
    plan.sets.push_back(std::move(q));
  }
  return true;
}

}  // namespace skws
