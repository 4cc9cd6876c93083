// ws_plan.hpp -- pair components, the multi-context pair split and the working-set planners of the host sketch store paths
// (host only, no CUDA: tests/emu/emu_partition.cpp, tests/emu/emu_ws_plan.cpp and tests/emu/emu_qr_plan.cpp run them on the CPU).
//
// pair_components groups a sorted pair list by connected component of the pair graph (a cluster of related genomes).
// partition_pairs splits a pair list over the contexts of sk_triangle_multi (multi.cu) by component, so that a context fetches a
// cluster's sketches once.  genomes_fit is the one refusal of a genome over budget / 2.
//
// The triangle's screened pairs are cut into working sets: groups of pairs whose genomes, gathered from the host sketch
// store, fit a device budget.  A pair's chain result depends only on its two sketches, so every pair is chained in exactly
// one working set and the union of the working sets' results is the triangle's.
//   1. Pairs are grouped by connected component (pair_components): a component's genomes are gathered once.
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

// The pairs of a sorted list of distinct pairs grouped by connected component of the pair graph: groups in order of their
// root (the component's smallest genome), pairs sorted inside a group.  Group k is pairs[first[k] .. first[k + 1]).
struct PairComponents {
  std::vector<uint64_t> pairs;
  std::vector<size_t> first;
};

inline PairComponents pair_components(const std::vector<uint64_t>& sorted_pairs, uint32_t n_genomes) {
  std::vector<uint32_t> parent(n_genomes);
  for (uint32_t g = 0; g < n_genomes; g++) parent[g] = g;
  auto find = [&](uint32_t x) { while (parent[x] != x) { parent[x] = parent[parent[x]]; x = parent[x]; } return x; };
  for (uint64_t p : sorted_pairs) {
    const uint32_t a = find((uint32_t)(p >> 32)), b = find((uint32_t)p);
    if (a != b) parent[std::max(a, b)] = std::min(a, b);            // root = smallest genome of the component
  }
  std::vector<std::pair<uint32_t, uint64_t>> keyed(sorted_pairs.size());
  for (size_t i = 0; i < sorted_pairs.size(); i++) keyed[i] = {find((uint32_t)(sorted_pairs[i] >> 32)), sorted_pairs[i]};
  std::stable_sort(keyed.begin(), keyed.end(), [](const std::pair<uint32_t, uint64_t>& a, const std::pair<uint32_t, uint64_t>& b) { return a.first < b.first; });
  PairComponents pc;
  pc.pairs.resize(keyed.size());
  for (size_t i = 0; i < keyed.size(); i++) {
    if (i == 0 || keyed[i].first != keyed[i - 1].first) pc.first.push_back(i);
    pc.pairs[i] = keyed[i].second;
  }
  pc.first.push_back(keyed.size());
  return pc;
}

// Pairs -> one list per context.  The pairs of one component stay together, so a context fetches that cluster's sketches once;
// with a genome order unrelated to relatedness a contiguous slice of the sorted list touches ~5x more genomes.  Components above
// half a context's fair share are cut into runs of consecutive pairs; items go to the least loaded context, largest first (ties:
// first pair).  Deterministic; every list comes out sorted.  (skani_b200/multi_gpu.py partition_pairs follows the same rule.)
inline void partition_pairs(const std::vector<uint64_t>& sorted_pairs, uint32_t W, uint32_t n_genomes, std::vector<std::vector<uint64_t>>& out) {
  out.assign(W, {});
  const size_t n = sorted_pairs.size();
  if (n == 0) return;
  if (W == 1) { out[0] = sorted_pairs; return; }
  const PairComponents pc = pair_components(sorted_pairs, n_genomes);
  const size_t cap = std::max<size_t>(1, (n + 2 * (size_t)W - 1) / (2 * (size_t)W));
  struct Item { size_t size, start; };
  std::vector<Item> items;
  for (size_t k = 0; k + 1 < pc.first.size(); k++)
    for (size_t s0 = pc.first[k]; s0 < pc.first[k + 1]; s0 += cap) items.push_back(Item{std::min(cap, pc.first[k + 1] - s0), s0});
  std::sort(items.begin(), items.end(), [&](const Item& a, const Item& b) { return a.size != b.size ? a.size > b.size : pc.pairs[a.start] < pc.pairs[b.start]; });
  std::vector<size_t> load(W, 0);
  for (const Item& it : items) {
    uint32_t r = 0;
    for (uint32_t k = 1; k < W; k++) if (load[k] < load[r]) r = k;
    out[r].insert(out[r].end(), pc.pairs.begin() + it.start, pc.pairs.begin() + it.start + it.size);
    load[r] += it.size;
  }
  for (auto& v : out) std::sort(v.begin(), v.end());
}

// false (and the refusal in err) if a genome is larger than budget / 2: it cannot be placed in every chunk pair.  Genome g is
// named "genome g"; with a split point n_refs >= 0, genomes [0, n_refs) are "reference g" and genome n_refs + q is "query q".
inline bool genomes_fit(const std::vector<uint64_t>& genome_bytes, uint64_t budget, std::string& err, int64_t n_refs = -1) {
  for (uint64_t g = 0; g < genome_bytes.size(); g++)
    if (genome_bytes[g] > budget / 2) {
      const std::string name = n_refs < 0 ? "genome " + std::to_string(g)
                               : g < (uint64_t)n_refs ? "reference " + std::to_string(g) : "query " + std::to_string(g - n_refs);
      err = name + " needs " + std::to_string(genome_bytes[g]) + " device bytes, more than half the working-set budget of " +
            std::to_string(budget) + " bytes";
      return false;
    }
  return true;
}

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
  if (!genomes_fit(genome_bytes, budget, err)) return false;
  if (sorted_pairs.empty()) return true;
  const uint32_t n = (uint32_t)genome_bytes.size();
  const PairComponents pc = pair_components(sorted_pairs, n);
  struct Comp { size_t p0, p1; std::vector<uint32_t> genomes; uint64_t bytes = 0; };
  std::vector<Comp> comps;
  for (size_t k = 0; k + 1 < pc.first.size(); k++) {
    Comp c; c.p0 = pc.first[k]; c.p1 = pc.first[k + 1];
    for (size_t i = c.p0; i < c.p1; i++) { c.genomes.push_back((uint32_t)(pc.pairs[i] >> 32)); c.genomes.push_back((uint32_t)pc.pairs[i]); }
    std::sort(c.genomes.begin(), c.genomes.end());
    c.genomes.erase(std::unique(c.genomes.begin(), c.genomes.end()), c.genomes.end());
    for (uint32_t g : c.genomes) c.bytes += genome_bytes[g];
    comps.push_back(std::move(c));
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
      ws.pairs.insert(ws.pairs.end(), pc.pairs.begin() + comps[c].p0, pc.pairs.begin() + comps[c].p1);
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
      const uint64_t p = pc.pairs[k];
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
  if (!genomes_fit(bytes, budget, err, (int64_t)NR)) return false;
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
