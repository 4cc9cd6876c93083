// sk_cluster's per-vertex logic (skani_b200/csrc/cluster_core.cuh) driven by host loops that emulate the kernels' rounds, against
// a sequential reference written independently here, on random graphs: Erdos-Renyi, cliques joined by bridges, paths in rank
// order and in reverse, stars, equal ANIs, ani == min_ani, NaN / -1 / <= 0.1 rows and isolated vertices.
// Greedy rounds visit the undecided vertices in a random order and read the states as they are at that moment (one
// emulation) or as they were when the round began (another: every lane of a warp reads at once).  Single-linkage passes hook
// the edges in a random order with live parents, then jump pointers in a random order.  Both methods must equal the
// reference for every visit order.  Development/test harness only.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <numeric>
#include <random>
#include <vector>

#include "../../skani_b200/csrc/cluster_core.cuh"

namespace {

using namespace sk;

int failures = 0, cs = 0;
#define CHECK(cond, ...) do { if (!(cond)) { failures++; if (failures < 20) { fprintf(stderr, "case %d: ", cs); fprintf(stderr, __VA_ARGS__); fputc('\n', stderr); } } } while (0)

struct Row { uint32_t a, b; float ani; };
struct Case { uint32_t n; std::vector<Row> rows; std::vector<uint32_t> rank; float min_ani; };
struct Out { std::vector<uint32_t> rep, cluster; std::vector<uint64_t> edge; };

const float NaN = std::nanf("");

Case make_case(std::mt19937_64& rng, int kind) {
  Case c;
  c.n = kind == 8 ? 0 : 1 + (uint32_t)(rng() % 300);
  c.min_ani = 0.95f;
  std::vector<std::pair<uint32_t, uint32_t>> pairs;
  auto rand_ani = [&] { return 0.9f + 0.1f * (float)(rng() % 1000) / 1000.f; };
  const uint32_t n = c.n;
  if (kind == 0) {                                   // Erdos-Renyi
    const double p = (double)(rng() % 100) / 100.0 * 8.0 / std::max<uint32_t>(n, 1);
    for (uint32_t a = 0; a < n; a++)
      for (uint32_t b = a + 1; b < n; b++)
        if ((double)(rng() % 1000000) / 1e6 < p) pairs.push_back({a, b});
  } else if (kind == 1) {                            // cliques (families) joined by bridges
    const uint32_t k = 1 + (uint32_t)(rng() % 20);
    for (uint32_t a = 0; a < n; a++)
      for (uint32_t b = a + 1; b < n; b++)
        if (a / k == b / k) pairs.push_back({a, b});
    for (uint32_t i = 0; i < n / k; i++) { const uint32_t a = (uint32_t)(rng() % n), b = (uint32_t)(rng() % n); if (a / k != b / k) pairs.push_back({a, b}); }
  } else if (kind == 2 || kind == 3) {               // paths (ranks set below: in path order or reversed)
    for (uint32_t a = 0; a + 1 < n; a++) pairs.push_back({a, a + 1});
  } else if (kind == 4) {                            // stars
    const uint32_t s = 1 + (uint32_t)(rng() % 5);
    for (uint32_t v = s; v < n; v++) pairs.push_back({v % s, v});
  } else {                                           // sparse random graphs with many isolated vertices
    for (uint32_t i = 0; i < n / 4; i++) pairs.push_back({(uint32_t)(rng() % n), (uint32_t)(rng() % n)});
  }
  // unique unordered pairs, no self pairs
  for (auto& p : pairs) if (p.first > p.second) std::swap(p.first, p.second);
  std::sort(pairs.begin(), pairs.end());
  pairs.erase(std::unique(pairs.begin(), pairs.end()), pairs.end());
  pairs.erase(std::remove_if(pairs.begin(), pairs.end(), [](auto& p) { return p.first == p.second; }), pairs.end());
  for (auto& p : pairs) {
    Row r{p.first, p.second, rand_ani()};
    if (rng() % 2) std::swap(r.a, r.b);                       // either direction
    const int special = (int)(rng() % 16);
    if (kind == 5) r.ani = 0.97f;                             // equal ANIs everywhere
    else if (kind == 6 && special < 6) r.ani = c.min_ani;     // exactly at the threshold
    if (special == 7) r.ani = NaN;
    else if (special == 8) r.ani = -1.f;
    else if (special == 9) r.ani = 0.1f;
    else if (special == 10 && kind == 7) r.ani = 0.5f;
    c.rows.push_back(r);
  }
  if (kind == 7) c.min_ani = 0.f;                             // every printed row is an edge: rows <= 0.1 still are not
  std::shuffle(c.rows.begin(), c.rows.end(), rng);
  c.rank.resize(n);
  std::iota(c.rank.begin(), c.rank.end(), 0u);
  if (kind == 3) std::reverse(c.rank.begin(), c.rank.end());
  else if (kind != 2) std::shuffle(c.rank.begin(), c.rank.end(), rng);
  return c;
}

// the symmetric CSR of the device: keys v << 32 | u ascending, values = edge index
struct Graph { std::vector<uint64_t> off, adj; std::vector<uint32_t> adj_e; std::vector<float> ani; std::vector<uint64_t> row, ekey; };
Graph build(const Case& c) {
  Graph g;
  std::vector<std::pair<uint64_t, uint32_t>> kv;
  for (uint64_t i = 0; i < c.rows.size(); i++) {
    const Row& r = c.rows[i];
    if (!cl_is_edge(r.ani, c.min_ani)) continue;
    const uint32_t e = (uint32_t)g.ani.size();
    const uint32_t a = std::min(r.a, r.b), b = std::max(r.a, r.b);
    g.ani.push_back(r.ani); g.row.push_back(i); g.ekey.push_back((uint64_t)a << 32 | b);
    kv.push_back({(uint64_t)a << 32 | b, e});
    kv.push_back({(uint64_t)b << 32 | a, e});
  }
  std::sort(kv.begin(), kv.end());
  g.off.assign(c.n + 1, 0);
  for (auto& x : kv) { g.adj.push_back(x.first); g.adj_e.push_back(x.second); g.off[(x.first >> 32) + 1]++; }
  for (uint32_t v = 0; v < c.n; v++) g.off[v + 1] += g.off[v];
  return g;
}

void number(const Case& c, const std::vector<bool>& is_rep_by_rank, Out& o) {
  std::vector<uint32_t> cid(c.n);
  uint32_t k = 0;
  for (uint32_t r = 0; r < c.n; r++) cid[r] = is_rep_by_rank[r] ? k++ : UINT32_MAX;
  o.cluster.resize(c.n);
  for (uint32_t v = 0; v < c.n; v++) o.cluster[v] = cid[c.rank[o.rep[v]]];
}

// ---- sequential references (independent of cluster_core.cuh)
Out reference(const Case& c, bool single) {
  const uint32_t n = c.n;
  std::vector<std::vector<std::pair<uint32_t, uint64_t>>> nb(n);   // (neighbour, row)
  for (uint64_t i = 0; i < c.rows.size(); i++) {
    const Row& r = c.rows[i];
    if (!(r.ani > 0.1f) || !(r.ani >= c.min_ani)) continue;
    nb[r.a].push_back({r.b, i}); nb[r.b].push_back({r.a, i});
  }
  std::vector<uint32_t> order(n);
  for (uint32_t v = 0; v < n; v++) order[c.rank[v]] = v;
  Out o;
  o.rep.assign(n, UINT32_MAX); o.edge.assign(n, UINT64_MAX);
  std::vector<bool> rep_by_rank(n, false);
  if (!single) {
    std::vector<bool> is_rep(n, false);
    for (uint32_t r = 0; r < n; r++) {
      const uint32_t v = order[r];
      bool hit = false;
      for (auto& x : nb[v]) hit |= is_rep[x.first];
      if (!hit) { is_rep[v] = true; rep_by_rank[r] = true; }
    }
    for (uint32_t v = 0; v < n; v++) {
      if (is_rep[v]) { o.rep[v] = v; continue; }
      float best = -1; uint32_t br = UINT32_MAX;
      for (auto& x : nb[v]) {
        if (!is_rep[x.first]) continue;
        const float a = c.rows[x.second].ani;
        if (a > best || (a == best && c.rank[x.first] < br)) { best = a; br = c.rank[x.first]; o.rep[v] = x.first; o.edge[v] = x.second; }
      }
    }
  } else {
    std::vector<uint32_t> comp(n, UINT32_MAX);
    for (uint32_t r = 0; r < n; r++) {            // BFS from each smallest-rank unvisited vertex
      const uint32_t s = order[r];
      if (comp[s] != UINT32_MAX) continue;
      rep_by_rank[r] = true;
      std::vector<uint32_t> q{s};
      comp[s] = s;
      for (size_t i = 0; i < q.size(); i++)
        for (auto& x : nb[q[i]]) if (comp[x.first] == UINT32_MAX) { comp[x.first] = s; q.push_back(x.first); }
    }
    for (uint32_t v = 0; v < n; v++) {
      o.rep[v] = comp[v];
      if (comp[v] != v) for (auto& x : nb[v]) if (x.first == comp[v]) o.edge[v] = x.second;
    }
  }
  number(c, rep_by_rank, o);
  return o;
}

// ---- emulations of cluster.cu's rounds through cluster_core.cuh
Out emulate_greedy(const Case& c, const Graph& g, std::mt19937_64& rng, bool snapshot, uint64_t& rounds) {
  const uint32_t n = c.n;
  std::vector<uint8_t> state(n, CL_UNDECIDED);
  std::vector<uint32_t> frontier(n);
  for (uint32_t v = 0; v < n; v++) frontier[c.rank[v]] = v;
  while (!frontier.empty()) {
    std::vector<uint32_t> visit = frontier;
    std::shuffle(visit.begin(), visit.end(), rng);
    const std::vector<uint8_t> before = state;
    for (uint32_t v : visit) {
      const uint8_t s = cl_greedy_decide(v, g.off.data(), g.adj.data(), c.rank.data(), snapshot ? before.data() : state.data());
      if (s != CL_UNDECIDED) state[v] = s;
    }
    rounds++;
    std::vector<uint32_t> next;
    for (uint32_t v : frontier) if (state[v] == CL_UNDECIDED) next.push_back(v);
    CHECK(next.size() < frontier.size(), "greedy round decided nothing");
    if (next.size() == frontier.size()) break;
    frontier.swap(next);
  }
  Out o;
  o.rep.resize(n); o.edge.assign(n, UINT64_MAX);
  std::vector<bool> rep_by_rank(n, false);
  for (uint32_t v = 0; v < n; v++) {
    uint32_t r = v;
    uint64_t at = 0;
    if (state[v] == CL_MEMBER && cl_assign(v, g.off.data(), g.adj.data(), g.adj_e.data(), g.ani.data(), c.rank.data(), state.data(), &r, &at))
      o.edge[v] = g.row[g.adj_e[at]];
    o.rep[v] = r;
    rep_by_rank[c.rank[v]] = state[v] == CL_REP;
  }
  number(c, rep_by_rank, o);
  return o;
}

Out emulate_single(const Case& c, const Graph& g, std::mt19937_64& rng, uint64_t& total_passes) {
  const uint32_t n = c.n;
  uint64_t passes = 0;
  std::vector<uint32_t> parent(n), order(n);
  std::iota(parent.begin(), parent.end(), 0u);
  for (uint32_t v = 0; v < n; v++) order[c.rank[v]] = v;
  std::vector<uint32_t> ev(g.ekey.size()), rv(n);
  std::iota(ev.begin(), ev.end(), 0u);
  std::iota(rv.begin(), rv.end(), 0u);
  for (bool changed = !ev.empty(); changed;) {
    changed = false;
    std::shuffle(ev.begin(), ev.end(), rng);
    for (uint32_t e : ev) {
      uint32_t slot, val;
      const uint64_t k = g.ekey[e];
      if (cl_hook(parent[c.rank[(uint32_t)(k >> 32)]], parent[c.rank[(uint32_t)k]], &slot, &val) && parent[slot] > val) { parent[slot] = val; changed = true; }
    }
    passes++;
    if (!changed) break;
    std::shuffle(rv.begin(), rv.end(), rng);
    for (uint32_t r : rv) parent[r] = cl_find(parent.data(), r);
    CHECK(passes <= (uint64_t)n + 1, "single linkage does not converge");
    if (passes > (uint64_t)n + 1) break;
  }
  total_passes += passes;
  Out o;
  o.rep.resize(n); o.edge.assign(n, UINT64_MAX);
  std::vector<bool> rep_by_rank(n, false);
  for (uint32_t v = 0; v < n; v++) {
    const uint32_t r = order[parent[c.rank[v]]];
    o.rep[v] = r;
    if (r != v) {
      const uint64_t want = (uint64_t)v << 32 | r;
      auto it = std::lower_bound(g.adj.begin() + g.off[v], g.adj.begin() + g.off[v + 1], want);
      if (it != g.adj.begin() + g.off[v + 1] && *it == want) o.edge[v] = g.row[g.adj_e[it - g.adj.begin()]];
    }
    rep_by_rank[c.rank[v]] = parent[c.rank[v]] == c.rank[v];
  }
  number(c, rep_by_rank, o);
  return o;
}

bool same(const Out& a, const Out& b) { return a.rep == b.rep && a.cluster == b.cluster && a.edge == b.edge; }

}  // namespace

int main() {
  std::mt19937_64 rng(20261017);
  const int KINDS = 9, CASES = 2250;
  uint64_t edges = 0, rounds = 0, passes = 0, path_rounds = 0, greedy_clusters = 0, single_clusters = 0;
  for (cs = 0; cs < CASES; cs++) {
    const int kind = cs % KINDS;
    const Case c = make_case(rng, kind);
    const Graph g = build(c);
    edges += g.ekey.size();
    const Out rg = reference(c, false), rs = reference(c, true);
    for (uint32_t v = 0; v < c.n; v++) { greedy_clusters += rg.rep[v] == v; single_clusters += rs.rep[v] == v; }
    for (int t = 0; t < 3; t++) {          // three visit orders: live, live, start-of-round snapshot
      uint64_t r = 0;
      const Out eg = emulate_greedy(c, g, rng, t == 2, r);
      rounds += r;
      if (kind == 2 && t == 0) path_rounds += r;
      CHECK(same(eg, rg), "greedy differs from the sequential loop (kind %d, n %u, visit order %d)", kind, c.n, t);
      const Out es = emulate_single(c, g, rng, passes);
      CHECK(same(es, rs), "single linkage differs from the components (kind %d, n %u, visit order %d)", kind, c.n, t);
    }
  }
  printf("%d cases, %llu edges, %llu greedy clusters, %llu components, %llu greedy rounds (%llu on rank-ordered paths), %llu hook passes, %d failures\n",
         CASES, (unsigned long long)edges, (unsigned long long)greedy_clusters, (unsigned long long)single_clusters, (unsigned long long)rounds,
         (unsigned long long)path_rounds, (unsigned long long)passes, failures);
  return failures ? 1 : 0;
}
