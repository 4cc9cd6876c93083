// sk_cluster_linkage's per-cluster logic (skani_b200/csrc/linkage_core.cuh) driven by host loops that emulate the kernels'
// rounds, on random graphs: Erdos-Renyi, cliques joined by bridges, paths, stars, equal ANIs, ani == min_ani, complete-linkage
// partial pairs, NaN / -1 / <= 0.1 rows, isolated genomes and n = 0 / 1.
// A round folds every cluster's pairs to its best partner in one of four visit orders (forward, reverse, random, and the
// warp's lane-strided partial bests reduced by xor shuffles), decides every cluster in a random order, then relabels and
// combines the pair list.  All orders must give the same merges and flat clusters; on graphs without ties they must equal a
// sequential HAC written independently here (exact sums and minima over member pairs, compared in 128 bits).
// Development/test harness only.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <map>
#include <numeric>
#include <random>
#include <vector>

#include "../../skani_b200/csrc/linkage_core.cuh"

namespace {

using namespace sk;

int failures = 0, cs = 0;
#define CHECK(cond, ...) do { if (!(cond)) { failures++; if (failures < 20) { fprintf(stderr, "case %d: ", cs); fprintf(stderr, __VA_ARGS__); fputc('\n', stderr); } } } while (0)

struct Row { uint32_t a, b; float ani; };
struct Case { uint32_t n; std::vector<Row> rows; std::vector<uint32_t> rank; float min_ani; int method; bool dendrogram; bool tie_free; };
struct Out {
  std::vector<uint32_t> root;             // by rank: the flat cluster's id
  std::vector<LkMerge> merges;            // dendrogram order
  uint32_t rounds = 0;
};

const float NaN = std::nanf("");

Case make_case(std::mt19937_64& rng, int kind) {
  Case c;
  c.n = kind == 9 ? (uint32_t)(rng() % 2) : 2 + (uint32_t)(rng() % 40);
  c.min_ani = 0.95f;
  c.method = (int)(rng() % 2);
  c.dendrogram = rng() % 2;
  const uint32_t n = c.n;
  std::vector<std::pair<uint32_t, uint32_t>> pairs;
  if (kind == 0 || kind == 6 || kind == 7) {            // Erdos-Renyi (dense for complete linkage's full pairs)
    const double p = kind == 7 ? 0.7 : (double)(rng() % 100) / 100.0 * 6.0 / n;
    for (uint32_t a = 0; a < n; a++)
      for (uint32_t b = a + 1; b < n; b++)
        if ((double)(rng() % 1000000) / 1e6 < p) pairs.push_back({a, b});
  } else if (kind == 1) {                               // cliques joined by bridges
    const uint32_t k = 1 + (uint32_t)(rng() % 8);
    for (uint32_t a = 0; a < n; a++)
      for (uint32_t b = a + 1; b < n; b++)
        if (a / k == b / k) pairs.push_back({a, b});
    for (uint32_t i = 0; i < n / k; i++) pairs.push_back({(uint32_t)(rng() % n), (uint32_t)(rng() % n)});
  } else if (kind == 2) {                               // paths
    for (uint32_t a = 0; a + 1 < n; a++) pairs.push_back({a, a + 1});
  } else if (kind == 3) {                               // stars
    const uint32_t s = 1 + (uint32_t)(rng() % 3);
    for (uint32_t v = s; v < n; v++) pairs.push_back({v % s, v});
  } else {                                              // sparse, many isolated genomes
    for (uint32_t i = 0; i < n / 3; i++) pairs.push_back({(uint32_t)(rng() % n), (uint32_t)(rng() % n)});
  }
  for (auto& p : pairs) if (p.first > p.second) std::swap(p.first, p.second);
  std::sort(pairs.begin(), pairs.end());
  pairs.erase(std::unique(pairs.begin(), pairs.end()), pairs.end());
  pairs.erase(std::remove_if(pairs.begin(), pairs.end(), [](auto& p) { return p.first == p.second; }), pairs.end());
  // tie-free kinds draw distinct ANIs; kind 4 uses ten values only, kind 5 one value, kind 6 puts many on the cut
  c.tie_free = kind == 0 || kind == 1 || kind == 2 || kind == 3 || kind == 7;
  std::vector<float> anis;
  for (size_t i = 0; i < pairs.size(); i++) anis.push_back(0.9f + 0.1f * (float)(i + 1) / (float)(pairs.size() + 1));
  std::shuffle(anis.begin(), anis.end(), rng);
  for (size_t i = 0; i < pairs.size(); i++) {
    Row r{pairs[i].first, pairs[i].second, anis[i]};
    if (rng() % 2) std::swap(r.a, r.b);
    if (kind == 4) r.ani = 0.9f + 0.01f * (float)(rng() % 10);
    else if (kind == 5) r.ani = 0.97f;
    else if (kind == 6) {
      const int sp = (int)(rng() % 8);
      if (sp < 3) r.ani = c.min_ani;
      else if (sp == 3) r.ani = NaN;
      else if (sp == 4) r.ani = -1.f;
      else if (sp == 5) r.ani = 0.1f;
    }
    c.rows.push_back(r);
  }
  std::shuffle(c.rows.begin(), c.rows.end(), rng);
  c.rank.resize(n);
  std::iota(c.rank.begin(), c.rank.end(), 0u);
  if (rng() % 3) std::shuffle(c.rank.begin(), c.rank.end(), rng);
  return c;
}

uint32_t find(const std::vector<uint32_t>& parent, uint32_t r) { while (parent[r] != r) r = parent[r]; return r; }

// ---- the kernels' rounds through linkage_core.cuh; order 0 forward, 1 reverse, 2 random, 3 lane-strided warp fold
Out emulate(const Case& c, int order, std::mt19937_64& rng) {
  const uint32_t n = c.n, qcut = lk_q(c.min_ani);
  std::map<std::pair<uint32_t, uint32_t>, LkVal> list;   // directed pairs in rank space, sorted like the device keys
  for (const Row& r : c.rows) {
    if (!(r.ani > 0.1f)) continue;
    const uint32_t a = c.rank[r.a], b = c.rank[r.b], q = lk_q(r.ani);
    list[{a, b}] = list[{b, a}] = LkVal{q, 1, q};
  }
  std::vector<uint32_t> size(n, 1), parent(n), lab(n), best(n, LK_NONE), best_at(n);
  std::iota(parent.begin(), parent.end(), 0u);
  std::iota(lab.begin(), lab.end(), 0u);
  Out o;
  for (uint32_t round = 0; !list.empty(); round++) {
    if (round > n + 1) { CHECK(false, "rounds do not converge"); break; }
    std::vector<std::pair<uint32_t, uint32_t>> key;
    std::vector<LkVal> val;
    for (auto& x : list) { key.push_back(x.first); val.push_back(x.second); }
    std::vector<uint32_t> seg;
    for (uint32_t i = 0; i < key.size(); i++) if (i == 0 || key[i].first != key[i - 1].first) seg.push_back(i);
    std::vector<uint8_t> drop(key.size(), 0);
    for (size_t w = 0; w < seg.size(); w++) {
      const uint32_t i0 = seg[w], i1 = w + 1 < seg.size() ? seg[w + 1] : (uint32_t)key.size(), A = key[i0].first;
      std::vector<uint32_t> visit(i1 - i0);
      std::iota(visit.begin(), visit.end(), i0);
      if (order == 1) std::reverse(visit.begin(), visit.end());
      if (order == 2) std::shuffle(visit.begin(), visit.end(), rng);
      struct Cand { bool found = false; uint64_t s = 0, p = 1; uint32_t id = 0, at = 0; };
      const auto fold = [&](Cand& b, uint32_t i) {
        uint64_t s, p;
        lk_value(c.method, val[i], size[A], size[key[i].second], &s, &p);
        if (lk_droppable(c.method, s, p, qcut, c.dendrogram)) { drop[i] = 1; return; }
        if (!b.found || lk_better(s, p, key[i].second, b.s, b.p, b.id)) b = Cand{true, s, p, key[i].second, i};
      };
      Cand b;
      if (order == 3) {
        Cand lane[32];
        for (uint32_t i = i0; i < i1; i++) fold(lane[(i - i0) % 32], i);
        for (int d = 16; d; d >>= 1) {
          Cand next[32];
          for (int l = 0; l < 32; l++) {
            next[l] = lane[l];
            const Cand& x = lane[l ^ d];
            if (x.found && (!next[l].found || lk_better(x.s, x.p, x.id, next[l].s, next[l].p, next[l].id))) next[l] = x;
          }
          std::copy(next, next + 32, lane);
        }
        b = lane[0];
      } else {
        for (uint32_t i : visit) fold(b, i);
      }
      best[A] = b.found && lk_qualifies(b.s, b.p, qcut, c.dendrogram) ? b.id : LK_NONE;
      best_at[A] = b.at;
    }
    // decisions in a random order; merges numbered in segment order (the device's scan)
    std::vector<uint32_t> ws(seg.size());
    std::iota(ws.begin(), ws.end(), 0u);
    std::shuffle(ws.begin(), ws.end(), rng);
    std::vector<uint8_t> flag(seg.size(), 0);
    for (uint32_t w : ws) {
      const uint32_t A = key[seg[w]].first;
      const int d = lk_decide(A, best.data());
      if (d == LK_DEACTIVATE) lab[A] = LK_NONE;
      else if (d == LK_MERGE_HIGH) lab[A] = best[A];
      else if (d == LK_MERGE_LOW) flag[w] = 1;
    }
    bool merged = false;
    std::vector<uint32_t> new_size = size;
    for (uint32_t w : ws) {
      if (!flag[w]) continue;
      const uint32_t A = key[seg[w]].first, B = best[A];
      uint64_t s, p;
      lk_value(c.method, val[best_at[A]], size[A], size[B], &s, &p);
      o.merges.push_back(LkMerge{s, p, round, A, B, size[A] + size[B]});
      if (lk_qualifies(s, p, qcut, false)) parent[B] = A;
      new_size[A] = size[A] + size[B];
      merged = true;
    }
    size = new_size;
    if (merged) o.rounds = round + 1;
    std::map<std::pair<uint32_t, uint32_t>, LkVal> next;
    std::vector<uint32_t> vi(key.size());
    std::iota(vi.begin(), vi.end(), 0u);
    std::shuffle(vi.begin(), vi.end(), rng);          // the combine is associative and commutative: any order
    for (uint32_t i : vi) {
      if (drop[i]) continue;
      const uint32_t a = lab[key[i].first], b = lab[key[i].second];
      if (a == LK_NONE || b == LK_NONE || a == b) continue;
      auto it = next.find({a, b});
      if (it == next.end()) next[{a, b}] = val[i];
      else it->second = lk_combine(it->second, val[i]);
    }
    list.swap(next);
  }
  std::sort(o.merges.begin(), o.merges.end(), LkMergeOrder{});
  o.root.resize(n);
  for (uint32_t r = 0; r < n; r++) o.root[r] = find(parent, r);
  return o;
}

// ---- sequential HAC, independent of linkage_core.cuh: the globally best qualifying pair merges, one at a time
using u128 = unsigned __int128;
Out sequential(const Case& c) {
  const uint32_t n = c.n;
  const u128 qcut = (u128)(uint64_t)((double)c.min_ani * 134217728.0);
  std::map<std::pair<uint32_t, uint32_t>, uint64_t> q;
  for (const Row& r : c.rows)
    if (r.ani > 0.1f) q[{c.rank[r.a], c.rank[r.b]}] = q[{c.rank[r.b], c.rank[r.a]}] = (uint64_t)((double)r.ani * 134217728.0);
  std::map<uint32_t, std::vector<uint32_t>> cl;
  for (uint32_t r = 0; r < n; r++) cl[r] = {r};
  std::vector<uint32_t> parent(n);
  std::iota(parent.begin(), parent.end(), 0u);
  Out o;
  for (uint32_t step = 0; cl.size() > 1; step++) {
    bool have = false;
    uint64_t bs = 0, bp = 1;
    uint32_t ba = 0, bb = 0;
    for (auto x = cl.begin(); x != cl.end(); ++x)
      for (auto y = std::next(x); y != cl.end(); ++y) {
        uint64_t sum = 0, cnt = 0, mn = UINT64_MAX;
        for (uint32_t u : x->second)
          for (uint32_t v : y->second) {
            auto it = q.find({u, v});
            if (it == q.end()) continue;
            sum += it->second; cnt++; mn = std::min(mn, it->second);
          }
        const uint64_t P = (uint64_t)x->second.size() * y->second.size();
        const uint64_t s = c.method == LK_AVERAGE ? sum : (cnt == P ? mn : 0), p = c.method == LK_AVERAGE ? P : 1;
        if (!have || (u128)s * bp > (u128)bs * p) { have = true; bs = s; bp = p; ba = x->first; bb = y->first; }
      }
    if (c.dendrogram ? bs == 0 : (u128)bs < qcut * bp) break;
    o.merges.push_back(LkMerge{bs, bp, step, ba, bb, (uint32_t)(cl[ba].size() + cl[bb].size())});
    if ((u128)bs >= qcut * bp) parent[bb] = ba;
    cl[ba].insert(cl[ba].end(), cl[bb].begin(), cl[bb].end());
    cl.erase(bb);
  }
  o.root.resize(n);
  for (uint32_t r = 0; r < n; r++) o.root[r] = find(parent, r);
  return o;
}

bool same_merges(const std::vector<LkMerge>& x, const std::vector<LkMerge>& y, bool rounds) {
  if (x.size() != y.size()) return false;
  for (size_t i = 0; i < x.size(); i++)
    if ((u128)x[i].s * y[i].p != (u128)y[i].s * x[i].p || x[i].a != y[i].a || x[i].b != y[i].b || x[i].size != y[i].size ||
        (rounds && x[i].round != y[i].round))
      return false;
  return true;
}

bool distinct_values(const std::vector<LkMerge>& m) {
  for (size_t i = 1; i < m.size(); i++) if ((u128)m[i].s * m[i - 1].p == (u128)m[i - 1].s * m[i].p) return false;
  return true;
}

}  // namespace

int main() {
  std::mt19937_64 rng(20261017);
  const int KINDS = 10, CASES = 2400;
  uint64_t merges = 0, rounds = 0, hac_checked = 0, complete_cases = 0;
  for (cs = 0; cs < CASES; cs++) {
    const int kind = cs % KINDS;
    const Case c = make_case(rng, kind);
    complete_cases += c.method == LK_COMPLETE;
    const Out base = emulate(c, 0, rng);
    merges += base.merges.size();
    rounds += base.rounds;
    if (c.dendrogram && c.n) CHECK(base.merges.size() <= c.n - 1, "more merges than n - 1");
    for (int order = 1; order < 4; order++) {
      const Out o = emulate(c, order, rng);
      CHECK(o.root == base.root && o.rounds == base.rounds && same_merges(o.merges, base.merges, true),
            "visit order %d differs (kind %d, n %u, method %d)", order, kind, c.n, c.method);
    }
    // the cut-mode partition equals the dendrogram-mode one
    Case other = c;
    other.dendrogram = !c.dendrogram;
    CHECK(emulate(other, 2, rng).root == base.root, "cut and dendrogram modes partition differently (kind %d)", kind);
    if (c.tie_free) {
      const Out h = sequential(c);
      if (distinct_values(h.merges)) {
        hac_checked++;
        CHECK(h.root == base.root && same_merges(h.merges, base.merges, false), "rounds differ from sequential HAC (kind %d, n %u, method %d)",
              kind, c.n, c.method);
      }
    }
  }
  printf("%d cases (%llu complete linkage), %llu merges, %llu rounds, %llu checked against sequential HAC, %d failures\n", CASES,
         (unsigned long long)complete_cases, (unsigned long long)merges, (unsigned long long)rounds, (unsigned long long)hac_checked, failures);
  return failures ? 1 : 0;
}
