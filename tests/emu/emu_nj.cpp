// sk_neighbor_joining's per-element arithmetic (skani_b200/csrc/nj_core.cuh) driven through whole runs on the host, the way
// nj.cu's kernels drive it: a padded square over slots (1.0, diagonal 0, both directions of every edge), row sums, dead slots
// marked with NJ_DEAD, the (Q, i << 32 | j) minimum over the upper triangle visited in a random order of elements, the update
// of every slot in a random order, compaction of the live slots into a smaller square when m <= 3/4 of its dimension, and the
// last two nodes joined at half their distance.
// Input (stdin): cases "n E" then E rows "a b bits" (bits = the float32 ANI's bit pattern, hex).  Output: per case "case n",
// then n - 1 rows "a b len_a len_b" with the lengths in hex-float notation.  Build with -ffp-contract=off.
// Development/test harness only.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "../../skani_b200/csrc/nj_core.cuh"

using namespace sk;

namespace {

constexpr uint32_t TILE = 64;
uint32_t padded(uint32_t s) { return (s + TILE - 1) / TILE * TILE; }

struct Join { uint32_t a, b; double la, lb; };

std::vector<Join> run(uint32_t n, const std::vector<uint32_t>& ea, const std::vector<uint32_t>& eb, const std::vector<float>& ani,
                      std::mt19937_64& rng) {
  std::vector<Join> out;
  if (n < 2) return out;
  uint32_t S = n, P = padded(n);
  std::vector<double> D((size_t)P * P), R(P);
  std::vector<uint32_t> node(P);
  for (size_t x = 0; x < D.size(); x++) D[x] = x / P == x % P ? 0.0 : 1.0;
  for (size_t e = 0; e < ea.size(); e++) {
    if (!(ani[e] > 0.1f)) continue;
    const double d = nj_dist(ani[e]);
    D[(size_t)ea[e] * P + eb[e]] = d;
    D[(size_t)eb[e] * P + ea[e]] = d;
  }
  for (uint32_t r = 0; r < P; r++) {
    double s = 0.0;
    for (uint32_t c = 0; c < n; c++) s = nj_add(s, D[(size_t)r * P + c]);
    R[r] = r < n ? s : NJ_DEAD;
    node[r] = r;
  }
  std::vector<uint64_t> cells;
  for (uint32_t t = 0; t + 2 < n; t++) {
    const uint32_t m = n - t;
    if (S > TILE && 4ull * m <= 3ull * S) {
      std::vector<uint32_t> src;
      for (uint32_t k = 0; k < S; k++) if (R[k] != NJ_DEAD) src.push_back(k);
      const uint32_t P2 = padded(m);
      std::vector<double> D2((size_t)P2 * P2), R2(P2);
      std::vector<uint32_t> node2(P2);
      for (uint32_t r = 0; r < P2; r++) {
        for (uint32_t c = 0; c < P2; c++)
          D2[(size_t)r * P2 + c] = r < m && c < m ? D[(size_t)src[r] * P + src[c]] : r == c ? 0.0 : 1.0;
        R2[r] = r < m ? R[src[r]] : NJ_DEAD;
        node2[r] = r < m ? node[src[r]] : 0;
      }
      D.swap(D2); R.swap(R2); node.swap(node2);
      S = m; P = P2;
    }
    cells.clear();
    for (uint32_t r = 0; r < P; r++)
      for (uint32_t c = r + 1; c < P; c++) cells.push_back((uint64_t)r << 32 | c);
    std::shuffle(cells.begin(), cells.end(), rng);
    double bq = __builtin_huge_val();
    uint64_t bk = UINT64_MAX;
    for (uint64_t key : cells) {
      const uint32_t r = (uint32_t)(key >> 32), c = (uint32_t)key;
      const double q = nj_q(m, D[(size_t)r * P + c], R[r], R[c]);
      if (nj_before(q, key, bq, bk)) { bq = q; bk = key; }
    }
    const uint32_t i = (uint32_t)(bk >> 32), j = (uint32_t)bk;
    const double dij = D[(size_t)i * P + j], ri = R[i], rj = R[j];
    const double di = nj_delta_i(m, dij, ri, rj), ru = nj_ru(m, ri, rj, dij);
    std::vector<uint32_t> ks(S);
    for (uint32_t k = 0; k < S; k++) ks[k] = k;
    std::shuffle(ks.begin(), ks.end(), rng);
    for (uint32_t k : ks) {
      if (k == j) { R[k] = NJ_DEAD; continue; }
      if (k == i) {
        out.push_back({node[i], node[j], di, nj_sub(dij, di)});
        node[k] = n + t;
        R[k] = ru;
        continue;
      }
      if (R[k] == NJ_DEAD) continue;
      const double dik = D[(size_t)i * P + k], djk = D[(size_t)j * P + k];
      const double duk = nj_duk(dik, djk, dij);
      D[(size_t)i * P + k] = duk;
      D[(size_t)k * P + i] = duk;
      R[k] = nj_rk(R[k], dik, djk, duk);
    }
  }
  uint32_t a = UINT32_MAX, b = UINT32_MAX;
  for (uint32_t k = 0; k < S && b == UINT32_MAX; k++)
    if (R[k] != NJ_DEAD) (a == UINT32_MAX ? a : b) = k;
  const double h = nj_mul(0.5, D[(size_t)a * P + b]);
  out.push_back({node[a], node[b], h, h});
  return out;
}

}  // namespace

int main() {
  std::mt19937_64 rng(12345);
  uint32_t n;
  unsigned long long E;
  while (scanf("%u %llu", &n, &E) == 2) {
    std::vector<uint32_t> a(E), b(E);
    std::vector<float> ani(E);
    for (unsigned long long e = 0; e < E; e++) {
      unsigned bits;
      if (scanf("%u %u %x", &a[e], &b[e], &bits) != 3) return 2;
      memcpy(&ani[e], &bits, 4);
    }
    printf("case %u\n", n);
    for (const Join& j : run(n, a, b, ani, rng)) printf("%u %u %a %a\n", j.a, j.b, j.la, j.lb);
  }
  return 0;
}
