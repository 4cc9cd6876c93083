// The row bands and scan tiles of neighbour joining on several contexts (skani_b200/csrc/nj_plan.hpp: plan_nj) for every
// square of 1 to 400 row tiles over 1 to 16 contexts (also more contexts than row tiles).  Checks that the bands cover the
// row tiles in order without overlap and are equal in size to within one, that every upper-triangle tile is scanned by
// exactly one context, that a context only scans tiles one of whose row tiles is in its band, and that no context's load
// is more than nt / 2 + N tiles (half a row of tiles) away from the mean.
// Development/test harness only.
#include <cmath>
#include <cstdio>
#include <vector>

#include "../../skani_b200/csrc/nj_plan.hpp"

int main() {
  int failures = 0;
  uint64_t cases = 0, tiles = 0, empty_bands = 0, transposed = 0;
  double worst = 0;   // largest |load - mean| / (nt / N + N)
#define CHECK(cond, ...) do { if (!(cond)) { if (++failures < 20) { fprintf(stderr, "nt %u N %u: ", nt, N); fprintf(stderr, __VA_ARGS__); fputc('\n', stderr); } } } while (0)
  for (uint32_t nt = 1; nt <= 400; nt++)
    for (uint32_t N = 1; N <= 16; N++) {
      cases++;
      const sknj::NjPlan p = sknj::plan_nj(nt, N);
      CHECK(p.band.size() == N + 1 && p.tiles.size() == N, "sizes");
      if (p.band.size() != N + 1 || p.tiles.size() != N) continue;
      CHECK(p.band[0] == 0 && p.band[N] == nt, "bands do not span the row tiles");
      for (uint32_t d = 0; d < N; d++) {
        CHECK(p.band[d] <= p.band[d + 1], "band %u out of order", d);
        const uint32_t w = p.band[d + 1] - p.band[d];
        CHECK(w == nt / N || w == nt / N + 1, "band %u has %u row tiles", d, w);
        empty_bands += w == 0;
      }
      std::vector<uint8_t> seen((size_t)nt * nt, 0);
      const double mean = (double)nt * (nt + 1) / 2 / N;
      for (uint32_t d = 0; d < N; d++) {
        const auto in_band = [&](uint32_t a) { return a >= p.band[d] && a < p.band[d + 1]; };
        for (uint64_t t : p.tiles[d]) {
          const uint32_t a = (uint32_t)(t >> 32), b = (uint32_t)t;
          CHECK(a <= b && b < nt, "tile (%u, %u) outside the upper triangle", a, b);
          if (a > b || b >= nt) continue;
          CHECK(in_band(a) || in_band(b), "context %u scans tile (%u, %u) without its rows", d, a, b);
          transposed += !in_band(a);
          seen[(size_t)a * nt + b]++;
        }
        const double off = std::fabs((double)p.tiles[d].size() - mean), bound = (double)nt / 2 + N;
        CHECK(off <= bound, "context %u scans %zu tiles, mean %.1f", d, p.tiles[d].size(), mean);
        if (off / bound > worst) worst = off / bound;
      }
      for (uint32_t b = 0; b < nt; b++)
        for (uint32_t a = 0; a <= b; a++) {
          CHECK(seen[(size_t)a * nt + b] == 1, "tile (%u, %u) scanned %u times", a, b, seen[(size_t)a * nt + b]);
          tiles++;
        }
    }
  printf("%llu cases, %llu tiles, %llu transposed, %llu empty bands, worst load %.3f of the bound, %d failures\n", (unsigned long long)cases,
         (unsigned long long)tiles, (unsigned long long)transposed, (unsigned long long)empty_bands, worst, failures);
  return failures != 0;
}
