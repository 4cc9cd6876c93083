// nj_plan.hpp -- the row bands and scan tiles of neighbour joining on several contexts (nj.cu, sk_neighbor_joining_multi).
// Host only, no CUDA: tests/emu/emu_nj_plan.cpp runs it on the CPU.
//
// The square of dimension P (a multiple of the scan tile) has nt = P / tile row tiles.  Context d owns the row tiles
// [band[d], band[d + 1]): equal in count to within one, in order, so the bands cover the slots in order without overlap
// (with more contexts than row tiles some bands are empty).  A context holds full rows of its band only.
//
// The upper-triangle tile (a, b), a <= b, is scanned by the owner of row tile a or of row tile b: the owner of b reads it
// transposed (D is symmetric bit for bit).  A tile whose row tiles share an owner goes to that owner; a tile between two
// bands goes to whichever of the two owners has the smaller load so far (ties: a's owner), the loads starting from the
// bands' own triangles.  Every context's load is then within nt / 2 + N tiles of the mean (under 1 % of it from a few
// hundred row tiles up).  Deterministic: the plan depends only on nt and N.
#pragma once
#include <cstdint>
#include <vector>

namespace sknj {

struct NjPlan {
  std::vector<uint32_t> band;                  // N + 1 row-tile boundaries
  std::vector<std::vector<uint64_t>> tiles;    // tiles[d]: a << 32 | b (a <= b), in column-major order of the upper triangle
};

// the N + 1 row-tile boundaries of the bands
inline std::vector<uint32_t> nj_bands(uint32_t nt, uint32_t n_ctx) {
  std::vector<uint32_t> band(n_ctx + 1);
  for (uint32_t d = 0; d <= n_ctx; d++) band[d] = (uint32_t)((uint64_t)d * nt / n_ctx);
  return band;
}

inline NjPlan plan_nj(uint32_t nt, uint32_t n_ctx) {
  NjPlan p;
  p.band = nj_bands(nt, n_ctx);
  std::vector<uint32_t> owner(nt);
  for (uint32_t d = 0; d < n_ctx; d++)
    for (uint32_t a = p.band[d]; a < p.band[d + 1]; a++) owner[a] = d;
  p.tiles.assign(n_ctx, {});
  std::vector<uint64_t> load(n_ctx, 0);
  for (uint32_t d = 0; d < n_ctx; d++) {
    const uint64_t w = p.band[d + 1] - p.band[d];
    load[d] = w * (w + 1) / 2;
  }
  for (uint32_t b = 0; b < nt; b++)
    for (uint32_t a = 0; a <= b; a++) {
      const uint32_t da = owner[a], db = owner[b];
      const uint32_t d = da == db || load[da] <= load[db] ? da : db;
      if (da != db) load[d]++;
      p.tiles[d].push_back((uint64_t)a << 32 | b);
    }
  return p;
}

}  // namespace sknj
