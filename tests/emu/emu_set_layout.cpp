// The sketch-set array table (skani_b200/csrc/set_layout.hpp) on the CPU: over random counts, zeros included, the blob
// layout equals the format's arithmetic written out by hand, the metadata encoder and decoder round-trip, the per-genome
// slices of a concatenation start where the sentinel rule says, and the store's genome bytes are 22 S + 8 U + 8 M + 8 C +
// 8 HT + 8.
#include <cstdio>
#include <cstring>
#include <random>

#include "../../skani_b200/csrc/set_layout.hpp"

using namespace sk;

static int failures = 0;
#define CHECK(cond)                                                        \
  do {                                                                     \
    if (!(cond)) {                                                         \
      if (failures++ < 20) fprintf(stderr, "%s:%d: %s\n", __FILE__, __LINE__, #cond); \
    }                                                                      \
  } while (0)

static uint64_t pick(std::mt19937_64& rng, uint64_t hi) {   // 0 one time in four, else uniform in [0, hi]
  return rng() % 4 == 0 ? 0 : rng() % (hi + 1);
}

// the blob layout, spelt out array by array
static void hand_layout(uint64_t G, uint64_t S, uint64_t U, uint64_t M, uint64_t C, uint64_t HT, uint64_t off[12], uint64_t* total) {
  const uint64_t n[12] = {S * 4, S * 4, S * 4, S * 2, S * 4, S * 4, U * 4, (U + G) * 4, M * 8, (C + G) * 4, C * 4, HT * 8};
  uint64_t o = 0;
  for (int a = 0; a < 12; a++) { off[a] = o; o += (n[a] + 255) / 256 * 256; }
  *total = o ? o : 256;
}

int main() {
  std::mt19937_64 rng(20261016);
  const int CASES = 20000;
  for (int t = 0; t < CASES; t++) {
    const uint64_t big = t % 3 == 0 ? (1ull << 34) : 1000;
    // ---- layout over raw totals
    const uint64_t G = pick(rng, t % 2 ? 40 : 1u << 20);
    const uint64_t n[N_COUNTS] = {pick(rng, big), pick(rng, big), pick(rng, big), pick(rng, big), pick(rng, big)};
    uint64_t off[12], total;
    hand_layout(G, n[CNT_S], n[CNT_U], n[CNT_M], n[CNT_C], n[CNT_HT], off, &total);
    const BlobLayout b = blob_layout(G, n);
    CHECK(b.total == total);
    for (int a = 0; a < 12; a++) {
      CHECK(b.off[a] == off[a]);
      CHECK(b.off[a] + b.bytes[a] <= (a < 11 ? off[a + 1] : total));
    }
    const bool tables = rng() & 1;
    CHECK(meta_words(G, n[CNT_C], tables) == 10 + 4 * (G + 1) + G + n[CNT_C] + (tables ? G + 1 : 0));

    // ---- genomes one by one: concatenation, sentinels, store records, metadata
    const uint32_t g = (uint32_t)pick(rng, 12);
    const bool mo = !tables && (rng() % 3 == 0);
    SetMeta m;
    m.c = 1 + rng() % 200; m.k = 1 + rng() % 16; m.marker_c = m.c + rng() % 1000; m.tables = tables;
    std::vector<std::vector<uint64_t>> cnt(g, std::vector<uint64_t>(N_COUNTS));
    std::vector<uint64_t> elems_before(BLOB_ARRAYS, 0);
    std::vector<uint32_t> ctg;
    for (uint32_t i = 0; i < g; i++) {
      for (int x = 0; x < N_COUNTS; x++) cnt[i][x] = pick(rng, x == CNT_C ? 30 : 5000);
      const uint64_t* c = cnt[i].data();
      // where genome i's slice begins in the concatenation of the genomes before it
      std::vector<uint64_t> prefix(N_COUNTS, 0);
      for (uint32_t j = 0; j < i; j++) for (int x = 0; x < N_COUNTS; x++) prefix[x] += cnt[j][x];
      for (int a = 0; a < BLOB_ARRAYS; a++) {
        CHECK(array_index(a, i, prefix[SET_ARRAYS[a].by]) == elems_before[a]);
        CHECK(array_index(a, i, prefix[SET_ARRAYS[a].by]) == prefix[SET_ARRAYS[a].by] + ((a == 7 || a == 9) ? i : 0));
        elems_before[a] += array_elems(a, 1, c);
      }
      // store record of one genome
      uint64_t slice[BLOB_ARRAYS];
      const uint64_t rec = genome_slices(c, slice);
      const uint64_t gb = genome_bytes(c);
      CHECK(gb == 22 * c[CNT_S] + 8 * c[CNT_U] + 8 * c[CNT_M] + 8 * c[CNT_C] + 8 * c[CNT_HT] + 8);
      CHECK(rec >= gb && rec % 16 == 0 && rec < gb + 16 * BLOB_ARRAYS);
      for (int a = 0; a < BLOB_ARRAYS; a++) {
        CHECK(slice[a] % 16 == 0);
        CHECK(slice[a] + array_elems(a, 1, c) * SET_ARRAYS[a].esz <= (a < 11 ? slice[a + 1] : rec));
      }
      ctg.assign(c[CNT_C], 0);
      for (auto& v : ctg) v = (uint32_t)rng();
      meta_push(m, c, mo, rng() % (1ull << 40), ctg.begin(), ctg.end());
      if (!mo)
        for (size_t j = 0; j < ctg.size(); j++) CHECK(m.ctg_len[m.ctg_len.size() - ctg.size() + j] == ctg[j]);
    }
    // whole-set totals of the concatenation = the per-genome sums (zeroed where the array does not travel)
    CHECK(m.G == g);
    for (int x = 0; x < N_COUNTS; x++) {
      uint64_t s = 0;
      for (uint32_t i = 0; i < g; i++) s += cnt[i][x];
      const bool travels = mo ? x == CNT_M : (x != CNT_HT || tables);
      CHECK(m.n[x] == (travels ? s : 0));
      CHECK(m.off[x].size() == g + 1 && m.off[x][g] == m.n[x]);
    }
    for (int a = 0; a < BLOB_ARRAYS; a++)
      if (array_travels(a, mo, tables)) CHECK(array_elems(a, g, m.n) == elems_before[a]);
    // encode -> decode -> encode
    std::vector<uint64_t> w(meta_words(m.G, m.n[CNT_C], m.tables) + 1, 0xDEADBEEFull);
    encode_meta(m, w.data());
    CHECK(w.back() == 0xDEADBEEFull);          // exactly meta_words words
    CHECK(w[0] == m.G && w[1] == m.n[CNT_S] && w[2] == m.n[CNT_U] && w[3] == m.n[CNT_M] && w[4] == m.n[CNT_C]);
    CHECK(w[5] == m.c && w[6] == m.k && w[7] == m.marker_c && w[8] == m.n[CNT_HT] && w[9] == (uint64_t)tables);
    CHECK(w[META_HEADER + (g + 1)] == m.off[CNT_U][0] && w[META_HEADER + 4 * (g + 1) - 1] == m.off[CNT_C][g]);
    const SetMeta d = decode_meta(w.data());
    CHECK(d.G == m.G && d.c == m.c && d.k == m.k && d.marker_c == m.marker_c && d.tables == m.tables);
    for (int x = 0; x < N_COUNTS; x++) CHECK(d.n[x] == m.n[x] && d.off[x] == m.off[x]);
    CHECK(d.total_len == m.total_len && d.ctg_len == m.ctg_len);
    std::vector<uint64_t> w2(w.size(), 0xDEADBEEFull);
    encode_meta(d, w2.data());
    CHECK(w2 == w);
  }
  printf("%d cases, %d failures\n", CASES, failures);
  return failures != 0;
}
