// emu_entry_layout.cpp -- skdb::entry_layout (skani_b200/csrc/entry_layout.cuh), the section arithmetic sk_sketch_set_encode
// lays entries out with, against what the host writer (put_params + put_sketch, put_sketch(markers_only(s))) writes:
// the entry length and the value found at every section offset, for both entry forms, on constructed sketches.
// Prints "<cases> cases, <failures> failures".
#include <cstdio>
#include <random>

#include "../../skani_b200/cli/sketch_db.hpp"
#include "../../skani_b200/csrc/entry_layout.cuh"

using namespace skdb;

static int failures = 0, cases = 0;
#define EXPECT(cond, what)                                                      \
  do {                                                                          \
    if (!(cond)) { failures++; printf("FAIL case %d: %s\n", cases, what); }     \
  } while (0)

// list lengths: one k-mer per entry of `lists` (1 = a single-position key); records in (contig, pos) order
static HostSketch make(std::mt19937_64& rng, size_t name_len, const std::vector<uint32_t>& lists, size_t n_contigs, size_t n_markers) {
  HostSketch s;
  for (size_t i = 0; i < name_len; i++) s.file_name += (char)('a' + i % 26);
  uint32_t km = 7;
  for (uint32_t n : lists) {
    km += 1 + (uint32_t)(rng() % 1000);
    for (uint32_t t = 0; t < n; t++) { s.kmer.push_back(km); s.pos.push_back(t * 17 + 3); s.cc.push_back((uint32_t)(t % 3) << 1 | (t & 1)); }
  }
  for (size_t c = 0; c < n_contigs; c++) {
    s.contigs.push_back(std::string(rng() % 40, 'x'));
    s.contig_lengths.push_back(500 + (uint32_t)(rng() % 100000));
    s.total_len += s.contig_lengths.back();
  }
  for (size_t m = 0; m < n_markers; m++) s.markers.push_back(1000 + 3 * m);
  s.c = s.marker_c = 30; s.k = 15; s.contig_order = rng() % 5;
  return s;
}

static void check(const HostSketch& s) {
  for (int form = 0; form < 2; form++) {
    cases++;
    const bool full = form == 0;
    Out o;
    if (full) {
      DiskParams p; p.c = 30; p.k = 15; p.marker_c = 200;
      put_params(o, p);
      put_sketch(o, s);
    } else {
      put_sketch(o, markers_only(s));
    }
    EntryCounts c;
    c.params = c.seeds = full;
    c.name_len = s.file_name.size();
    for (size_t i = 0; i < s.kmer.size();) {
      size_t j = i + 1;
      while (j < s.kmer.size() && s.kmer[j] == s.kmer[i]) j++;
      c.n_keys++;
      if (j - i > 1) c.n_multi++;
      i = j;
    }
    if (!full) c.n_keys = c.n_multi = 0;
    c.n_records = full ? s.kmer.size() : 0;
    c.n_contigs = s.contigs.size();
    for (auto& x : s.contigs) c.contig_name_bytes += x.size();
    c.n_contig_lengths = full ? s.contig_lengths.size() : 0;
    c.n_markers = s.markers.size();
    const EntryLayout l = entry_layout(c);
    const uint8_t* b = o.b.data();
    EXPECT(l.length == o.b.size(), "length");
    if (l.length != o.b.size()) { printf("  %llu != %zu\n", (unsigned long long)l.length, o.b.size()); continue; }
    EXPECT(!full || l.name_at == 626, "params bytes");
    EXPECT(load_u64(b + l.name_at) == s.file_name.size(), "name length");
    EXPECT(b[l.tag_at] == (full ? 1 : 0), "Option tag");
    if (full) {
      EXPECT(load_u64(b + l.keys_at) == c.n_keys, "n_keys");
      if (c.n_keys) EXPECT(load_u32(b + l.keys_at + 8) == s.kmer[0], "first k-mer");
    }
    EXPECT(load_u64(b + l.multi_at) == c.n_multi, "n_multi");
    EXPECT(load_u64(b + l.contigs_at) == s.contigs.size(), "contig count");
    EXPECT(load_u64(b + l.total_len_at) == s.total_len, "total_len");
    EXPECT(load_u64(b + l.ctg_len_at) == c.n_contig_lengths, "contig length count");
    if (c.n_contig_lengths) EXPECT(load_u32(b + l.ctg_len_at + 8) == s.contig_lengths[0], "first contig length");
    EXPECT(load_u64(b + l.repetitive_at) == 0, "repetitive_kmers");
    EXPECT(load_u64(b + l.markers_at) == s.markers.size(), "marker count");
    if (c.n_markers) EXPECT(load_u64(b + l.markers_at + 8) == s.markers[0], "first marker");
    EXPECT(load_u64(b + l.tail_at) == s.marker_c && load_u64(b + l.tail_at + 8) == s.c && load_u64(b + l.tail_at + 16) == s.k &&
           load_u64(b + l.tail_at + 24) == s.contig_order, "tail");
  }
}

int main() {
  std::mt19937_64 rng(5);
  for (size_t name = 0; name <= 17; name++) check(make(rng, name, {1, 2, 1}, 2, 3));   // names of 0 to 17 bytes
  check(make(rng, 4, {}, 1, 10));                                                       // zero records
  check(make(rng, 4, std::vector<uint32_t>(500, 1), 3, 40));                            // all single
  check(make(rng, 4, {2, 3, 7, 2, 1000}, 3, 40));                                       // all multi
  std::vector<uint32_t> mixed;
  for (uint32_t n = 2; n <= 1000; n += 37) { mixed.push_back(n); mixed.push_back(1); }   // lists of 2 to 1000 positions
  mixed.push_back(1000);
  check(make(rng, 9, mixed, 5, 0));                                                     // zero markers
  check(make(rng, 9, {1, 4, 1}, 0, 2));                                                 // zero contigs
  check(make(rng, 0, {}, 0, 0));                                                        // nothing at all
  printf("%d cases, %d failures\n", cases, failures);
  return failures != 0;
}
