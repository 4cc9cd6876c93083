// emu_db_scan.cpp -- host checks of the sketch-entry framing walk (skani_b200/cli/sketch_db.hpp: scan_entry, expand_records,
// get_sketch) on blobs written by the host writer (put_params + put_sketch).  Built with AddressSanitizer by
// tests/test_emu_db_scan.py, so a read past the end of a blob is caught.
//   emu_db_scan <out dir>   writes case<i>.sketch (the blob) and case<i>.txt (the scan and expansion, for the independent
//                           Python decoder) and prints "<n> cases, <f> failures"
#include <cstdio>
#include <memory>
#include <random>
#include <string>

#include "../../skani_b200/cli/sketch_db.hpp"

using namespace skdb;

static int failures = 0, cases = 0;
#define CHECK(c, what)                                                          \
  do {                                                                          \
    if (!(c)) { failures++; printf("FAIL case %d: %s\n", cases, what); }        \
  } while (0)

// records grouped by k-mer (ascending distinct k-mers): list_lens[j] records for the j-th multi-position k-mer, singles
// single-position k-mers, interleaved at random
static HostSketch make(std::mt19937_64& rng, const std::vector<uint32_t>& list_lens, size_t singles, size_t n_contigs,
                       size_t n_markers, bool seeds = true) {
  HostSketch s;
  s.file_name = "g/case" + std::to_string(cases) + ".fa";
  s.has_seeds = seeds;
  std::vector<uint32_t> groups(list_lens);
  groups.insert(groups.end(), singles, 1);
  std::shuffle(groups.begin(), groups.end(), rng);
  uint32_t kmer = (uint32_t)(rng() % 1000);
  for (uint32_t n : groups) {
    kmer += 1 + (uint32_t)(rng() % 50000);
    for (uint32_t t = 0; t < n; t++) {
      s.kmer.push_back(kmer);
      s.pos.push_back(rng() % 7 == 0 ? 0xFFFFFFFFu - (uint32_t)(rng() % 3) : (uint32_t)(rng() % 5000000));
      s.cc.push_back((uint32_t)(rng() % std::max<size_t>(2 * n_contigs, 2)) | (rng() % 11 == 0 ? 0x7FFFFFF0u : 0u));
    }
  }
  if (!seeds) s.kmer.clear(), s.pos.clear(), s.cc.clear();
  for (size_t c = 0; c < n_contigs; c++) {
    s.contigs.push_back("contig " + std::to_string(c) + std::string(rng() % 9, 'x'));
    s.contig_lengths.push_back(500 + (uint32_t)(rng() % 100000));
    s.total_len += s.contig_lengths.back();
  }
  for (size_t m = 0; m < n_markers; m++) s.markers.push_back(rng() >> 22);
  s.repetitive_kmers = rng() % 100;
  s.contig_order = rng() % 5;
  s.c = 30; s.marker_c = 30; s.k = 15;
  return s;
}

static std::vector<uint8_t> blob_of(const HostSketch& s) {
  Out o;
  DiskParams p; p.c = 30; p.k = 15; p.marker_c = 200;
  put_params(o, p);
  put_sketch(o, s);
  return o.b;
}

// scan_entry + expand_records + get_sketch against the writer's input; the text form for the Python decoder
static void check_case(const HostSketch& s, const std::string& dir) {
  const std::vector<uint8_t> b = blob_of(s);
  std::unique_ptr<uint8_t[]> exact(new uint8_t[b.size()]);     // exactly sized: AddressSanitizer sees any over-read
  memcpy(exact.get(), b.data(), b.size());
  SketchScan sc;
  try { sc = scan_entry(exact.get(), b.size()); }
  catch (const std::exception& e) { CHECK(false, e.what()); cases++; return; }
  HostSketch h;
  expand_records(exact.get(), sc, h);
  CHECK(sc.params.c == 30 && sc.params.k == 15 && sc.params.marker_c == 200 && !sc.params.use_aa, "params");
  CHECK(sc.file_name == s.file_name && sc.has_seeds == s.has_seeds && sc.contigs == s.contigs, "names");
  CHECK(sc.total_len == s.total_len && sc.contig_order == s.contig_order && sc.repetitive_kmers == s.repetitive_kmers, "metadata");
  CHECK(h.kmer == s.kmer && h.pos == s.pos && h.cc == s.cc, "records (writer's input order)");
  CHECK(sc.n_records == h.kmer.size(), "scan record count == expansion");
  CHECK(sc.n_ctg_len == s.contig_lengths.size() && sc.n_markers == s.markers.size(), "list counts");
  size_t n_keys = 0, n_multi = 0;
  for (size_t i = 0; i < s.kmer.size(); i++)
    if (i == 0 || s.kmer[i] != s.kmer[i - 1]) { n_keys++; n_multi += i + 1 < s.kmer.size() && s.kmer[i + 1] == s.kmer[i]; }
  CHECK(sc.n_keys == n_keys && sc.multi_at.size() == n_multi, "key and list counts");
  In in(exact.get(), b.size());
  get_params(in);
  const HostSketch d = get_sketch(in, true);
  CHECK(in.p == exact.get() + b.size(), "get_sketch consumes the blob");
  CHECK(d.kmer == s.kmer && d.pos == s.pos && d.cc == s.cc && d.contig_lengths == s.contig_lengths && d.markers == s.markers &&
        d.contigs == s.contigs && d.total_len == s.total_len && d.marker_c == s.marker_c && d.c == s.c && d.k == s.k, "get_sketch");
  // every truncation throws (inside the blob: AddressSanitizer)
  bool all_throw = true;
  for (size_t n = 0; n < b.size(); n++) {
    std::unique_ptr<uint8_t[]> t(new uint8_t[std::max<size_t>(n, 1)]);
    memcpy(t.get(), b.data(), n);
    bool threw = false;
    try { scan_entry(t.get(), n); } catch (const std::runtime_error& e) { threw = std::string(e.what()) == "truncated sketch data" || std::string(e.what()) == "corrupt length prefix"; }
    all_throw &= threw;
  }
  CHECK(all_throw, "every truncation throws");
  const std::string base = dir + "/case" + std::to_string(cases);
  write_file(base + ".sketch", b);
  FILE* f = fopen((base + ".txt").c_str(), "w");
  fprintf(f, "N %llu %llu %zu %llu %llu\nR", (unsigned long long)sc.n_keys, (unsigned long long)sc.n_records, sc.multi_at.size(),
          (unsigned long long)sc.n_ctg_len, (unsigned long long)sc.n_markers);
  for (size_t i = 0; i < h.kmer.size(); i++) fprintf(f, " %u %u %u", h.kmer[i], h.pos[i], h.cc[i]);
  fprintf(f, "\n");
  fclose(f);
  cases++;
}

static std::string error_of(const std::vector<uint8_t>& b, bool expand) {
  std::unique_ptr<uint8_t[]> t(new uint8_t[b.size()]);
  memcpy(t.get(), b.data(), b.size());
  try {
    SketchScan sc = scan_entry(t.get(), b.size());
    if (expand) { HostSketch h; expand_records(t.get(), sc, h); }
  } catch (const std::runtime_error& e) { return e.what(); }
  return "";
}

int main(int argc, char** argv) {
  if (argc < 2) { fprintf(stderr, "usage: emu_db_scan <out dir>\n"); return 2; }
  const std::string dir = argv[1];
  std::mt19937_64 rng(20261017);
  check_case(make(rng, {2, 3, 2, 5}, 200, 3, 40), dir);                          // typical
  check_case(make(rng, {2, 3, 4, 10, 100, 999, 1000}, 50, 2, 10), dir);          // long multi-position lists
  check_case(make(rng, {}, 0, 2, 5), dir);                                       // zero keys
  check_case(make(rng, {}, 0, 4, 30, false), dir);                               // markers only (Option None)
  check_case(make(rng, {}, 0, 0, 0, false), dir);                                // nothing at all
  check_case(make(rng, {2, 7}, 30, 0, 3), dir);                                  // zero contigs
  check_case(make(rng, {}, 1, 1, 1), dir);                                       // one record
  check_case(make(rng, {1000}, 0, 1, 0), dir);                                   // one key, one list

  // corruptions: (byte offset, new u64) -> the reader's messages (sketch_db.hpp In::len, scan_sketch)
  HostSketch s = make(rng, {2, 3}, 20, 2, 4);
  const std::vector<uint8_t> b = blob_of(s);
  const size_t P = 626, name = P, tag = name + 8 + s.file_name.size(), nkeys = tag + 1;
  const size_t n_keys = 22, nmulti = nkeys + 8 + 12 * n_keys, list0 = nmulti + 8;
  auto with = [&](size_t at, uint64_t v) { std::vector<uint8_t> c = b; memcpy(c.data() + at, &v, 8); return c; };
  CHECK(error_of(b, true).empty(), "corruption base case decodes");
  uint64_t got_keys; memcpy(&got_keys, b.data() + nkeys, 8);
  CHECK(got_keys == n_keys, "layout of the corruption case");
  for (size_t at : {name, nkeys, nmulti, list0})
    for (uint64_t v : {(uint64_t)1 << 60, (uint64_t)~0ull, (uint64_t)b.size()})
      CHECK(error_of(with(at, v), false) == "corrupt length prefix", ("length prefix at " + std::to_string(at)).c_str());
  std::vector<uint8_t> t2 = b;
  t2[tag] = 2;
  CHECK(error_of(t2, false) == "corrupt Option tag (a pre-0.3 .sketch file?)", "Option tag 2");
  t2[tag] = 255;
  CHECK(error_of(t2, false) == "corrupt Option tag (a pre-0.3 .sketch file?)", "Option tag 255");
  // a multi-position index past the lists: the scan accepts it, the expansion refuses it
  size_t k0 = nkeys + 8;
  while (true) { uint64_t v; memcpy(&v, b.data() + k0 + 4, 8); if (!value_is_single(v)) break; k0 += 12; }
  std::vector<uint8_t> bad = with(k0 + 4, multi_value(2));
  CHECK(error_of(bad, false).empty(), "scan leaves multi indices to the expansion");
  CHECK(error_of(bad, true) == "multi-position index out of range", "multi index out of range");
  cases++;
  printf("%d cases, %d failures\n", cases, failures);
  return failures != 0;
}
