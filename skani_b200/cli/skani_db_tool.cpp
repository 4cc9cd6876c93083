// skani_db_tool.cpp -- host-only helper around sketch_db.hpp (no CUDA): lets the CPU test-suite exercise the skani v0.3.0
// database writer and reader without a GPU.
//   skani-db-tool write <dir> <c> <k> <marker_c>   < sketches in the text form below  -> sketches.db, index.db, markers.bin
//   skani-db-tool dump  <dir>                       -> the same text form, read back through index.db / sketches.db /
//                                                      markers.bin (records sorted by (kmer, contig, pos), markers ascending)
//   skani-db-tool fastx <file>                      -> the CLI's FASTA/FASTQ(.gz) reader (fastx.hpp): "OK n" then one line per
//                                                      record "<length> <fnv1a64 of the sequence> <id>", or "ERR"
//   skani-db-tool groups <max_records> <threads> <input>...
//                                                   -> the sketch inputs of triangle / dist (.sketch files and databases) as
//                                                      the CLI opens and groups them: "PARAMS c k marker_c", "N entries", then
//                                                      per group "G <first entry> <sketches> <records>" and per sketch
//                                                      "S <records> <contig_order> <file name>"; ERROR and exit 1 on a refusal
// Text form, one sketch = the lines
//   S <contig_order> <total_len> <file name>
//   C <contig header>            (one line per contig)
//   L <n> <len> ...              contig lengths
//   R <n> <kmer> <pos> <cc> ...  seed records grouped by k-mer
//   M <n> <marker> ...
//   E
#include <algorithm>
#include <iostream>
#include <numeric>
#include <sstream>

#include "fastx.hpp"
#include "sketch_db.hpp"

using namespace skdb;

static void print_sketch(const HostSketch& s0, const char* tag) {
  HostSketch s = s0;
  std::vector<size_t> ord(s.kmer.size());
  std::iota(ord.begin(), ord.end(), 0);
  std::sort(ord.begin(), ord.end(), [&](size_t a, size_t b) {
    if (s.kmer[a] != s.kmer[b]) return s.kmer[a] < s.kmer[b];
    if ((s.cc[a] >> 1) != (s.cc[b] >> 1)) return (s.cc[a] >> 1) < (s.cc[b] >> 1);
    return s.pos[a] < s.pos[b];
  });
  std::sort(s.markers.begin(), s.markers.end());
  printf("%s %llu %llu %s\n", tag, (unsigned long long)s.contig_order, (unsigned long long)s.total_len, s.file_name.c_str());
  for (auto& c : s.contigs) printf("C %s\n", c.c_str());
  printf("L %zu", s.contig_lengths.size());
  for (uint32_t l : s.contig_lengths) printf(" %u", l);
  printf("\nR %zu", ord.size());
  for (size_t i : ord) printf(" %u %u %u", s.kmer[i], s.pos[i], s.cc[i]);
  printf("\nM %zu", s.markers.size());
  for (uint64_t m : s.markers) printf(" %llu", (unsigned long long)m);
  printf("\nP %d %llu %llu %llu %llu %d %d\nE\n", (int)s.has_seeds, (unsigned long long)s.marker_c, (unsigned long long)s.c,
         (unsigned long long)s.k, (unsigned long long)s.repetitive_kmers, (int)s.individual_contig, (int)s.amino_acid);
}

int main(int argc, char** argv) {
  try {
    if (argc >= 6 && std::string(argv[1]) == "write") {
      DiskParams dp;
      dp.c = strtoull(argv[3], nullptr, 10); dp.k = strtoull(argv[4], nullptr, 10); dp.marker_c = strtoull(argv[5], nullptr, 10);
      DbWriter w;
      if (!w.open(argv[2], dp)) { fprintf(stderr, "cannot create %s/sketches.db\n", argv[2]); return 1; }
      std::string line;
      HostSketch s;
      while (std::getline(std::cin, line)) {
        if (line.empty()) continue;
        std::istringstream is(line.substr(line.size() > 1 ? 2 : 1));
        switch (line[0]) {
          case 'S': {
            s = HostSketch();
            s.c = dp.c; s.k = dp.k; s.marker_c = dp.c;
            is >> s.contig_order >> s.total_len;
            std::getline(is, s.file_name);
            if (!s.file_name.empty() && s.file_name[0] == ' ') s.file_name.erase(0, 1);
            break;
          }
          case 'C': s.contigs.push_back(line.substr(2)); break;
          case 'L': { size_t n; is >> n; s.contig_lengths.resize(n); for (auto& x : s.contig_lengths) is >> x; break; }
          case 'R': { size_t n; is >> n; s.kmer.resize(n); s.pos.resize(n); s.cc.resize(n); for (size_t i = 0; i < n; i++) is >> s.kmer[i] >> s.pos[i] >> s.cc[i]; break; }
          case 'M': { size_t n; is >> n; s.markers.resize(n); for (auto& x : s.markers) is >> x; break; }
          case 'E': if (!w.add(s, dp)) { fprintf(stderr, "write failed\n"); return 1; } break;
          default: break;
        }
      }
      return w.finalize() ? 0 : 1;
    }
    if (argc >= 3 && std::string(argv[1]) == "dump") {
      const std::string dir = argv[2];
      DiskParams dp;
      std::vector<HostSketch> mk;
      read_markers_bin(dir + "/markers.bin", dp, mk);
      std::vector<IndexEntry> ix;
      read_index_db(dir + "/index.db", ix);
      std::vector<uint8_t> db;
      if (!read_file(dir + "/sketches.db", db)) { fprintf(stderr, "cannot read sketches.db\n"); return 1; }
      printf("PARAMS %llu %llu %llu %d %d %llu\n", (unsigned long long)dp.c, (unsigned long long)dp.k, (unsigned long long)dp.marker_c,
             (int)dp.use_syncs, (int)dp.use_aa, (unsigned long long)dp.orf_size);
      printf("N %zu %zu\n", ix.size(), mk.size());
      for (size_t i = 0; i < ix.size(); i++) {
        if (ix[i].offset + ix[i].length > db.size()) { fprintf(stderr, "index entry out of range\n"); return 1; }
        DiskParams p2;
        HostSketch s = read_blob(db.data() + ix[i].offset, ix[i].length, &p2);
        if (!(p2 == dp) || s.file_name != ix[i].file_name) { fprintf(stderr, "entry %zu disagrees with index.db / markers.bin\n", i); return 1; }
        print_sketch(s, "S");
      }
      for (auto& m : mk) print_sketch(m, "K");
      return 0;
    }
    if (argc >= 5 && std::string(argv[1]) == "groups") {
      SketchInputs si;
      if (!open_sketch_inputs(std::vector<std::string>(argv + 4, argv + argc), si)) return 1;
      printf("PARAMS %llu %llu %llu\nN %zu\n", (unsigned long long)si.params.c, (unsigned long long)si.params.k,
             (unsigned long long)si.params.marker_c, si.entries.size());
      std::vector<size_t> all(si.entries.size());
      std::iota(all.begin(), all.end(), 0);
      SketchGroupReader rd(si, std::move(all), atoi(argv[3]), strtoull(argv[2], nullptr, 10));
      SketchGroup g;
      while (rd.next(g)) {
        printf("G %zu %zu %llu\n", rd.first, g.size(), (unsigned long long)g.records);
        for (auto& h : g.scan) printf("S %llu %llu %s\n", (unsigned long long)h.n_records, (unsigned long long)h.contig_order, h.file_name.c_str());
      }
      return rd.failed ? 1 : 0;
    }
    if (argc >= 3 && std::string(argv[1]) == "fastx") {
      std::vector<fastx::Record> recs;
      if (!fastx::read_fastx(argv[2], recs, argc >= 4 ? std::max(1, atoi(argv[3])) : 1)) { printf("ERR\n"); return 0; }    // [threads]
      printf("OK %zu\n", recs.size());
      for (auto& r : recs) {
        uint64_t h = 0xcbf29ce484222325ull;
        for (unsigned char ch : r.seq) { h ^= ch; h *= 0x100000001b3ull; }
        printf("%zu %llu %s\n", r.seq.size(), (unsigned long long)h, r.id.c_str());
      }
      return 0;
    }
  } catch (const std::exception& e) {
    fprintf(stderr, "ERROR %s\n", e.what());
    return 1;
  }
  fprintf(stderr, "usage: skani-db-tool write <dir> <c> <k> <marker_c> < text | skani-db-tool dump <dir> | "
                  "skani-db-tool groups <max_records> <threads> <input>...\n");
  return 2;
}
