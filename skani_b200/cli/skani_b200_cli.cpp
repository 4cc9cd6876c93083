// skani_b200_cli.cpp -- `skani-b200 triangle|dist|sketch|search|cluster`: host driver over the C ABI (include/skani_b200.h).
//
// Mirrors the reference's command drivers:
//   triangle  src/triangle.rs:13-169  (flags src/cli.rs:236-330, defaults src/parse.rs:790-921)
//   dist      src/dist.rs:12-190      (flags src/cli.rs:100-232, defaults src/parse.rs:628-788)
//   sketch    src/sketch.rs:15-201    (consolidated sketches.db / index.db / markers.bin, or --separate-sketches)
//   search    src/search.rs:16-300    (flags src/cli.rs:332-448, defaults src/parse.rs:380-500)
// and their writers (TSV src/file_io.rs:15-139,608-678; phylip + .af matrices src/file_io.rs:364-539).
// FASTA/FASTQ(.gz) record rules follow needletail as skani uses it (ids = whole header line, sequences with line
// breaks removed, records < 500 bp dropped, src/file_io.rs:141-362).  On-disk formats: sketch_db.hpp.
// All heavy work happens on the GPU through libskani_b200.so.  search keeps the reference's structure but not its memory
// model: instead of deserialising a reference sketch from the mmap'd database for every passing pair
// (src/search.rs:142-166) it screens each group of queries against all marker sketches, indexed once on the GPU, loads each
// reference sketch that passed for some query exactly once (per block of queries), imports them to the device in groups
// through the same reader as triangle's and dist's sketch inputs, and chains every pair there.
// --gpus N: dist and search split the references into contiguous blocks, one per GPU, and copy the query set to every GPU
// (sk_screen_query_ref_multi / sk_chain_pairs_multi); the output is byte-identical to one GPU's.
// sketch encodes the database entries on the GPU (sk_sketch_set_encode) and, with --gpus N, sketches each group of files
// in N contiguous runs, one per GPU; the database is byte-identical for every N.
// triangle and dist take pre-sketched inputs as .sketch files and as consolidated databases (sketch_db.hpp: SketchInputs),
// read as stored and imported in groups of < 2^28 records (sk_sketch_set_import_blobs expands them on the device), so that
// host memory holds one group's bytes at a time.
#include <dirent.h>
#include <sys/stat.h>
#include <zlib.h>

#include <algorithm>
#include <array>
#include <chrono>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <numeric>
#include <set>
#include <string>
#include <thread>
#include <vector>

#include "../../include/skani_b200.h"
#include "fastx.hpp"
#include "search_plan.hpp"
#include "sketch_db.hpp"

namespace {

using fastx::Record;
using fastx::read_fastx;

struct Genome {          // one Sketch-to-be (src/types.rs:253-277 metadata kept on the host)
  std::string file_name;
  std::vector<std::string> contigs;  // header lines
  uint64_t contig_order = 0;
  uint64_t total_len = 0;
};

struct Inputs {
  std::vector<Genome> genomes;       // sorted by (file_name, contig_order) (src/types.rs:360-364)
  std::vector<uint8_t, fastx::no_init_alloc<uint8_t>> bases;      // filled (and first touched) by the parallel copies of load_inputs
  std::vector<uint64_t> contig_off{0};
  std::vector<uint32_t> genome_of_contig;
};

// file_io::fastx_to_sketches / fastx_to_multiple_sketch_rewrite record rules (src/file_io.rs:141-362)
void load_inputs(std::vector<std::string> files, bool individual, int threads, Inputs& in) {
  std::sort(files.begin(), files.end());                      // final order = (file_name, contig_order)
  // step 1 (files in parallel): open / inflate and LOCATE the records; the text stays alive.  Step 2 (serial, metadata only):
  // record rules + layout.  Step 3 (parallel): line breaks are stripped straight into the flat buffer -- one copy per base.
  std::vector<fastx::LoadedFile> loaded(files.size());
  std::vector<int> status(files.size(), 0);
  threads = std::max(threads, 1);
  {   // files in parallel (dynamic); threads left over when there are few files go to member-parallel BGZF inflate
    std::atomic<size_t> next{0};
    const int per_file = std::max<int>(1, threads / (int)std::max<size_t>(files.size(), 1));
    auto worker = [&] { for (size_t i; (i = next.fetch_add(1)) < files.size();) status[i] = fastx::open_fastx(files[i], loaded[i], per_file) ? 1 : -1; };
    std::vector<std::thread> pool;
    for (int t = 1; t < threads && (size_t)t < files.size(); t++) pool.emplace_back(worker);
    worker();
    for (auto& t : pool) t.join();
  }
  // record rules + layout (serial, metadata only), then one parallel copy of the sequences into the flat buffer
  struct Copy { size_t file; const fastx::RecordView* rec; uint64_t off; };
  std::vector<Copy> copies;
  uint64_t total = in.bases.size();
  for (size_t i = 0; i < files.size(); i++) {
    if (status[i] < 0) { fprintf(stderr, "WARN %s is not a valid fasta/fastq file; skipping.\n", files[i].c_str()); continue; }
    size_t kept = 0;
    if (!individual) {
      Genome g; g.file_name = files[i];
      for (auto& r : loaded[i].recs) {
        if (r.n_bases < 500) continue;                        // MIN_LENGTH_CONTIG (src/params.rs:42, src/file_io.rs:176)
        g.contigs.push_back(r.id); g.total_len += r.n_bases;
        copies.push_back(Copy{i, &r, total});
        total += r.n_bases;
        in.contig_off.push_back(total);
        in.genome_of_contig.push_back((uint32_t)in.genomes.size());
        kept++;
      }
      if (kept) in.genomes.push_back(std::move(g));
      else fprintf(stderr, "WARN File %s consists of only contigs < 500 bp. Skipping this file.\n", files[i].c_str());
    } else {
      bool warned = false;
      for (auto& r : loaded[i].recs) {
        if (r.n_bases < 500) {
          if (!warned) { fprintf(stderr, "WARN At least one sequence in file %s has < 500 bp. These sequences will be skipped.\n", files[i].c_str()); warned = true; }
          continue;
        }
        Genome g; g.file_name = files[i]; g.contigs.push_back(r.id); g.total_len = r.n_bases; g.contig_order = kept++;
        copies.push_back(Copy{i, &r, total});
        total += r.n_bases;
        in.contig_off.push_back(total);
        in.genome_of_contig.push_back((uint32_t)in.genomes.size());
        in.genomes.push_back(std::move(g));
      }
    }
  }
  in.bases.resize(total);
  {
    std::atomic<size_t> next{0};
    auto worker = [&] { for (size_t i; (i = next.fetch_add(1)) < copies.size();) fastx::copy_sequence(loaded[copies[i].file].data, *copies[i].rec, (char*)in.bases.data() + copies[i].off); };
    std::vector<std::thread> pool;
    for (int t = 1; t < threads && (size_t)t < copies.size(); t++) pool.emplace_back(worker);
    worker();
    for (auto& t : pool) t.join();
  }
}

std::vector<std::string> read_list(const std::string& path) {
  std::vector<std::string> v;
  FILE* f = fopen(path.c_str(), "r");
  if (!f) { fprintf(stderr, "ERROR cannot open list file %s\n", path.c_str()); exit(1); }
  char line[1 << 16];
  while (fgets(line, sizeof(line), f)) {
    std::string s(line);
    while (!s.empty() && (s.back() == '\n' || s.back() == '\r')) s.pop_back();
    if (!s.empty()) v.push_back(s);
  }
  fclose(f);
  return v;
}

std::string short_name(const std::string& s, bool short_header) {   // truncate_contig_name (src/types.rs:197-203)
  if (!short_header) return s;
  size_t b = s.find_first_not_of(" \t");
  if (b == std::string::npos) return s;
  size_t e = s.find_first_of(" \t", b);
  return s.substr(b, e == std::string::npos ? std::string::npos : e - b);
}

std::string f32_display(float v) {   // Rust `{}` / `{:0}` for an f32 holding an integer value
  if (v == std::floor(v) && std::fabs(v) < 1e15) { char b[64]; snprintf(b, sizeof(b), "%.0f", (double)v); return b; }
  char b[64]; snprintf(b, sizeof(b), "%g", (double)v); return b;
}

struct Opts {
  std::string cmd, out;
  std::vector<std::string> files, queries, refs;
  uint32_t c = 125, k = 15, m = 1000;
  bool c_set = false, m_set = false, k_set = false;
  double s = 0.0, min_af = -1e9, both_min_af = -1.0;
  bool individual = false, qi = false, ri = false, sparse = false, full_matrix = false, diagonal = false, ci = false, detailed = false,
       short_header = false, distance = false, robust = false, median = false, no_learned = false, faster_small = false,
       small_genomes = false, fast = false, medium = false, slow = false, no_marker_index = false;
  uint64_t n = 1000000000000ull;
  int threads = 3, device = 0, gpus = 1;
  std::string db_dir;               // search -d
  bool separate_sketches = false;   // sketch --separate-sketches
  double cluster_ani = 95.0;        // cluster --ani (percent)
  bool single_linkage = false;      // cluster --single-linkage
  std::string linkage;              // cluster --linkage average|complete
  std::string dendrogram;           // cluster --dendrogram FILE
  std::string representatives;      // dereplicate --representatives FILE
  bool host_store = false;          // dereplicate --host-store
  std::vector<std::string> fixed_reps;   // dereplicate --fixed-reps PATH / --fixed-reps-list FILE
  bool fixed_given = false;              // either flag was given
  std::string tree_method = "nj";   // tree --method nj|average|complete
  std::string mappings;             // triangle / dist / search --mappings FILE
};

void write_header(FILE* o, bool ci, bool detailed) {   // src/file_io.rs:15-23
  if (!ci && !detailed) fprintf(o, "Ref_file\tQuery_file\tANI\tAlign_fraction_ref\tAlign_fraction_query\tRef_name\tQuery_name\n");
  else if (!detailed) fprintf(o, "Ref_file\tQuery_file\tANI\tAlign_fraction_ref\tAlign_fraction_query\tRef_name\tQuery_name\tANI_5_percentile\tANI_95_percentile\n");
  else fprintf(o, "Ref_file\tQuery_file\tANI\tAlign_fraction_ref\tAlign_fraction_query\tRef_name\tQuery_name\tNum_ref_contigs\tNum_query_contigs\t"
                  "ANI_5_percentile\tANI_95_percentile\tStandard_deviation\tRef_90_ctg_len\tRef_50_ctg_len\tRef_10_ctg_len\tQuery_90_ctg_len\t"
                  "Query_50_ctg_len\tQuery_10_ctg_len\tAvg_chain_len\tTotal_bases_covered\n");
}
void write_row(FILE* o, const sk_ani_result& r, const Genome& ref, const Genome& qry, const Opts& op) {   // write_ani_res, src/file_io.rs:83-139
  fprintf(o, "%s\t%s\t%.2f\t%.2f\t%.2f\t%s\t%s", ref.file_name.c_str(), qry.file_name.c_str(), (double)(r.ani * 100.f),
          (double)(r.af_ref * 100.f), (double)(r.af_query * 100.f), short_name(ref.contigs[0], op.short_header).c_str(),
          short_name(qry.contigs[0], op.short_header).c_str());
  if (op.detailed) {
    fprintf(o, "\t%u\t%u\t%.2f\t%.2f\t%.2f\t%s\t%s\t%s\t%s\t%s\t%s\t%u\t%u", r.num_contigs_r, r.num_contigs_q, (double)(r.ci_lower * 100.f),
            (double)(r.ci_upper * 100.f), (double)(r.std * 100.f), f32_display(r.q90_r).c_str(), f32_display(r.q50_r).c_str(),
            f32_display(r.q10_r).c_str(), f32_display(r.q90_q).c_str(), f32_display(r.q50_q).c_str(), f32_display(r.q10_q).c_str(),
            r.avg_chain_int_len, r.total_bases_covered);
  } else if (op.ci) {
    fprintf(o, "\t%.2f\t%.2f", (double)(r.ci_lower * 100.f), (double)(r.ci_upper * 100.f));
  }
  fputc('\n', o);
}
void write_perfect(FILE* o, const Genome& g, const Opts& op) {   // write_ani_res_perfect, src/file_io.rs:25-81
  std::string nm = short_name(g.contigs[0], op.short_header);
  fprintf(o, "%s\t%s\t100.00\t100.00\t100.00\t%s\t%s", g.file_name.c_str(), g.file_name.c_str(), nm.c_str(), nm.c_str());
  if (op.detailed) fprintf(o, "\t%zu\t%zu\t100.00\t100.00\t0.00\t-1\t-1\t-1\t-1\t-1\t-1\t0\t%llu", g.contigs.size(), g.contigs.size(), (unsigned long long)g.total_len);
  else if (op.ci) fprintf(o, "\t100.00\t100.00");
  fputc('\n', o);
}

// --mappings FILE: one row per kept chain interval of every printed pair, 0-based half-open base coordinates.  A seed's
// position is the last base of its k-mer, so seed positions p0..p1 cover [p0 - k + 1, p1 + 1).
struct MappingFile {
  FILE* f = nullptr;
  uint32_t k = 0;
  bool open(const std::string& path, uint32_t k_) {
    k = k_;
    f = fopen(path.c_str(), "w");
    if (!f) { fprintf(stderr, "ERROR cannot open %s\n", path.c_str()); return false; }
    fprintf(f, "Ref_file\tQuery_file\tRef_contig\tRef_start\tRef_end\tQuery_contig\tQuery_start\tQuery_end\tStrand\tAnchors\t"
               "Chunk_genome\tChunk\tChunk_ANI\tChunk_weight\n");
    return true;
  }
  static const std::string& contig(const Genome& g, uint32_t i) { static const std::string none; return i < g.contigs.size() ? g.contigs[i] : none; }
  void write(const sk_mapping* m, uint64_t n, const Genome& ref, const Genome& qry, const Opts& op) {
    for (uint64_t i = 0; i < n; i++) {
      const sk_mapping& x = m[i];
      char ani[32];
      if (x.chunk_valid) snprintf(ani, sizeof(ani), "%.2f", x.chunk_est * 100.);
      else snprintf(ani, sizeof(ani), "NA");
      fprintf(f, "%s\t%s\t%s\t%u\t%u\t%s\t%u\t%u\t%c\t%u\t%c\t%u\t%s\t%u\n", ref.file_name.c_str(), qry.file_name.c_str(),
              short_name(contig(ref, x.ref_contig), op.short_header).c_str(), x.r0 + 1 - k, x.r1 + 1,
              short_name(contig(qry, x.query_contig), op.short_header).c_str(), x.q0 + 1 - k, x.q1 + 1, x.reverse ? '-' : '+',
              x.num_anchors, x.switched ? 'R' : 'Q', x.chunk, ani, x.chunk_weight);
    }
  }
  void flush() { if (f) fflush(f); }
  ~MappingFile() { if (f) fclose(f); }
};

// the mapping records of a block of result rows: row i owns recs[off[i] .. off[i + 1])
struct RowMaps {
  std::vector<uint64_t> off{0};
  std::vector<sk_mapping> recs;
  void clear() { off.assign(1, 0); recs.clear(); }
  void add(const sk_mapping* m, uint64_t n) { recs.insert(recs.end(), m, m + n); off.push_back(recs.size()); }
};

#define CK(ctx, call) do { int rc__ = (call); if (rc__ != 0) { fprintf(stderr, "ERROR %s failed (%d): %s\n", #call, rc__, sk_last_error(ctx)); exit(1); } } while (0)

// the genomes [g0, g1) of in sketched on ctx (genome g becomes the set's genome g - g0)
sk_sketch_set* sketch(sk_ctx* ctx, const Inputs& in, const sk_sketch_params& sp, size_t g0, size_t g1) {
  const auto& goc = in.genome_of_contig;
  const size_t c0 = std::lower_bound(goc.begin(), goc.end(), (uint32_t)g0) - goc.begin();
  const size_t c1 = std::lower_bound(goc.begin(), goc.end(), (uint32_t)g1) - goc.begin();
  std::vector<uint32_t> gl(c1 - c0);
  for (size_t i = c0; i < c1; i++) gl[i - c0] = goc[i] - (uint32_t)g0;
  sk_sketch_set* set = nullptr;
  CK(ctx, sk_sketch_batch(ctx, in.bases.data(), in.contig_off.data() + c0, (uint32_t)(c1 - c0), gl.data(), (uint32_t)(g1 - g0), &sp, &set));
  return set;
}
sk_sketch_set* sketch(sk_ctx* ctx, const Inputs& in, const sk_sketch_params& sp) { return sketch(ctx, in, sp, 0, in.genomes.size()); }

// INTERMEDIATE_WRITE_COUNT (src/params.rs:9): results are appended to the output every this many processed rows / queries
// (src/triangle.rs:113-138, src/dist.rs:151-175, src/search.rs:255-279).  SK_INTERMEDIATE_WRITE_COUNT overrides it (tests).
size_t intermediate_write_count() {
  if (const char* e = getenv("SK_INTERMEDIATE_WRITE_COUNT")) return (size_t)std::max(1ll, atoll(e));
  return 5000;
}

void resolve_presets(Opts& op) {   // src/parse.rs:829-853 / 680-710
  if (op.fast && op.slow) { fprintf(stderr, "ERROR Both --slow and --fast were set. This is not allowed.\n"); exit(1); }
  if (op.fast) op.c = 200;
  if (op.slow) op.c = 30;
  if (op.medium) op.c = 70;
  if (op.small_genomes) { op.c = 30; op.m = 200; }
  if (op.c > op.m) { fprintf(stderr, "ERROR We currently don't allow c (%u) > m (%u). -m should be larger than c.\n", op.c, op.m); exit(1); }  // src/params.rs:183
}

// flatten host sketches for sk_sketch_set_import_batch
struct Flat {
  std::vector<uint64_t> rec_off{0}, mk_off{0}, ctg_off{0}, total_len;
  std::vector<uint32_t> kmer, pos, cc, ctg_len;
  std::vector<uint64_t> markers;
  void add(const skdb::HostSketch& h, bool seeds) {
    if (seeds) {
      kmer.insert(kmer.end(), h.kmer.begin(), h.kmer.end()); pos.insert(pos.end(), h.pos.begin(), h.pos.end());
      cc.insert(cc.end(), h.cc.begin(), h.cc.end()); ctg_len.insert(ctg_len.end(), h.contig_lengths.begin(), h.contig_lengths.end());
    }
    markers.insert(markers.end(), h.markers.begin(), h.markers.end());
    rec_off.push_back(kmer.size()); mk_off.push_back(markers.size()); ctg_off.push_back(ctg_len.size());
    total_len.push_back(h.total_len);
  }
  sk_sketch_set* import(sk_ctx* ctx, const sk_sketch_params& sp) {
    sk_sketch_set* set = nullptr;
    CK(ctx, sk_sketch_set_import_batch(ctx, &sp, (uint32_t)total_len.size(), rec_off.data(), kmer.data(), pos.data(), cc.data(), mk_off.data(),
                                       markers.data(), ctg_off.data(), ctg_len.data(), total_len.data(), &set));
    return set;
  }
};

// inputs given as sketches (refs_are_sketch / queries_are_sketch, src/parse.rs:264-275): every file name contains
// ".sketch" or "markers.bin", or is a consolidated sketch database (a directory with index.db and sketches.db).  A
// database among FASTA inputs is refused.
bool sketch_inputs_given(const std::vector<std::string>& files) {
  if (files.empty()) return false;
  const std::string* db = nullptr;
  bool all = true;
  for (auto& f : files) {
    if (skdb::is_sketch_db(f)) { if (!db) db = &f; }
    else if (f.find(".sketch") == std::string::npos && f.find("markers.bin") == std::string::npos) all = false;
  }
  if (db && !all) { fprintf(stderr, "ERROR Sketch database %s cannot be mixed with FASTA/FASTQ inputs. Exiting.\n", db->c_str()); exit(1); }
  return all;
}

// group bound of the sketch readers: < `bound` seed records per sk_sketch_set_import_blobs call (2^28 for triangle and
// dist).  SK_SKETCH_GROUP_RECORDS lowers it (a test hook: many groups from a small input).
uint64_t sketch_group_records(uint64_t bound = 1ull << 28) {
  if (const char* e = getenv("SK_SKETCH_GROUP_RECORDS")) return (uint64_t)std::max(1ll, atoll(e));
  return bound;
}

// the metadata of a scanned (skdb::SketchScan) or decoded (skdb::HostSketch) sketch
template <class S>
Genome genome_of(const S& h) {
  Genome g; g.file_name = h.file_name; g.contigs = h.contigs; g.contig_order = h.contig_order; g.total_len = h.total_len;
  if (g.contigs.empty()) g.contigs.push_back("");   // a sketch without contig names still prints
  return g;
}

// a group of sketches as stored -> one device set (sk_sketch_set_import_blobs); nullptr after an ERROR line naming the
// sketch (name_of(i) for blob i) when one does not decode on the device
template <class N>
sk_sketch_set* import_group(sk_ctx* ctx, const skdb::SketchGroup& g, const sk_sketch_params& sp, N name_of) {
  sk_sketch_set* set = nullptr;
  uint32_t bad = UINT32_MAX;
  const int rc = sk_sketch_set_import_blobs(ctx, &sp, g.bytes.data(), g.off.data(), g.len.data(), (uint32_t)g.size(), &set, &bad);
  if (rc != 0 && bad < g.size()) { fprintf(stderr, "ERROR Failed to load sketch %s\n", name_of(bad).c_str()); return nullptr; }
  if (rc != 0) { fprintf(stderr, "ERROR sk_sketch_set_import_blobs failed (%d): %s\n", rc, sk_last_error(ctx)); exit(1); }
  return set;
}

// sketch inputs [a, b) read group by group: fn(set) gets each group imported as one device set on ctx and owns it;
// meta[i - a] gets entry i's metadata.  A group's bytes are freed before the next one is read.  false (after an ERROR
// line) when an entry cannot be loaded: the caller ends the run from the main thread.  One INFO line reports the time
// spent reading + decoding (reading the entries as stored and walking their framing) and importing (fn included).
template <class F>
bool for_each_sketch_group(sk_ctx* ctx, const skdb::SketchInputs& si, size_t a, size_t b, int threads, const sk_sketch_params& sp, Genome* meta, F fn) {
  using clk = std::chrono::steady_clock;
  std::vector<size_t> list(b - a);
  std::iota(list.begin(), list.end(), a);
  skdb::SketchGroupReader rd(si, std::move(list), threads, sketch_group_records());
  skdb::SketchGroup g;
  double t_read = 0, t_import = 0;
  size_t groups = 0;
  for (auto t0 = clk::now(); rd.next(g); t0 = clk::now()) {
    for (size_t i = 0; i < g.size(); i++) meta[rd.first + i] = genome_of(g.scan[i]);
    const auto t1 = clk::now();
    sk_sketch_set* s = import_group(ctx, g, sp, [&](size_t i) { return si.entries[a + rd.first + i].file_name; });
    if (!s) return false;
    fn(s);
    t_read += std::chrono::duration<double>(t1 - t0).count();
    t_import += std::chrono::duration<double>(clk::now() - t1).count();
    groups++;
  }
  if (rd.failed) return false;
  fprintf(stderr, "INFO %zu sketches loaded in %zu group(s): read + decode %.2f s, import %.2f s.\n", b - a, groups, t_read, t_import);
  return true;
}

// sketch inputs [a, b) -> one device set on ctx, grown group by group with sk_sketch_set_append (which holds the old and the
// merged set at once: about twice the set at its peak, see the estimate of sketch_bytes_estimate).  ok = false when an
// entry cannot be loaded.
sk_sketch_set* import_sketch_inputs(sk_ctx* ctx, const skdb::SketchInputs& si, size_t a, size_t b, int threads, const sk_sketch_params& sp, Genome* meta,
                                    bool& ok) {
  sk_sketch_set* set = nullptr;
  ok = for_each_sketch_group(ctx, si, a, b, threads, sp, meta, [&](sk_sketch_set* s) {
    if (!set) { set = s; return; }
    CK(ctx, sk_sketch_set_append(set, s));
    sk_sketch_set_free(s);
  });
  return set;
}

// sketch inputs -> a host sketch store (a new one, or `into` grown after its genomes): each group's set is added and freed
// before the next group is read, so host memory holds one group of stored sketches besides the pinned store, and the device
// one imported group.  meta gets the entries' metadata appended.  nullptr when an entry cannot be loaded (a new store is
// then freed; `into` stays the caller's).
sk_sketch_store* store_sketch_inputs(sk_ctx* ctx, const skdb::SketchInputs& si, int threads, const sk_sketch_params& sp, std::vector<Genome>& meta,
                                     sk_sketch_store* into = nullptr) {
  sk_sketch_store* st = into;
  if (!st) CK(ctx, sk_sketch_store_create(&sp, &st));
  const size_t m0 = meta.size();
  meta.resize(m0 + si.entries.size());
  const bool ok = for_each_sketch_group(ctx, si, 0, si.entries.size(), threads, sp, meta.data() + m0, [&](sk_sketch_set* s) {
    CK(ctx, sk_sketch_store_add(st, s));
    sk_sketch_set_free(s);
  });
  if (!ok) { if (!into) sk_sketch_store_free(st); return nullptr; }
  return st;
}

// the parameters of sketch inputs, as sk_sketch_params
sk_sketch_params params_of(const skdb::SketchInputs& si) {
  return sk_sketch_params{(uint32_t)si.params.c, (uint32_t)si.params.k, (uint32_t)si.params.marker_c};
}

// the number of inputs as the reference counts query files, where a database counts once per sketch
size_t n_inputs(const std::vector<std::string>& files, const skdb::SketchInputs& si) {
  size_t n = files.size();
  for (auto& e : si.entries) if (si.db_fd[e.input] >= 0) n++;
  for (int fd : si.db_fd) if (fd >= 0) n--;
  return n;
}

// --gpus N: per_device contexts on each of n devices, device d being (device + d) % device count, ctx0 (on --device) first.
// With fewer devices than N the contexts share devices (same code path; copies between them stay on the device).
std::vector<sk_ctx*> make_contexts(sk_ctx* ctx0, const Opts& op, size_t n, int per_device = 1) {
  const int ndev = std::max(sk_device_count(), 1);
  if (ndev < op.gpus) fprintf(stderr, "WARN --gpus %d but %d CUDA device(s) visible: contexts share devices.\n", op.gpus, ndev);
  std::vector<sk_ctx*> ctxs(1, ctx0);
  for (size_t d = 0; d < n; d++)
    for (int k = d == 0; k < per_device; k++) {
      const int dev = (op.device + (int)d) % ndev;
      sk_ctx* c = nullptr;
      if (sk_ctx_create(dev, &c) != 0) { fprintf(stderr, "ERROR cannot create a context on GPU %d\n", dev); exit(1); }
      ctxs.push_back(c);
    }
  return ctxs;
}

// the share of -t threads of context d of n
int context_threads(const Opts& op, size_t d, size_t n) {
  const int t = std::max(op.threads, 1);
  return std::max(1, t / (int)n + ((int)d < t % (int)n ? 1 : 0));
}

// fn(d) for d < n, one host thread per context
template <class F>
void per_context(size_t n, F fn) {
  if (n == 1) { fn((size_t)0); return; }
  std::vector<std::thread> th;
  for (size_t d = 0; d < n; d++) th.emplace_back(fn, d);
  for (auto& t : th) t.join();
}

// [0, w.size()) cut into W contiguous blocks of about equal total weight: bounds[d], bounds[d + 1] delimit block d.  A block
// is empty only when there are fewer items than blocks.
std::vector<size_t> split_balanced(const std::vector<uint64_t>& w, size_t W) {
  const size_t n = w.size();
  uint64_t total = 0;
  for (uint64_t x : w) total += x;
  std::vector<size_t> b(W + 1, 0);
  uint64_t acc = 0;
  size_t d = 1;
  for (size_t g = 0; g < n && d < W; g++) {
    acc += w[g];
    if (acc * W >= total * d || n - (g + 1) <= W - d) b[d++] = g + 1;
  }
  for (; d < W; d++) b[d] = b[d - 1];
  b[W] = n;
  return b;
}

// the file bound of a group: 4096 files; SK_SKETCH_GROUP_FILES lowers it (a test hook: many groups from a few files)
size_t group_max_files() {
  static const size_t max_files = [] {
    const char* e = getenv("SK_SKETCH_GROUP_FILES");
    return e ? (size_t)std::max(1ll, std::min(4096ll, atoll(e))) : (size_t)4096;
  }();
  return max_files;
}

// sorted files [f0, end) form the next group that goes through the GPU at once: at most group_max_files() files and about
// max_bytes (8 GiB) of sequence (file sizes x 4, as gz inflates ~4x), at least one file.
size_t file_group_end(const std::vector<std::string>& files, size_t f0, uint64_t max_bytes = 8ull << 30) {
  const size_t max_files = group_max_files();
  size_t f1 = f0;
  uint64_t bytes = 0;
  while (f1 < files.size() && (f1 == f0 || (f1 - f0 < max_files && bytes < max_bytes))) {
    struct stat st;
    bytes += stat(files[f1].c_str(), &st) == 0 ? (uint64_t)st.st_size * 4 : 0;
    f1++;
  }
  return f1;
}

// triangle: whether the sketches are expected to exceed the device (the estimate of sk_triangle's memory guard: 56 B per
// seed, 24 B per marker and 6 GB of workspace against 92 % of the device, from the file sizes, x 4 for .gz; .sketch files
// about triple on the device; a database counts the bytes of its sketches.db) or SK_DEVICE_BUDGET_MB asks for the store
// path.  --gpus N with FASTA inputs keeps sk_triangle_multi; with sketch inputs it always takes the store path.
double sketch_bytes_estimate(const Opts& op, const std::vector<std::string>& files, bool sketches) {
  uint64_t bytes = 0;
  for (auto& f : files) {
    struct stat st;
    if (stat(skdb::is_sketch_db(f) ? (f + "/sketches.db").c_str() : f.c_str(), &st) != 0) continue;
    const bool gz = f.size() > 3 && f.compare(f.size() - 3, 3, ".gz") == 0;
    bytes += (uint64_t)st.st_size * (gz ? 4 : 1);
  }
  return sketches ? 3.0 * bytes : (double)bytes / op.c * 56.0 + (double)bytes / op.m * 24.0;
}
// SK_DEVICE_BUDGET_MB: the device bytes the store paths' working sets may take, and a request for the store path (a test
// hook: the store path on small inputs); 0 when unset (the working sets are then sized from the free device memory)
uint64_t device_budget() {
  const char* e = getenv("SK_DEVICE_BUDGET_MB");
  return e ? (uint64_t)std::max(1ll, atoll(e)) << 20 : 0;
}
// need bytes against 92 % of the device, or SK_DEVICE_BUDGET_MB asks for the store path
bool exceeds_device(const Opts& op, double need) {
  if (device_budget()) return true;
  uint64_t free_b = 0, total_b = 0;
  if (sk_device_memory(op.device, &free_b, &total_b) != 0) return false;
  return need > 0.92 * (double)total_b;
}
// Sketch inputs of more records than one import group are grown into one set by sk_sketch_set_append, which holds the old
// and the merged set on the device at once: their estimate then counts twice.  records = the inputs' (or one context's
// share of the) SketchEntry weights.
double append_peak(uint64_t records) { return records >= sketch_group_records() ? 2.0 : 1.0; }
uint64_t total_weight(const skdb::SketchInputs& si) {
  uint64_t w = 0;
  for (auto& e : si.entries) w += e.weight;
  return w;
}

bool triangle_needs_store(const Opts& op, bool sketches, const skdb::SketchInputs& si, double* need_gb) {
  const double need = sketch_bytes_estimate(op, op.files, sketches) * (sketches ? append_peak(total_weight(si)) : 1.0) + 6.0e9;
  *need_gb = need / 1e9;
  if (op.gpus > 1 && !sketches) return false;
  return (op.gpus > 1 && sketches) || exceeds_device(op, need);
}

// dist: the same estimate per context, where the references are split over --gpus contexts and every context holds the
// whole query set
bool dist_needs_store(const Opts& op, bool refs_sketch, bool queries_sketch, const skdb::SketchInputs& rsi, const skdb::SketchInputs& qsi, double* need_gb) {
  const int gpus = std::max(op.gpus, 1);
  const double need = sketch_bytes_estimate(op, op.refs, refs_sketch) / gpus * (refs_sketch ? append_peak(total_weight(rsi) / gpus) : 1.0) +
                      sketch_bytes_estimate(op, op.queries, queries_sketch) * (queries_sketch ? append_peak(total_weight(qsi)) : 1.0) + 6.0e9;
  *need_gb = need / 1e9;
  return exceeds_device(op, need);
}

// the INFO line of the store paths (dist: the estimate per context, one store per side)
void info_store_path(const Opts& op, double need_gb, bool dist) {
  char on[64];
  if (dist || op.gpus > 1) snprintf(on, sizeof(on), "%d GPU(s) from GPU %d", op.gpus, op.device);
  else snprintf(on, sizeof(on), "GPU %d", op.device);
  fprintf(stderr, "INFO Store path: sketches (~%.1f GB%s estimated) are kept in %s and chained in working sets on %s%s.\n", need_gb,
          dist ? " per context" : "", dist ? "host sketch stores" : "a host sketch store", on, device_budget() ? " (SK_DEVICE_BUDGET_MB set)" : "");
}

// The store path of triangle and dist on FASTA inputs: files are sketched in groups, each group's set is added to a host
// sketch store and freed, so device memory holds one group at a time and host memory one group of sequence plus the
// sketches.  genomes gets the metadata of every genome appended in store order (= the order of the in-memory path).  The
// store is a new one, or `into` grown after its genomes.  nullptr when the files hold no genome (a new store is then freed;
// `into` stays the caller's).  Sketch inputs fill their store through store_sketch_inputs.
sk_sketch_store* fill_store(sk_ctx* ctx, const Opts& op, const std::vector<std::string>& input_files, bool individual,
                            std::vector<Genome>& genomes, sk_sketch_params& sp, sk_sketch_store* into = nullptr) {
  sk_sketch_store* st = into;
  if (!st) CK(ctx, sk_sketch_store_create(&sp, &st));
  const size_t g0 = genomes.size();
  std::vector<std::string> files = input_files;
  std::sort(files.begin(), files.end());
  for (size_t f0 = 0; f0 < files.size();) {
    const size_t f1 = file_group_end(files, f0);
    Inputs in;
    load_inputs(std::vector<std::string>(files.begin() + f0, files.begin() + f1), individual, std::max(op.threads, 1), in);
    f0 = f1;
    if (in.genomes.empty()) continue;
    sk_sketch_set* set = sketch(ctx, in, sp);
    CK(ctx, sk_sketch_store_add(st, set));
    sk_sketch_set_free(set);
    for (auto& g : in.genomes) genomes.push_back(std::move(g));
  }
  if (genomes.size() == g0) { if (!into) sk_sketch_store_free(st); return nullptr; }
  return st;
}

// "WARN Input parameter ..." of triangle's sketch inputs (src/triangle.rs:16-24); the sketches' parameters are used
void warn_sketch_params(const Opts& op, const skdb::SketchInputs& si) {
  if (si.params.c != op.c || si.params.marker_c != op.m)
    fprintf(stderr, "WARN Input parameter c = %u, m = %u is not equal to the sketch parameter c = %llu,m = %llu. Using sketch parameters.\n", op.c, op.m,
            (unsigned long long)si.params.c, (unsigned long long)si.params.marker_c);
}

// the map parameters of triangle and dist (search sets its own); learned_ani = regression::use_learned_ani
// (src/regression.rs:8-10) as the command decides it
sk_map_params map_params(const Opts& op, bool learned_ani) {
  sk_map_params mp{};
  mp.screen_val = op.s / 100.0;
  mp.min_aligned_frac = (op.min_af > -1e8 ? op.min_af : 15.0) / 100.0;
  mp.both_min_aligned_frac = op.both_min_af / 100.0;
  mp.robust = op.robust; mp.median = op.median;
  mp.rescue_small = !op.faster_small && !op.small_genomes;
  mp.learned_ani = learned_ani;
  if (mp.learned_ani) fprintf(stderr, "INFO Learned ANI mode detected. ANI may be adjusted according to a regression model trained on MAGs.\n");
  return mp;
}

// file-name order for the switch_qr tie-break (src/chain.rs:19-21): the names of a and b ranked together, equal names
// sharing a rank (with -i all records of a file share its name); [0] holds a's ranks, [1] b's
std::array<std::vector<uint64_t>, 2> name_ranks(const std::vector<Genome>& a, const std::vector<Genome>& b = {}) {
  std::vector<std::pair<const std::string*, uint64_t*>> names;
  std::array<std::vector<uint64_t>, 2> ranks{std::vector<uint64_t>(a.size()), std::vector<uint64_t>(b.size())};
  for (size_t i = 0; i < a.size(); i++) names.push_back({&a[i].file_name, &ranks[0][i]});
  for (size_t i = 0; i < b.size(); i++) names.push_back({&b[i].file_name, &ranks[1][i]});
  std::sort(names.begin(), names.end(), [](auto& x, auto& y) { return *x.first < *y.first; });
  uint64_t rank = 0;
  for (size_t i = 0; i < names.size(); i++) {
    if (i && *names[i].first != *names[i - 1].first) rank++;
    *names[i].second = rank;
  }
  return ranks;
}

// One block of chained rows of the in-memory triangle; more = further blocks follow.  false ends the run (after an ERROR line).
using BlockWriter = std::function<bool(const std::vector<sk_ani_result>& rows, bool more)>;

// The triangle up to its writers, on every path (in memory, --gpus N through sk_triangle_multi, the host sketch store, sketch
// inputs): in.genomes gets the genomes in genome-index order ((file_name, contig_order)), res the result of every screened pair
// in the order the writers print them (they keep ani > 0.1), ctx the context on --device, which the caller destroys.  With
// `stream`, the in-memory path chains and hands over the rows in blocks of INTERMEDIATE_WRITE_COUNT rows instead
// (src/triangle.rs:113-138), so a long run leaves its finished rows on disk and holds at most one block of results in memory.
// Returns 0, or the exit code after an ERROR line.
// The inputs of a triangle (triangle, cluster, tree, dereplicate) in two halves.  open_triangle_inputs resolves the presets,
// opens sketch inputs and decides whether the run takes the host sketch store path; load_triangle_inputs then reads FASTA
// inputs (in memory), creates the context on --device and fills the store or imports the sketch inputs.  Both return 0, or
// the exit code after an ERROR line.
struct TriangleInputs {
  bool sketches = false;              // .sketch files and databases
  skdb::SketchInputs si;
  bool use_store = false;
  double need_gb = 0;                 // the store path's estimate
  sk_sketch_params sp{};
  sk_sketch_set* loaded = nullptr;    // sketch inputs imported in memory (FASTA inputs are sketched by the caller)
  sk_sketch_store* store = nullptr;   // the store path's sketches
  // dereplicate --fixed-reps: the fixed group (op.fixed_reps), whose genomes come first; the fields above then describe the
  // new group (op.files), and loaded / store hold both groups
  bool fixed_sketches = false;
  skdb::SketchInputs fsi;
  uint32_t n_fixed = 0;
};

// the names a group of inputs gives its genomes: its paths (FASTA), or its sketches' file names
std::set<std::string> group_names(const std::vector<std::string>& files, bool sketches, const skdb::SketchInputs& si) {
  std::set<std::string> names;
  if (sketches) for (auto& e : si.entries) names.insert(e.file_name);
  else names.insert(files.begin(), files.end());
  return names;
}

// dereplicate --fixed-reps: the fixed group opened beside the new one.  Each group follows the triangle's input rules on its
// own; a FASTA group is sketched with a sketch group's (c, k, m), so an explicit -c / -k / -m that differs from them is
// refused, as are two sketch groups whose parameters differ and a genome file name in both groups.  Both groups are held in
// one set at the end, joined by sk_sketch_set_append (the fixed group's set and the joined one at once): the estimate counts
// both groups twice.
int open_fixed_inputs(Opts& op, TriangleInputs& ti) {
  if (op.fixed_reps.empty()) { fprintf(stderr, "ERROR --fixed-reps / --fixed-reps-list: no fixed representatives given.\n"); return 1; }
  ti.fixed_sketches = sketch_inputs_given(op.fixed_reps);
  if (ti.fixed_sketches) {
    fprintf(stderr, "INFO Sketches detected among the fixed representatives.\n");
    if (!skdb::open_sketch_inputs(op.fixed_reps, ti.fsi)) return 1;
    if (ti.fsi.entries.empty()) { fprintf(stderr, "ERROR No genomes/sketches found among the fixed representatives.\n"); return 1; }
  }
  if (ti.fixed_sketches && ti.sketches) {
    const skdb::DiskParams &a = ti.fsi.params, &b = ti.si.params;
    if (a.c != b.c || a.k != b.k || a.marker_c != b.marker_c) {
      fprintf(stderr, "ERROR Sketch parameters of %s (c = %llu, k = %llu, m = %llu) differ from those of %s (c = %llu, k = %llu, m = %llu). Exiting.\n",
              op.files[0].c_str(), (unsigned long long)b.c, (unsigned long long)b.k, (unsigned long long)b.marker_c, op.fixed_reps[0].c_str(),
              (unsigned long long)a.c, (unsigned long long)a.k, (unsigned long long)a.marker_c);
      return 1;
    }
  } else if (ti.fixed_sketches || ti.sketches) {   // one FASTA group, sketched with the sketch group's parameters
    const skdb::SketchInputs& si = ti.fixed_sketches ? ti.fsi : ti.si;
    const char* who = ti.fixed_sketches ? "fixed representatives" : "new genomes";
    const struct { bool set; uint32_t given; uint64_t used; const char* flag; } ps[] = {
        {op.c_set, op.c, si.params.c, "-c"}, {op.k_set, op.k, si.params.k, "-k"}, {op.m_set, op.m, si.params.marker_c, "-m"}};
    for (auto& p : ps)
      if (p.set && p.given != p.used) {
        fprintf(stderr, "ERROR %s %u differs from the sketch parameter %s %llu of the %s, with which the FASTA inputs are sketched.\n",
                p.flag, p.given, p.flag, (unsigned long long)p.used, who);
        return 1;
      }
  }
  const std::set<std::string> fixed = group_names(op.fixed_reps, ti.fixed_sketches, ti.fsi);
  for (auto& name : group_names(op.files, ti.sketches, ti.si))
    if (fixed.count(name)) { fprintf(stderr, "ERROR %s is both a fixed representative and a new genome.\n", name.c_str()); return 1; }
  if (ti.fixed_sketches || ti.sketches) warn_sketch_params(op, ti.fixed_sketches ? ti.fsi : ti.si);
  const double need = 2.0 * (sketch_bytes_estimate(op, op.fixed_reps, ti.fixed_sketches) + sketch_bytes_estimate(op, op.files, ti.sketches)) + 6.0e9;
  ti.need_gb = need / 1e9;
  ti.use_store = exceeds_device(op, need);
  return 0;
}

int open_triangle_inputs(Opts& op, TriangleInputs& ti) {
  resolve_presets(op);
  if (op.files.empty()) { fprintf(stderr, "ERROR No reference inputs found.\n"); return 1; }
  ti.sketches = sketch_inputs_given(op.files);
  if (ti.sketches) {      // .sketch files and databases (src/triangle.rs:16-24): opened here, decoded in groups below
    fprintf(stderr, "INFO Sketches detected.\n");
    if (!skdb::open_sketch_inputs(op.files, ti.si)) return 1;   // file_io::sketches_from_sketch (src/file_io.rs:680-717)
    if (ti.si.entries.empty()) { fprintf(stderr, "ERROR No genomes/sketches found.\n"); return 1; }
    if (!op.fixed_given) warn_sketch_params(op, ti.si);
  }
  if (op.fixed_given) return open_fixed_inputs(op, ti);
  ti.use_store = triangle_needs_store(op, ti.sketches, ti.si, &ti.need_gb);
  return 0;
}

int load_triangle_inputs(Opts& op, Inputs& in, sk_ctx*& ctx, TriangleInputs& ti) {
  if (!ti.sketches && !ti.use_store) {
    load_inputs(op.files, op.individual, std::max(op.threads, 1), in);
    if (in.genomes.empty()) { fprintf(stderr, "ERROR No genomes/sketches found.\n"); return 1; }   // src/triangle.rs:46-49
  }
  if (sk_ctx_create(op.device, &ctx) != 0) { fprintf(stderr, "ERROR a CUDA device is required (no CPU fallback)\n"); return 1; }
  ti.sp = ti.sketches ? params_of(ti.si) : sk_sketch_params{op.c, op.k, op.m};
  if (ti.use_store) {
    info_store_path(op, ti.need_gb, false);
    ti.store = ti.sketches ? store_sketch_inputs(ctx, ti.si, std::max(op.threads, 1), ti.sp, in.genomes)
                           : fill_store(ctx, op, op.files, op.individual, in.genomes, ti.sp);
    if (!ti.store) {      // sketch inputs: an entry could not be loaded (reported)
      if (!ti.sketches) fprintf(stderr, "ERROR No genomes/sketches found.\n");
      return 1;
    }
  } else if (ti.sketches) {
    in.genomes.resize(ti.si.entries.size());
    bool ok = true;
    ti.loaded = import_sketch_inputs(ctx, ti.si, 0, ti.si.entries.size(), std::max(op.threads, 1), ti.sp, in.genomes.data(), ok);
    if (!ok) return 1;
  }
  return 0;
}

// One group of dereplicate --fixed-reps' inputs, its genomes' metadata appended to genomes: in memory, one device set on ctx
// (FASTA sketched, sketch inputs imported) joined to *set with sk_sketch_set_append; on the store path, added to *store.
// false after an ERROR line.
bool load_fixed_group(const Opts& op, sk_ctx* ctx, const std::vector<std::string>& files, bool sketches, const skdb::SketchInputs& si,
                      sk_sketch_params& sp, bool use_store, const char* what, std::vector<Genome>& genomes, sk_sketch_set** set,
                      sk_sketch_store** store) {
  const int threads = std::max(op.threads, 1);
  const size_t g0 = genomes.size();
  if (use_store) {
    sk_sketch_store* st = sketches ? store_sketch_inputs(ctx, si, threads, sp, genomes, *store) : fill_store(ctx, op, files, op.individual, genomes, sp, *store);
    if (!st) {
      if (!sketches) fprintf(stderr, "ERROR No genomes/sketches found among the %s.\n", what);
      return false;
    }
    *store = st;
    return true;
  }
  sk_sketch_set* s = nullptr;
  if (sketches) {
    genomes.resize(g0 + si.entries.size());
    bool ok = true;
    s = import_sketch_inputs(ctx, si, 0, si.entries.size(), threads, sp, genomes.data() + g0, ok);
    if (!ok) { if (s) sk_sketch_set_free(s); return false; }
  } else {
    Inputs in;
    load_inputs(files, op.individual, threads, in);
    if (in.genomes.empty()) { fprintf(stderr, "ERROR No genomes/sketches found among the %s.\n", what); return false; }
    s = sketch(ctx, in, sp);
    for (auto& g : in.genomes) genomes.push_back(std::move(g));
  }
  if (!*set) { *set = s; return true; }
  CK(ctx, sk_sketch_set_append(*set, s));
  sk_sketch_set_free(s);
  return true;
}

// load_triangle_inputs of dereplicate --fixed-reps: the fixed group, then the new one, into one set (in memory, ti.loaded) or
// one host sketch store (ti.store); in.genomes gets the metadata of both and ti.n_fixed the fixed group's genome count
int load_fixed_inputs(Opts& op, Inputs& in, sk_ctx*& ctx, TriangleInputs& ti) {
  if (sk_ctx_create(op.device, &ctx) != 0) { fprintf(stderr, "ERROR a CUDA device is required (no CPU fallback)\n"); return 1; }
  ti.sp = ti.fixed_sketches ? params_of(ti.fsi) : ti.sketches ? params_of(ti.si) : sk_sketch_params{op.c, op.k, op.m};
  if (ti.use_store) info_store_path(op, ti.need_gb, false);
  const bool ok = load_fixed_group(op, ctx, op.fixed_reps, ti.fixed_sketches, ti.fsi, ti.sp, ti.use_store, "fixed representatives", in.genomes,
                                   &ti.loaded, &ti.store);
  ti.n_fixed = (uint32_t)in.genomes.size();
  if (!ok || !load_fixed_group(op, ctx, op.files, ti.sketches, ti.si, ti.sp, ti.use_store, "new genomes", in.genomes, &ti.loaded, &ti.store)) {
    if (ti.store) sk_sketch_store_free(ti.store);
    if (ti.loaded) sk_sketch_set_free(ti.loaded);
    ti.store = nullptr;
    ti.loaded = nullptr;
    return 1;
  }
  return 0;
}

int triangle_results(Opts& op, Inputs& in, sk_ctx*& ctx, std::vector<sk_ani_result>& res, const BlockWriter* stream) {
  TriangleInputs ti;
  if (const int rc = open_triangle_inputs(op, ti)) return rc;
  if (!op.mappings.empty() && ti.use_store) {
    fprintf(stderr, "ERROR --mappings is not supported when the sketches exceed device memory (host sketch store path); "
                    "split the inputs into runs that fit the device.\n");
    return 1;
  }
  if (!op.mappings.empty() && op.gpus > 1 && !ti.sketches) {
    fprintf(stderr, "ERROR --mappings is not supported with triangle --gpus N > 1 (the multi-GPU triangle); run it on one GPU.\n");
    return 1;
  }
  if (const int rc = load_triangle_inputs(op, in, ctx, ti)) return rc;
  const bool refs_are_sketch = ti.sketches;
  const sk_sketch_params sp = ti.sp;
  sk_sketch_set* loaded = ti.loaded;
  sk_sketch_store* store = ti.store;
  if (op.cmd == "triangle" && in.genomes.size() > 500 && !op.sparse) fprintf(stderr, "WARN > 500 genomes detected. The output matrix will be large. Consider using -E or --sparse for a tsv output instead.\n");
  const sk_map_params mp = map_params(op, !op.no_learned && op.c >= 70 && !op.individual && !op.median);
  const std::vector<uint64_t> ranks = name_ranks(in.genomes)[0];
  // sketch inputs: one INFO line gives the time of the screen and the chaining (with the "sketches loaded" line, the split
  // of a run from a database)
  using clk = std::chrono::steady_clock;
  double t_work = 0;
  auto timed = [&](clk::time_point t0) { t_work += std::chrono::duration<double>(clk::now() - t0).count(); };
  if (store) {
    // two contexts on each of the --gpus devices: one gathers its next working set over PCIe while the other chains.  Every
    // row is written at the end (no intermediate "Writing results" flushes in sparse mode).
    CK(ctx, sk_sketch_store_set_name_ranks(store, ranks.data()));
    std::vector<sk_ctx*> sctx = make_contexts(ctx, op, op.gpus, 2);
    sk_ani_result* r = nullptr; uint64_t nr = 0;
    const auto t0 = clk::now();
    CK(ctx, sk_triangle_store(sctx.data(), (uint32_t)sctx.size(), store, &mp, device_budget(), &r, &nr, nullptr));
    timed(t0);
    res.assign(r, r + nr);
    sk_free(r);
    std::sort(res.begin(), res.end(), [](const sk_ani_result& a, const sk_ani_result& b) { return a.ref_id != b.ref_id ? a.ref_id < b.ref_id : a.query_id < b.query_id; });
    for (size_t d = sctx.size(); d-- > 1;) sk_ctx_destroy(sctx[d]);
    sk_sketch_store_free(store);
  } else if (op.gpus > 1 && !loaded) {
    // --gpus N: one context per GPU, genome blocks + marker exchange + cross-block slices (sk_triangle_multi).  With fewer
    // physical devices than N the contexts share devices (same code path; the exchange then stays on the device).
    std::vector<sk_ctx*> ctxs = make_contexts(ctx, op, op.gpus);
    sk_ani_result* r = nullptr; uint64_t nr = 0;
    CK(ctx, sk_triangle_multi(ctxs.data(), (uint32_t)ctxs.size(), in.bases.data(), in.contig_off.data(), (uint32_t)in.genome_of_contig.size(),
                              in.genome_of_contig.data(), (uint32_t)in.genomes.size(), &sp, &mp, ranks.data(), &r, &nr, nullptr));
    res.assign(r, r + nr);
    sk_free(r);
    std::sort(res.begin(), res.end(), [](const sk_ani_result& a, const sk_ani_result& b) { return a.ref_id != b.ref_id ? a.ref_id < b.ref_id : a.query_id < b.query_id; });
    for (size_t d = 1; d < ctxs.size(); d++) sk_ctx_destroy(ctxs[d]);
  } else {
    sk_sketch_set* set = loaded ? loaded : sketch(ctx, in, sp);
    sk_sketch_set_set_name_ranks(set, ranks.data());
    uint64_t* pairs = nullptr; uint64_t np = 0;
    const auto t0 = clk::now();
    CK(ctx, sk_screen_triangle(ctx, set, &mp, &pairs, &np));
    timed(t0);
    // rows in blocks of FL: with `stream` each block is handed over and replaced by the next, without it the one block of
    // all rows stays in res
    const size_t N = in.genomes.size(), FL = stream ? intermediate_write_count() : N;
    // --mappings: the records of the rows the sparse output prints (ani > 0.1, in (i, j) order), written block by block
    MappingFile mf;
    if (!op.mappings.empty() && !mf.open(op.mappings, sp.k)) return 1;
    std::vector<uint64_t> off;
    uint64_t p0 = 0;
    bool ok = true;
    for (size_t r0 = 0; r0 < N && ok; r0 += FL) {
      uint64_t p1 = p0;
      while (p1 < np && (uint32_t)(pairs[p1] >> 32) < r0 + FL) p1++;      // pairs are sorted by (i, j)
      res.resize(p1 - p0);
      const auto t1 = clk::now();
      if (mf.f) {
        off.resize(p1 - p0 + 1);
        sk_mapping* maps = nullptr;
        CK(ctx, sk_chain_pairs_mappings(ctx, set, set, pairs + p0, p1 - p0, &mp, res.data(), off.data(), &maps));
        for (size_t i = 0; i < res.size(); i++)
          if (res[i].ani > 0.1f) mf.write(maps + off[i], off[i + 1] - off[i], in.genomes[res[i].ref_id], in.genomes[res[i].query_id], op);
        mf.flush();
        sk_free(maps);
      } else {
        CK(ctx, sk_chain_pairs(ctx, set, set, pairs + p0, p1 - p0, &mp, res.data()));
      }
      timed(t1);
      if (stream) ok = (*stream)(res, r0 + FL < N);
      p0 = p1;
    }
    sk_free(pairs);
    sk_sketch_set_free(set);
    if (!ok) return 1;
  }
  if (refs_are_sketch) fprintf(stderr, "INFO Screen + chain %.2f s.\n", t_work);
  return 0;
}

int run_triangle(Opts& op) {
  Inputs in;
  sk_ctx* ctx = nullptr;
  std::vector<sk_ani_result> res;
  FILE* so = nullptr;   // the sparse output, opened with the first block
  const BlockWriter stream = [&](const std::vector<sk_ani_result>& rows, bool more) {
    if (!so) {
      so = op.out.empty() ? stdout : fopen(op.out.c_str(), "w");
      if (!so) { fprintf(stderr, "ERROR cannot open %s\n", op.out.c_str()); return false; }
      write_header(so, op.ci, op.detailed);
      if (op.diagonal) for (auto& g : in.genomes) write_perfect(so, g, op);
    }
    for (auto& r : rows) if (r.ani > 0.1f) write_row(so, r, in.genomes[r.ref_id], in.genomes[r.query_id], op);
    fflush(so);
    if (more) fprintf(stderr, "INFO Writing results for %zu query sequences.\n", intermediate_write_count());
    return true;
  };
  if (const int rc = triangle_results(op, in, ctx, res, op.sparse ? &stream : nullptr)) return rc;
  // write_sparse_matrix (src/file_io.rs:541-606): rows in (i, j) order (the reference's order is arbitrary), written block by
  // block on the in-memory path and here at once on the store and --gpus N paths
  if (op.sparse && !so && !stream(res, false)) return 1;
  FILE* o = so;
  if (!op.sparse) {           // write_phyllip_matrix (src/file_io.rs:364-539)
    const size_t N = in.genomes.size();
    o = op.out.empty() ? stdout : fopen(op.out.c_str(), "w");
    if (!o) { fprintf(stderr, "ERROR cannot open %s\n", op.out.c_str()); return 1; }
    std::map<std::pair<uint32_t, uint32_t>, const sk_ani_result*> m;
    for (auto& r : res) if (r.ani > 0.1f) m[{r.ref_id, r.query_id}] = &r;
    const double perfect = op.distance ? 0. : 100., none = 100. - perfect;
    std::string af_name = op.out.empty() ? "skani_matrix.af" : op.out + ".af";
    FILE* af = fopen(af_name.c_str(), "w");
    fprintf(o, "%zu\n", N);
    if (af) fprintf(af, "%zu\n", N);
    for (size_t i = 0; i < N; i++) {
      const std::string& name = op.individual ? in.genomes[i].contigs[0] : in.genomes[i].file_name;
      fputs(name.c_str(), o);
      if (af) fputs(name.c_str(), af);
      for (size_t j = 0; j < N; j++) {
        bool full_cond = op.full_matrix || (i > j);
        auto it = m.find({(uint32_t)std::min(i, j), (uint32_t)std::max(i, j)});
        if (i == j) {
          if (full_cond || op.diagonal) fprintf(o, "\t%.2f", perfect);
          if (af) fprintf(af, "\t%.2f", 100.);
          continue;
        }
        if (it == m.end()) {
          if (full_cond) fprintf(o, "\t%.2f", none);
          if (af) fprintf(af, "\t%.2f", 0.);
        } else {
          if (full_cond) { double val = (double)(it->second->ani * 100.f); fprintf(o, "\t%.2f", op.distance ? 100. - val : val); }
          if (af) fprintf(af, "\t%.2f", (double)((j > i ? it->second->af_ref : it->second->af_query) * 100.f));
        }
      }
      fputc('\n', o);
      if (af) fputc('\n', af);
    }
    if (af) fclose(af);
    fprintf(stderr, "INFO Aligned fraction matrix written to %s\n", af_name.c_str());
  }
  if (o != stdout) fclose(o);
  sk_ctx_destroy(ctx);
  return 0;
}

// genomes ranked by total sequence length, longest first, ties by genome index (cluster's choice of representatives).  With
// n_first > 0 (dereplicate --fixed-reps) genomes 0 .. n_first - 1 take ranks 0 .. n_first - 1 by that rule, and the others
// the ranks after them.
std::vector<uint32_t> length_rank(const Inputs& in, uint32_t n_first = 0) {
  const uint32_t N = (uint32_t)in.genomes.size();
  std::vector<uint32_t> order(N), rank(N);
  for (uint32_t g = 0; g < N; g++) order[g] = g;
  const auto longer = [&](uint32_t a, uint32_t b) { return in.genomes[a].total_len > in.genomes[b].total_len; };
  std::stable_sort(order.begin(), order.begin() + n_first, longer);
  std::stable_sort(order.begin() + n_first, order.end(), longer);
  for (uint32_t i = 0; i < N; i++) rank[order[i]] = i;
  return rank;
}

// The TSV of cluster and dereplicate (-o or stdout): one row per genome in genome-index order with its representative, its
// cluster and the ANI / aligned fractions of row(g), the result row joining g to rep[g] (nullptr: NA).  false after an ERROR line.
bool write_clusters(const Opts& op, const Inputs& in, const std::vector<uint32_t>& rep, const std::vector<uint32_t>& cluster,
                    const std::function<const sk_ani_result*(uint32_t)>& row) {
  FILE* o = op.out.empty() ? stdout : fopen(op.out.c_str(), "w");
  if (!o) { fprintf(stderr, "ERROR cannot open %s\n", op.out.c_str()); return false; }
  fprintf(o, "Genome_file\tRepresentative_file\tCluster\tANI\tAlign_fraction_genome\tAlign_fraction_representative\tGenome_name\tRepresentative_name\n");
  for (uint32_t g = 0; g < (uint32_t)rep.size(); g++) {
    const Genome &gg = in.genomes[g], &rg = in.genomes[rep[g]];
    fprintf(o, "%s\t%s\t%u\t", gg.file_name.c_str(), rg.file_name.c_str(), cluster[g]);
    const sk_ani_result* r = rep[g] == g ? nullptr : row(g);
    if (rep[g] == g) fputs("100.00\t100.00\t100.00", o);
    else if (!r) fputs("NA\tNA\tNA", o);
    else {
      const bool is_ref = r->ref_id == g;
      fprintf(o, "%.2f\t%.2f\t%.2f", (double)(r->ani * 100.f), (double)((is_ref ? r->af_ref : r->af_query) * 100.f),
              (double)((is_ref ? r->af_query : r->af_ref) * 100.f));
    }
    fprintf(o, "\t%s\t%s\n", short_name(gg.contigs[0], op.short_header).c_str(), short_name(rg.contigs[0], op.short_header).c_str());
  }
  if (o != stdout) fclose(o);
  return true;
}

// cluster: the triangle's results (the rows `triangle -E` prints) clustered on the GPU by sk_cluster at ANI >= --ani, greedy
// representatives or --single-linkage, or by sk_cluster_linkage (--linkage average|complete: every printed row is a
// similarity, --ani the cut; --dendrogram FILE writes the scipy linkage matrix), genomes ranked by total sequence length
// (longest first, ties by genome index).  One TSV row per genome in genome-index order: its representative, cluster, and the
// ANI / aligned fractions of the row joining them.
int run_cluster(Opts& op) {
  if (op.sparse || op.full_matrix || op.diagonal || op.distance || op.ci || op.detailed) {
    fprintf(stderr, "ERROR -E/--sparse, --full-matrix, --diagonal, --distance, --ci and --detailed are triangle output options; cluster does not take them.\n");
    return 2;
  }
  if (!op.linkage.empty() && op.linkage != "average" && op.linkage != "complete") {
    fprintf(stderr, "ERROR --linkage %s: the methods are average and complete.\n", op.linkage.c_str());
    return 2;
  }
  if (!op.linkage.empty() && op.single_linkage) { fprintf(stderr, "ERROR --linkage and --single-linkage exclude each other.\n"); return 2; }
  if (!op.dendrogram.empty() && op.linkage.empty()) { fprintf(stderr, "ERROR --dendrogram needs --linkage average|complete.\n"); return 2; }
  Inputs in;
  sk_ctx* ctx = nullptr;
  std::vector<sk_ani_result> all;
  if (const int rc = triangle_results(op, in, ctx, all, nullptr)) return rc;
  std::vector<sk_ani_result> res;
  for (auto& r : all) if (r.ani > 0.1f) res.push_back(r);
  all = std::vector<sk_ani_result>();
  const uint32_t N = (uint32_t)in.genomes.size();
  const std::vector<uint32_t> rank = length_rank(in);
  std::vector<uint32_t> rep(N), cluster(N);
  std::vector<uint64_t> edge(N);
  sk_cluster_stats st{};
  std::vector<sk_merge> merges;
  if (op.linkage.empty()) {
    const sk_cluster_params cp{(float)(op.cluster_ani / 100.0), op.single_linkage ? 1 : 0};
    CK(ctx, sk_cluster(ctx, N, res.data(), res.size(), rank.data(), &cp, rep.data(), cluster.data(), edge.data(), &st));
  } else {
    const sk_linkage_params lp{(float)(op.cluster_ani / 100.0), op.linkage == "complete" ? SK_LINKAGE_COMPLETE : SK_LINKAGE_AVERAGE,
                               op.dendrogram.empty() ? 0 : 1};
    if (!op.dendrogram.empty()) merges.resize(N ? N - 1 : 0);
    CK(ctx, sk_cluster_linkage(ctx, N, res.data(), res.size(), rank.data(), &lp, rep.data(), cluster.data(), edge.data(),
                               merges.empty() ? nullptr : merges.data(), &st));
  }
  if (!op.dendrogram.empty()) {   // scipy linkage matrix, heights in percent distance as `triangle --distance` prints them
    FILE* z = fopen(op.dendrogram.c_str(), "w");
    if (!z) { fprintf(stderr, "ERROR cannot open %s\n", op.dendrogram.c_str()); return 1; }
    for (const sk_merge& m : merges) fprintf(z, "%u\t%u\t%.6f\t%llu\n", m.a, m.b, 100.0 * m.height, (unsigned long long)m.size);
    fclose(z);
  }
  if (!write_clusters(op, in, rep, cluster, [&](uint32_t g) { return edge[g] == UINT64_MAX ? nullptr : &res[edge[g]]; })) return 1;
  if (op.linkage.empty())
    fprintf(stderr, "INFO %u genomes in %u clusters at ANI >= %g (%s), clustering %.1f ms\n", N, st.n_clusters, op.cluster_ani,
            op.single_linkage ? "single linkage" : "greedy", st.t_device * 1e3);
  else
    fprintf(stderr, "INFO %u genomes in %u clusters at ANI >= %g (%s linkage, %u rounds), clustering %.1f ms\n", N, st.n_clusters,
            op.cluster_ani, op.linkage.c_str(), st.rounds, st.t_device * 1e3);
  sk_ctx_destroy(ctx);
  return 0;
}

// dereplicate: cluster's greedy clusters (same inputs, presets, name ranks, length ranking and TSV) from sk_dereplicate, which
// screens and chains only genome x representative pairs instead of the whole triangle.  By default an in-memory set on one
// GPU: inputs that need the host sketch store, and --gpus N, are refused.  --host-store takes the store path whatever the
// input size: sketches in a host sketch store, sk_dereplicate_store on two contexts per GPU of --gpus N, the same output.
// --representatives FILE: one line per representative in cluster-id order, its file name (-i: its first contig name).
// --fixed-reps PATH / --fixed-reps-list FILE: genomes that are representatives already (sk_dereplicate_fixed): they come
// first in genome-index and rank order and keep cluster ids 0 .. n - 1; the positional inputs and -l are the new genomes.
int run_dereplicate(Opts& op) {
  if (op.single_linkage || !op.linkage.empty() || !op.dendrogram.empty()) {
    fprintf(stderr, "ERROR --single-linkage, --linkage and --dendrogram are cluster options; dereplicate is greedy clustering only: use cluster.\n");
    return 2;
  }
  if (op.sparse || op.full_matrix || op.diagonal || op.distance || op.ci || op.detailed) {
    fprintf(stderr, "ERROR -E/--sparse, --full-matrix, --diagonal, --distance, --ci and --detailed are triangle output options; dereplicate does not take them.\n");
    return 2;
  }
  if (op.gpus > 1 && !op.host_store) {
    fprintf(stderr, "ERROR --gpus %d: dereplicate keeps the sketches on one GPU; use cluster --gpus %d, or dereplicate --host-store --gpus %d.\n", op.gpus,
            op.gpus, op.gpus);
    return 2;
  }
  TriangleInputs ti;
  if (const int rc = open_triangle_inputs(op, ti)) return rc;
  if (ti.use_store && !op.host_store) {
    fprintf(stderr, "ERROR dereplicate keeps the sketches on the GPU, and these inputs (~%.1f GB estimated%s) need the host sketch store: use cluster, "
            "which takes the store path, or dereplicate --host-store.\n", ti.need_gb, device_budget() ? ", SK_DEVICE_BUDGET_MB set" : "");
    return 1;
  }
  if (op.host_store) ti.use_store = true;
  Inputs in;
  sk_ctx* ctx = nullptr;
  if (const int rc = op.fixed_given ? load_fixed_inputs(op, in, ctx, ti) : load_triangle_inputs(op, in, ctx, ti)) return rc;
  const sk_map_params mp = map_params(op, !op.no_learned && op.c >= 70 && !op.individual && !op.median);
  const std::vector<uint64_t> ranks = name_ranks(in.genomes)[0];
  const uint32_t N = (uint32_t)in.genomes.size();
  const std::vector<uint32_t> rank = length_rank(in, ti.n_fixed);
  std::vector<uint32_t> rep(N), cluster(N);
  std::vector<sk_ani_result> join(N);
  // SK_DEREP_WAVE: genomes per wave (a test hook: many waves on small inputs); it only sizes the waves
  const char* w = getenv("SK_DEREP_WAVE");
  const sk_derep_params dp{(float)(op.cluster_ani / 100.0), w ? (uint32_t)std::max(1ll, atoll(w)) : 0u};
  sk_derep_stats st{};
  sk_store_stats sst{};
  size_t n_ctx = 1;
  if (ti.store) {
    // two contexts on each of the --gpus devices, as the triangle's store path: one gathers its next working set while the
    // other chains
    CK(ctx, sk_sketch_store_set_name_ranks(ti.store, ranks.data()));
    std::vector<sk_ctx*> sctx = make_contexts(ctx, op, op.gpus, 2);
    n_ctx = sctx.size();
    if (op.fixed_given)
      CK(ctx, sk_dereplicate_store_fixed(sctx.data(), (uint32_t)sctx.size(), ti.store, &mp, rank.data(), ti.n_fixed, &dp, device_budget(), rep.data(),
                                         cluster.data(), join.data(), &st, &sst));
    else
      CK(ctx, sk_dereplicate_store(sctx.data(), (uint32_t)sctx.size(), ti.store, &mp, rank.data(), &dp, device_budget(), rep.data(), cluster.data(),
                                   join.data(), &st, &sst));
    for (size_t d = sctx.size(); d-- > 1;) sk_ctx_destroy(sctx[d]);
    sk_sketch_store_free(ti.store);
  } else {
    sk_sketch_set* set = ti.loaded ? ti.loaded : sketch(ctx, in, ti.sp);
    sk_sketch_set_set_name_ranks(set, ranks.data());
    if (op.fixed_given) CK(ctx, sk_dereplicate_fixed(ctx, set, &mp, rank.data(), ti.n_fixed, &dp, rep.data(), cluster.data(), join.data(), &st));
    else CK(ctx, sk_dereplicate(ctx, set, &mp, rank.data(), &dp, rep.data(), cluster.data(), join.data(), &st));
    sk_sketch_set_free(set);
  }
  if (!write_clusters(op, in, rep, cluster, [&](uint32_t g) { return &join[g]; })) return 1;
  if (!op.representatives.empty()) {
    FILE* f = fopen(op.representatives.c_str(), "w");
    if (!f) { fprintf(stderr, "ERROR cannot open %s\n", op.representatives.c_str()); return 1; }
    std::vector<uint32_t> by_cluster(st.n_clusters);
    for (uint32_t g = 0; g < N; g++) if (rep[g] == g) by_cluster[cluster[g]] = g;
    for (uint32_t g : by_cluster) fprintf(f, "%s\n", (op.individual ? in.genomes[g].contigs[0] : in.genomes[g].file_name).c_str());
    fclose(f);
  }
  char fixed[64] = "";
  if (op.fixed_given) snprintf(fixed, sizeof(fixed), ", %u fixed representatives", ti.n_fixed);
  fprintf(stderr, "INFO %u genomes in %u clusters at ANI >= %g (greedy)%s, %u waves, %llu pairs screened, %llu chained; "
          "screen %.2f s, chain %.2f s, decide %.2f s, total %.2f s\n", N, st.n_clusters, op.cluster_ani, fixed, st.waves,
          (unsigned long long)st.pairs_screened, (unsigned long long)st.pairs_chained, st.t_screen, st.t_chain, st.t_decide, st.t_total);
  if (op.host_store)
    fprintf(stderr, "INFO Store path: %u working sets, %.2f GB gathered (largest working set %.2f GB); marker gather %.2f s, gather %.2f s, chain %.2f s "
            "(summed over %zu contexts)\n", sst.n_working_sets, sst.gathered_bytes / 1e9, sst.max_working_set_bytes / 1e9, sst.t_screen, sst.t_gather,
            sst.t_chain, n_ctx);
  sk_ctx_destroy(ctx);
  return 0;
}

// a Newick label: as is, or single-quoted with every ' doubled when it holds whitespace or any of ()[]':;,
std::string newick_label(const std::string& s) {
  if (!s.empty() && s.find_first_of(" \t\r\n()[]':;,") == std::string::npos) return s;
  std::string q = "'";
  for (char c : s) q += c == '\'' ? std::string("''") : std::string(1, c);
  return q + "'";
}

// Newick text of a tree whose internal nodes list their (child, branch length) pairs: nodes < n_leaves are leaves, `root`
// is written without a length.  An explicit stack, not recursion: a caterpillar of 50 000 leaves nests 50 000 deep.
std::string newick(uint32_t n_leaves, const std::vector<std::string>& labels,
                   const std::vector<std::vector<std::pair<uint32_t, double>>>& kids, uint32_t root) {
  if (root < n_leaves) return labels[root] + ";\n";
  std::string out = "(";
  char len[64];
  struct Frame { uint32_t v; size_t next; double len; };
  std::vector<Frame> st{{root, 0, 0.0}};
  while (!st.empty()) {
    Frame& f = st.back();
    if (f.next < kids[f.v].size()) {
      if (f.next) out += ',';
      const std::pair<uint32_t, double> c = kids[f.v][f.next++];
      if (c.first < n_leaves) {
        snprintf(len, sizeof(len), ":%.6f", 100.0 * c.second);
        out += labels[c.first];
        out += len;
      } else {
        out += '(';
        st.push_back({c.first, 0, c.second});
      }
      continue;
    }
    out += ')';
    if (st.size() > 1) { snprintf(len, sizeof(len), ":%.6f", 100.0 * f.len); out += len; }
    st.pop_back();
  }
  return out + ";\n";
}

// tree: the triangle's genomes (every row `triangle -E` prints) as a Newick tree, branch lengths in percent distance.
// --method nj (default): sk_neighbor_joining (with --gpus N > 1 sk_neighbor_joining_multi on N contexts, the same tree), written unrooted with the basal trifurcation (X, Y, K): X and Y the children
// of the last internal node, K the other last node at the full last-edge length.  --method average | complete:
// sk_cluster_linkage's dendrogram (genomes ranked as cluster ranks them), rooted, a child at (h_parent - h_child) / 2 below
// its parent, so that patristic distances are the cophenetic ones.  Labels as triangle's matrix names its rows.
int run_tree(Opts& op) {
  if (op.sparse || op.full_matrix || op.diagonal || op.distance || op.ci || op.detailed) {
    fprintf(stderr, "ERROR -E/--sparse, --full-matrix, --diagonal, --distance, --ci and --detailed are triangle output options; tree does not take them.\n");
    return 2;
  }
  if (op.tree_method != "nj" && op.tree_method != "average" && op.tree_method != "complete") {
    fprintf(stderr, "ERROR --method %s: the methods are nj, average and complete.\n", op.tree_method.c_str());
    return 2;
  }
  Inputs in;
  sk_ctx* ctx = nullptr;
  std::vector<sk_ani_result> all;
  if (const int rc = triangle_results(op, in, ctx, all, nullptr)) return rc;
  std::vector<sk_ani_result> res;
  for (auto& r : all) if (r.ani > 0.1f) res.push_back(r);
  all = std::vector<sk_ani_result>();
  const uint32_t N = (uint32_t)in.genomes.size();
  std::vector<std::string> labels(N);
  for (uint32_t g = 0; g < N; g++) labels[g] = newick_label(op.individual ? in.genomes[g].contigs[0] : in.genomes[g].file_name);
  std::vector<std::vector<std::pair<uint32_t, double>>> kids(N ? 2 * N : 0);   // node 2N - 1: the NJ trifurcation
  uint32_t root = N ? 2 * N - 2 : 0, steps = 0;
  double t_device = 0;
  size_t n_ctx = 1;
  if (op.tree_method == "nj") {
    std::vector<sk_nj_join> joins(N > 1 ? N - 1 : 0);
    sk_nj_stats st{};
    if (op.gpus > 1) {   // the distance matrix split over one context per GPU
      std::vector<sk_ctx*> ctxs = make_contexts(ctx, op, op.gpus);
      n_ctx = ctxs.size();
      CK(ctx, sk_neighbor_joining_multi(ctxs.data(), (uint32_t)n_ctx, N, res.data(), res.size(), joins.empty() ? nullptr : joins.data(), &st));
      for (size_t d = 1; d < ctxs.size(); d++) sk_ctx_destroy(ctxs[d]);
    } else {
      CK(ctx, sk_neighbor_joining(ctx, N, res.data(), res.size(), joins.empty() ? nullptr : joins.data(), &st));
    }
    for (uint32_t t = 0; t < joins.size(); t++) kids[N + t] = {{joins[t].a, joins[t].len_a}, {joins[t].b, joins[t].len_b}};
    if (N >= 3) {   // unroot: the last internal node's children and the other last node, at the whole last edge
      const sk_nj_join& l = joins[N - 2];
      const uint32_t last = 2 * N - 3, other = l.a == last ? l.b : l.a;
      root = 2 * N - 1;
      kids[root] = kids[last];
      kids[root].push_back({other, l.len_a + l.len_b});
    }
    steps = st.compactions;
    t_device = st.t_device;
  } else {
    std::vector<uint32_t> rep(N), cluster(N);
    std::vector<uint64_t> edge(N);
    std::vector<sk_merge> merges(N > 1 ? N - 1 : 0);
    const std::vector<uint32_t> rank = length_rank(in);
    const sk_linkage_params lp{(float)(op.cluster_ani / 100.0), op.tree_method == "complete" ? SK_LINKAGE_COMPLETE : SK_LINKAGE_AVERAGE, 1};
    sk_cluster_stats st{};
    CK(ctx, sk_cluster_linkage(ctx, N, res.data(), res.size(), rank.data(), &lp, rep.data(), cluster.data(), edge.data(),
                               merges.empty() ? nullptr : merges.data(), &st));
    const auto height = [&](uint32_t v) { return v < N ? 0.0 : merges[v - N].height; };
    for (uint32_t j = 0; j < merges.size(); j++) {
      const double h = merges[j].height;
      kids[N + j] = {{merges[j].a, (h - height(merges[j].a)) / 2}, {merges[j].b, (h - height(merges[j].b)) / 2}};
    }
    steps = st.rounds;
    t_device = st.t_device;
  }
  FILE* o = op.out.empty() ? stdout : fopen(op.out.c_str(), "w");
  if (!o) { fprintf(stderr, "ERROR cannot open %s\n", op.out.c_str()); return 1; }
  if (N) fputs(newick(N, labels, kids, root).c_str(), o);
  if (o != stdout) fclose(o);
  const std::string on = n_ctx > 1 ? " on " + std::to_string(n_ctx) + " contexts" : "";
  fprintf(stderr, "INFO %u genomes, tree by %s (%u %s)%s, %.1f ms on the device\n", N, op.tree_method.c_str(), steps,
          op.tree_method == "nj" ? "compactions" : "rounds", on.c_str(), t_device * 1e3);
  sk_ctx_destroy(ctx);
  return 0;
}

// write_query_ref_list (src/file_io.rs:608-678) of dist and search, one block of queries at a time: the block's rows (rows of
// equal ANI in the order they print) are grouped by the query's first contig name, each group sorted by ANI (descending,
// stable) and its top n written, with their mapping records under --mappings (rm.recs[rm.off[i] .. rm.off[i + 1]) belong to
// row i), then flushed.  more() prints the line the reference prints between two blocks.
struct DistWriter {
  const Opts& op;
  const std::vector<Genome>& refs;
  const std::vector<Genome>& queries;
  MappingFile mf;
  FILE* o = nullptr;
  DistWriter(const Opts& op_, const std::vector<Genome>& refs_, const std::vector<Genome>& queries_) : op(op_), refs(refs_), queries(queries_) {}
  // false after an ERROR line; k = the sketches' k
  bool open(uint32_t k) {
    if (!op.mappings.empty() && !mf.open(op.mappings, k)) return false;
    o = op.out.empty() ? stdout : fopen(op.out.c_str(), "w");
    if (!o) { fprintf(stderr, "ERROR cannot open %s\n", op.out.c_str()); return false; }
    write_header(o, op.ci, op.detailed);
    return true;
  }
  bool mappings() const { return mf.f != nullptr; }
  void write(const std::vector<sk_ani_result>& res, const RowMaps& rm) {
    std::map<std::string, std::vector<const sk_ani_result*>> groups;
    for (auto& r : res) if (r.ani > 0.1f) groups[queries[r.query_id].contigs[0]].push_back(&r);
    for (auto& kv : groups) {
      auto v = kv.second;
      std::stable_sort(v.begin(), v.end(), [](const sk_ani_result* a, const sk_ani_result* b) { return a->ani > b->ani; });
      for (size_t i = 0; i < v.size() && i < op.n; i++) {
        write_row(o, *v[i], refs[v[i]->ref_id], queries[v[i]->query_id], op);
        if (mf.f) {
          const size_t row = v[i] - res.data();
          mf.write(rm.recs.data() + rm.off[row], rm.off[row + 1] - rm.off[row], refs[v[i]->ref_id], queries[v[i]->query_id], op);
        }
      }
    }
    fflush(o);
    mf.flush();
  }
  void more() { fprintf(stderr, "INFO Writing results for %zu query sequences.\n", intermediate_write_count()); }
  ~DistWriter() { if (o && o != stdout) fclose(o); }
};

// dist's queries in blocks of INTERMEDIATE_WRITE_COUNT (src/dist.rs:151-175).  block(q0, q1, res, rm) fills res with the
// results of the queries [q0, q1), rows of equal ANI in the order they print, and with --mappings (rm non-null, k = the
// sketches' k) rm with their mapping records; or returns false (after an ERROR line) to end the run with exit code 1.
template <class F>
int write_dist(const Opts& op, const std::vector<Genome>& refs, const std::vector<Genome>& queries, uint32_t k, F block) {
  DistWriter w(op, refs, queries);
  if (!w.open(k)) return 1;
  const size_t FL = intermediate_write_count(), NQ = queries.size();
  std::vector<sk_ani_result> res;
  RowMaps rm;
  RowMaps* rmp = w.mappings() ? &rm : nullptr;
  for (size_t q0 = 0; q0 < NQ; q0 += FL) {
    rm.clear();
    if (!block(q0, std::min(q0 + FL, NQ), res, rmp)) return 1;
    w.write(res, rm);
    if (q0 + FL < NQ) w.more();
  }
  return 0;
}

int run_dist(Opts& op) {
  resolve_presets(op);
  if (op.refs.empty() || op.queries.empty()) { fprintf(stderr, "ERROR No reference sketches/genomes or query sketches/genomes found.\n"); return 1; }
  Inputs rin, qin;
  const bool refs_are_sketch = sketch_inputs_given(op.refs), queries_are_sketch = sketch_inputs_given(op.queries);
  sk_sketch_params sp{op.c, op.k, op.m};
  // sketch inputs (.sketch files, databases) carry their own parameters, which then also apply to FASTA inputs on the other
  // side (src/dist.rs:17-50).  They are opened on the host here and decoded and imported in groups once the contexts exist.
  skdb::SketchInputs rsi, qsi;
  if (refs_are_sketch) {
    fprintf(stderr, "INFO Sketches detected.\n");
    if (!skdb::open_sketch_inputs(op.refs, rsi)) return 1;   // file_io::sketches_from_sketch (src/file_io.rs:680-717)
    if (!rsi.entries.empty()) {
      const sk_sketch_params dp = params_of(rsi);
      if (dp.c != sp.c || dp.k != sp.k || dp.marker_c != sp.marker_c)
        fprintf(stderr, "WARN Parameters from .sketch files not equal to the input parameters. Using parameters from .sketch files.\n");
      sp = dp;
    }
  }
  if (queries_are_sketch) {
    if (!skdb::open_sketch_inputs(op.queries, qsi)) return 1;   // file_io::sketches_from_sketch (src/file_io.rs:680-717)
    const sk_sketch_params dp = params_of(qsi);
    if (!qsi.entries.empty() && (dp.c != sp.c || dp.k != sp.k || dp.marker_c != sp.marker_c)) {
      if (refs_are_sketch) { fprintf(stderr, "ERROR Query sketch parameters were not equal to reference sketch parameters. Exiting.\n"); return 1; }
      fprintf(stderr, "WARN Parameters from .sketch files not equal to the input parameters. Using parameters from .sketch files.\n");
      sp = dp;
    }
  }
  sk_ctx* ctx = nullptr;
  if (sk_ctx_create(op.device, &ctx) != 0) { fprintf(stderr, "ERROR a CUDA device is required (no CPU fallback)\n"); return 1; }
  // store path: both sides go into host sketch stores in groups and are chained in working sets (sk_query_ref_store)
  double need_gb = 0;
  const bool use_store = dist_needs_store(op, refs_are_sketch, queries_are_sketch, rsi, qsi, &need_gb);
  if (use_store && !op.mappings.empty()) {
    fprintf(stderr, "ERROR --mappings is not supported when the sketches exceed device memory (host sketch store path); "
                    "split the inputs into runs that fit the device.\n");
    return 1;
  }
  sk_sketch_store *rstore = nullptr, *qstore = nullptr;
  const int threads = std::max(op.threads, 1);
  if (use_store) {
    info_store_path(op, need_gb, true);
    rstore = refs_are_sketch ? store_sketch_inputs(ctx, rsi, threads, sp, rin.genomes) : fill_store(ctx, op, op.refs, op.ri, rin.genomes, sp);
    if (refs_are_sketch && !rstore) return 1;      // an entry could not be loaded (reported)
    qstore = queries_are_sketch ? store_sketch_inputs(ctx, qsi, threads, sp, qin.genomes) : fill_store(ctx, op, op.queries, op.qi, qin.genomes, sp);
    if (queries_are_sketch && !qstore) return 1;
  } else {
    // sketch inputs: names now (for the name ranks), the rest of the metadata when each side is imported below
    if (!refs_are_sketch) load_inputs(op.refs, op.ri, threads, rin);
    else for (auto& e : rsi.entries) { Genome g; g.file_name = e.file_name; rin.genomes.push_back(std::move(g)); }
    if (!queries_are_sketch) load_inputs(op.queries, op.qi, threads, qin);
    else for (auto& e : qsi.entries) { Genome g; g.file_name = e.file_name; qin.genomes.push_back(std::move(g)); }
  }
  if (rin.genomes.empty() || qin.genomes.empty()) { fprintf(stderr, "ERROR No reference sketches/genomes or query sketches/genomes found.\n"); return 1; }
  const sk_map_params mp = map_params(op, !op.no_learned && op.c >= 70 && !op.qi && !op.ri && !op.median);
  const bool use_index = (n_inputs(op.queries, qsi) > 50 || op.qi) && !op.no_marker_index;   // FULL_INDEX_THRESH (src/parse.rs:750)
  const auto ranks = name_ranks(rin.genomes, qin.genomes);
  const std::vector<uint64_t> &rr = ranks[0], &qr = ranks[1];
  if (use_store) {
    // two contexts on each of the --gpus devices: one gathers its next working set over PCIe while the other chains.  Every
    // block of queries is written at the end, through the same writer as the in-memory path.
    CK(ctx, sk_sketch_store_set_name_ranks(rstore, rr.data()));
    CK(ctx, sk_sketch_store_set_name_ranks(qstore, qr.data()));
    std::vector<sk_ctx*> sctx = make_contexts(ctx, op, op.gpus, 2);
    sk_ani_result* r = nullptr; uint64_t nr = 0;
    CK(ctx, sk_query_ref_store(sctx.data(), (uint32_t)sctx.size(), rstore, qstore, &mp, use_index ? 2 : 0, device_budget(), &r, &nr, nullptr));
    std::vector<sk_ani_result> all(r, r + nr);
    sk_free(r);
    std::sort(all.begin(), all.end(), [](const sk_ani_result& a, const sk_ani_result& b) { return a.query_id != b.query_id ? a.query_id < b.query_id : a.ref_id < b.ref_id; });
    size_t p0 = 0;
    const int rc = write_dist(op, rin.genomes, qin.genomes, sp.k, [&](size_t, size_t q1, std::vector<sk_ani_result>& res, RowMaps*) {
      size_t p1 = p0;
      while (p1 < all.size() && all[p1].query_id < q1) p1++;
      res.assign(all.begin() + p0, all.begin() + p1);
      p0 = p1;
      return true;
    });
    sk_sketch_store_free(rstore);
    sk_sketch_store_free(qstore);
    for (size_t d = sctx.size(); d-- > 0;) sk_ctx_destroy(sctx[d]);
    return rc;
  }
  // --gpus N: the references in W contiguous blocks (genome order, balanced by bases, or by records for sketch inputs), each
  // sketched or imported on its own context; the queries once on context 0, then copied to the others.  Sketch inputs are
  // decoded and imported in groups (-t threads split over the contexts), so host memory holds one group per context.
  const size_t NR = rin.genomes.size(), W = std::min<size_t>(std::max(op.gpus, 1), NR);
  std::vector<sk_ctx*> ctxs = make_contexts(ctx, op, W);
  std::vector<uint64_t> weight(NR);
  for (size_t g = 0; g < NR; g++) weight[g] = refs_are_sketch ? rsi.entries[g].weight : rin.genomes[g].total_len;
  const std::vector<size_t> gb = split_balanced(weight, W);
  std::vector<sk_sketch_set*> rsets(W, nullptr), qsets(W, nullptr);
  std::vector<uint32_t> ref_first(W);
  for (size_t d = 0; d < W; d++) ref_first[d] = (uint32_t)gb[d];
  std::atomic<bool> load_failed{false};     // a sketch entry could not be loaded (reported); the run ends below
  per_context(W, [&](size_t d) {
    sk_ctx* c = ctxs[d];
    const int t_ctx = context_threads(op, d, W);
    bool ok = true;
    if (refs_are_sketch) rsets[d] = import_sketch_inputs(c, rsi, gb[d], gb[d + 1], t_ctx, sp, rin.genomes.data() + gb[d], ok);
    else rsets[d] = sketch(c, rin, sp, gb[d], gb[d + 1]);
    if (!ok) { load_failed = true; return; }
    sk_sketch_set_set_name_ranks(rsets[d], rr.data() + gb[d]);
    if (d == 0) {
      qsets[0] = queries_are_sketch ? import_sketch_inputs(c, qsi, 0, qsi.entries.size(), t_ctx, sp, qin.genomes.data(), ok) : sketch(c, qin, sp);
      if (!ok) { load_failed = true; return; }
      sk_sketch_set_set_name_ranks(qsets[0], qr.data());
    }
  });
  if (load_failed) return 1;
  for (size_t d = 1; d < W; d++) CK(ctxs[d], sk_sketch_set_copy(ctxs[d], qsets[0], &qsets[d]));
  uint64_t* pairs = nullptr; uint64_t np = 0;
  CK(ctx, sk_screen_query_ref_multi(ctxs.data(), (uint32_t)W, rsets.data(), ref_first.data(), qsets.data(), &mp, use_index ? 2 : 0, &pairs, &np));
  // queries are processed, and their results appended, in blocks of INTERMEDIATE_WRITE_COUNT (src/dist.rs:151-175)
  std::vector<uint64_t> byq(pairs, pairs + np);
  sk_free(pairs);
  std::sort(byq.begin(), byq.end(), [](uint64_t a, uint64_t b) { return (uint32_t)a != (uint32_t)b ? (uint32_t)a < (uint32_t)b : a < b; });
  size_t p0 = 0;
  const int rc = write_dist(op, rin.genomes, qin.genomes, sp.k, [&](size_t, size_t q1, std::vector<sk_ani_result>& res, RowMaps* rm) {
    size_t p1 = p0;
    while (p1 < byq.size() && (uint32_t)byq[p1] < q1) p1++;
    res.resize(p1 - p0);
    if (rm) {
      std::vector<uint64_t> off(p1 - p0 + 1);
      sk_mapping* maps = nullptr;
      CK(ctx, sk_chain_pairs_multi_mappings(ctxs.data(), (uint32_t)W, rsets.data(), ref_first.data(), qsets.data(), byq.data() + p0, p1 - p0, &mp,
                                            res.data(), off.data(), &maps));
      for (size_t i = 0; i < res.size(); i++) rm->add(maps + off[i], off[i + 1] - off[i]);
      sk_free(maps);
    } else {
      CK(ctx, sk_chain_pairs_multi(ctxs.data(), (uint32_t)W, rsets.data(), ref_first.data(), qsets.data(), byq.data() + p0, p1 - p0, &mp, res.data()));
    }
    p0 = p1;
    return true;
  });
  for (size_t d = 0; d < W; d++) { sk_sketch_set_free(rsets[d]); sk_sketch_set_free(qsets[d]); }
  for (size_t d = W; d-- > 0;) sk_ctx_destroy(ctxs[d]);
  return rc;
}

// ---- sketch / search (src/sketch.rs, src/search.rs) --------------------------------------------------------------
std::string base_name(const std::string& p) { size_t i = p.find_last_of('/'); return i == std::string::npos ? p : p.substr(i + 1); }
bool path_exists(const std::string& p) { struct stat st; return stat(p.c_str(), &st) == 0; }
void make_dirs(const std::string& p) {
  for (size_t i = 1; i <= p.size(); i++)
    if (i == p.size() || p[i] == '/') mkdir(p.substr(0, i).c_str(), 0777);
}

// genomes [a, b) of a group as sk_entry_meta (the arrays it points into)
struct EntryMetaArrays {
  std::string names, contig_names;
  std::vector<uint64_t> name_off{0}, contig_name_off{0}, contig_first{0}, contig_order;
  EntryMetaArrays(const std::vector<Genome>& gs, size_t a, size_t b) {
    for (size_t g = a; g < b; g++) {
      names += gs[g].file_name;
      name_off.push_back(names.size());
      for (auto& c : gs[g].contigs) { contig_names += c; contig_name_off.push_back(contig_names.size()); }
      contig_first.push_back(contig_name_off.size() - 1);
      contig_order.push_back(gs[g].contig_order);
    }
  }
  sk_entry_meta meta() const {
    return sk_entry_meta{names.data(), name_off.data(), contig_names.data(), contig_name_off.data(), contig_first.data(), contig_order.data()};
  }
};

// one context's run of a group encoded on the device (sk_sketch_set_encode): full entries and markers-only entries, each
// form back to back
struct EncodedRun {
  std::vector<uint8_t, skdb::uninit_alloc<uint8_t>> full, mk;
  std::vector<uint64_t> full_len, mk_len;
};

void encode_run(sk_ctx* ctx, const sk_sketch_set* set, const EntryMetaArrays& ma, EncodedRun& out) {
  const uint32_t n = sk_sketch_set_n_genomes(set);
  const sk_entry_meta m = ma.meta();
  auto encode = [&](int form, std::vector<uint8_t, skdb::uninit_alloc<uint8_t>>& bytes, std::vector<uint64_t>& len) {
    len.resize(n);
    CK(ctx, sk_sketch_set_encode_sizes(set, 0, n, form, &m, len.data()));
    uint64_t total = 0;
    for (uint64_t l : len) total += l;
    bytes.resize(total);
    CK(ctx, sk_sketch_set_encode(set, 0, n, form, &m, bytes.data(), total, nullptr));
  };
  encode(SK_ENTRY_FULL, out.full, out.full_len);
  encode(SK_ENTRY_MARKERS, out.mk, out.mk_len);
}

// `sketch`: the files go through the GPU in groups (file_group_end), three stages deep.  While the contexts sketch and encode
// group n, a reader thread loads group n + 1 and a writer thread appends group n - 1's entries in database order,
// (file_name, contig_order).  A group's genomes are cut into --gpus contiguous runs balanced by bases, one per context, and
// the runs are written in order, so the output does not depend on --gpus.  Encoding waits for the previous group's writer:
// host memory holds at most two groups of sequence (the one sketched, the one read) and one group's encoded entries.
int run_sketch(Opts& op) {
  using clk = std::chrono::steady_clock;
  auto secs = [](clk::time_point t0) { return std::chrono::duration<double>(clk::now() - t0).count(); };
  resolve_presets(op);
  if (op.files.empty()) { fprintf(stderr, "ERROR No reference inputs found.\n"); return 1; }
  if (op.out.empty()) { fprintf(stderr, "ERROR an output folder is required (-o)\n"); return 1; }
  if (path_exists(op.out)) { fprintf(stderr, "ERROR Output directory exists; output directory must not be an existing directory. Exiting.\n"); return 1; }   // src/sketch.rs:19-22
  make_dirs(op.out);
  if (op.separate_sketches && op.individual)
    fprintf(stderr, "WARN --separate-sketches combined with -i (individual contigs) is NOT compatible with `skani search`.\n");
  sk_ctx* ctx = nullptr;
  if (sk_ctx_create(op.device, &ctx) != 0) { fprintf(stderr, "ERROR a CUDA device is required (no CPU fallback)\n"); return 1; }
  const size_t W = (size_t)std::max(op.gpus, 1);
  std::vector<sk_ctx*> ctxs = make_contexts(ctx, op, W);
  sk_sketch_params sp{op.c, op.k, op.m};
  skdb::DiskParams dp;
  dp.c = op.c; dp.k = op.k; dp.marker_c = op.m;
  skdb::DbWriter w;
  if (!w.open(op.out, dp, op.separate_sketches)) { fprintf(stderr, "ERROR Failed to create the sketch database writer in %s\n", op.out.c_str()); return 1; }
  std::vector<std::string> files = op.files;
  std::sort(files.begin(), files.end());
  std::vector<size_t> fb{0};
  while (fb.back() < files.size()) fb.push_back(file_group_end(files, fb.back()));
  const size_t n_groups = fb.size() - 1;
  double t_read = 0, t_sketch = 0, t_encode = 0, t_write = 0;
  auto load = [&](size_t k, Inputs* in) {
    const auto t0 = clk::now();
    load_inputs(std::vector<std::string>(files.begin() + fb[k], files.begin() + fb[k + 1]), op.individual, std::max(op.threads, 1), *in);
    t_read += secs(t0);
  };
  // the writer's group: its genomes, its runs' first genomes and their encoded entries
  std::vector<Genome> wr_genomes;
  std::vector<size_t> wr_bounds;
  std::vector<EncodedRun> wr_enc;
  std::atomic<bool> write_failed{false};
  size_t total = 0;
  auto write_group = [&] {
    const auto t0 = clk::now();
    size_t j_in_file = 0;
    for (size_t d = 0; d + 1 < wr_bounds.size() && !write_failed; d++) {
      const EncodedRun& e = wr_enc[d];
      uint64_t fo = 0, mo = 0;
      for (size_t i = 0; i < wr_bounds[d + 1] - wr_bounds[d]; i++) {
        const size_t g = wr_bounds[d] + i;
        const Genome& ge = wr_genomes[g];
        j_in_file = (g && ge.file_name == wr_genomes[g - 1].file_name) ? j_in_file + 1 : 0;
        std::string path;        // src/sketch.rs:38-101: <basename>.sketch, or <j>_<basename>.sketch with -i
        if (op.separate_sketches) path = op.out + "/" + (op.individual ? std::to_string(j_in_file) + "_" : std::string()) + base_name(ge.file_name) + ".sketch";
        if (!w.add(ge.file_name, path, e.full.data() + fo, e.full_len[i], e.mk.data() + mo, e.mk_len[i])) {
          if (op.separate_sketches) fprintf(stderr, "ERROR cannot write %s\n", path.c_str());
          else fprintf(stderr, "ERROR Failed to add sketch to database\n");
          write_failed = true;
          break;
        }
        fo += e.full_len[i]; mo += e.mk_len[i];
        if (++total % 100 == 0) fprintf(stderr, "INFO %zu sequences sketched.\n", total);
      }
    }
    wr_enc.clear();
    t_write += secs(t0);
  };
  Inputs cur, next;
  std::thread reader, writer;
  if (n_groups) load(0, &cur);
  for (size_t k = 0; k < n_groups; k++) {
    if (k + 1 < n_groups) reader = std::thread(load, k + 1, &next);
    const size_t G = cur.genomes.size(), R = std::min(W, G);
    std::vector<uint64_t> weight(G);
    for (size_t g = 0; g < G; g++) weight[g] = cur.genomes[g].total_len;
    const std::vector<size_t> gb = R ? split_balanced(weight, R) : std::vector<size_t>{0};
    std::vector<sk_sketch_set*> sets(R, nullptr);
    auto t0 = clk::now();
    per_context(R, [&](size_t d) { sets[d] = sketch(ctxs[d], cur, sp, gb[d], gb[d + 1]); });
    t_sketch += secs(t0);
    std::vector<Genome> genomes = std::move(cur.genomes);
    cur = Inputs();                                           // the group's sequence is no longer needed
    if (writer.joinable()) writer.join();
    if (write_failed) { if (reader.joinable()) reader.join(); return 1; }
    std::vector<EncodedRun> enc(R);
    t0 = clk::now();
    per_context(R, [&](size_t d) {
      encode_run(ctxs[d], sets[d], EntryMetaArrays(genomes, gb[d], gb[d + 1]), enc[d]);
      sk_sketch_set_free(sets[d]);
    });
    t_encode += secs(t0);
    wr_genomes = std::move(genomes); wr_bounds = gb; wr_enc = std::move(enc);
    writer = std::thread(write_group);
    if (reader.joinable()) reader.join();
    cur = std::move(next);
    next = Inputs();
  }
  if (writer.joinable()) writer.join();
  if (write_failed) return 1;
  if (!w.finalize()) { fprintf(stderr, op.separate_sketches ? "ERROR cannot write markers.bin\n" : "ERROR Failed to finalize consolidated database\n"); return 1; }
  fprintf(stderr, "INFO %zu sketches written in %zu group(s): read %.2f s, sketch %.2f s, encode %.2f s, write %.2f s.\n", total, n_groups, t_read,
          t_sketch, t_encode, t_write);
  fprintf(stderr, "INFO Successfully wrote %zu sketches to %s\n", total, op.out.c_str());
  for (size_t d = ctxs.size(); d-- > 0;) sk_ctx_destroy(ctxs[d]);
  return 0;
}

// the bases bound of a query group of search: 8 GiB.  SK_SEARCH_GROUP_BASES lowers it (a test hook: one multi-record file
// cut into several query groups with --qi).
uint64_t search_group_bases() {
  if (const char* e = getenv("SK_SEARCH_GROUP_BASES")) return (uint64_t)std::max(1ll, atoll(e));
  return 8ull << 30;
}

// search streams its queries: they are read in groups of files, each query group is sketched (or imported), copied to the
// --gpus contexts, screened against a reference marker index built once on ctx (sk_ref_index_screen) and chained, and the
// results are written in blocks of INTERMEDIATE_WRITE_COUNT queries as each block's last query is done.  The output is that
// of one pass over all queries: name ranks come from search_plan::NameRanks, which needs the reference names only.
int run_search(Opts& op) {
  if (op.db_dir.empty()) { fprintf(stderr, "ERROR search needs -d <sketched database folder>\n"); return 1; }
  if (op.queries.empty()) { fprintf(stderr, "ERROR No query files found.\n"); return 1; }
  const std::string marker_file = op.db_dir + "/markers.bin";
  if (!path_exists(marker_file)) { fprintf(stderr, "ERROR markers.bin not found in the folder. Ensure that the folder was generated by `skani sketch`.\n"); return 1; }
  skdb::DiskParams dp;
  std::vector<skdb::HostSketch> ref_mk;
  try { skdb::read_markers_bin(marker_file, dp, ref_mk); }
  catch (const std::exception& e) { fprintf(stderr, "ERROR Problem reading %s. Exiting. (%s)\n", marker_file.c_str(), e.what()); return 1; }
  if (dp.use_aa) { fprintf(stderr, "ERROR amino-acid databases are not supported\n"); return 1; }
  if (ref_mk.empty()) { fprintf(stderr, "ERROR No valid reference fastas or sketches found.\n"); return 1; }
  std::vector<Genome> refs;
  for (auto& h : ref_mk) refs.push_back(genome_of(h));
  // the references' sketches as stored, entry r = reference r of markers.bin: the entries of index.db in index order, or the
  // .sketch files <dir>/<basename(file_name)>.sketch (src/search.rs:157-166), whose sizes are read when a block of queries
  // first needs them
  const bool consolidated = path_exists(op.db_dir + "/sketches.db") && path_exists(op.db_dir + "/index.db");   // src/sketch_db.rs:142-146
  skdb::SketchInputs rsi;
  if (consolidated) {
    std::vector<skdb::IndexEntry> index;
    int fd = -1;
    if (!skdb::open_db(op.db_dir, index, fd)) return 1;   // the reader of triangle's and dist's database inputs
    rsi.paths.push_back(op.db_dir);
    rsi.db_fd.push_back(fd);
    for (auto& e : index) rsi.entries.push_back(skdb::SketchEntry{0, e.file_name, e.offset, e.length, e.length / 12});
  } else {
    for (size_t r = 0; r < refs.size(); r++) {
      rsi.paths.push_back(op.db_dir + "/" + base_name(refs[r].file_name) + ".sketch");
      rsi.db_fd.push_back(-1);
      rsi.entries.push_back(skdb::SketchEntry{(uint32_t)r, refs[r].file_name, 0, 0, 0});
    }
  }
  sk_sketch_params sp{(uint32_t)dp.c, (uint32_t)dp.k, (uint32_t)dp.marker_c};
  sk_ctx* ctx = nullptr;
  if (sk_ctx_create(op.device, &ctx) != 0) { fprintf(stderr, "ERROR a CUDA device is required (no CPU fallback)\n"); return 1; }
  // ---- queries: FASTA/FASTQ sketched with the DATABASE's parameters (src/search.rs:112-123), or .sketch files.  qfiles holds
  //      them in query order: paths sorted (genomes then follow in (file_name, contig_order) order, as load_inputs gives
  //      them), or .sketch files stably sorted by the name stored inside (src/file_io.rs:715).
  bool queries_are_sketch = true;
  for (auto& q : op.queries) if (q.find(".sketch") == std::string::npos && q.find("markers.bin") == std::string::npos) { queries_are_sketch = false; break; }
  std::vector<std::string> qfiles;
  if (queries_are_sketch) {
    // first pass: the stored names (and the warnings, in argument order); the sketches are decoded again group by group below
    std::vector<std::pair<std::string, std::string>> named;   // (file_name stored inside, path)
    for (auto& q : op.queries) {
      if (q.find("markers.bin") != std::string::npos) continue;
      std::vector<uint8_t> b;
      if (!skdb::read_file(q, b)) { fprintf(stderr, "ERROR Problem reading sketch file %s. Perhaps your file path is wrong? Exiting.\n", q.c_str()); return 1; }
      skdb::DiskParams qp;
      skdb::HostSketch h;
      try { h = skdb::read_blob(b.data(), b.size(), &qp); }
      catch (const std::exception&) { fprintf(stderr, "ERROR %s is not a valid .sketch file or is corrupted.\n", q.c_str()); continue; }
      if (!(qp == dp)) fprintf(stderr, "WARN Query sketch parameters for %s not equal to reference sketch parameters; no ANI calculated\n", q.c_str());
      named.emplace_back(h.file_name, q);
    }
    std::stable_sort(named.begin(), named.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
    if (named.empty()) { fprintf(stderr, "ERROR No query sketches found.\n"); return 1; }
    for (auto& n : named) qfiles.push_back(n.second);
  } else {
    qfiles = op.queries;
    std::sort(qfiles.begin(), qfiles.end());
  }
  sk_map_params mp{};
  mp.screen_val = op.s == 0.0 ? 0.80 : op.s / 100.0;              // SEARCH_ANI_CUTOFF_DEFAULT (src/search.rs:40-49)
  mp.min_aligned_frac = (op.min_af > -1e8 ? op.min_af : -100.0) / 100.0;   // src/parse.rs:444-449; < 0 -> 15 % (src/chain.rs:101-107)
  mp.both_min_aligned_frac = -0.01;
  mp.robust = op.robust; mp.median = op.median;
  mp.rescue_small = 0;
  // use_learned_ani(c, individual_contig_q, false, median) alone picks the model in search (src/search.rs:52-53);
  // --no-learned-ani never reaches map_params_from_sketch there, so the reference ignores the flag: so do we
  mp.learned_ani = dp.c >= 70 && !op.qi && !op.median;
  if (mp.learned_ani) fprintf(stderr, "INFO Learned ANI mode detected. ANI may be adjusted according to a regression model trained on MAGs.\n");
  const bool use_index = (op.queries.size() > 50 || op.qi) && !op.no_marker_index;   // src/parse.rs:436-442
  const int mode = use_index ? 3 : 1;
  // ---- marker sketches of every reference -> one index on ctx, sorted once; every query group is screened against it
  sk_ref_index* idx = nullptr;
  {
    Flat f;
    for (auto& h : ref_mk) f.add(h, false);
    sk_sketch_set* rmk = f.import(ctx, sp);
    CK(ctx, sk_ref_index_create(ctx, rmk, &idx));
    sk_sketch_set_free(rmk);
    uint32_t n_parts = 0; uint64_t bytes = 0;
    sk_ref_index_info(idx, nullptr, &n_parts, &bytes);
    fprintf(stderr, "INFO Reference marker index: %zu references in %u part(s), %.1f MB on GPU %d.\n", refs.size(), n_parts, bytes / 1e6, op.device);
  }
  const search_plan::NameRanks ranks([&] { std::vector<std::string> v; for (auto& g : refs) v.push_back(g.file_name); return v; }());
  std::vector<uint64_t> ref_rank(refs.size());
  for (size_t r = 0; r < refs.size(); r++) ref_rank[r] = ranks.ref(refs[r].file_name);
  const size_t W = op.gpus;
  std::vector<sk_ctx*> ctxs = make_contexts(ctx, op, W);
  const uint64_t group_records = sketch_group_records((1ull << 31) - 1);
  // ---- chaining: the references that passed for at least one of a run of queries ("hits") are loaded ONCE each and their
  //      pairs chained (the reference deserialises a sketch per passing PAIR, src/search.rs:142-166).  The hits are cut into
  //      W contiguous runs balanced by estimated records (marker counts), one per context, and each context reads its run in
  //      groups of < 2^31 - 1 records.  Every round, each context imports its next group (-t threads split over the contexts
  //      read it), then one sk_chain_pairs_multi call chains the round's pairs on all contexts.  chain_run chains the group
  //      queries [q0, q1) (gpairs: the group's screen pairs, qsets: the group on every context) and appends the rows that
  //      pass, with global query ids (the group's first query is q_first), to rows and, with --mappings, to rowmaps.
  std::vector<sk_ani_result> rows;
  std::vector<std::vector<sk_mapping>> rowmaps;
  auto chain_run = [&](size_t q0, size_t q1, size_t q_first, const std::vector<uint64_t>& gpairs, const std::vector<sk_sketch_set*>& qsets, bool maps_on) {
    std::vector<uint64_t> blockp;
    for (uint64_t x : gpairs) if ((uint32_t)x >= q0 && (uint32_t)x < q1) blockp.push_back(x);   // stays sorted by (ref, query)
    std::vector<uint32_t> hits;
    std::vector<size_t> hit_pairs;          // pairs of hits[h]: blockp[hit_pairs[h], hit_pairs[h + 1])
    for (size_t i = 0; i < blockp.size(); i++)
      if (hits.empty() || hits.back() != (uint32_t)(blockp[i] >> 32)) { hits.push_back((uint32_t)(blockp[i] >> 32)); hit_pairs.push_back(i); }
    hit_pairs.push_back(blockp.size());
    std::vector<uint64_t> est(hits.size());
    for (size_t h = 0; h < hits.size(); h++) est[h] = ref_mk[hits[h]].markers.size() + 1;
    const std::vector<size_t> run = split_balanced(est, W);     // context d: hits [run[d], run[d + 1])
    if (!consolidated)
      for (uint32_t r : hits) { struct stat st; rsi.entries[r].length = stat(rsi.paths[r].c_str(), &st) == 0 ? (uint64_t)st.st_size : 0; }
    std::vector<skdb::SketchGroupReader> rd;
    rd.reserve(W);
    for (size_t d = 0; d < W; d++)
      rd.emplace_back(rsi, std::vector<size_t>(hits.begin() + run[d], hits.begin() + run[d + 1]), context_threads(op, d, W), group_records);
    for (;;) {
      std::vector<size_t> lo(W, 0), hi(W, 0);                   // this round: context d imports hits [lo[d], hi[d])
      std::vector<sk_sketch_set*> rsets(W, nullptr);
      std::atomic<bool> load_failed{false};                     // a reference that cannot be loaded ends the run (reported)
      per_context(W, [&](size_t d) {
        skdb::SketchGroup g;
        if (!rd[d].next(g)) { if (rd[d].failed) load_failed = true; return; }
        lo[d] = run[d] + rd[d].first;
        hi[d] = lo[d] + g.size();
        std::vector<uint64_t> rk(g.size());
        for (size_t i = 0; i < g.size(); i++) rk[i] = ref_rank[hits[lo[d] + i]];
        rsets[d] = import_group(ctxs[d], g, sp, [&](size_t i) { return rsi.entries[hits[lo[d] + i]].file_name; });
        if (!rsets[d]) { load_failed = true; return; }
        sk_sketch_set_set_name_ranks(rsets[d], rk.data());
      });
      if (load_failed) return false;
      // the round's refs are numbered run after run: context d's block starts at ref_first[d]
      std::vector<uint32_t> ref_first(W), round_hit;
      std::vector<uint64_t> local;
      for (size_t d = 0; d < W; d++) {
        ref_first[d] = (uint32_t)round_hit.size();
        for (size_t h = lo[d]; h < hi[d]; h++) {
          for (size_t i = hit_pairs[h]; i < hit_pairs[h + 1]; i++) local.push_back(((uint64_t)round_hit.size() << 32) | (uint32_t)blockp[i]);
          round_hit.push_back((uint32_t)h);
        }
      }
      if (round_hit.empty()) break;
      std::vector<sk_ani_result> round(local.size());
      std::vector<uint64_t> off(maps_on ? local.size() + 1 : 0);
      sk_mapping* maps = nullptr;
      if (maps_on) CK(ctx, sk_chain_pairs_multi_mappings(ctxs.data(), (uint32_t)W, rsets.data(), ref_first.data(), qsets.data(), local.data(), local.size(),
                                                         &mp, round.data(), off.data(), &maps));
      else CK(ctx, sk_chain_pairs_multi(ctxs.data(), (uint32_t)W, rsets.data(), ref_first.data(), qsets.data(), local.data(), local.size(), &mp, round.data()));
      for (size_t i = 0; i < round.size(); i++) {
        sk_ani_result& r = round[i];
        if (!(r.ani > 0.5f)) continue;                                                        // src/search.rs:174
        r.ref_id = hits[round_hit[r.ref_id]];
        r.query_id += (uint32_t)q_first;
        rows.push_back(r);
        if (maps_on) rowmaps.emplace_back(maps + off[i], maps + off[i + 1]);
      }
      sk_free(maps);
      for (auto* s : rsets) sk_sketch_set_free(s);
    }
    return true;
  };
  // ---- queries are processed, and their results appended, in blocks of INTERMEDIATE_WRITE_COUNT (src/search.rs:255-279).
  //      A block that spans two query groups keeps its rows until its last query is chained.
  std::vector<Genome> qmeta;                // every query so far, in global order
  DistWriter w(op, refs, qmeta);
  bool opened = false;
  const size_t FL = intermediate_write_count();
  size_t blocks_written = 0;
  auto write_block = [&] {
    // rows of equal ANI print in (ref, query) order, as one context chaining the hits in order produces them
    std::vector<size_t> ord(rows.size());
    std::iota(ord.begin(), ord.end(), 0);
    std::sort(ord.begin(), ord.end(), [&](size_t a, size_t b) { return rows[a].ref_id != rows[b].ref_id ? rows[a].ref_id < rows[b].ref_id : rows[a].query_id < rows[b].query_id; });
    std::vector<sk_ani_result> res(rows.size());
    RowMaps rm;
    for (size_t i = 0; i < ord.size(); i++) {
      res[i] = rows[ord[i]];
      if (w.mappings()) rm.add(rowmaps[ord[i]].data(), rowmaps[ord[i]].size());
    }
    if (blocks_written++) w.more();
    w.write(res, rm);
    rows.clear();
    rowmaps.clear();
  };
  // one query group: its genomes' metadata appended to qmeta, the group as a device set on ctx (which process() owns)
  size_t n_groups = 0;
  auto process = [&](sk_sketch_set* qset, uint64_t bases) {
    const size_t q_end = qmeta.size(), q_first = q_end - sk_sketch_set_n_genomes(qset);
    fprintf(stderr, "INFO Query group %zu: genomes %zu-%zu (%llu bases).\n", ++n_groups, q_first, q_end - 1, (unsigned long long)bases);
    if (!opened) { if (!w.open(sp.k)) return false; opened = true; }
    std::vector<uint64_t> qr(q_end - q_first);
    for (size_t i = 0; i < qr.size(); i++) qr[i] = ranks.query(qmeta[q_first + i].file_name);
    sk_sketch_set_set_name_ranks(qset, qr.data());
    uint64_t* pairs = nullptr; uint64_t np = 0;
    CK(ctx, sk_ref_index_screen(ctx, idx, qset, &mp, mode, &pairs, &np));
    std::vector<uint64_t> gpairs(pairs, pairs + np);
    sk_free(pairs);
    // --gpus N: the group is copied to every context; each run's references are spread over them in chain_run
    std::vector<sk_sketch_set*> qsets(W, qset);
    for (size_t d = 1; d < W; d++) CK(ctxs[d], sk_sketch_set_copy(ctxs[d], qset, &qsets[d]));
    bool ok = true;
    for (size_t s0 = q_first; s0 < q_end && ok;) {
      const size_t block_end = (s0 / FL + 1) * FL, s1 = std::min(block_end, q_end);
      ok = chain_run(s0 - q_first, s1 - q_first, q_first, gpairs, qsets, w.mappings());
      if (ok && s1 == block_end) write_block();
      s0 = s1;
    }
    for (size_t d = 1; d < W; d++) sk_sketch_set_free(qsets[d]);
    sk_sketch_set_free(qset);
    return ok;
  };
  // ---- the queries in read groups of files (file_group_end; a group of .sketch files is one query group, a group of FASTA
  //      files is cut into query groups by search_plan::cut_groups).  The next read group is read and laid out on a host
  //      thread while the current one is sketched, screened and chained: host memory holds at most two groups of queries.
  const uint64_t max_bases = search_group_bases();
  std::vector<size_t> fb{0};
  while (fb.back() < qfiles.size()) fb.push_back(file_group_end(qfiles, fb.back(), max_bases));
  const size_t n_reads = fb.size() - 1;
  struct QueryRead {
    Inputs in;                        // FASTA: the files' genomes, cut into query groups at bounds
    std::vector<size_t> bounds{0};
    Flat flat;                        // .sketch files: one query group
    std::vector<Genome> meta;
    bool failed = false;
  };
  auto load = [&](size_t k, QueryRead* r) {
    const std::vector<std::string> files(qfiles.begin() + fb[k], qfiles.begin() + fb[k + 1]);
    if (!queries_are_sketch) {
      load_inputs(files, op.qi, std::max(op.threads, 1), r->in);
      const auto& gs = r->in.genomes;
      std::vector<uint32_t> gfile(gs.size());
      std::vector<uint64_t> gbases(gs.size());
      for (size_t g = 0; g < gs.size(); g++) {
        gfile[g] = g == 0 ? 0 : gfile[g - 1] + (gs[g].file_name != gs[g - 1].file_name);
        gbases[g] = gs[g].total_len;
      }
      r->bounds = search_plan::cut_groups(gfile, gbases, group_max_files(), max_bases, op.qi);
      return;
    }
    for (auto& q : files) {
      std::vector<uint8_t> b;
      skdb::HostSketch h;
      try {
        if (!skdb::read_file(q, b)) throw std::runtime_error("read");
        h = skdb::read_blob(b.data(), b.size());
      } catch (const std::exception&) {
        fprintf(stderr, "ERROR Problem reading sketch file %s. Exiting.\n", q.c_str());
        r->failed = true;
        return;
      }
      r->flat.add(h, true);
      r->meta.push_back(genome_of(h));
    }
    r->bounds = {0, r->meta.size()};
  };
  QueryRead cur, next;
  std::thread reader;
  int rc = 0;
  if (n_reads) load(0, &cur);
  for (size_t k = 0; k < n_reads && rc == 0; k++) {
    if (k + 1 < n_reads) reader = std::thread(load, k + 1, &next);
    if (cur.failed) rc = 1;
    for (size_t j = 0; j + 1 < cur.bounds.size() && rc == 0; j++) {
      const size_t g0 = cur.bounds[j], g1 = cur.bounds[j + 1];
      sk_sketch_set* qset = nullptr;
      uint64_t bases = 0;
      if (queries_are_sketch) {
        qset = cur.flat.import(ctx, sp);
        for (auto& g : cur.meta) { bases += g.total_len; qmeta.push_back(std::move(g)); }
      } else {
        qset = sketch(ctx, cur.in, sp, g0, g1);
        for (size_t g = g0; g < g1; g++) { bases += cur.in.genomes[g].total_len; qmeta.push_back(std::move(cur.in.genomes[g])); }
      }
      if (!process(qset, bases)) rc = 1;
    }
    cur = QueryRead();                  // the group's sequence is no longer needed
    if (reader.joinable()) reader.join();
    cur = std::move(next);
    next = QueryRead();
  }
  if (reader.joinable()) reader.join();
  if (rc == 0 && qmeta.empty()) { fprintf(stderr, "ERROR No query sequences found.\n"); rc = 1; }
  if (rc == 0 && qmeta.size() > blocks_written * FL) write_block();   // the last, partial block
  sk_ref_index_free(idx);
  for (size_t d = W; d-- > 0;) sk_ctx_destroy(ctxs[d]);
  return rc;
}

// `skani-b200 ingest [-t T] files...`: parse the inputs exactly as triangle / dist / sketch do (no GPU work) and report the
// ingestion rate -- the host-side bound of an end-to-end run on FASTA(.gz) files (SURVEY.md section 8f rank 2)
int run_ingest(Opts& op) {
  if (op.files.empty()) { fprintf(stderr, "ERROR No inputs.\n"); return 1; }
  uint64_t file_bytes = 0;
  for (auto& f : op.files) { struct stat st; if (stat(f.c_str(), &st) == 0) file_bytes += (uint64_t)st.st_size; }
  const auto t0 = std::chrono::steady_clock::now();
  Inputs in;
  load_inputs(op.files, op.individual, std::max(op.threads, 1), in);
  const double dt = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  printf("{\"files\": %zu, \"threads\": %d, \"file_bytes\": %llu, \"bases\": %zu, \"genomes\": %zu, \"seconds\": %.4f, "
         "\"file_MB_per_s\": %.1f, \"bases_MB_per_s\": %.1f}\n", op.files.size(), std::max(op.threads, 1), (unsigned long long)file_bytes,
         in.bases.size(), in.genomes.size(), dt, file_bytes / dt / 1e6, in.bases.size() / dt / 1e6);
  return 0;
}

void usage() {
  fprintf(stderr,
          "skani-b200 (H100 CUDA implementation of skani v0.3.0's ANI hot path)\n"
          "  skani-b200 triangle [fasta ... | -l list] [-i] [-E|--sparse] [-o out] [--full-matrix] [--diagonal] [--distance]\n"
          "  skani-b200 dist [query] [refs ...] [-q ...] [-r ...] [--ql list] [--rl list] [--qi] [--ri] [-n N] [-o out]\n"
          "      triangle and dist also take sketches: .sketch files and sketch databases (folders written by `sketch`, with\n"
          "      index.db and sketches.db), mixed freely; a database stands for all of its sketches\n"
          "  skani-b200 sketch [fasta ... | -l list] -o new_folder [-i] [--separate-sketches]\n"
          "  skani-b200 search -d sketch_folder [query ... | -q ... | --ql list] [--qi] [-n N] [-o out]\n"
          "      queries are read, sketched, screened and chained in groups of whole files (up to 4096 files, about 8 GiB of\n"
          "      sequence; with --qi a larger file is cut between records) against the database's markers indexed once\n"
          "  skani-b200 cluster [fasta | sketch ... | -l list] [-i] [--ani T] [--single-linkage | --linkage average|complete]\n"
          "                    [--dendrogram Z.tsv] [-o out]\n"
          "      the triangle's genomes clustered at ANI >= T %% (default 95, 10 < T <= 100): greedy representatives, longest\n"
          "      genomes first, --single-linkage components, or --linkage average / complete (UPGMA / complete linkage of\n"
          "      100 - ANI, 100 for pairs not printed, cut at 100 - T); one TSV row per genome with its representative and\n"
          "      cluster; --dendrogram writes the linkage matrix (a b height size, heights in percent) that scipy takes\n"
          "  skani-b200 dereplicate [fasta | sketch ... | -l list] [-i] [--ani T] [-o out] [--representatives FILE] [--host-store]\n"
          "      cluster's greedy clusters (same TSV), screening and chaining only genome x representative pairs instead of\n"
          "      the whole triangle; --representatives writes one representative per line in cluster order.  By default one\n"
          "      GPU with the sketches in device memory; --host-store keeps them in host memory and chains in working sets\n"
          "      (inputs beyond device memory, and --gpus N), with the same output\n"
          "  skani-b200 dereplicate [fasta | sketch ... | -l list] --fixed-reps PATH [--fixed-reps PATH ...] [--fixed-reps-list FILE]\n"
          "                        [-i] [--ani T] [-o out] [--representatives FILE] [--host-store] [--gpus N]\n"
          "      adds new genomes (the positional inputs and -l) to representatives that exist already (--fixed-reps, one\n"
          "      FASTA or sketch input each, and --fixed-reps-list, one per line): every fixed genome stays a representative\n"
          "      and keeps cluster ids 0 .. n - 1 (fixed genomes ranked longest first, ties in file-name order), the new\n"
          "      genomes join them or form new clusters by the greedy rule, and no pair of two fixed genomes is screened or\n"
          "      chained.  Each group is FASTA files or .sketch files and databases; a FASTA group is sketched with a sketch\n"
          "      group's parameters (an explicit -c / -k / -m that differs is refused).  An earlier run's --representatives\n"
          "      file passed back as --fixed-reps-list keeps its clusters' ids; with -i that file lists contig names, so pass\n"
          "      the catalogue as files (or a sketch database) instead\n"
          "  skani-b200 tree [fasta | sketch ... | -l list] [-i] [--method nj|average|complete] [-o tree.nwk]\n"
          "      the triangle's genomes as a Newick tree of 100 - ANI (100 for pairs not printed), branch lengths in percent:\n"
          "      neighbour joining (default; unrooted, basal trifurcation) or the average / complete linkage dendrogram\n"
          "      (rooted, a node at half its merge height)\n"
          "  common: -c C -m M -k K -s SCREEN%% --min-af P --both-min-af P --robust --median --no-learned-ani --faster-small\n"
          "          --small-genomes --fast --medium --slow --ci --detailed --short-header --no-marker-index -t THREADS --device D\n"
          "          --gpus N (triangle, dist, search, sketch, cluster, tree, dereplicate --host-store: one context per GPU, devices\n"
          "          D, D+1, ...)\n"
          "  --mappings FILE (triangle, dist, search): where each printed pair aligns, one TSV row per chain interval kept by the\n"
          "          ANI estimate: contigs, 0-based half-open coordinates, strand, anchors, and the identity of the 20 kb chunk it\n"
          "          was chained in.  Pairs, order and orientation are those of the main output (triangle: those of -E).  A few\n"
          "          hundred rows per related 5 Mbp pair: on large triangles the file runs to gigabytes.  Not with inputs beyond\n"
          "          device memory, nor with triangle --gpus N > 1\n");
}

}  // namespace

int main(int argc, char** argv) {
  if (argc < 2) { usage(); return 2; }
  Opts op;
  op.cmd = argv[1];
  if (op.cmd != "triangle" && op.cmd != "dist" && op.cmd != "sketch" && op.cmd != "search" && op.cmd != "ingest" && op.cmd != "cluster" &&
      op.cmd != "tree" && op.cmd != "dereplicate") { usage(); return 2; }
  std::vector<std::string> positional;
  enum { NONE, QS, RS } multi = NONE;
  for (int i = 2; i < argc; i++) {
    std::string a = argv[i];
    auto val = [&]() -> std::string { if (i + 1 >= argc) { fprintf(stderr, "ERROR missing value for %s\n", a.c_str()); exit(2); } return argv[++i]; };
    if (a[0] != '-') {
      if (multi == QS) op.queries.push_back(a); else if (multi == RS) op.refs.push_back(a); else positional.push_back(a);
      continue;
    }
    multi = NONE;
    if (a == "-c") { op.c = (uint32_t)atoi(val().c_str()); op.c_set = true; }
    else if (a == "-m") { op.m = (uint32_t)atof(val().c_str()); op.m_set = true; }
    else if (a == "-k") { op.k = (uint32_t)atoi(val().c_str()); op.k_set = true; }
    else if (a == "-s") op.s = atof(val().c_str());
    else if (a == "-t") op.threads = atoi(val().c_str());
    else if (a == "-o") op.out = val();
    else if (a == "-n") op.n = strtoull(val().c_str(), nullptr, 10);
    else if (a == "-l") { auto v = read_list(val()); op.files.insert(op.files.end(), v.begin(), v.end()); }
    else if (a == "--ql") { auto v = read_list(val()); op.queries.insert(op.queries.end(), v.begin(), v.end()); }
    else if (a == "--rl") { auto v = read_list(val()); op.refs.insert(op.refs.end(), v.begin(), v.end()); }
    else if (a == "-q") multi = QS;
    else if (a == "-r") multi = RS;
    else if (a == "-i") op.individual = true;
    else if (a == "--qi") op.qi = true;
    else if (a == "--ri") op.ri = true;
    else if (a == "-E" || a == "--sparse") op.sparse = true;
    else if (a == "--full-matrix") op.full_matrix = true;
    else if (a == "--diagonal") op.diagonal = true;
    else if (a == "--min-af") op.min_af = atof(val().c_str());
    else if (a == "--both-min-af") op.both_min_af = atof(val().c_str());
    else if (a == "--ci") op.ci = true;
    else if (a == "--detailed") op.detailed = true;
    else if (a == "--short-header") op.short_header = true;
    else if (a == "--distance") op.distance = true;
    else if (a == "--robust") op.robust = true;
    else if (a == "--median") op.median = true;
    else if (a == "--no-learned-ani") op.no_learned = true;
    else if (a == "--gpus") op.gpus = std::max(1, atoi(val().c_str()));
    else if (a == "--faster-small") op.faster_small = true;
    else if (a == "--small-genomes") op.small_genomes = true;
    else if (a == "--fast") op.fast = true;
    else if (a == "--medium") op.medium = true;
    else if (a == "--slow") op.slow = true;
    else if (a == "--no-marker-index") op.no_marker_index = true;
    else if (a == "--device") op.device = atoi(val().c_str());
    else if (a == "-d") op.db_dir = val();
    else if (a == "--separate-sketches") op.separate_sketches = true;
    else if (a == "--ani" && (op.cmd == "cluster" || op.cmd == "dereplicate")) {
      const std::string v = val();
      char* end = nullptr;
      op.cluster_ani = strtod(v.c_str(), &end);
      if (v.empty() || *end || !(op.cluster_ani > 10.0 && op.cluster_ani <= 100.0)) {
        fprintf(stderr, "ERROR --ani %s: the threshold is a percentage in (10, 100] (rows with ANI <= 10 %% are never reported).\n", v.c_str());
        return 2;
      }
    }
    else if (a == "--single-linkage" && (op.cmd == "cluster" || op.cmd == "dereplicate")) op.single_linkage = true;
    else if (a == "--linkage" && (op.cmd == "cluster" || op.cmd == "dereplicate")) op.linkage = val();
    else if (a == "--dendrogram" && (op.cmd == "cluster" || op.cmd == "dereplicate")) op.dendrogram = val();
    else if (a == "--representatives" && op.cmd == "dereplicate") op.representatives = val();
    else if (a == "--host-store" && op.cmd == "dereplicate") op.host_store = true;
    else if (a == "--fixed-reps" && op.cmd == "dereplicate") { op.fixed_reps.push_back(val()); op.fixed_given = true; }
    else if (a == "--fixed-reps-list" && op.cmd == "dereplicate") {
      auto v = read_list(val());
      op.fixed_reps.insert(op.fixed_reps.end(), v.begin(), v.end());
      op.fixed_given = true;
    }
    else if (a == "--method" && op.cmd == "tree") op.tree_method = val();
    else if (a == "--mappings" && (op.cmd == "triangle" || op.cmd == "dist" || op.cmd == "search")) op.mappings = val();
    else if (a == "--keep-refs") {}   // search already loads every passing reference exactly once
    else if (a == "-v" || a == "--debug" || a == "--trace") {}
    else { fprintf(stderr, "ERROR unknown option %s\n", a.c_str()); usage(); return 2; }
  }
  if (op.cmd == "triangle" || op.cmd == "sketch" || op.cmd == "ingest" || op.cmd == "cluster" || op.cmd == "tree" || op.cmd == "dereplicate") {
    op.files.insert(op.files.end(), positional.begin(), positional.end());
    return op.cmd == "triangle" ? run_triangle(op) : op.cmd == "sketch" ? run_sketch(op) : op.cmd == "cluster" ? run_cluster(op)
         : op.cmd == "tree" ? run_tree(op) : op.cmd == "dereplicate" ? run_dereplicate(op) : run_ingest(op);
  }
  if (op.cmd == "search") {
    op.queries.insert(op.queries.end(), positional.begin(), positional.end());
    return run_search(op);
  }
  // dist: first positional is the query, the rest are references (src/cli.rs:115-121)
  if (!positional.empty()) {
    if (op.queries.empty()) { op.queries.push_back(positional[0]); op.refs.insert(op.refs.end(), positional.begin() + 1, positional.end()); }
    else op.refs.insert(op.refs.end(), positional.begin(), positional.end());
  }
  return run_dist(op);
}
