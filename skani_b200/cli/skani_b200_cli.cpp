// skani_b200_cli.cpp -- `skani-b200 triangle|dist|sketch|search`: host driver over the C ABI (include/skani_b200.h).
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
// (src/search.rs:142-166) it screens ALL queries against ALL marker sketches in one GPU pass, loads each reference sketch
// that passed for some query exactly once, imports them to the device in one batch and chains every pair there.
#include <dirent.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>
#include <zlib.h>

#include <algorithm>
#include <chrono>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <thread>
#include <vector>

#include "../../include/skani_b200.h"
#include "fastx.hpp"
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
  bool c_set = false, m_set = false;
  double s = 0.0, min_af = -1e9, both_min_af = -1.0;
  bool individual = false, qi = false, ri = false, sparse = false, full_matrix = false, diagonal = false, ci = false, detailed = false,
       short_header = false, distance = false, robust = false, median = false, no_learned = false, faster_small = false,
       small_genomes = false, fast = false, medium = false, slow = false, no_marker_index = false;
  uint64_t n = 1000000000000ull;
  int threads = 3, device = 0, gpus = 1;
  std::string db_dir;               // search -d
  bool separate_sketches = false;   // sketch --separate-sketches
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

#define CK(ctx, call) do { int rc__ = (call); if (rc__ != 0) { fprintf(stderr, "ERROR %s failed (%d): %s\n", #call, rc__, sk_last_error(ctx)); exit(1); } } while (0)

sk_sketch_set* sketch(sk_ctx* ctx, const Inputs& in, const sk_sketch_params& sp) {
  sk_sketch_set* set = nullptr;
  CK(ctx, sk_sketch_batch(ctx, in.bases.data(), in.contig_off.data(), (uint32_t)in.genome_of_contig.size(), in.genome_of_contig.data(),
                          (uint32_t)in.genomes.size(), &sp, &set));
  return set;
}

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

// inputs given as .sketch files (refs_are_sketch / queries_are_sketch, src/parse.rs:264-275): every file name contains
// ".sketch" or "markers.bin"
bool all_sketch_files(const std::vector<std::string>& files) {
  if (files.empty()) return false;
  for (auto& f : files) if (f.find(".sketch") == std::string::npos && f.find("markers.bin") == std::string::npos) return false;
  return true;
}

// file_io::sketches_from_sketch (src/file_io.rs:680-717): one (SketchParams, Sketch) blob per file, markers.bin skipped,
// result sorted by file name; the sketches' parameters replace the command line's.  Then straight to the device.
sk_sketch_set* load_sketch_files(sk_ctx* ctx, const std::vector<std::string>& files, skdb::DiskParams& dp, std::vector<Genome>& meta) {
  std::vector<skdb::HostSketch> hs;
  for (auto& f : files) {
    if (f.find("markers.bin") != std::string::npos) continue;
    std::vector<uint8_t> b;
    if (!skdb::read_file(f, b)) { fprintf(stderr, "ERROR Problem reading sketch file %s. Perhaps your file path is wrong? Exiting.\n", f.c_str()); exit(1); }
    try { hs.push_back(skdb::read_blob(b.data(), b.size(), &dp)); }
    catch (const std::exception&) {
      fprintf(stderr, "ERROR %s is not a valid .sketch file or is corrupted. Skani v0.3+ is not compatible with older sketch files.\n", f.c_str());
    }
  }
  if (hs.empty()) return nullptr;
  if (dp.use_aa) { fprintf(stderr, "ERROR amino-acid sketches are not supported\n"); exit(1); }
  std::stable_sort(hs.begin(), hs.end(), [](const skdb::HostSketch& x, const skdb::HostSketch& y) { return x.file_name < y.file_name; });
  Flat f;
  for (auto& h : hs) {
    f.add(h, true);
    Genome g; g.file_name = h.file_name; g.contigs = h.contigs; g.contig_order = h.contig_order; g.total_len = h.total_len;
    if (g.contigs.empty()) g.contigs.push_back("");
    meta.push_back(std::move(g));
  }
  sk_sketch_params sp{(uint32_t)dp.c, (uint32_t)dp.k, (uint32_t)dp.marker_c};
  return f.import(ctx, sp);
}

int run_triangle(Opts& op) {
  resolve_presets(op);
  if (op.files.empty()) { fprintf(stderr, "ERROR No reference inputs found.\n"); return 1; }
  Inputs in;
  const bool refs_are_sketch = all_sketch_files(op.files);
  if (!refs_are_sketch) {
    load_inputs(op.files, op.individual, std::max(op.threads, 1), in);
    if (in.genomes.empty()) { fprintf(stderr, "ERROR No genomes/sketches found.\n"); return 1; }   // src/triangle.rs:46-49
  }
  sk_ctx* ctx = nullptr;
  if (sk_ctx_create(op.device, &ctx) != 0) { fprintf(stderr, "ERROR a CUDA device is required (no CPU fallback)\n"); return 1; }
  sk_sketch_params sp{op.c, op.k, op.m};
  sk_sketch_set* loaded = nullptr;
  if (refs_are_sketch) {      // src/triangle.rs:16-24
    fprintf(stderr, "INFO Sketches detected.\n");
    skdb::DiskParams dp;
    loaded = load_sketch_files(ctx, op.files, dp, in.genomes);
    if (!loaded) { fprintf(stderr, "ERROR No genomes/sketches found.\n"); return 1; }
    if (dp.c != op.c || dp.marker_c != op.m)
      fprintf(stderr, "WARN Input parameter c = %u, m = %u is not equal to the sketch parameter c = %llu,m = %llu. Using sketch parameters.\n", op.c, op.m,
              (unsigned long long)dp.c, (unsigned long long)dp.marker_c);
    sp = sk_sketch_params{(uint32_t)dp.c, (uint32_t)dp.k, (uint32_t)dp.marker_c};
  }
  if (in.genomes.size() > 500 && !op.sparse) fprintf(stderr, "WARN > 500 genomes detected. The output matrix will be large. Consider using -E or --sparse for a tsv output instead.\n");
  sk_map_params mp{};
  mp.screen_val = op.s / 100.0;
  mp.min_aligned_frac = (op.min_af > -1e8 ? op.min_af : 15.0) / 100.0;
  mp.both_min_aligned_frac = op.both_min_af / 100.0;
  mp.robust = op.robust; mp.median = op.median;
  mp.rescue_small = !op.faster_small && !op.small_genomes;
  mp.learned_ani = !op.no_learned && op.c >= 70 && !op.individual && !op.median;   // regression::use_learned_ani (src/regression.rs:8-10)
  if (mp.learned_ani) fprintf(stderr, "INFO Learned ANI mode detected. ANI may be adjusted according to a regression model trained on MAGs.\n");
  // file-name order for the switch_qr tie-break (src/chain.rs:19-21): with -i all records of a file share its name
  std::vector<uint64_t> ranks(in.genomes.size());
  {
    uint64_t rank = 0;
    for (size_t i = 0; i < in.genomes.size(); i++) {
      if (i && in.genomes[i].file_name != in.genomes[i - 1].file_name) rank++;
      ranks[i] = rank;
    }
  }
  std::vector<sk_ani_result> res;
  sk_sketch_set* set = nullptr;
  if (op.gpus > 1 && !loaded) {
    // --gpus N: one context per GPU, genome blocks + marker exchange + cross-block slices (sk_triangle_multi).  With fewer
    // physical devices than N the contexts share devices (same code path; the exchange then stays on the device).
    const int ndev = sk_device_count();
    if (ndev < op.gpus) fprintf(stderr, "WARN --gpus %d but %d CUDA device(s) visible: contexts share devices.\n", op.gpus, ndev);
    std::vector<sk_ctx*> ctxs(1, ctx);
    for (int d = 1; d < op.gpus; d++) {
      sk_ctx* c = nullptr;
      if (sk_ctx_create((op.device + d) % std::max(ndev, 1), &c) != 0) { fprintf(stderr, "ERROR cannot create a context on GPU %d\n", (op.device + d) % std::max(ndev, 1)); return 1; }
      ctxs.push_back(c);
    }
    sk_ani_result* r = nullptr; uint64_t nr = 0;
    CK(ctx, sk_triangle_multi(ctxs.data(), (uint32_t)ctxs.size(), in.bases.data(), in.contig_off.data(), (uint32_t)in.genome_of_contig.size(),
                              in.genome_of_contig.data(), (uint32_t)in.genomes.size(), &sp, &mp, ranks.data(), &r, &nr, nullptr));
    res.assign(r, r + nr);
    sk_free(r);
    std::sort(res.begin(), res.end(), [](const sk_ani_result& a, const sk_ani_result& b) { return a.ref_id != b.ref_id ? a.ref_id < b.ref_id : a.query_id < b.query_id; });
    for (size_t d = 1; d < ctxs.size(); d++) sk_ctx_destroy(ctxs[d]);
  } else {
    set = loaded ? loaded : sketch(ctx, in, sp);
    sk_sketch_set_set_name_ranks(set, ranks.data());
    uint64_t* pairs = nullptr; uint64_t np = 0;
    CK(ctx, sk_screen_triangle(ctx, set, &mp, &pairs, &np));
    if (op.sparse) {
      // sparse output: rows are chained and APPENDED in blocks of INTERMEDIATE_WRITE_COUNT rows (src/triangle.rs:113-138),
      // so a long run leaves its finished rows on disk and holds at most one block of results in memory
      FILE* o = op.out.empty() ? stdout : fopen(op.out.c_str(), "w");
      if (!o) { fprintf(stderr, "ERROR cannot open %s\n", op.out.c_str()); return 1; }
      write_header(o, op.ci, op.detailed);
      if (op.diagonal) for (auto& g : in.genomes) write_perfect(o, g, op);
      const size_t FL = intermediate_write_count(), Nrows = in.genomes.size();
      uint64_t p0 = 0;
      for (size_t r0 = 0; r0 < Nrows; r0 += FL) {
        uint64_t p1 = p0;
        while (p1 < np && (uint32_t)(pairs[p1] >> 32) < r0 + FL) p1++;      // pairs are sorted by (i, j)
        res.resize(p1 - p0);
        CK(ctx, sk_chain_pairs(ctx, set, set, pairs + p0, p1 - p0, &mp, res.data()));
        for (auto& r : res) if (r.ani > 0.1f) write_row(o, r, in.genomes[r.ref_id], in.genomes[r.query_id], op);
        fflush(o);
        if (r0 + FL < Nrows) fprintf(stderr, "INFO Writing results for %zu query sequences.\n", FL);
        p0 = p1;
      }
      sk_free(pairs);
      if (o != stdout) fclose(o);
      sk_sketch_set_free(set);
      sk_ctx_destroy(ctx);
      return 0;
    }
    res.resize(np);
    CK(ctx, sk_chain_pairs(ctx, set, set, pairs, np, &mp, res.data()));
    sk_free(pairs);
  }
  const size_t N = in.genomes.size();
  FILE* o = op.out.empty() ? stdout : fopen(op.out.c_str(), "w");
  if (!o) { fprintf(stderr, "ERROR cannot open %s\n", op.out.c_str()); return 1; }
  if (op.sparse) {   // write_sparse_matrix (src/file_io.rs:541-606); rows emitted in (i, j) order (the reference's order is arbitrary)
    write_header(o, op.ci, op.detailed);
    if (op.diagonal) for (auto& g : in.genomes) write_perfect(o, g, op);
    for (auto& r : res) if (r.ani > 0.1f) write_row(o, r, in.genomes[r.ref_id], in.genomes[r.query_id], op);
  } else {           // write_phyllip_matrix (src/file_io.rs:364-539)
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
  if (set) sk_sketch_set_free(set);
  sk_ctx_destroy(ctx);
  return 0;
}

int run_dist(Opts& op) {
  resolve_presets(op);
  if (op.refs.empty() || op.queries.empty()) { fprintf(stderr, "ERROR No reference sketches/genomes or query sketches/genomes found.\n"); return 1; }
  Inputs rin, qin;
  const bool refs_are_sketch = all_sketch_files(op.refs), queries_are_sketch = all_sketch_files(op.queries);
  sk_ctx* ctx = nullptr;
  if (sk_ctx_create(op.device, &ctx) != 0) { fprintf(stderr, "ERROR a CUDA device is required (no CPU fallback)\n"); return 1; }
  sk_sketch_params sp{op.c, op.k, op.m};
  sk_sketch_set *rset = nullptr, *qset = nullptr;
  // .sketch inputs carry their own parameters, which then also apply to FASTA inputs on the other side (src/dist.rs:17-50)
  if (refs_are_sketch) {
    fprintf(stderr, "INFO Sketches detected.\n");
    skdb::DiskParams dp;
    rset = load_sketch_files(ctx, op.refs, dp, rin.genomes);
    if (rset) {
      if (dp.c != sp.c || dp.k != sp.k || dp.marker_c != sp.marker_c)
        fprintf(stderr, "WARN Parameters from .sketch files not equal to the input parameters. Using parameters from .sketch files.\n");
      sp = sk_sketch_params{(uint32_t)dp.c, (uint32_t)dp.k, (uint32_t)dp.marker_c};
    }
  }
  if (queries_are_sketch) {
    skdb::DiskParams dp;
    qset = load_sketch_files(ctx, op.queries, dp, qin.genomes);
    if (qset && (dp.c != sp.c || dp.k != sp.k || dp.marker_c != sp.marker_c)) {
      if (refs_are_sketch) { fprintf(stderr, "ERROR Query sketch parameters were not equal to reference sketch parameters. Exiting.\n"); return 1; }
      fprintf(stderr, "WARN Parameters from .sketch files not equal to the input parameters. Using parameters from .sketch files.\n");
      sp = sk_sketch_params{(uint32_t)dp.c, (uint32_t)dp.k, (uint32_t)dp.marker_c};
    }
  }
  if (!refs_are_sketch) load_inputs(op.refs, op.ri, std::max(op.threads, 1), rin);
  if (!queries_are_sketch) load_inputs(op.queries, op.qi, std::max(op.threads, 1), qin);
  if (rin.genomes.empty() || qin.genomes.empty()) { fprintf(stderr, "ERROR No reference sketches/genomes or query sketches/genomes found.\n"); return 1; }
  sk_map_params mp{};
  mp.screen_val = op.s / 100.0;
  mp.min_aligned_frac = (op.min_af > -1e8 ? op.min_af : 15.0) / 100.0;
  mp.both_min_aligned_frac = op.both_min_af / 100.0;
  mp.robust = op.robust; mp.median = op.median;
  mp.rescue_small = !op.faster_small && !op.small_genomes;
  mp.learned_ani = !op.no_learned && op.c >= 70 && !op.qi && !op.ri && !op.median;
  if (mp.learned_ani) fprintf(stderr, "INFO Learned ANI mode detected. ANI may be adjusted according to a regression model trained on MAGs.\n");
  const bool use_index = (op.queries.size() > 50 || op.qi) && !op.no_marker_index;   // FULL_INDEX_THRESH (src/parse.rs:750)
  if (!rset) rset = sketch(ctx, rin, sp);
  if (!qset) qset = sketch(ctx, qin, sp);
  // file-name order for the switch_qr tie-break (src/chain.rs:19-21): rank all names together
  {
    std::vector<std::pair<std::string, std::pair<int, size_t>>> names;
    for (size_t i = 0; i < rin.genomes.size(); i++) names.push_back({rin.genomes[i].file_name, {0, i}});
    for (size_t i = 0; i < qin.genomes.size(); i++) names.push_back({qin.genomes[i].file_name, {1, i}});
    std::sort(names.begin(), names.end(), [](auto& a, auto& b) { return a.first < b.first; });
    std::vector<uint64_t> rr(rin.genomes.size()), qr(qin.genomes.size());
    uint64_t rank = 0;
    for (size_t i = 0; i < names.size(); i++) {
      if (i && names[i].first != names[i - 1].first) rank++;
      (names[i].second.first ? qr : rr)[names[i].second.second] = rank;
    }
    sk_sketch_set_set_name_ranks(rset, rr.data());
    sk_sketch_set_set_name_ranks(qset, qr.data());
  }
  uint64_t* pairs = nullptr; uint64_t np = 0;
  CK(ctx, sk_screen_query_ref(ctx, rset, qset, &mp, use_index ? 2 : 0, &pairs, &np));
  // queries are processed, and their results appended, in blocks of INTERMEDIATE_WRITE_COUNT (src/dist.rs:151-175)
  std::vector<uint64_t> byq(pairs, pairs + np);
  sk_free(pairs);
  std::sort(byq.begin(), byq.end(), [](uint64_t a, uint64_t b) { return (uint32_t)a != (uint32_t)b ? (uint32_t)a < (uint32_t)b : a < b; });
  FILE* o = op.out.empty() ? stdout : fopen(op.out.c_str(), "w");
  if (!o) { fprintf(stderr, "ERROR cannot open %s\n", op.out.c_str()); return 1; }
  write_header(o, op.ci, op.detailed);
  const size_t FL = intermediate_write_count(), NQ = qin.genomes.size();
  size_t p0 = 0;
  std::vector<sk_ani_result> res;
  for (size_t q0 = 0; q0 < NQ; q0 += FL) {
    size_t p1 = p0;
    while (p1 < byq.size() && (uint32_t)byq[p1] < q0 + FL) p1++;
    res.resize(p1 - p0);
    CK(ctx, sk_chain_pairs(ctx, rset, qset, byq.data() + p0, p1 - p0, &mp, res.data()));
    // write_query_ref_list (src/file_io.rs:608-678): group by the query's first contig name, sort each group by ANI desc, top n
    std::map<std::string, std::vector<const sk_ani_result*>> groups;
    for (auto& r : res) if (r.ani > 0.1f) groups[qin.genomes[r.query_id].contigs[0]].push_back(&r);
    for (auto& kv : groups) {
      auto v = kv.second;
      std::stable_sort(v.begin(), v.end(), [](const sk_ani_result* a, const sk_ani_result* b) { return a->ani > b->ani; });
      for (size_t i = 0; i < v.size() && i < op.n; i++) write_row(o, *v[i], rin.genomes[v[i]->ref_id], qin.genomes[v[i]->query_id], op);
    }
    fflush(o);
    if (q0 + FL < NQ) fprintf(stderr, "INFO Writing results for %zu query sequences.\n", FL);
    p0 = p1;
  }
  if (o != stdout) fclose(o);
  sk_sketch_set_free(rset); sk_sketch_set_free(qset);
  sk_ctx_destroy(ctx);
  return 0;
}

// ---- sketch / search (src/sketch.rs, src/search.rs) --------------------------------------------------------------
std::string base_name(const std::string& p) { size_t i = p.find_last_of('/'); return i == std::string::npos ? p : p.substr(i + 1); }
bool path_exists(const std::string& p) { struct stat st; return stat(p.c_str(), &st) == 0; }
void make_dirs(const std::string& p) {
  for (size_t i = 1; i <= p.size(); i++)
    if (i == p.size() || p[i] == '/') mkdir(p.substr(0, i).c_str(), 0777);
}

// device sketch g -> the host form the database writer takes (records grouped by k-mer, src/types.rs:253-277)
skdb::HostSketch export_sketch(sk_ctx* ctx, const sk_sketch_set* set, uint32_t g, const Genome& meta, const sk_sketch_params& sp) {
  uint64_t nr = 0, nk = 0, nm = 0, nc = 0, tl = 0;
  CK(ctx, sk_sketch_set_genome_info(set, g, &nr, &nk, &nm, &nc, &tl));
  skdb::HostSketch h;
  h.file_name = meta.file_name; h.contigs = meta.contigs; h.contig_order = meta.contig_order; h.total_len = tl;
  h.kmer.resize(nr); h.pos.resize(nr); h.cc.resize(nr); h.markers.resize(nm); h.contig_lengths.resize(nc);
  CK(ctx, sk_sketch_set_export(set, g, h.kmer.data(), h.pos.data(), h.cc.data(), h.markers.data(), h.contig_lengths.data()));
  h.c = sp.c; h.k = sp.k; h.marker_c = sp.c;     // the sketch's marker_c field holds c (Sketch::new, src/types.rs:347)
  return h;
}

int run_sketch(Opts& op) {
  resolve_presets(op);
  if (op.files.empty()) { fprintf(stderr, "ERROR No reference inputs found.\n"); return 1; }
  if (op.out.empty()) { fprintf(stderr, "ERROR an output folder is required (-o)\n"); return 1; }
  if (path_exists(op.out)) { fprintf(stderr, "ERROR Output directory exists; output directory must not be an existing directory. Exiting.\n"); return 1; }   // src/sketch.rs:19-22
  make_dirs(op.out);
  if (op.separate_sketches && op.individual)
    fprintf(stderr, "WARN --separate-sketches combined with -i (individual contigs) is NOT compatible with `skani search`.\n");
  sk_ctx* ctx = nullptr;
  if (sk_ctx_create(op.device, &ctx) != 0) { fprintf(stderr, "ERROR a CUDA device is required (no CPU fallback)\n"); return 1; }
  sk_sketch_params sp{op.c, op.k, op.m};
  skdb::DiskParams dp;
  dp.c = op.c; dp.k = op.k; dp.marker_c = op.m;
  skdb::DbWriter w;
  std::vector<skdb::HostSketch> sep_markers;
  if (!op.separate_sketches && !w.open(op.out, dp)) { fprintf(stderr, "ERROR Failed to create consolidated database writer\n"); return 1; }
  std::vector<std::string> files = op.files;
  std::sort(files.begin(), files.end());
  size_t total = 0;
  // files go through the GPU in groups (bounds the host copy of the sequences); database order = (file_name, contig_order)
  for (size_t f0 = 0; f0 < files.size();) {
    size_t f1 = f0;
    uint64_t bytes = 0;
    while (f1 < files.size() && (f1 == f0 || (f1 - f0 < 4096 && bytes < (8ull << 30)))) {
      struct stat st;
      bytes += stat(files[f1].c_str(), &st) == 0 ? (uint64_t)st.st_size * 4 : 0;   // gz inflates ~4x
      f1++;
    }
    Inputs in;
    load_inputs(std::vector<std::string>(files.begin() + f0, files.begin() + f1), op.individual, std::max(op.threads, 1), in);
    f0 = f1;
    if (in.genomes.empty()) continue;
    sk_sketch_set* set = sketch(ctx, in, sp);
    size_t j_in_file = 0;
    for (size_t g = 0; g < in.genomes.size(); g++) {
      skdb::HostSketch h = export_sketch(ctx, set, (uint32_t)g, in.genomes[g], sp);
      j_in_file = (g && in.genomes[g].file_name == in.genomes[g - 1].file_name) ? j_in_file + 1 : 0;
      if (op.separate_sketches) {      // src/sketch.rs:38-101: <basename>.sketch, or <j>_<basename>.sketch with -i
        std::string name = op.out + "/" + (op.individual ? std::to_string(j_in_file) + "_" : std::string()) + base_name(h.file_name) + ".sketch";
        skdb::Out o;
        skdb::put_params(o, dp);
        skdb::put_sketch(o, h);
        if (!skdb::write_file(name, o.b)) { fprintf(stderr, "ERROR cannot write %s\n", name.c_str()); return 1; }
        sep_markers.push_back(skdb::markers_only(h));
      } else if (!w.add(h)) { fprintf(stderr, "ERROR Failed to add sketch to database\n"); return 1; }
      if (++total % 100 == 0) fprintf(stderr, "INFO %zu sequences sketched.\n", total);
    }
    sk_sketch_set_free(set);
  }
  if (op.separate_sketches) {
    skdb::Out mk;
    skdb::put_params(mk, dp);
    mk.u64(sep_markers.size());
    for (auto& m : sep_markers) skdb::put_sketch(mk, m);
    if (!skdb::write_file(op.out + "/markers.bin", mk.b)) { fprintf(stderr, "ERROR cannot write markers.bin\n"); return 1; }
  } else if (!w.finalize()) { fprintf(stderr, "ERROR Failed to finalize consolidated database\n"); return 1; }
  fprintf(stderr, "INFO Successfully wrote %zu sketches to %s\n", total, op.out.c_str());
  sk_ctx_destroy(ctx);
  return 0;
}

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
  const bool consolidated = path_exists(op.db_dir + "/sketches.db") && path_exists(op.db_dir + "/index.db");   // src/sketch_db.rs:142-146
  std::vector<skdb::IndexEntry> index;
  int db_fd = -1;
  if (consolidated) {
    try { skdb::read_index_db(op.db_dir + "/index.db", index); }
    catch (const std::exception& e) { fprintf(stderr, "ERROR Failed to load consolidated database: %s\n", e.what()); return 1; }
    if (index.size() != ref_mk.size()) { fprintf(stderr, "ERROR index.db and markers.bin disagree on the number of sketches\n"); return 1; }
    db_fd = open((op.db_dir + "/sketches.db").c_str(), O_RDONLY);
    if (db_fd < 0) { fprintf(stderr, "ERROR Failed to load consolidated database\n"); return 1; }
  }
  sk_sketch_params sp{(uint32_t)dp.c, (uint32_t)dp.k, (uint32_t)dp.marker_c};
  sk_ctx* ctx = nullptr;
  if (sk_ctx_create(op.device, &ctx) != 0) { fprintf(stderr, "ERROR a CUDA device is required (no CPU fallback)\n"); return 1; }
  // ---- queries: FASTA/FASTQ sketched with the DATABASE's parameters (src/search.rs:112-123), or .sketch files
  bool queries_are_sketch = true;
  for (auto& q : op.queries) if (q.find(".sketch") == std::string::npos && q.find("markers.bin") == std::string::npos) { queries_are_sketch = false; break; }
  std::vector<Genome> qmeta;
  sk_sketch_set* qset = nullptr;
  if (queries_are_sketch) {
    std::vector<skdb::HostSketch> qs;
    for (auto& q : op.queries) {
      if (q.find("markers.bin") != std::string::npos) continue;
      std::vector<uint8_t> b;
      if (!skdb::read_file(q, b)) { fprintf(stderr, "ERROR Problem reading sketch file %s. Perhaps your file path is wrong? Exiting.\n", q.c_str()); return 1; }
      skdb::DiskParams qp;
      try { qs.push_back(skdb::read_blob(b.data(), b.size(), &qp)); }
      catch (const std::exception&) { fprintf(stderr, "ERROR %s is not a valid .sketch file or is corrupted.\n", q.c_str()); continue; }
      if (!(qp == dp)) fprintf(stderr, "WARN Query sketch parameters for %s not equal to reference sketch parameters; no ANI calculated\n", q.c_str());
    }
    std::stable_sort(qs.begin(), qs.end(), [](const skdb::HostSketch& a, const skdb::HostSketch& b) { return a.file_name < b.file_name; });   // src/file_io.rs:715
    if (qs.empty()) { fprintf(stderr, "ERROR No query sketches found.\n"); return 1; }
    Flat f;
    for (auto& h : qs) {
      f.add(h, true);
      Genome g; g.file_name = h.file_name; g.contigs = h.contigs; g.contig_order = h.contig_order; g.total_len = h.total_len;
      if (g.contigs.empty()) g.contigs.push_back("");   // a .sketch without contig names still prints (as load_sketch_files does)
      qmeta.push_back(std::move(g));
    }
    qset = f.import(ctx, sp);
  } else {
    Inputs qin;
    load_inputs(op.queries, op.qi, std::max(op.threads, 1), qin);
    if (qin.genomes.empty()) { fprintf(stderr, "ERROR No query sequences found.\n"); return 1; }
    qset = sketch(ctx, qin, sp);
    qmeta = std::move(qin.genomes);
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
  // ---- marker sketches of every reference -> device, one screen of all queries against all references
  sk_sketch_set* rmk = nullptr;
  {
    Flat f;
    for (auto& h : ref_mk) f.add(h, false);
    rmk = f.import(ctx, sp);
  }
  uint64_t* pairs = nullptr; uint64_t np = 0;
  CK(ctx, sk_screen_query_ref(ctx, rmk, qset, &mp, use_index ? 3 : 1, &pairs, &np));
  sk_sketch_set_free(rmk);
  // file-name order for the switch_qr tie-break (src/chain.rs:19-21): rank all names together
  std::vector<uint64_t> rrank(ref_mk.size()), qrank(qmeta.size());
  {
    std::vector<std::pair<const std::string*, std::pair<int, size_t>>> names;
    for (size_t i = 0; i < ref_mk.size(); i++) names.push_back({&ref_mk[i].file_name, {0, i}});
    for (size_t i = 0; i < qmeta.size(); i++) names.push_back({&qmeta[i].file_name, {1, i}});
    std::sort(names.begin(), names.end(), [](auto& a, auto& b) { return *a.first < *b.first; });
    uint64_t rank = 0;
    for (size_t i = 0; i < names.size(); i++) {
      if (i && *names[i].first != *names[i - 1].first) rank++;
      (names[i].second.first ? qrank : rrank)[names[i].second.second] = rank;
    }
    sk_sketch_set_set_name_ranks(qset, qrank.data());
  }
  // ---- queries are processed, and their results appended, in blocks of INTERMEDIATE_WRITE_COUNT (src/search.rs:255-279).
  //      Inside a block: the references that passed for at least one of its queries are loaded ONCE each, imported in
  //      batches, and their pairs chained (the reference deserialises a sketch per passing PAIR, src/search.rs:142-166)
  FILE* o = op.out.empty() ? stdout : fopen(op.out.c_str(), "w");
  if (!o) { fprintf(stderr, "ERROR cannot open %s\n", op.out.c_str()); return 1; }
  write_header(o, op.ci, op.detailed);
  std::vector<uint64_t> all_pairs(pairs, pairs + np);
  sk_free(pairs);
  const size_t FL = intermediate_write_count(), NQ = qmeta.size();
  for (size_t q0 = 0; q0 < NQ; q0 += FL) {
  std::vector<uint64_t> blockp;
  for (uint64_t x : all_pairs) if ((uint32_t)x >= q0 && (uint32_t)x < q0 + FL) blockp.push_back(x);   // stays sorted by (ref, query)
  const uint64_t* pairs = blockp.data();
  const uint64_t np = blockp.size();
  std::vector<uint32_t> hits;
  for (uint64_t i = 0; i < np; i++) hits.push_back((uint32_t)(pairs[i] >> 32));   // pairs are sorted by (ref, query)
  hits.erase(std::unique(hits.begin(), hits.end()), hits.end());
  std::vector<sk_ani_result> kept;
  size_t pi = 0;
  for (size_t h0 = 0; h0 < hits.size();) {
    size_t h1 = h0;
    std::vector<skdb::HostSketch> loaded;
    uint64_t recs = 0;
    while (h1 < hits.size() && h1 - h0 < 60000 && recs < (1ull << 30)) h1++, recs += 45000;   // provisional bound, refined below
    loaded.resize(h1 - h0);
    std::vector<int> ok(h1 - h0, 1);
    {
      const int T = std::max(op.threads, 1);
      std::vector<std::thread> pool;
      for (int t = 0; t < T; t++) pool.emplace_back([&, t] {
        for (size_t i = h0 + t; i < h1; i += T) {
          const uint32_t r = hits[i];
          std::vector<uint8_t> b;
          bool good;
          if (consolidated) {
            b.resize(index[r].length);
            good = pread(db_fd, b.data(), b.size(), (off_t)index[r].offset) == (ssize_t)b.size();
          } else {                     // <dir>/<basename(file_name)>.sketch (src/search.rs:157-166)
            good = skdb::read_file(op.db_dir + "/" + base_name(ref_mk[r].file_name) + ".sketch", b);
          }
          try { if (good) loaded[i - h0] = skdb::read_blob(b.data(), b.size()); }
          catch (const std::exception&) { good = false; }
          if (!good) { ok[i - h0] = 0; fprintf(stderr, "ERROR Failed to load sketch %s\n", ref_mk[r].file_name.c_str()); }
        }
      });
      for (auto& th : pool) th.join();
    }
    // keep the batch under 2^31 records: shrink it if the real sizes exceed the estimate
    uint64_t real = 0;
    size_t cut = h0;
    while (cut < h1 && real + loaded[cut - h0].kmer.size() < (1ull << 31) - 1) real += loaded[cut - h0].kmer.size(), cut++;
    if (cut == h0) { fprintf(stderr, "ERROR reference sketch too large\n"); return 1; }
    h1 = cut;
    Flat f;
    std::vector<uint64_t> ranks;
    for (size_t i = h0; i < h1; i++) {
      if (!ok[i - h0]) loaded[i - h0] = skdb::HostSketch();     // unreadable reference: chains to "no anchors", dropped below
      f.add(loaded[i - h0], true);
      ranks.push_back(rrank[hits[i]]);
    }
    sk_sketch_set* rset = f.import(ctx, sp);
    sk_sketch_set_set_name_ranks(rset, ranks.data());
    std::vector<uint64_t> local;
    while (pi < np && (uint32_t)(pairs[pi] >> 32) <= hits[h1 - 1]) {
      const uint32_t r = (uint32_t)(pairs[pi] >> 32);
      const size_t li = std::lower_bound(hits.begin() + h0, hits.begin() + h1, r) - (hits.begin() + h0);
      local.push_back(((uint64_t)li << 32) | (uint32_t)pairs[pi]);
      pi++;
    }
    std::vector<sk_ani_result> res(local.size());
    CK(ctx, sk_chain_pairs(ctx, rset, qset, local.data(), local.size(), &mp, res.data()));
    for (auto& r : res) if (r.ani > 0.5f) { r.ref_id = hits[h0 + r.ref_id]; kept.push_back(r); }   // src/search.rs:174
    sk_sketch_set_free(rset);
    h0 = h1;
  }
  // write_query_ref_list (src/file_io.rs:608-678): group by the query's first contig name, ANI descending, top n
  std::map<std::string, std::vector<const sk_ani_result*>> groups;
  for (auto& r : kept) groups[qmeta[r.query_id].contigs[0]].push_back(&r);
  for (auto& kv : groups) {
    auto v = kv.second;
    std::stable_sort(v.begin(), v.end(), [](const sk_ani_result* a, const sk_ani_result* b) { return a->ani > b->ani; });
    for (size_t i = 0; i < v.size() && i < op.n; i++) {
      Genome ref; ref.file_name = ref_mk[v[i]->ref_id].file_name; ref.contigs = ref_mk[v[i]->ref_id].contigs;
      if (ref.contigs.empty()) ref.contigs.push_back("");
      write_row(o, *v[i], ref, qmeta[v[i]->query_id], op);
    }
  }
  fflush(o);
  if (q0 + FL < NQ) fprintf(stderr, "INFO Writing results for %zu query sequences.\n", FL);
  }
  if (db_fd >= 0) close(db_fd);
  if (o != stdout) fclose(o);
  sk_sketch_set_free(qset);
  sk_ctx_destroy(ctx);
  return 0;
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
          "  skani-b200 sketch [fasta ... | -l list] -o new_folder [-i] [--separate-sketches]\n"
          "  skani-b200 search -d sketch_folder [query ... | -q ... | --ql list] [--qi] [-n N] [-o out]\n"
          "  common: -c C -m M -k K -s SCREEN%% --min-af P --both-min-af P --robust --median --no-learned-ani --faster-small\n"
          "          --small-genomes --fast --medium --slow --ci --detailed --short-header --no-marker-index -t THREADS --device D\n");
}

}  // namespace

int main(int argc, char** argv) {
  if (argc < 2) { usage(); return 2; }
  Opts op;
  op.cmd = argv[1];
  if (op.cmd != "triangle" && op.cmd != "dist" && op.cmd != "sketch" && op.cmd != "search" && op.cmd != "ingest") { usage(); return 2; }
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
    else if (a == "-k") op.k = (uint32_t)atoi(val().c_str());
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
    else if (a == "--keep-refs") {}   // search already loads every passing reference exactly once
    else if (a == "-v" || a == "--debug" || a == "--trace") {}
    else { fprintf(stderr, "ERROR unknown option %s\n", a.c_str()); usage(); return 2; }
  }
  if (op.cmd == "triangle" || op.cmd == "sketch" || op.cmd == "ingest") {
    op.files.insert(op.files.end(), positional.begin(), positional.end());
    return op.cmd == "triangle" ? run_triangle(op) : op.cmd == "sketch" ? run_sketch(op) : run_ingest(op);
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
