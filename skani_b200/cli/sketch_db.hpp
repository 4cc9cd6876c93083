// sketch_db.hpp -- skani v0.3.0 on-disk sketch formats (host only; no CUDA).
//
// Byte layout = bincode 1.3 with default options (little endian, fixed-width integers, usize -> u64, u64 length
// prefixes, Option tag u8, bool u8, String = length + UTF-8 bytes) applied to the reference's serde structs:
//   (SketchParams, Sketch)                each `.sketch` file (src/sketch.rs:85) and each entry of `sketches.db`
//                                         (src/sketch_db.rs:45-47); SketchParams src/params.rs:137-146, Sketch
//                                         src/types.rs:253-277, SeedPosition src/types.rs:125-128
//   Vec<IndexEntry{file_name, offset, length}>   `index.db` (src/sketch_db.rs:10-15, 72-77)
//   (SketchParams, Vec<Sketch>)           `markers.bin`, sketches reduced by Sketch::get_markers_only
//                                         (src/types.rs:322-340, src/sketch.rs:141-146)
// The k-mer map is a Rust HashMap, so entry order in a file is arbitrary and carries no meaning; this writer emits
// ascending k-mers.  Map value (src/types.rs:207-244): csrc/sketch_value.cuh, shared with the device expansion of
// sk_sketch_set_import_blobs.
#pragma once
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "../csrc/sketch_value.cuh"

namespace skdb {

struct DiskParams {            // SketchParams, src/params.rs:137-146
  uint64_t c = 125, k = 15, marker_c = 1000;
  bool use_syncs = false, use_aa = false;
  uint64_t orf_size = 30;      // ORF_SIZE src/params.rs:32
  bool operator==(const DiskParams& o) const {
    return c == o.c && k == o.k && marker_c == o.marker_c && use_syncs == o.use_syncs && use_aa == o.use_aa && orf_size == o.orf_size;
  }
};

struct HostSketch {            // Sketch, src/types.rs:253-277 (records flattened: one entry per seed position)
  std::string file_name;
  bool has_seeds = true;       // kmer_seeds_k is Some(..) (false for get_markers_only)
  std::vector<uint32_t> kmer, pos, cc;      // cc = contig_index << 1 | canonical
  std::vector<std::string> contigs;
  uint64_t total_len = 0;
  std::vector<uint32_t> contig_lengths;
  uint64_t repetitive_kmers = 0;
  std::vector<uint64_t> markers;
  uint64_t marker_c = 125, c = 125, k = 15;  // marker_c field = c (quirk, src/types.rs:347)
  uint64_t contig_order = 0;
  bool individual_contig = false, amino_acid = false;
};

struct IndexEntry { std::string file_name; uint64_t offset = 0, length = 0; };

// ---------------------------------------------------------------- writer
struct Out {
  std::vector<uint8_t> b;
  void u8(uint8_t v) { b.push_back(v); }
  void u32(uint32_t v) { uint8_t t[4]; memcpy(t, &v, 4); b.insert(b.end(), t, t + 4); }
  void u64(uint64_t v) { uint8_t t[8]; memcpy(t, &v, 8); b.insert(b.end(), t, t + 8); }
  void str(const std::string& s) { u64(s.size()); b.insert(b.end(), s.begin(), s.end()); }
};

// DNA_TO_AA (src/types.rs:27-28) and its integer encoding (src/params.rs:150-180; the duplicated 'R' key keeps the later value 15)
inline const char* dna_to_aa() { return "KNKNTTTTRSRSIIMIQHQHPPPPRRRRLLLLEDEDAAAAGGGGVVVV*Y*YSSSS*CWCLFLF"; }
inline uint64_t aa_code(char a) {
  switch (a) {
    case 'A': return 0; case 'R': return 15; case 'N': return 2; case 'D': return 3; case 'C': return 4; case 'E': return 5;
    case 'F': return 6; case 'G': return 7; case 'H': return 8; case 'I': return 9; case 'K': return 10; case 'L': return 11;
    case 'M': return 12; case 'P': return 13; case 'Q': return 14; case 'S': return 16; case 'T': return 17; case 'V': return 18;
    case 'W': return 19; case 'Y': return 20; default: return 21;   // '*' = STOP_CODON src/params.rs:14
  }
}

inline void put_params(Out& o, const DiskParams& p) {
  o.u64(p.c); o.u64(p.k); o.u64(p.marker_c); o.u8(p.use_syncs); o.u8(p.use_aa);
  o.u64(64);
  for (int i = 0; i < 64; i++) o.u64(aa_code(dna_to_aa()[i]));
  o.u64(64);
  for (int i = 0; i < 64; i++) o.u8((uint8_t)dna_to_aa()[i]);
  o.u64(p.orf_size);
}

// records must be grouped by k-mer (any order inside a group); this is what sk_sketch_set_export returns
inline void put_sketch(Out& o, const HostSketch& s) {
  o.str(s.file_name);
  const size_t n = s.kmer.size();
  if (!s.has_seeds) {
    o.u8(0);
    o.u64(0);                                   // multi_position_storage
  } else {
    o.u8(1);
    size_t n_keys = 0, n_multi = 0;
    for (size_t i = 0; i < n;) {
      size_t j = i + 1;
      while (j < n && s.kmer[j] == s.kmer[i]) j++;
      n_keys++;
      if (j - i > 1) n_multi++;
      i = j;
    }
    o.u64(n_keys);
    size_t storage = 0;
    for (size_t i = 0; i < n;) {
      size_t j = i + 1;
      while (j < n && s.kmer[j] == s.kmer[i]) j++;
      o.u32(s.kmer[i]);
      if (j - i == 1) o.u64(single_value(s.pos[i], s.cc[i]));
      else o.u64(multi_value(storage++));
      i = j;
    }
    o.u64(n_multi);
    for (size_t i = 0; i < n;) {
      size_t j = i + 1;
      while (j < n && s.kmer[j] == s.kmer[i]) j++;
      if (j - i > 1) {
        o.u64(j - i);
        for (size_t t = i; t < j; t++) { o.u32(s.pos[t]); o.u32(s.cc[t]); }
      }
      i = j;
    }
  }
  o.u64(s.contigs.size());
  for (auto& c : s.contigs) o.str(c);
  o.u64(s.total_len);
  o.u64(s.contig_lengths.size());
  for (uint32_t l : s.contig_lengths) o.u32(l);
  o.u64(s.repetitive_kmers);
  o.u64(s.markers.size());
  for (uint64_t m : s.markers) o.u64(m);
  o.u64(s.marker_c); o.u64(s.c); o.u64(s.k); o.u64(s.contig_order);
  o.u8(s.individual_contig); o.u8(s.amino_acid);
}

inline HostSketch markers_only(const HostSketch& s) {   // Sketch::get_markers_only, src/types.rs:322-340
  HostSketch m;
  m.file_name = s.file_name; m.has_seeds = false; m.contigs = s.contigs; m.total_len = s.total_len;
  m.repetitive_kmers = s.repetitive_kmers; m.markers = s.markers; m.marker_c = s.marker_c; m.c = s.c; m.k = s.k;
  m.contig_order = s.contig_order; m.individual_contig = s.individual_contig; m.amino_acid = s.amino_acid;
  return m;
}

// ---------------------------------------------------------------- reader
struct In {
  const uint8_t* p; const uint8_t* e;
  In(const uint8_t* b, size_t n) : p(b), e(b + n) {}
  void need(size_t n) const { if ((size_t)(e - p) < n) throw std::runtime_error("truncated sketch data"); }
  uint8_t u8() { need(1); return *p++; }
  uint32_t u32() { need(4); uint32_t v; memcpy(&v, p, 4); p += 4; return v; }
  uint64_t u64() { need(8); uint64_t v; memcpy(&v, p, 8); p += 8; return v; }
  uint64_t len(size_t elem) { uint64_t n = u64(); if (elem && n > (uint64_t)(e - p) / elem) throw std::runtime_error("corrupt length prefix"); return n; }
  std::string str() { uint64_t n = len(1); std::string s((const char*)p, (size_t)n); p += n; return s; }
};

inline DiskParams get_params(In& in) {
  DiskParams p;
  p.c = in.u64(); p.k = in.u64(); p.marker_c = in.u64(); p.use_syncs = in.u8() != 0; p.use_aa = in.u8() != 0;
  uint64_t n = in.len(8); in.need(n * 8); in.p += n * 8;
  n = in.len(1); in.need(n); in.p += n;
  p.orf_size = in.u64();
  return p;
}

// The framing of one Sketch, walked without materialising its records or markers.  Byte offsets are relative to the
// start of what was scanned (scan_entry: the blob).  The key block holds n_keys x {u32 k-mer, u64 value}
// (sketch_value.cuh); multi-position list j holds multi_len[j] x {u32 pos, u32 contig_index_canonical} at multi_at[j].
struct SketchScan {
  DiskParams params;                 // scan_entry only
  std::string file_name;
  bool has_seeds = true;
  uint64_t keys_at = 0, n_keys = 0;
  std::vector<uint64_t> multi_at, multi_len;
  std::vector<std::string> contigs;
  uint64_t total_len = 0;
  uint64_t ctg_len_at = 0, n_ctg_len = 0;      // u32 each
  uint64_t repetitive_kmers = 0;
  uint64_t markers_at = 0, n_markers = 0;      // u64 each
  uint64_t marker_c = 125, c = 125, k = 15, contig_order = 0;
  bool individual_contig = false, amino_acid = false;
  // seed records: n_keys - n_multi + sum of the list lengths, exact when every list belongs to exactly one key (as
  // skani writes them; the expansions count what the keys actually reference)
  uint64_t n_records = 0;
};

inline uint32_t load_u32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
inline uint64_t load_u64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }

// one Sketch at in.p (in is advanced past it); offsets relative to base.  Throws where the data cannot be a Sketch:
// truncated, a length prefix longer than the bytes left, an Option tag > 1.  Whether the keys' multi-position indices
// are in range is left to the expansion, which reads the values.
inline SketchScan scan_sketch(In& in, const uint8_t* base) {
  SketchScan s;
  s.file_name = in.str();
  const uint8_t tag = in.u8();
  if (tag > 1) throw std::runtime_error("corrupt Option tag (a pre-0.3 .sketch file?)");
  s.has_seeds = tag == 1;
  if (tag == 1) {
    s.n_keys = in.len(12);
    s.keys_at = (uint64_t)(in.p - base);
    in.p += s.n_keys * 12;
  }
  const uint64_t n_multi = in.len(8);
  s.multi_at.resize(n_multi);
  s.multi_len.resize(n_multi);
  uint64_t listed = 0;
  for (uint64_t i = 0; i < n_multi; i++) {
    s.multi_len[i] = in.len(8);
    s.multi_at[i] = (uint64_t)(in.p - base);
    in.p += s.multi_len[i] * 8;
    listed += s.multi_len[i];
  }
  s.n_records = s.n_keys + listed >= n_multi ? s.n_keys + listed - n_multi : 0;
  uint64_t n = in.len(8);
  for (uint64_t i = 0; i < n; i++) s.contigs.push_back(in.str());
  s.total_len = in.u64();
  s.n_ctg_len = in.len(4);
  s.ctg_len_at = (uint64_t)(in.p - base);
  in.p += s.n_ctg_len * 4;
  s.repetitive_kmers = in.u64();
  s.n_markers = in.len(8);
  s.markers_at = (uint64_t)(in.p - base);
  in.p += s.n_markers * 8;
  s.marker_c = in.u64(); s.c = in.u64(); s.k = in.u64(); s.contig_order = in.u64();
  s.individual_contig = in.u8() != 0; s.amino_acid = in.u8() != 0;
  return s;
}

// one (SketchParams, Sketch) blob: a `.sketch` file or a slice of sketches.db
inline SketchScan scan_entry(const uint8_t* p, size_t n) {
  In in(p, n);
  const DiskParams dp = get_params(in);
  SketchScan s = scan_sketch(in, p);
  s.params = dp;
  return s;
}

// the seed records of a scanned Sketch in file order (keys as stored, each multi-position list expanded in place), the
// order the device expansion of sk_sketch_set_import_blobs writes too
inline void expand_records(const uint8_t* base, const SketchScan& s, HostSketch& h) {
  for (uint64_t i = 0; i < s.n_keys; i++) {
    const uint8_t* e = base + s.keys_at + 12 * i;
    const uint32_t key = load_u32(e);
    const uint64_t v = load_u64(e + 4);
    if (value_is_single(v)) {
      h.kmer.push_back(key); h.pos.push_back(value_pos(v)); h.cc.push_back(value_cc(v));
      continue;
    }
    const uint64_t si = value_multi_index(v);
    if (si >= s.multi_at.size()) throw std::runtime_error("multi-position index out of range");
    const uint8_t* l = base + s.multi_at[si];
    for (uint64_t t = 0; t < s.multi_len[si]; t++) {
      h.kmer.push_back(key); h.pos.push_back(load_u32(l + 8 * t)); h.cc.push_back(load_u32(l + 8 * t + 4));
    }
  }
}

// seeds = false skips materialising the records (markers.bin entries have none anyway)
inline HostSketch get_sketch(In& in, bool seeds = true) {
  const uint8_t* base = in.p;
  const SketchScan sc = scan_sketch(in, base);
  HostSketch s;
  s.file_name = sc.file_name;
  s.has_seeds = sc.has_seeds;
  if (seeds) expand_records(base, sc, s);
  s.contigs = sc.contigs;
  s.total_len = sc.total_len;
  s.contig_lengths.resize(sc.n_ctg_len);
  for (uint64_t i = 0; i < sc.n_ctg_len; i++) s.contig_lengths[i] = load_u32(base + sc.ctg_len_at + 4 * i);
  s.repetitive_kmers = sc.repetitive_kmers;
  s.markers.resize(sc.n_markers);
  for (uint64_t i = 0; i < sc.n_markers; i++) s.markers[i] = load_u64(base + sc.markers_at + 8 * i);
  s.marker_c = sc.marker_c; s.c = sc.c; s.k = sc.k; s.contig_order = sc.contig_order;
  s.individual_contig = sc.individual_contig; s.amino_acid = sc.amino_acid;
  return s;
}

// ---------------------------------------------------------------- files
inline bool read_file(const std::string& path, std::vector<uint8_t>& out) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return false;
  fseek(f, 0, SEEK_END);
  long n = ftell(f);
  fseek(f, 0, SEEK_SET);
  out.resize(n > 0 ? (size_t)n : 0);
  size_t got = out.empty() ? 0 : fread(out.data(), 1, out.size(), f);
  fclose(f);
  return got == out.size();
}
inline bool write_file(const std::string& path, const std::vector<uint8_t>& b) {
  FILE* f = fopen(path.c_str(), "wb");
  if (!f) return false;
  size_t w = b.empty() ? 0 : fwrite(b.data(), 1, b.size(), f);
  return fclose(f) == 0 && w == b.size();
}

// Database writer over encoded entries (SketchDbWriter, src/sketch_db.rs:17-84, + markers.bin, src/sketch.rs:141-146).
// add() takes one full entry, (SketchParams, Sketch) as put_params + put_sketch or sk_sketch_set_encode write it, and the
// same sketch's markers-only Sketch (put_sketch(markers_only(s))).  Consolidated, the entry is appended to sketches.db and
// listed in index.db; with separate sketches it becomes the file sketch_path.  markers.bin is appended entry by entry and
// its count filled in by finalize(), so the writer holds no sketches.
struct DbWriter {
  std::string dir;
  bool separate = false;
  FILE* concat = nullptr;
  FILE* markers = nullptr;
  long count_at = 0;                 // markers.bin: where the Vec<Sketch> length goes
  std::vector<IndexEntry> index;
  uint64_t offset = 0, n_markers = 0;
  bool open(const std::string& d, const DiskParams& p, bool separate_sketches = false) {
    dir = d; separate = separate_sketches;
    if (!separate && !(concat = fopen((dir + "/sketches.db").c_str(), "wb"))) return false;
    if (!(markers = fopen((dir + "/markers.bin").c_str(), "wb"))) return false;
    Out head;
    put_params(head, p);
    count_at = (long)head.b.size();
    head.u64(0);
    return fwrite(head.b.data(), 1, head.b.size(), markers) == head.b.size();
  }
  bool add(const std::string& file_name, const std::string& sketch_path, const uint8_t* entry, uint64_t len, const uint8_t* marker_entry,
           uint64_t marker_len) {
    if (separate) {
      FILE* f = fopen(sketch_path.c_str(), "wb");
      if (!f) return false;
      const bool ok = fwrite(entry, 1, len, f) == len;
      if (fclose(f) != 0 || !ok) return false;
    } else {
      if (fwrite(entry, 1, len, concat) != len) return false;
      index.push_back(IndexEntry{file_name, offset, len});
      offset += len;
    }
    n_markers++;
    return fwrite(marker_entry, 1, marker_len, markers) == marker_len;
  }
  bool add(const HostSketch& s, const DiskParams& p, const std::string& sketch_path = std::string()) {   // the host encoder
    Out o, m;
    put_params(o, p);
    put_sketch(o, s);
    put_sketch(m, markers_only(s));
    return add(s.file_name, sketch_path, o.b.data(), o.b.size(), m.b.data(), m.b.size());
  }
  bool finalize() {
    if (concat) {
      if (fclose(concat) != 0) return false;
      concat = nullptr;
      Out ix;
      ix.u64(index.size());
      for (auto& e : index) { ix.str(e.file_name); ix.u64(e.offset); ix.u64(e.length); }
      if (!write_file(dir + "/index.db", ix.b)) return false;
    }
    Out n;
    n.u64(n_markers);
    const bool ok = fseek(markers, count_at, SEEK_SET) == 0 && fwrite(n.b.data(), 1, 8, markers) == 8;
    const bool closed = fclose(markers) == 0;
    markers = nullptr;
    return ok && closed;
  }
};

// (SketchParams, Vec<Sketch>) of markers.bin (file_io::marker_sketches_from_marker_file, src/file_io.rs:719-729)
inline void read_markers_bin(const std::string& path, DiskParams& params, std::vector<HostSketch>& out) {
  std::vector<uint8_t> b;
  if (!read_file(path, b)) throw std::runtime_error("cannot read " + path);
  In in(b.data(), b.size());
  params = get_params(in);
  uint64_t n = in.len(8);
  out.clear();
  for (uint64_t i = 0; i < n; i++) out.push_back(get_sketch(in, false));
}

inline void read_index_db(const std::string& path, std::vector<IndexEntry>& out) {
  std::vector<uint8_t> b;
  if (!read_file(path, b)) throw std::runtime_error("cannot read " + path);
  In in(b.data(), b.size());
  uint64_t n = in.len(8);
  out.clear();
  for (uint64_t i = 0; i < n; i++) { IndexEntry e; e.file_name = in.str(); e.offset = in.u64(); e.length = in.u64(); out.push_back(e); }
}

// one (SketchParams, Sketch) blob: a `.sketch` file or a slice of sketches.db
inline HostSketch read_blob(const uint8_t* p, size_t n, DiskParams* params = nullptr) {
  In in(p, n);
  DiskParams dp = get_params(in);
  if (params) *params = dp;
  return get_sketch(in, true);
}

// one entry of sketches.db (open as fd): pread of its slice, then read_blob.  false if it cannot be read or decoded.
inline bool read_db_entry(int fd, const IndexEntry& e, HostSketch& out, DiskParams* params = nullptr) {
  std::vector<uint8_t> b(e.length);
  if (pread(fd, b.data(), b.size(), (off_t)e.offset) != (ssize_t)b.size()) return false;
  try { out = read_blob(b.data(), b.size(), params); }
  catch (const std::exception&) { return false; }
  return true;
}

// the sketch count of markers.bin, read from its head only (the marker sketches themselves are not decoded)
inline bool markers_bin_count(const std::string& path, uint64_t& n) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return false;
  std::vector<uint8_t> b(4096);
  b.resize(fread(b.data(), 1, b.size(), f));
  fclose(f);
  try { In in(b.data(), b.size()); get_params(in); n = in.u64(); }
  catch (const std::exception&) { return false; }
  return true;
}

// A consolidated database: index.db read, checked against markers.bin's sketch count when markers.bin exists, and
// sketches.db opened read-only as fd.  false after an ERROR line (the messages of `search`).
inline bool open_db(const std::string& dir, std::vector<IndexEntry>& index, int& fd) {
  try { read_index_db(dir + "/index.db", index); }
  catch (const std::exception& e) { fprintf(stderr, "ERROR Failed to load consolidated database: %s\n", e.what()); return false; }
  uint64_t n_markers = 0;
  struct stat st;
  if (stat((dir + "/markers.bin").c_str(), &st) == 0 && (!markers_bin_count(dir + "/markers.bin", n_markers) || n_markers != index.size())) {
    fprintf(stderr, "ERROR index.db and markers.bin disagree on the number of sketches\n");
    return false;
  }
  fd = open((dir + "/sketches.db").c_str(), O_RDONLY);
  if (fd < 0) { fprintf(stderr, "ERROR Failed to load consolidated database\n"); return false; }
  return true;
}

// ---------------------------------------------------------------- sketch inputs of triangle / dist / search
// A consolidated database (a directory holding index.db and sketches.db, src/sketch_db.rs:142-146) stands for all of its
// sketches, exactly as if each entry were a .sketch file.  Opening the inputs reads index.db (and checks it against
// markers.bin and the size of sketches.db) but decodes only a database's first entry; the sketches themselves are read
// later, in groups and as stored (SketchGroupReader), so host memory holds one group's bytes at a time.
inline bool is_sketch_db(const std::string& p) {
  struct stat st;
  return stat(p.c_str(), &st) == 0 && S_ISDIR(st.st_mode) && stat((p + "/index.db").c_str(), &st) == 0 &&
         stat((p + "/sketches.db").c_str(), &st) == 0;
}

struct SketchEntry {            // one sketch of the inputs
  uint32_t input = 0;           // index into SketchInputs::paths
  std::string file_name;        // sort key: the name in index.db, or the one stored in the .sketch file
  uint64_t offset = 0, length = 0;   // slice of sketches.db (a .sketch file: the whole file)
  uint64_t weight = 0;          // seed records (.sketch files, decoded when opened) or length / 12 (a database entry, not
                                // yet decoded: a single-position record takes 12 bytes on disk)
};

struct SketchInputs {
  std::vector<std::string> paths;    // .sketch files and database directories (open_sketch_inputs: in command-line order)
  std::vector<int> db_fd;            // sketches.db of paths[i], or -1 for a .sketch file
  std::vector<SketchEntry> entries;  // every sketch (open_sketch_inputs: stably sorted by file name, src/file_io.rs:715)
  DiskParams params;                 // of the first input (all inputs agree on c, k and marker_c)
  SketchInputs() = default;
  SketchInputs(const SketchInputs&) = delete;
  SketchInputs& operator=(const SketchInputs&) = delete;
  ~SketchInputs() { for (int fd : db_fd) if (fd >= 0) close(fd); }
};

// Opens the inputs (.sketch files, markers.bin names, which are skipped, and databases) into si.  Problems are reported
// on stderr with an ERROR line; false means the run must stop.  A .sketch file that does not decode is skipped, as
// file_io::sketches_from_sketch does (src/file_io.rs:680-717).
inline bool open_sketch_inputs(const std::vector<std::string>& files, SketchInputs& si) {
  std::string params_of;        // the input whose parameters si.params holds
  auto take_params = [&](const DiskParams& p, const std::string& path, bool db) {
    if (p.use_aa) { fprintf(stderr, db ? "ERROR amino-acid databases are not supported\n" : "ERROR amino-acid sketches are not supported\n"); return false; }
    if (params_of.empty()) { si.params = p; params_of = path; return true; }
    if (p.c == si.params.c && p.k == si.params.k && p.marker_c == si.params.marker_c) return true;
    fprintf(stderr, "ERROR Sketch parameters of %s (c = %llu, k = %llu, m = %llu) differ from those of %s (c = %llu, k = %llu, m = %llu). Exiting.\n",
            path.c_str(), (unsigned long long)p.c, (unsigned long long)p.k, (unsigned long long)p.marker_c, params_of.c_str(),
            (unsigned long long)si.params.c, (unsigned long long)si.params.k, (unsigned long long)si.params.marker_c);
    return false;
  };
  for (auto& f : files) {
    const uint32_t input = (uint32_t)si.paths.size();
    if (is_sketch_db(f)) {
      std::vector<IndexEntry> index;
      int fd = -1;
      if (!open_db(f, index, fd)) return false;
      si.paths.push_back(f);
      si.db_fd.push_back(fd);
      struct stat st;
      if (fstat(fd, &st) != 0) { fprintf(stderr, "ERROR Failed to load consolidated database\n"); return false; }
      for (auto& e : index)
        if (e.offset > (uint64_t)st.st_size || e.length > (uint64_t)st.st_size - e.offset) {
          fprintf(stderr, "ERROR Failed to load consolidated database: the entry of %s runs past the end of %s/sketches.db\n", e.file_name.c_str(), f.c_str());
          return false;
        }
      if (index.empty()) continue;
      HostSketch first;
      DiskParams p;
      if (!read_db_entry(fd, index[0], first, &p)) { fprintf(stderr, "ERROR Failed to load sketch %s\n", index[0].file_name.c_str()); return false; }
      if (!take_params(p, f, true)) return false;
      for (auto& e : index) si.entries.push_back(SketchEntry{input, e.file_name, e.offset, e.length, e.length / 12});
    } else {
      if (f.find("markers.bin") != std::string::npos) continue;
      std::vector<uint8_t> b;
      if (!read_file(f, b)) { fprintf(stderr, "ERROR Problem reading sketch file %s. Perhaps your file path is wrong? Exiting.\n", f.c_str()); return false; }
      HostSketch h;
      DiskParams p;
      try { h = read_blob(b.data(), b.size(), &p); }
      catch (const std::exception&) {
        fprintf(stderr, "ERROR %s is not a valid .sketch file or is corrupted. Skani v0.3+ is not compatible with older sketch files.\n", f.c_str());
        continue;
      }
      if (!take_params(p, f, false)) return false;
      si.paths.push_back(f);
      si.db_fd.push_back(-1);
      si.entries.push_back(SketchEntry{input, h.file_name, 0, (uint64_t)b.size(), (uint64_t)h.kmer.size()});
    }
  }
  std::stable_sort(si.entries.begin(), si.entries.end(), [](const SketchEntry& x, const SketchEntry& y) { return x.file_name < y.file_name; });
  return true;
}

// bytes that are written before they are read: growing the buffer does not clear it
template <class T>
struct uninit_alloc : std::allocator<T> {
  template <class U> struct rebind { using other = uninit_alloc<U>; };
  template <class U> void construct(U* p) noexcept { ::new ((void*)p) U; }
  template <class U, class... A> void construct(U* p, A&&... a) { ::new ((void*)p) U(std::forward<A>(a)...); }
};

// A group of sketch inputs as stored: blob i (a .sketch file or a sketches.db entry, SketchParams included) is
// bytes[off[i], off[i] + len[i]), scan[i] its framing.  records = the sum of the scans' record counts.
struct SketchGroup {
  std::vector<uint8_t, uninit_alloc<uint8_t>> bytes;
  std::vector<uint64_t> off, len;
  std::vector<SketchScan> scan;
  uint64_t records = 0;
  size_t size() const { return scan.size(); }
  void clear() { bytes.clear(); off.clear(); len.clear(); scan.clear(); records = 0; }
};

// Reads the entries of si listed in `list` (entry indices), in list order, and hands them out in groups of < max_records
// seed records (a group holds at least one sketch), each group's blobs read into one buffer as stored and scanned
// (scan_entry), not decoded.  Entries are read and scanned in batches by `threads` threads; the entries of a batch that
// the current group cannot take are carried into the next one.  An entry that cannot be read or scanned, or whose name
// differs from its index entry, ends the reading with an ERROR line: next() then returns false with failed set.
class SketchGroupReader {
 public:
  SketchGroupReader(const SketchInputs& si, std::vector<size_t> list, int threads, uint64_t max_records)
      : si_(si), list_(std::move(list)), threads_(std::max(threads, 1)), max_records_(max_records) {}
  bool failed = false;
  size_t first = 0;             // position in the list of g's first blob after next()

  bool next(SketchGroup& g) {
    g = std::move(carry_);        // the previous group's buffer is freed here
    carry_ = SketchGroup();
    first = consumed_;
    size_t take = 0;            // g's blobs [0, take) fit the group
    uint64_t recs = 0;
    for (;;) {
      while (take < g.size() && (take == 0 || recs + g.scan[take].n_records < max_records_)) recs += g.scan[take++].n_records;
      if (take < g.size() || !read_batch(g)) break;
      if (failed) { g.clear(); return false; }
    }
    for (size_t i = take; i < g.size(); i++) {             // the rest of the last batch opens the next group
      carry_.off.push_back(carry_.bytes.size());
      carry_.bytes.insert(carry_.bytes.end(), g.bytes.begin() + g.off[i], g.bytes.begin() + g.off[i] + g.len[i]);
      carry_.len.push_back(g.len[i]);
      carry_.scan.push_back(std::move(g.scan[i]));
      carry_.records += carry_.scan.back().n_records;
    }
    if (take < g.size()) {
      g.bytes.resize(g.off[take]);
      g.off.resize(take); g.len.resize(take); g.scan.resize(take);
    }
    g.records = recs;
    consumed_ += g.size();
    return g.size() != 0;
  }

 private:
  // the next entries (at most 8 per thread and about 256 MiB on disk) appended to g: read, then scanned
  bool read_batch(SketchGroup& g) {
    const size_t listed = list_.size();
    if (next_ >= listed) return false;
    size_t b = next_;
    uint64_t bytes = 0;
    while (b < listed && (b == next_ || (b - next_ < 8 * (size_t)threads_ && bytes < (256ull << 20)))) bytes += si_.entries[list_[b++]].length;
    const size_t n0 = g.size(), n = b - next_;
    if (g.bytes.capacity() < g.bytes.size() + bytes) {   // room for the rest of the inputs, up to about a group's worth
      uint64_t rest = 0;
      for (size_t i = next_; i < listed && rest < 16 * max_records_; i++) rest += si_.entries[list_[i]].length;
      g.bytes.reserve(g.bytes.size() + std::max<uint64_t>(bytes, rest));
    }
    uint64_t end = g.bytes.size();
    for (size_t i = 0; i < n; i++) {
      g.off.push_back(end);
      g.len.push_back(si_.entries[list_[next_ + i]].length);
      end += g.len.back();
    }
    g.bytes.resize(end);
    g.scan.resize(n0 + n);
    std::atomic<size_t> at{0};
    std::atomic<bool> bad{false};
    auto worker = [&] {
      for (size_t i; (i = at.fetch_add(1)) < n;) {
        const SketchEntry& e = si_.entries[list_[next_ + i]];
        const int fd = si_.db_fd[e.input];
        uint8_t* dst = g.bytes.data() + g.off[n0 + i];
        bool good;
        if (fd >= 0) good = pread(fd, dst, e.length, (off_t)e.offset) == (ssize_t)e.length;
        else {                   // a .sketch file: the size its entry records
          FILE* f = fopen(si_.paths[e.input].c_str(), "rb");
          good = f && fread(dst, 1, e.length, f) == e.length;
          if (f) fclose(f);
        }
        try { if (good) g.scan[n0 + i] = scan_entry(dst, e.length); }
        catch (const std::exception&) { good = false; }
        if (good && fd >= 0) good = g.scan[n0 + i].file_name == e.file_name;
        if (!good) { bad = true; fprintf(stderr, "ERROR Failed to load sketch %s\n", e.file_name.c_str()); }
      }
    };
    std::vector<std::thread> pool;
    for (int t = 1; t < threads_ && (size_t)t < n; t++) pool.emplace_back(worker);
    worker();
    for (auto& t : pool) t.join();
    next_ = b;
    if (bad) failed = true;
    return true;
  }
  const SketchInputs& si_;
  std::vector<size_t> list_;
  size_t next_ = 0, consumed_ = 0;   // positions in list_: the next entry to read, the first not yet handed out
  int threads_;
  uint64_t max_records_;
  SketchGroup carry_;
};

}  // namespace skdb
