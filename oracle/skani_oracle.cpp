// ============================================================================
// skani_oracle.cpp -- TEST INFRASTRUCTURE ONLY (CPU oracle / CPU baseline).
// See skani_oracle.hpp for the scope statement.  Citations are into /root/reference
// (bluenote-1577/skani @ c57dbe7, crate v0.3.0).
// ============================================================================
#include "skani_oracle.hpp"
#if defined(__x86_64__)
#include <immintrin.h>
#endif

#include <zlib.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <limits>
#include <map>
#include <unordered_map>

#ifdef _OPENMP
#include <omp.h>
#endif

namespace orc {

// ------------------------------------------------------------------------------------------------
// types.rs:40-49  BYTE_TO_SEQ: A/a=0 C/c=1 G/g=2 T/t/U/u=3, bytes 0..3 map to themselves, else 0
// ------------------------------------------------------------------------------------------------
namespace {
struct ByteToSeqTable {
  uint8_t t[256];
  ByteToSeqTable() {
    std::memset(t, 0, sizeof(t));
    t[1] = 1; t[2] = 2; t[3] = 3;
    t['C'] = t['c'] = 1;
    t['G'] = t['g'] = 2;
    t['T'] = t['t'] = t['U'] = t['u'] = 3;
  }
};
const ByteToSeqTable g_b2s;
}  // namespace
const uint8_t* const BYTE_TO_SEQ = g_b2s.t;

// types.rs:86-96  Thomas Wang 64-bit mix (as used by minimap2)
uint64_t mm_hash64(uint64_t key) {
  key = ~(key + (key << 21));
  key = key ^ (key >> 24);
  key = (key + (key << 3)) + (key << 8);
  key = key ^ (key >> 14);
  key = (key + (key << 2)) + (key << 4);
  key = key ^ (key >> 28);
  key = key + (key << 31);
  return key;
}

// ------------------------------------------------------------------------------------------------
// hash containers (stand-ins for hashbrown with MMHasher, types.rs:56-69, 394-427)
// ------------------------------------------------------------------------------------------------
KmerSeeds::KmerSeeds() {}
void KmerSeeds::grow() {
  size_t ncap = keys_.empty() ? 1024 : keys_.size() * 2;
  std::vector<uint32_t> ok;
  std::vector<uint64_t> ov;
  std::vector<uint8_t> ou;
  ok.swap(keys_); ov.swap(vals_); ou.swap(used_);
  keys_.assign(ncap, 0); vals_.assign(ncap, 0); used_.assign(ncap, 0);
  mask_ = ncap - 1;
  for (size_t s = 0; s < ok.size(); s++) {
    if (!ou[s]) continue;
    size_t h = mm_hash64(ok[s]) & mask_;
    while (used_[h]) h = (h + 1) & mask_;
    used_[h] = 1; keys_[h] = ok[s]; vals_[h] = ov[s];
  }
}
uint64_t* KmerSeeds::find(uint32_t key) {
  if (keys_.empty()) return nullptr;
  size_t h = mm_hash64(key) & mask_;
  while (used_[h]) {
    if (keys_[h] == key) return &vals_[h];
    h = (h + 1) & mask_;
  }
  return nullptr;
}
const uint64_t* KmerSeeds::find(uint32_t key) const { return const_cast<KmerSeeds*>(this)->find(key); }
void KmerSeeds::insert(uint32_t key, uint64_t val) {
  if ((n_ + 1) * 2 > keys_.size()) grow();
  size_t h = mm_hash64(key) & mask_;
  while (used_[h]) h = (h + 1) & mask_;
  used_[h] = 1; keys_[h] = key; vals_[h] = val; n_++;
}

MarkerSet::MarkerSet() {}
void MarkerSet::grow() {
  size_t ncap = keys_.empty() ? 256 : keys_.size() * 2;
  std::vector<uint64_t> ok;
  ok.swap(keys_);
  keys_.assign(ncap, EMPTY);
  mask_ = ncap - 1;
  for (uint64_t k : ok) {
    if (k == EMPTY) continue;
    size_t h = mm_hash64(k) & mask_;
    while (keys_[h] != EMPTY) h = (h + 1) & mask_;
    keys_[h] = k;
  }
}
bool MarkerSet::contains(uint64_t key) const {
  if (keys_.empty()) return false;
  size_t h = mm_hash64(key) & mask_;
  while (keys_[h] != EMPTY) {
    if (keys_[h] == key) return true;
    h = (h + 1) & mask_;
  }
  return false;
}
void MarkerSet::insert(uint64_t key) {
  if ((n_ + 1) * 2 > keys_.size()) grow();
  size_t h = mm_hash64(key) & mask_;
  while (keys_[h] != EMPTY) {
    if (keys_[h] == key) return;
    h = (h + 1) & mask_;
  }
  keys_[h] = key; n_++;
}

// ------------------------------------------------------------------------------------------------
// types.rs:207-244 TaggedIndex, types.rs:281-320 Sketch::add_seed_position / get_seed_positions
// ------------------------------------------------------------------------------------------------
static inline uint64_t tagged_single(const SeedPosition& p) {
  uint64_t packed = ((uint64_t)p.pos << 31) | (uint64_t)p.contig_index_canonical;  // types.rs:177-180
  return 1ull | (packed << 1);                                                       // types.rs:214-216
}
static inline SeedPosition tagged_get_single(uint64_t t) {
  uint64_t packed = t >> 1;
  return SeedPosition{(uint32_t)(packed >> 31), (uint32_t)(packed & 0x7FFFFFFFull)};  // types.rs:184-191
}

void Sketch::add_seed_position(uint32_t seed, SeedPosition p) {
  if (!has_seeds) return;
  uint64_t* t = kmer_seeds_k.find(seed);
  if (t) {
    if (*t & 1ull) {  // single -> promote to multiple (types.rs:286-291)
      SeedPosition existing = tagged_get_single(*t);
      size_t idx = multi_position_storage.size();
      multi_position_storage.push_back({existing, p});
      *t = (uint64_t)idx << 1;
    } else {
      multi_position_storage[(size_t)(*t >> 1)].push_back(p);  // types.rs:293-295
    }
  } else {
    kmer_seeds_k.insert(seed, tagged_single(p));  // types.rs:299-301
  }
}

size_t Sketch::get_seed_positions(uint32_t seed, const SeedPosition** out, SeedPosition* tmp) const {
  if (has_seeds) {
    const uint64_t* t = kmer_seeds_k.find(seed);
    if (t) {
      if (*t & 1ull) {
        *tmp = tagged_get_single(*t);
        *out = tmp;
        return 1;
      }
      const auto& v = multi_position_storage[(size_t)(*t >> 1)];
      *out = v.data();
      return v.size();
    }
  }
  *out = nullptr;
  return 0;
}

// ------------------------------------------------------------------------------------------------
// seeding.rs:225-323  scalar FracMinHash seeding of one contig
// ------------------------------------------------------------------------------------------------
void fmh_seeds_scalar(const uint8_t* s, size_t n, const SketchParams& sp, uint32_t contig_index, Sketch& sk) {
  sk.has_seeds = true;  // seeding.rs:232-234 (seed == true at every call site)
  const size_t marker_k = K_MARKER_DNA;
  const size_t k = sp.k;
  if (k > 16) return;  // reference panics (seeding.rs:239-241); the oracle refuses
  if (n < 2 * marker_k) return;  // seeding.rs:242-244
  uint64_t f = 0, r = 0;
  const uint64_t seed_mask = ~0ull >> (64 - 2 * k);
  const unsigned rshift = 2 * (marker_k - 1);
  const uint64_t marker_mask = ~0ull >> (64 - 2 * marker_k);
  const uint64_t marker_rev_mask = ~(3ull << (2 * marker_k - 2));
  const uint64_t threshold = ~0ull / sp.c;                // seeding.rs:258
  const uint64_t threshold_marker = ~0ull / sp.marker_c;  // seeding.rs:259
  for (size_t i = 0; i < marker_k - 1; i++) {  // seeding.rs:260-269
    uint64_t nf = BYTE_TO_SEQ[s[i]];
    uint64_t nr = 3 - nf;
    f = (f << 2) | nf;
    r = (r >> 2) | (nr << rshift);
  }
  size_t resume_ind = 0;
  for (size_t i = marker_k - 1; i < n; i++) {  // seeding.rs:271-322
    uint8_t b = s[i];
    if (b == 78 || b == 110) resume_ind = i + k;  // 'N' or 'n' (seeding.rs:273-275)
    uint64_t nf = BYTE_TO_SEQ[b];
    uint64_t nr = 3 - nf;
    f = ((f << 2) | nf) & marker_mask;
    r = ((r >> 2) & marker_rev_mask) | (nr << rshift);
    uint64_t fs = f & seed_mask, rs = r & seed_mask;
    bool canonical_seed = fs < rs;
    uint64_t seed = canonical_seed ? fs : rs;
    uint64_t h = mm_hash64(seed);
    if (h < threshold && resume_ind <= i) {
      sk.add_seed_position((uint32_t)seed, SeedPosition{(uint32_t)i, (contig_index << 1) | (canonical_seed ? 1u : 0u)});
      uint64_t marker = (f < r) ? f : r;  // seeding.rs:311-316
      if (h < threshold_marker) sk.marker_seeds.insert(marker);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// avx2_seeding.rs:33-272  the 4-lane path, restated lane by lane (what x86-64+AVX2 hosts execute)
// ------------------------------------------------------------------------------------------------
// The same function with the reference's actual instruction mix: one __m256i holds the four lanes, mm_hash256 runs on
// all four per step and the hits are taken out with per-lane extracts (avx2_seeding.rs:7-30, 108-272).  Selected with
// set_avx2_intrinsics(true) for the CPU BASELINE (bench.py); parity tests keep the lane-by-lane form above as the
// definition and check that both produce identical sketches (tests/test_oracle_goldens.py).
static bool g_avx2_intrinsics = false;
void set_avx2_intrinsics(bool on) { g_avx2_intrinsics = on && __builtin_cpu_supports("avx2"); }
bool avx2_intrinsics() { return g_avx2_intrinsics; }

#if defined(__x86_64__)
__attribute__((target("avx2"))) static inline __m256i mm_hash256(__m256i key) {  // avx2_seeding.rs:7-30
  key = _mm256_add_epi64(key, _mm256_slli_epi64(key, 21));
  key = _mm256_xor_si256(key, _mm256_cmpeq_epi64(key, key));
  key = _mm256_xor_si256(key, _mm256_srli_epi64(key, 24));
  key = _mm256_add_epi64(_mm256_add_epi64(key, _mm256_slli_epi64(key, 3)), _mm256_slli_epi64(key, 8));
  key = _mm256_xor_si256(key, _mm256_srli_epi64(key, 14));
  key = _mm256_add_epi64(_mm256_add_epi64(key, _mm256_slli_epi64(key, 2)), _mm256_slli_epi64(key, 4));
  key = _mm256_xor_si256(key, _mm256_srli_epi64(key, 28));
  key = _mm256_add_epi64(key, _mm256_slli_epi64(key, 31));
  return key;
}

__attribute__((target("avx2"))) static void fmh_seeds_avx2_intrin(const uint8_t* s, size_t n, const SketchParams& sp, uint32_t contig_index, Sketch& sk) {
  sk.has_seeds = true;
  const size_t marker_k = K_MARKER_DNA;
  const size_t k = sp.k;
  if (k > 16) return;
  if (n < 2 * marker_k) return;
  const size_t len = (n - marker_k + 1) / 4;
  const uint8_t* str[4] = {s, s + len, s + 2 * len, s + 3 * len};
  const int64_t seed_mask = (int64_t)(~0ull >> (64 - 2 * k));
  const int64_t marker_mask = (int64_t)(~0ull >> (64 - 2 * marker_k));
  const int64_t rev_marker_mask = (int64_t)~(3ull << (2 * marker_k - 2));
  const uint64_t threshold = ~0ull / sp.c, threshold_marker = ~0ull / sp.marker_c;
  const __m256i rev_sub = _mm256_set1_epi64x(3), m_seed = _mm256_set1_epi64x(seed_mask), m_marker = _mm256_set1_epi64x(marker_mask),
                m_rev = _mm256_set1_epi64x(rev_marker_mask);
  __m256i f = _mm256_setzero_si256(), r = _mm256_setzero_si256();
  for (size_t i = 0; i < marker_k - 1; i++) {  // :63-81
    const __m256i fn = _mm256_set_epi64x(BYTE_TO_SEQ[str[3][i]], BYTE_TO_SEQ[str[2][i]], BYTE_TO_SEQ[str[1][i]], BYTE_TO_SEQ[str[0][i]]);
    const __m256i rn = _mm256_sub_epi64(rev_sub, fn);
    f = _mm256_or_si256(_mm256_slli_epi64(f, 2), fn);
    r = _mm256_or_si256(_mm256_srli_epi64(r, 2), _mm256_slli_epi64(rn, 40));
  }
  size_t resume[4] = {0, 0, 0, 0};
  for (size_t i = marker_k - 1; i < len + marker_k - 1; i++) {  // :108
    const uint8_t b0 = str[0][i], b1 = str[1][i], b2 = str[2][i], b3 = str[3][i];
    if (b0 == 78) resume[0] = i + marker_k;
    if (b1 == 78) resume[1] = i + marker_k;
    if (b2 == 78) resume[2] = i + marker_k;
    if (b3 == 78) resume[3] = i + marker_k;
    const __m256i fn = _mm256_set_epi64x(BYTE_TO_SEQ[b3], BYTE_TO_SEQ[b2], BYTE_TO_SEQ[b1], BYTE_TO_SEQ[b0]);
    const __m256i rn = _mm256_sub_epi64(rev_sub, fn);
    f = _mm256_and_si256(_mm256_or_si256(_mm256_slli_epi64(f, 2), fn), m_marker);
    r = _mm256_or_si256(_mm256_and_si256(_mm256_srli_epi64(r, 2), m_rev), _mm256_slli_epi64(rn, 40));
    const __m256i fs = _mm256_and_si256(f, m_seed), rs = _mm256_and_si256(r, m_seed);
    const __m256i cmp = _mm256_cmpgt_epi64(rs, fs), cmp_marker = _mm256_cmpgt_epi64(r, f);
    const __m256i seeds = _mm256_blendv_epi8(rs, fs, cmp);
    alignas(32) uint64_t hv[4], sv[4], cv[4];
    _mm256_store_si256((__m256i*)hv, mm_hash256(seeds));
    _mm256_store_si256((__m256i*)sv, seeds);
    _mm256_store_si256((__m256i*)cv, cmp);
    for (int lane = 0; lane < 4; lane++) {   // the four unrolled blocks of :179-269
      if (hv[lane] < threshold && resume[lane] <= i) {
        sk.add_seed_position((uint32_t)sv[lane], SeedPosition{(uint32_t)(i + len * lane), (contig_index << 1) | (cv[lane] ? 1u : 0u)});
        if (hv[lane] < threshold_marker) {
          alignas(32) uint64_t fv[4], rv[4], mv[4];
          _mm256_store_si256((__m256i*)fv, f); _mm256_store_si256((__m256i*)rv, r); _mm256_store_si256((__m256i*)mv, cmp_marker);
          sk.marker_seeds.insert(mv[lane] ? fv[lane] : rv[lane]);
        }
      }
    }
  }
}
#endif

void fmh_seeds_avx2sem(const uint8_t* s, size_t n, const SketchParams& sp, uint32_t contig_index, Sketch& sk) {
#if defined(__x86_64__)
  if (g_avx2_intrinsics) { fmh_seeds_avx2_intrin(s, n, sp, contig_index, sk); return; }
#endif
  sk.has_seeds = true;  // avx2_seeding.rs:40-42
  const size_t marker_k = K_MARKER_DNA;
  const size_t k = sp.k;
  if (k > 16) return;  // keeps the u32 SeedBits cast lossless; reference allows k<=21 here but CLI k is 15
  if (n < 2 * marker_k) return;  // avx2_seeding.rs:56-58 (slices at :49-52 need n >= 20; guaranteed by n >= 42)
  const size_t len = (n - marker_k + 1) / 4;  // avx2_seeding.rs:48
  const uint64_t seed_mask = ~0ull >> (64 - 2 * k);
  const uint64_t marker_mask = ~0ull >> (64 - 2 * marker_k);
  const uint64_t rev_marker_mask = ~(3ull << (2 * marker_k - 2));
  const uint64_t threshold = ~0ull / sp.c;
  const uint64_t threshold_marker = ~0ull / sp.marker_c;
  for (size_t lane = 0; lane < 4; lane++) {
    const uint8_t* str = s + lane * len;  // substring [lane*len, lane*len + len + 20)  (avx2_seeding.rs:49-52)
    uint64_t f = 0, r = 0;
    for (size_t i = 0; i < marker_k - 1; i++) {  // avx2_seeding.rs:63-81 (no N detection, no masking)
      uint64_t nf = BYTE_TO_SEQ[str[i]];
      uint64_t nr = 3 - nf;
      f = (f << 2) | nf;
      r = (r >> 2) | (nr << 40);
    }
    size_t resume = 0;  // avx2_seeding.rs:107
    for (size_t i = marker_k - 1; i < len + marker_k - 1; i++) {  // avx2_seeding.rs:108
      uint8_t b = str[i];
      if (b == 78) resume = i + marker_k;  // only 'N' (avx2_seeding.rs:115-126)
      uint64_t nf = BYTE_TO_SEQ[b];
      uint64_t nr = 3 - nf;
      f = ((f << 2) | nf) & marker_mask;                 // :137-139
      r = ((r >> 2) & rev_marker_mask) | (nr << 40);     // :140-143
      uint64_t fs = f & seed_mask, rs = r & seed_mask;   // :145-146
      bool canonical = rs > fs;                          // :147 (signed compare of <2^42 operands)
      uint64_t seed = canonical ? fs : rs;               // :149-150 blendv picks f where compare is set
      uint64_t h = mm_hash64(seed);
      if (h < threshold && resume <= i) {                // :179,202,225,248
        sk.add_seed_position((uint32_t)seed,
                             SeedPosition{(uint32_t)(i + len * lane), (contig_index << 1) | (canonical ? 1u : 0u)});
        uint64_t marker = (r > f) ? f : r;               // :148,188-194
        if (h < threshold_marker) sk.marker_seeds.insert(marker);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// needletail 0.5.1 parse_fastx_file, restated (SURVEY App. D.6): gz via zlib (multi-member ok),
// format sniffed from the first byte, FASTA seq() with \n / \r removed, id() = whole header line.
// ------------------------------------------------------------------------------------------------
namespace {
struct FastxRecord { std::string id; std::string seq; };

bool read_whole_file(const std::string& path, std::string& out) {
  gzFile f = gzopen(path.c_str(), "rb");
  if (!f) return false;
  gzbuffer(f, 1 << 20);
  out.clear();
  std::vector<char> buf(1 << 22);
  while (true) {
    int got = gzread(f, buf.data(), (unsigned)buf.size());
    if (got < 0) { gzclose(f); return false; }
    if (got == 0) break;
    out.append(buf.data(), (size_t)got);
  }
  gzclose(f);
  return true;
}

// returns false on a parse error (file is then skipped with a warning); records are appended
bool parse_fastx(const std::string& data, std::vector<FastxRecord>& recs) {
  size_t p = 0, n = data.size();
  // needletail skips nothing: first byte decides
  if (n == 0) return false;  // EmptyFile error
  char first = data[0];
  if (first != '>' && first != '@') return false;
  auto read_line = [&](size_t& pos, size_t& b, size_t& e) {  // [b,e) without terminator
    b = pos;
    const char* nl = (const char*)memchr(data.data() + pos, '\n', n - pos);
    size_t end = nl ? (size_t)(nl - data.data()) : n;
    pos = nl ? end + 1 : n;
    e = end;
    if (e > b && data[e - 1] == '\r') e--;
  };
  if (first == '>') {
    while (p < n) {
      if (data[p] != '>') return false;
      size_t b, e;
      read_line(p, b, e);
      FastxRecord r;
      r.id.assign(data, b + 1, e - b - 1);
      // sequence: everything up to the next line that starts with '>'
      while (p < n && data[p] != '>') {
        size_t lb, le;
        read_line(p, lb, le);
        r.seq.append(data, lb, le - lb);
      }
      recs.push_back(std::move(r));
    }
  } else {
    while (p < n) {
      // tolerate trailing blank lines at EOF
      if (data[p] == '\n' || data[p] == '\r') { p++; continue; }
      if (data[p] != '@') return false;
      size_t b, e;
      read_line(p, b, e);
      FastxRecord r;
      r.id.assign(data, b + 1, e - b - 1);
      if (p >= n) return false;
      size_t sb, se;
      read_line(p, sb, se);
      r.seq.assign(data, sb, se - sb);
      if (p >= n || data[p] != '+') return false;
      size_t pb, pe;
      read_line(p, pb, pe);
      size_t qb, qe;
      if (p > n) return false;
      read_line(p, qb, qe);
      if (qe - qb != se - sb) return false;
      recs.push_back(std::move(r));
    }
  }
  return true;
}
}  // namespace

Sketch sketch_from_contigs(const std::string& file_name, const std::vector<std::pair<const uint8_t*, size_t>>& contigs,
                           const std::vector<std::string>* names, const SketchParams& sp, bool use_avx2_semantics) {
  Sketch sk;  // Sketch::new (types.rs:342-351): marker_c field is set to c (quirk, types.rs:347)
  sk.file_name = file_name;
  sk.c = sp.c; sk.k = sp.k; sk.marker_c = sp.c;
  uint32_t j = 0;
  for (size_t i = 0; i < contigs.size(); i++) {
    if (contigs[i].second < MIN_LENGTH_CONTIG) continue;  // file_io.rs:176
    sk.contigs.push_back(names ? (*names)[i] : ("contig" + std::to_string(i)));
    sk.contig_lengths.push_back((uint32_t)contigs[i].second);
    sk.total_sequence_length += contigs[i].second;
    if (use_avx2_semantics) fmh_seeds_avx2sem(contigs[i].first, contigs[i].second, sp, j, sk);
    else fmh_seeds_scalar(contigs[i].first, contigs[i].second, sp, j, sk);
    j++;
  }
  return sk;
}

std::vector<Sketch> fastx_to_sketches(const std::vector<std::string>& files, const SketchParams& sp,
                                      bool individual_contig, bool use_avx2_semantics, int threads,
                                      std::vector<std::string>* warn) {
  std::vector<std::vector<Sketch>> per_file(files.size());
  std::vector<std::string> warns(files.size());
  (void)threads;
#pragma omp parallel for schedule(dynamic) num_threads(threads > 0 ? threads : 1)
  for (long fi = 0; fi < (long)files.size(); fi++) {
    const std::string& path = files[fi];
    std::string data;
    std::vector<FastxRecord> recs;
    if (!read_whole_file(path, data) || !parse_fastx(data, recs)) {
      warns[fi] = path + " is not a valid fasta/fastq file; skipping.";  // file_io.rs:159-166,232-236
      continue;
    }
    if (!individual_contig) {  // file_io.rs:141-252
      std::vector<std::pair<const uint8_t*, size_t>> ctgs;
      std::vector<std::string> names;
      for (auto& r : recs) { ctgs.push_back({(const uint8_t*)r.seq.data(), r.seq.size()}); names.push_back(r.id); }
      Sketch sk = sketch_from_contigs(path, ctgs, &names, sp, use_avx2_semantics);
      if (sk.contigs.empty()) {
        warns[fi] = "File " + path + " consists of only contigs < 500 bp. Skipping this file.";  // file_io.rs:244-246
        continue;
      }
      per_file[fi].push_back(std::move(sk));
    } else {  // file_io.rs:253-362: one sketch per kept record, contig_index 0, contig_order = rank
      uint64_t j = 0;
      for (auto& r : recs) {
        if (r.seq.size() < MIN_LENGTH_CONTIG) continue;
        Sketch sk;
        sk.file_name = path;
        sk.c = sp.c; sk.k = sp.k; sk.marker_c = sp.c;
        sk.contigs.push_back(r.id);
        sk.contig_lengths.push_back((uint32_t)r.seq.size());
        sk.total_sequence_length = r.seq.size();
        if (use_avx2_semantics) fmh_seeds_avx2sem((const uint8_t*)r.seq.data(), r.seq.size(), sp, 0, sk);
        else fmh_seeds_scalar((const uint8_t*)r.seq.data(), r.seq.size(), sp, 0, sk);
        sk.contig_order = j;
        sk.individual_contig = true;
        per_file[fi].push_back(std::move(sk));
        j++;
      }
    }
  }
  std::vector<Sketch> out;
  for (size_t fi = 0; fi < files.size(); fi++) {
    if (!warns[fi].empty() && warn) warn->push_back(warns[fi]);
    for (auto& s : per_file[fi]) out.push_back(std::move(s));
  }
  // types.rs:360-364: order by (file_name bytes, contig_order)
  std::stable_sort(out.begin(), out.end(), [](const Sketch& a, const Sketch& b) {
    if (a.file_name != b.file_name) return a.file_name < b.file_name;
    return a.contig_order < b.contig_order;
  });
  return out;
}

// ------------------------------------------------------------------------------------------------
// screen.rs
// ------------------------------------------------------------------------------------------------
struct KmerToSketch {
  std::unordered_map<uint64_t, std::vector<uint32_t>> map;
};

KmerToSketch* kmer_to_sketch_from_refs(const std::vector<const Sketch*>& refs) {  // screen.rs:190-210 (serial)
  auto* idx = new KmerToSketch();
  size_t total = 0;
  for (auto* r : refs) total += r->marker_seeds.size();
  idx->map.reserve(total);
  for (size_t i = 0; i < refs.size(); i++) {
    const MarkerSet& ms = refs[i]->marker_seeds;
    for (size_t s = 0; s < ms.capacity(); s++)
      if (ms.slot_used(s)) idx->map[ms.slot_key(s)].push_back((uint32_t)i);
  }
  return idx;
}
void kmer_to_sketch_free(KmerToSketch* p) { delete p; }

static inline double powi21(double x) {  // f64::powi(x, 21): repeated multiplication (llvm.powi), not libm pow
  // llvm's __powidf2: square-and-multiply from the low bit upward
  double r = 1.0, a = x;
  int b = K_MARKER_DNA;
  while (true) {
    if (b & 1) r *= a;
    b /= 2;
    if (b == 0) break;
    a *= a;
  }
  return r;
}

static std::vector<uint32_t> screen_common(double identity, const KmerToSketch& idx, const Sketch& q,
                                           const std::vector<const Sketch*>& refs) {
  std::unordered_map<uint32_t, size_t> count;
  const MarkerSet& ms = q.marker_seeds;
  for (size_t s = 0; s < ms.capacity(); s++) {
    if (!ms.slot_used(s)) continue;
    auto it = idx.map.find(ms.slot_key(s));
    if (it == idx.map.end()) continue;
    for (uint32_t id : it->second) count[id]++;
  }
  double cutoff = powi21(identity);  // screen.rs:60,176
  std::vector<uint32_t> ret;
  for (auto& kv : count) {
    size_t mn = std::min(refs[kv.first]->marker_seeds.size(), q.marker_seeds.size());
    size_t thr = std::max((size_t)(cutoff * (double)mn), (size_t)1);  // screen.rs:65-70,180-185
    if (kv.second > thr) ret.push_back(kv.first);
  }
  std::sort(ret.begin(), ret.end());
  return ret;
}

std::vector<uint32_t> screen_refs(double identity, const KmerToSketch& idx, const Sketch& q,
                                  const std::vector<const Sketch*>& refs, bool rescue_small) {
  if (q.marker_seeds.size() < 20 && rescue_small) {  // screen.rs:158-160
    std::vector<uint32_t> all(refs.size());
    for (size_t i = 0; i < refs.size(); i++) all[i] = (uint32_t)i;
    return all;
  }
  return screen_common(identity, idx, q, refs);
}

std::vector<uint32_t> screen_refs_indices(double identity, const KmerToSketch& idx, const Sketch& q,
                                          const std::vector<const Sketch*>& refs) {
  return screen_common(identity, idx, q, refs);
}

bool check_markers_quickly(const Sketch& ref, const Sketch& query, double screen_val, bool rescue_small) {
  if (screen_val == 0.) return true;  // screen.rs:91-93
  const MarkerSet *seeds1, *seeds2;
  size_t min_card;
  if (query.marker_seeds.size() > ref.marker_seeds.size()) {  // screen.rs:98-107
    seeds1 = &ref.marker_seeds; seeds2 = &query.marker_seeds; min_card = ref.marker_seeds.size();
  } else {
    seeds2 = &ref.marker_seeds; seeds1 = &query.marker_seeds; min_card = query.marker_seeds.size();
  }
  if (min_card < SCREEN_MINIMUM_KMERS && rescue_small) return true;  // screen.rs:108-110
  if (min_card == 0) return rescue_small;                            // screen.rs:112-119
  size_t ratio = (size_t)(powi21(screen_val) * (double)min_card);    // screen.rs:124-125
  if (ratio == 0) ratio = 1;
  size_t inter = 0;
  for (size_t s = 0; s < seeds1->capacity(); s++) {  // screen.rs:131-138
    if (!seeds1->slot_used(s)) continue;
    if (seeds2->contains(seeds1->slot_key(s))) inter++;
    if (inter >= ratio) return true;
  }
  return false;
}

// ------------------------------------------------------------------------------------------------
// gbdt 0.1.1 GBDT::predict for LAD loss, initial_guess disabled (SURVEY App. D.5)
// ------------------------------------------------------------------------------------------------
#include "gbdt_tables.inc"
static inline float bits2f(uint32_t b) { float f; std::memcpy(&f, &b, 4); return f; }

float gbdt_predict(int model, const float x[5]) {
  const unsigned char* feat = model == 0 ? SK_GBDT_C125_FEAT : SK_GBDT_C200_FEAT;
  const unsigned int* thr = model == 0 ? SK_GBDT_C125_THR : SK_GBDT_C200_THR;
  const unsigned int* leaf = model == 0 ? SK_GBDT_C125_LEAF : SK_GBDT_C200_LEAF;
  const int ntrees = model == 0 ? SK_GBDT_C125_NTREES : SK_GBDT_C200_NTREES;
  const float shrink = bits2f(model == 0 ? SK_GBDT_C125_SHRINK_BITS : SK_GBDT_C200_SHRINK_BITS);
  volatile float v = bits2f(model == 0 ? SK_GBDT_C125_BIAS_BITS : SK_GBDT_C200_BIAS_BITS);
  for (int t = 0; t < ntrees; t++) {
    const unsigned char* f = feat + 7 * t;
    const unsigned int* th = thr + 7 * t;
    // heap-ordered complete depth-3 tree: node 0 root; children of i are 2i+1 (x < thr) and 2i+2
    int node = 0;
    for (int d = 0; d < 3; d++) node = 2 * node + ((x[f[node]] < bits2f(th[node])) ? 1 : 2);
    float pred = bits2f(leaf[8 * t + (node - 7)]);
    volatile float prod = shrink * pred;  // f32 multiply, then f32 add (no fma contraction)
    v = v + prod;
  }
  return v;
}

int get_model_id(uint64_t c, bool learned_ani) {  // regression.rs:12-28
  if (!learned_ani) return -1;
  long d125 = std::labs((long)c - 125), d200 = std::labs((long)c - 200);
  return d125 < d200 ? 0 : 1;
}

// ------------------------------------------------------------------------------------------------
// chain.rs
// ------------------------------------------------------------------------------------------------
MapParams map_params_from_sketch(const Sketch& ref, const CommandParams& cp, int model) {  // chain.rs:88-142
  MapParams mp;
  mp.max_gap_length = D_MAX_GAP_LENGTH;
  mp.anchor_score = D_ANCHOR_SCORE_ANI;
  mp.min_anchors = D_MIN_ANCHORS_ANI;
  mp.min_length_cover = MIN_LENGTH_COVER;
  mp.fragment_length = CHUNK_SIZE_DNA;  // params.rs:125-134
  double fcc = cp.min_aligned_frac;
  if (fcc < 0.) fcc = 15.0 / 100.;  // chain.rs:101-107
  mp.frac_cover_cutoff = fcc;
  mp.both_frac_cover_cutoff = cp.both_min_aligned_frac;
  mp.bp_chain_band = BP_CHAIN_BAND;
  mp.index_chain_band = BP_CHAIN_BAND / ref.c;              // chain.rs:112
  mp.min_score = (double)mp.min_anchors * mp.anchor_score * 0.75;  // chain.rs:113
  mp.k = ref.k;
  mp.robust = cp.robust;
  mp.median = cp.median;
  mp.model = model;
  return mp;
}

static bool switch_qr(double med_ctg_len_r, double med_ctg_len_q, double q_sk_len, double r_sk_len,
                      const std::string& qname, const std::string& rname) {  // chain.rs:15-26
  double score_query = q_sk_len * std::min(med_ctg_len_q, 300000.);
  double score_ref = r_sk_len * std::min(med_ctg_len_r, 300000.);
  if (score_query == score_ref) return qname > rname;
  return score_query > score_ref;
}

static inline bool anchor_less(const Anchor& a, const Anchor& b) {  // derived Ord (types.rs:499-506)
  if (a.query_contig != b.query_contig) return a.query_contig < b.query_contig;
  if (a.query_pos != b.query_pos) return a.query_pos < b.query_pos;
  if (a.ref_contig != b.ref_contig) return a.ref_contig < b.ref_contig;
  if (a.ref_pos != b.ref_pos) return a.ref_pos < b.ref_pos;
  return a.reverse_match < b.reverse_match;
}

struct AnchorChunks {  // types.rs:545-550
  std::vector<std::vector<Anchor>> chunks;
  std::vector<uint32_t> lengths;
  std::vector<std::vector<uint32_t>> seeds_in_chunk;
};

static bool get_anchors(const Sketch& ref_sketch, const Sketch& query_sketch, const MapParams& mp,
                        AnchorChunks& out, std::vector<Anchor>* dbg_anchors) {  // chain.rs:608-836; returns `switched`
  if (ref_sketch.contig_lengths.empty() || query_sketch.contig_lengths.empty()) return true;  // :618-620
  auto mean_len = [](const Sketch& s) {
    double sum = 0;
    for (uint32_t x : s.contig_lengths) sum += (double)x;
    return sum / (double)s.contig_lengths.size();
  };
  double mean_q = mean_len(query_sketch), mean_r = mean_len(ref_sketch);  // :626-633
  double qproxy, rproxy;
  if (query_sketch.total_sequence_length > 100000 && ref_sketch.total_sequence_length > 100000) {  // :643-650
    qproxy = (double)query_sketch.marker_seeds.size() * (double)query_sketch.c;
    rproxy = (double)ref_sketch.marker_seeds.size() * (double)ref_sketch.c;
  } else {
    qproxy = (double)query_sketch.total_sequence_length;
    rproxy = (double)ref_sketch.total_sequence_length;
  }
  bool switched = switch_qr(mean_r, mean_q, qproxy, rproxy, query_sketch.file_name, ref_sketch.file_name);  // :651
  const Sketch& Q = switched ? ref_sketch : query_sketch;  // iterated + chunked side
  const Sketch& R = switched ? query_sketch : ref_sketch;  // probed side
  std::vector<std::vector<uint32_t>> qpos_all(Q.contigs.size());  // :656,662
  std::vector<Anchor> anchors;
  const KmerSeeds& qmap = Q.kmer_seeds_k;
  SeedPosition tq, tr;
  for (size_t s = 0; s < qmap.capacity(); s++) {  // :668-713
    if (!qmap.slot_used(s)) continue;
    uint32_t kmer = qmap.slot_key(s);
    const SeedPosition* qp;
    size_t nq = Q.get_seed_positions(kmer, &qp, &tq);
    if (nq > mp.index_chain_band) continue;  // :676-678
    const SeedPosition* rp;
    size_t nr = R.get_seed_positions(kmer, &rp, &tr);
    if (nr == 0) {  // !contains (:684-687)
      for (size_t a = 0; a < nq; a++) qpos_all[qp[a].contig_index()].push_back(qp[a].pos);
    } else {
      if (nr > mp.index_chain_band) continue;  // :695-697
      for (size_t a = 0; a < nq; a++) qpos_all[qp[a].contig_index()].push_back(qp[a].pos);
      for (size_t a = 0; a < nq; a++)
        for (size_t b = 0; b < nr; b++)
          anchors.push_back(Anchor{qp[a].contig_index(), qp[a].pos, rp[b].contig_index(), rp[b].pos,
                                   rp[b].canonical() != qp[a].canonical()});  // :704-711
    }
  }
  if (anchors.empty()) return true;  // :714-720 (returns switched = true)
  std::sort(anchors.begin(), anchors.end(), anchor_less);  // :721
  for (auto& v : qpos_all) std::sort(v.begin(), v.end());  // :722-724
  if (dbg_anchors) *dbg_anchors = anchors;

  // chunking, :738-836
  const uint32_t F = mp.fragment_length;
  std::vector<Anchor> cur;
  uint32_t last_ctg = anchors[0].query_contig;
  uint32_t end = anchors[0].query_pos + F;
  size_t rc = 0;
  for (const Anchor& a : anchors) {
    if (last_ctg != a.query_contig || a.query_pos > end) {
      const auto& qv = qpos_all[last_ctg];
      // (:749-752 warn-and-continue branch is unreachable: a contig with anchors has query positions)
      std::vector<uint32_t> seeds;
      while (rc < qv.size() && qv[rc] <= end) { seeds.push_back(qv[rc]); rc++; }  // :756-782
      out.seeds_in_chunk.push_back(std::move(seeds));
      end += F;                                  // :784
      out.chunks.push_back(std::move(cur));      // :785
      cur.clear();
      out.lengths.push_back(F);                  // :787
      if (last_ctg != a.query_contig) {          // :788-791
        end = a.query_pos + F;
        rc = 0;
      }
    }
    last_ctg = a.query_contig;
    cur.push_back(a);
  }
  if (!cur.empty()) {  // :796-824
    const auto& qv = qpos_all[last_ctg];
    std::vector<uint32_t> seeds;
    uint32_t lastpos = cur.back().query_pos;
    while (rc < qv.size() && qv[rc] <= lastpos) { seeds.push_back(qv[rc]); rc++; }
    out.lengths.push_back(cur.back().query_pos - cur.front().query_pos);
    out.chunks.push_back(std::move(cur));
    out.seeds_in_chunk.push_back(std::move(seeds));
  }
  return switched;
}

// partitions 0.2.4 (git adf36eea) PartitionVec, restated (SURVEY App. D.1)
struct PartitionVec {
  std::vector<uint32_t> parent, rank, link;
  void push() {
    uint32_t i = (uint32_t)parent.size();
    parent.push_back(i); rank.push_back(0); link.push_back(i);
  }
  uint32_t find(uint32_t i) {
    while (parent[i] != i) { parent[i] = parent[parent[i]]; i = parent[i]; }  // path halving: order of link list unaffected
    return i;
  }
  void unite(uint32_t a, uint32_t b) {
    uint32_t i = find(a), j = find(b);
    if (i == j) return;
    std::swap(link[i], link[j]);  // splice the two circular lists
    if (rank[i] < rank[j]) parent[i] = j;
    else if (rank[i] == rank[j]) { parent[i] = j; rank[j] += 1; }
    else parent[j] = i;
  }
  size_t len_of_set(uint32_t i) {
    size_t n = 1;
    for (uint32_t c = link[i]; c != i; c = link[c]) n++;
    return n;
  }
};

struct ChainingResult {  // types.rs:488-493
  std::vector<size_t> pointer_vec;
  PartitionVec chain_part;
  std::vector<double> score_vec;
};

static inline double score_anchors(const Anchor& cur, const Anchor& past, const MapParams& mp) {  // chain.rs:557-603
  const double NEG = std::numeric_limits<double>::lowest();  // f64::MIN
  if (cur.reverse_match != past.reverse_match) return NEG;
  if (cur.ref_pos == past.ref_pos || cur.query_pos == past.query_pos) return NEG;
  double acq = cur.query_pos, apq = past.query_pos, acr = cur.ref_pos, apr = past.ref_pos;
  double d_q = std::fabs(acq - apq);
  double d_r = cur.reverse_match ? (apr - acr) : (acr - apr);
  if (d_q > D_MAX_LIN_LENGTH || d_r > D_MAX_LIN_LENGTH) return NEG;
  if (d_r <= 0.) return NEG;
  double gap = std::fabs(d_r - d_q);
  if (gap > mp.max_gap_length) return NEG;
  return mp.anchor_score - gap;
}

static std::vector<ChainingResult> chain_anchors_ani(const std::vector<std::vector<Anchor>>& chunks,
                                                     const MapParams& mp) {  // chain.rs:838-896
  std::vector<ChainingResult> res;
  const double NEG = std::numeric_limits<double>::lowest();
  uint32_t past_chain_length = std::min<uint32_t>(mp.fragment_length / 2, mp.bp_chain_band);  // :842
  for (const auto& chunk : chunks) {
    ChainingResult cr;
    size_t n = chunk.size();
    cr.pointer_vec.assign(n, 0);
    cr.score_vec.assign(n, 0.);
    for (size_t i = 0; i < n; i++) {
      cr.chain_part.push();
      const Anchor& cur = chunk[i];
      double best = 0.;
      size_t best_prev = i;
      for (size_t jj = i; jj-- > 0;) {
        const Anchor& past = chunk[jj];
        if (cur.ref_contig != past.ref_contig) continue;  // :856-858 (before the break test)
        if (cur.query_pos - past.query_pos > past_chain_length || i - jj > mp.index_chain_band) break;  // :859-863
        double sc = score_anchors(cur, past, mp);
        if (sc == NEG) continue;
        double ns = sc + cr.score_vec[jj];
        if (ns > best) { best = ns; best_prev = jj; }  // strict > : first met (largest j) wins ties
      }
      cr.score_vec[i] = best;
      cr.pointer_vec[i] = best_prev;
      if (best_prev != i) cr.chain_part.unite((uint32_t)i, (uint32_t)best_prev);  // :883-885
    }
    res.push_back(std::move(cr));
  }
  return res;
}

static void get_chain_intervals(std::vector<ChainInterval>& good, ChainingResult& cr, const std::vector<Anchor>& anchors,
                                const MapParams& mp, size_t chunk_id) {  // chain.rs:939-1007
  size_t n = anchors.size();
  std::vector<uint8_t> done(n, 0);
  for (uint32_t s = 0; s < n; s++) {  // all_sets(): sets in order of first appearance of their root
    uint32_t root = cr.chain_part.find(s);
    if (done[root]) continue;
    done[root] = 1;
    bool small_chain = false, first_iter = true;
    double max_score = std::numeric_limits<double>::lowest();
    size_t best_index = SIZE_MAX;
    size_t num_anchors = 1;
    uint32_t idx = root;
    do {  // iterate the set: root first, then along `link`
      if (first_iter) {
        if (cr.chain_part.len_of_set(idx) < mp.min_anchors) { small_chain = true; break; }
        first_iter = false;
      }
      if (cr.score_vec[idx] > max_score) { max_score = cr.score_vec[idx]; best_index = idx; }
      idx = cr.chain_part.link[idx];
    } while (idx != root);
    if (small_chain) continue;
    size_t index = best_index;
    while (cr.pointer_vec[index] != index) { index = cr.pointer_vec[index]; num_anchors++; }  // :969-973
    small_chain = num_anchors < mp.min_anchors;
    if (small_chain || max_score < mp.min_score) continue;  // :974-977
    size_t smallest = index, largest = best_index;
    ChainInterval ci;
    ci.q0 = anchors[smallest].query_pos; ci.q1 = anchors[largest].query_pos;
    uint32_t e1 = anchors[smallest].ref_pos, e2 = anchors[largest].ref_pos;
    ci.r0 = std::min(e1, e2); ci.r1 = std::max(e1, e2);
    ci.ref_contig = anchors[smallest].ref_contig;
    ci.query_contig = anchors[smallest].query_contig;
    ci.score = max_score;
    ci.num_anchors = num_anchors;
    ci.chunk_id = chunk_id;
    ci.reverse_chain = anchors[smallest].reverse_match;
    ci.overlap = 0;
    good.push_back(ci);
  }
}

static inline int cmp_interval(const ChainInterval& x, const ChainInterval& y) {  // derived PartialOrd, types.rs:508-519
#define ORC_CMP(f) if (x.f < y.f) return -1; if (x.f > y.f) return 1;
  ORC_CMP(score) ORC_CMP(num_anchors) ORC_CMP(q0) ORC_CMP(q1) ORC_CMP(r0) ORC_CMP(r1)
  ORC_CMP(ref_contig) ORC_CMP(query_contig) ORC_CMP(chunk_id) ORC_CMP(reverse_chain) ORC_CMP(overlap)
#undef ORC_CMP
  return 0;
}

std::vector<std::vector<ChainInterval>> get_nonoverlapping_chains(std::vector<ChainInterval>& intervals, size_t num_chunks,
                                                                  std::vector<uint8_t>* kept, std::vector<uint32_t>* hits_out) {
  // chain.rs:1008-1099.  bio IntervalTree (half-open overlap query) is restated as per-contig lists.
  std::stable_sort(intervals.begin(), intervals.end(),
                   [](const ChainInterval& a, const ChainInterval& b) { return cmp_interval(b, a) < 0; });  // :1012 descending
  std::unordered_map<size_t, std::vector<size_t>> tree_q, tree_r;
  std::vector<std::vector<ChainInterval>> good(num_chunks);
  if (kept) kept->assign(intervals.size(), 0);
  if (hits_out) hits_out->assign(2 * intervals.size(), 0);
  for (size_t i = 0; i < intervals.size(); i++) {
    const ChainInterval& it = intervals[i];
    auto& tr = tree_r[it.ref_contig];
    auto& tq = tree_q[it.query_contig];
    uint32_t sum_r = 0, sum_q = 0;
    bool no_overlap_ref, no_overlap_query;
    size_t hits = 0;
    for (size_t o : tr) {
      const ChainInterval& ol = intervals[o];
      if (ol.r0 < it.r1 && it.r0 < ol.r1) {  // half-open overlap
        hits++;
        sum_r += std::min(it.r1 - ol.r0, ol.r1 - it.r0);  // :1034-1038
      }
    }
    if (hits_out) (*hits_out)[2 * i] = (uint32_t)hits;
    if (hits == 0) no_overlap_ref = true;
    else no_overlap_ref = ((float)sum_r < (float)(it.r1 - it.r0) * OVERLAP_ORTHOLOGOUS_FRACTION);  // :1042
    hits = 0;
    for (size_t o : tq) {
      const ChainInterval& ol = intervals[o];
      if (ol.q0 < it.q1 && it.q0 < ol.q1) {
        hits++;
        sum_q += std::min(it.q1 - ol.q0, ol.q1 - it.q0);  // :1064-1068
      }
    }
    if (hits_out) (*hits_out)[2 * i + 1] = (uint32_t)hits;
    if (hits == 0) no_overlap_query = true;
    else no_overlap_query = ((float)sum_q < (float)(it.q1 - it.q0) * OVERLAP_ORTHOLOGOUS_FRACTION);  // :1072
    if (no_overlap_ref && no_overlap_query) {
      tq.push_back(i);
      // same contig key may alias tr/tq only across the two maps, never within one
      tree_r[it.ref_contig].push_back(i);
      good[it.chunk_id].push_back(it);  // pushed with overlap left at 0 (:1091-1093)
      if (kept) (*kept)[i] = 1;
    }
  }
  return good;
}

// fastrand 1.9.0 (WyRand + Lemire), SURVEY App. D.4
struct WyRand {
  uint64_t state;
  uint64_t next() {
    state += 0xA0761D6478BD642Full;
    __uint128_t t = (__uint128_t)state * (__uint128_t)(state ^ 0xE7037ED1A0B428DBull);
    return (uint64_t)t ^ (uint64_t)(t >> 64);
  }
  uint64_t below(uint64_t n) {  // usize(..n)
    uint64_t r = next();
    __uint128_t m = (__uint128_t)r * n;
    uint64_t hi = (uint64_t)(m >> 64), lo = (uint64_t)m;
    if (lo < n) {
      uint64_t t = (0 - n) % n;
      while (lo < t) {
        r = next();
        m = (__uint128_t)r * n;
        hi = (uint64_t)(m >> 64); lo = (uint64_t)m;
      }
    }
    return hi;
  }
};

static void bootstrap_interval(const std::vector<std::pair<double, size_t>>& ani_ests, double& lo, double& hi, double& sd) {
  // chain.rs:57-86 (+ mean :28-37, std_deviation :39-55)
  size_t n = ani_ests.size();
  double sum = 0;
  for (auto& e : ani_ests) sum += e.first;
  if (n == 0) sd = 0.;
  else {
    double mean = sum / (double)n;
    double var = 0;
    for (auto& e : ani_ests) { double d = mean - e.first; var += d * d; }
    sd = std::sqrt(var / (double)n);
  }
  if (n < 10) { lo = 0.; hi = 1.; return; }  // :65-67
  std::vector<double> pool;
  for (auto& e : ani_ests) for (size_t m = 0; m < e.second; m++) pool.push_back(e.first);
  WyRand rng{7};  // fastrand::seed(7)
  const int iters = 100;
  std::vector<double> res;
  std::vector<size_t> rand_vec(n);
  for (int it = 0; it < iters; it++) {
    for (size_t s = 0; s < n; s++) rand_vec[s] = (size_t)rng.below(pool.size());
    double ssum = 0;
    for (size_t s = 0; s < n; s++) ssum += pool[rand_vec[s]];
    res.push_back(ssum / (double)n);
  }
  std::sort(res.begin(), res.end());
  lo = res[iters * 5 / 100 - 1];
  hi = res[iters * 95 / 100 - 1];
}

static void predict_from_ani_res(AniEstResult& a, int model) {  // regression.rs:30-64
  if (a.ani > 0.9f && a.total_bases_covered > TOTAL_BASES_REGRESS_CUTOFF) {
    float x[5];
    x[0] = a.ani * 100.f;
    x[1] = a.std;
    if (a.quant_50_contig_len_r > a.quant_50_contig_len_q) { x[2] = a.quant_90_contig_len_r; x[3] = a.quant_90_contig_len_q; }
    else { x[2] = a.quant_90_contig_len_q; x[3] = a.quant_90_contig_len_r; }
    x[4] = (float)a.avg_chain_int_len;
    float pred = gbdt_predict(model, x);
    if (pred < 100.f) {
      a.ci_upper = (a.ci_upper - a.ani) + pred / 100.f;
      a.ci_lower = (a.ci_lower - a.ani) + pred / 100.f;
      a.ani = pred / 100.f;
    }
  }
}

AniEstResult final_estimate(const std::vector<std::pair<double, size_t>>& ani_ests, uint32_t total_query_bases,
                            uint32_t avg_chain_int_len, uint64_t query_total_len, uint64_t ref_total_len,
                            const float quant_q[3], const float quant_r[3], const MapParams& mp) {  // chain.rs:422-555
  if (ani_ests.empty()) {  // :416-420
    AniEstResult r;
    r.ani = std::numeric_limits<float>::quiet_NaN();
    return r;
  }
  size_t total_mult = 0;
  for (auto& e : ani_ests) total_mult += e.second;
  double lower, upper;
  if (mp.median) { lower = 0.499; upper = 0.501; }
  else if (mp.robust) { lower = 0.10; upper = 0.90; }
  else { lower = 0.; upper = 1.; }
  size_t lower_i = 0, upper_i = ani_ests.size() - 1;
  bool changed_l = false, changed_u = false;
  size_t curr = 0;
  for (size_t i = 0; i < ani_ests.size(); i++) {  // :448-460
    curr += ani_ests[i].second;
    if (curr >= (size_t)((double)total_mult * lower) && !changed_l) { lower_i = i; changed_l = true; }
    if (curr >= (size_t)((double)total_mult * upper) && !changed_u) { upper_i = i + 1; changed_u = true; break; }
  }
  size_t tm2 = 0;
  double weighted = 0.;
  for (size_t i = lower_i; i < upper_i; i++) {  // :462-469
    weighted += ani_ests[i].first * (double)ani_ests[i].second;
    tm2 += ani_ests[i].second;
  }
  double final_ani = weighted / (double)tm2;
  double ci_lo, ci_hi, sd;
  bootstrap_interval(ani_ests, ci_lo, ci_hi, sd);
  double covered_query = std::min(1., (double)total_query_bases / (double)query_total_len);  // :477-480
  double covered_ref = std::min(1., (double)total_query_bases / (double)ref_total_len);      // :481-484
  if (mp.both_frac_cover_cutoff > 0.0) {  // :500-505
    if (covered_query < mp.both_frac_cover_cutoff || covered_ref < mp.both_frac_cover_cutoff) final_ani = -1.;
  } else if (covered_query < mp.frac_cover_cutoff && covered_ref < mp.frac_cover_cutoff) {  // :513-516
    final_ani = -1.;
  }
  AniEstResult r;
  r.ani = (float)final_ani;
  r.align_fraction_query = (float)covered_query;
  r.align_fraction_ref = (float)covered_ref;
  r.ci_upper = (float)ci_hi;
  r.ci_lower = (float)ci_lo;
  r.quant_10_contig_len_q = quant_q[0];
  r.quant_50_contig_len_q = quant_q[1];
  r.quant_90_contig_len_q = quant_q[2];
  r.quant_10_contig_len_r = quant_r[0];
  r.quant_50_contig_len_r = quant_r[1];
  r.quant_90_contig_len_r = quant_r[2];
  r.std = (float)sd;
  r.avg_chain_int_len = avg_chain_int_len;
  r.total_bases_covered = total_query_bases;
  if (mp.model >= 0) predict_from_ani_res(r, mp.model);
  return r;
}

uint32_t padded_start(uint32_t q0, uint32_t c) {  // chain.rs:239-240: i32::max(q0 as i32 - c as i32, 0), wrapping i32 subtraction
  const uint32_t d = q0 - c;                       // the same wrap in u32 (no signed overflow)
  return (int32_t)d > 0 ? d : 0u;
}

void chunk_estimate(ChunkStats& s, uint32_t c, size_t k, uint32_t min_length_cover) {  // chain.rs:253-394
  s.valid = s.filtered = false;
  s.est = 0.; s.weight = 0;
  if (s.total_anchors == 0) return;                  // :253-255
  if (s.rq1 - s.rq0 < min_length_cover) return;      // :257-259
  size_t considered = s.n_seeds;
  double putative = std::pow((double)s.total_anchors / (double)s.num_in, 1. / (double)k);  // :331-335
  if (putative > 0.950 && s.tbcq > c * 4 && s.rq1 - s.rq0 < (uint32_t)(CHUNK_SIZE_DNA * 9 / 10) &&
      (double)considered > 1.05 * (double)s.upper_lower) {  // :336-347
    considered = s.upper_lower;
    s.filtered = true;
  }
  double ml_hits = std::min(1., (double)s.total_anchors / (double)considered);  // :368-372
  s.est = std::pow(ml_hits, 1. / (double)k);                                     // :373-377
  s.weight = considered;                                                         // :394
  s.valid = true;
}

ChunkStats chunk_stats(const std::vector<ChainInterval>& intervals, const std::vector<uint32_t>& seeds, uint32_t c, size_t k,
                       uint32_t min_length_cover, bool switched) {  // chain.rs:204-394
  ChunkStats s;
  std::vector<std::pair<uint32_t, uint32_t>> all_intervals;  // closed intervals; union realised lazily (only contains() matters)
  for (const auto& in : intervals) {
    s.total_anchors += in.num_anchors;
    if (in.q0 < s.rq0) s.rq0 = in.q0;
    if (in.q1 > s.rq1) s.rq1 = in.q1;
    if (!switched) s.tbcq += in.q1 - in.q0 + (uint32_t)k + 2 * c;  // :223-237
    else s.tbcq += in.r1 - in.r0 + (uint32_t)k + 2 * c;
    all_intervals.push_back({padded_start(in.q0, c), in.q1 + c});  // :239-240
    s.n_int++;
  }
  s.n_seeds = seeds.size();
  if (s.n_int) {
    for (uint32_t pos : seeds) {
      bool in = false;
      for (auto& iv : all_intervals) if (iv.first <= pos && pos <= iv.second) { in = true; break; }
      if (in) s.num_in++;
      if (pos >= s.rq0 && pos <= s.rq1) s.upper_lower++;  // :322-328 with both spacing estimates 0 (extend = 0, :295)
    }
  }
  chunk_estimate(s, c, k, min_length_cover);
  return s;
}

std::vector<ChainInterval> chain_chunks(const std::vector<std::vector<Anchor>>& chunks, const MapParams& mp,
                                        std::vector<double>* score, std::vector<uint32_t>* pointer) {  // chain.rs:151-153
  std::vector<ChainingResult> crs = chain_anchors_ani(chunks, mp);
  std::vector<ChainInterval> good;
  for (size_t i = 0; i < chunks.size(); i++) {
    get_chain_intervals(good, crs[i], chunks[i], mp, i);
    if (score) score->insert(score->end(), crs[i].score_vec.begin(), crs[i].score_vec.end());
    if (pointer) for (size_t p : crs[i].pointer_vec) pointer->push_back((uint32_t)p);
  }
  return good;
}

void chain_len_sums(const std::vector<std::vector<ChainInterval>>& int_chunks, uint32_t c, size_t k, uint32_t* sum,
                    uint32_t* n) {  // chain.rs:244-249
  uint32_t s = 0, m = 0;
  for (const auto& v : int_chunks)
    for (const auto& in : v) { s += (in.q1 - in.q0) - in.overlap + 2 * c + (uint32_t)k; m += 1; }
  *sum = s; *n = m;
}

static AniEstResult calculate_ani(const std::vector<std::vector<ChainInterval>>& int_chunks, const Sketch& ref_sketch,
                                  const Sketch& query_sketch, const AnchorChunks& ac, const MapParams& mp, bool switched,
                                  ChainDebug* dbg) {  // chain.rs:173-555
  const size_t k = mp.k;
  std::vector<std::pair<double, size_t>> ani_ests;
  const uint32_t c = (uint32_t)ref_sketch.c;
  const bool sensitive_af = c < 200;
  uint32_t total_query_bases = 0, total_ref_range = 0;
  uint32_t avg_chain_int_len = 0, num_chains = 0;
  chain_len_sums(int_chunks, c, k, &avg_chain_int_len, &num_chains);  // :249
  if (sensitive_af) total_query_bases = total_ref_range = avg_chain_int_len;  // :244-247 add the same terms
  for (size_t i = 0; i < int_chunks.size(); i++) {
    const ChunkStats cs = chunk_stats(int_chunks[i], ac.seeds_in_chunk[i], c, k, mp.min_length_cover, switched);
    if (dbg) {
      const uint32_t row[9] = {(uint32_t)cs.total_anchors, cs.rq0, cs.rq1, cs.tbcq, cs.n_int, (uint32_t)cs.n_seeds,
                               (uint32_t)cs.num_in, (uint32_t)cs.upper_lower, cs.filtered ? 1u : 0u};
      dbg->chunk_stats.insert(dbg->chunk_stats.end(), row, row + 9);
    }
    if (!cs.valid) continue;                             // :253-259
    if (!sensitive_af) {                                 // :261-264
      total_query_bases += cs.rq1 - cs.rq0 + 2 * c + (uint32_t)k;
      total_ref_range += cs.rq1 - cs.rq0 + 2 * c + (uint32_t)k;
    }
    ani_ests.push_back({cs.est, cs.weight});             // :394
  }
  std::sort(ani_ests.begin(), ani_ests.end());  // :414 (f64, usize) lexicographic
  if (dbg) dbg->ani_ests = ani_ests;
  if (ani_ests.empty() || num_chains == 0) {  // :416-420
    AniEstResult r;
    r.ani = std::numeric_limits<float>::quiet_NaN();
    return r;
  }
  avg_chain_int_len /= num_chains;  // :421
  // total_ref_range == total_query_bases: both grow by the same amounts above
  std::vector<uint32_t> sq = query_sketch.contig_lengths, sr = ref_sketch.contig_lengths;
  std::sort(sq.begin(), sq.end());
  std::sort(sr.begin(), sr.end());
  const size_t ql = sq.size(), rl = sr.size();
  const float quant_q[3] = {(float)sq[ql * 10 / 100], (float)sq[ql * 50 / 100], (float)sq[ql * 90 / 100]};
  const float quant_r[3] = {(float)sr[rl * 10 / 100], (float)sr[rl * 50 / 100], (float)sr[rl * 90 / 100]};
  AniEstResult r = final_estimate(ani_ests, total_query_bases, avg_chain_int_len, query_sketch.total_sequence_length,
                                  ref_sketch.total_sequence_length, quant_q, quant_r, mp);
  r.num_contigs_r = (uint32_t)ref_sketch.contigs.size();
  r.num_contigs_q = (uint32_t)query_sketch.contigs.size();
  return r;
}

AniEstResult chain_seeds(const Sketch& ref, const Sketch& query, const MapParams& mp, ChainDebug* dbg) {  // chain.rs:144-171
  AnchorChunks ac;
  bool switched = get_anchors(ref, query, mp, ac, dbg ? &dbg->anchors : nullptr);
  std::vector<ChainInterval> good = chain_chunks(ac.chunks, mp, dbg ? &dbg->score : nullptr, dbg ? &dbg->pointer : nullptr);
  std::vector<uint8_t> kept;
  auto good_chunks = get_nonoverlapping_chains(good, ac.chunks.size(), dbg ? &kept : nullptr);
  if (dbg) {
    dbg->switched = switched;
    uint32_t off = 0;
    for (size_t i = 0; i < ac.chunks.size(); i++) {
      dbg->chunk_first.push_back(off);
      dbg->chunk_nseeds.push_back((uint32_t)ac.seeds_in_chunk[i].size());
      off += (uint32_t)ac.chunks[i].size();
    }
    dbg->chunk_first.push_back(off);
    dbg->intervals_all = good;
    dbg->interval_kept = kept;
  }
  return calculate_ani(good_chunks, ref, query, ac, mp, switched, dbg);
}

// ------------------------------------------------------------------------------------------------
// drivers
// ------------------------------------------------------------------------------------------------
static double now_s() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

std::vector<PairResult> triangle(const std::vector<const Sketch*>& sk, const CommandParams& cp, int threads,
                                 uint64_t* n_chained, double* t_screen, double* t_chain) {  // triangle.rs:13-169
  std::vector<PairResult> out;
  if (sk.empty()) return out;
  double screen_val = cp.screen_val == 0. ? SEARCH_ANI_CUTOFF_DEFAULT : cp.screen_val;  // triangle.rs:34-42
  double t0 = now_s();
  KmerToSketch* idx = kmer_to_sketch_from_refs(sk);  // triangle.rs:55
  int model = get_model_id(sk[0]->c, cp.learned_ani);
  std::vector<std::vector<uint32_t>> rows(sk.size());
  const long nrow = (long)sk.size() - 1;
  if (threads < 1) threads = 1;
#pragma omp parallel for schedule(dynamic, 4) num_threads(threads)
  for (long i = 0; i < nrow; i++) {  // triangle.rs:71-74
    auto pass = screen_refs(screen_val, *idx, *sk[i], sk, cp.rescue_small);
    for (uint32_t j : pass) if ((long)j > i) rows[i].push_back(j);  // triangle.rs:90
  }
  std::vector<std::pair<uint32_t, uint32_t>> pairs;
  for (long i = 0; i < nrow; i++) for (uint32_t j : rows[i]) pairs.push_back({(uint32_t)i, j});
  double t1 = now_s();
  std::vector<PairResult> res(pairs.size());
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads)
  for (long p = 0; p < (long)pairs.size(); p++) {
    const Sketch& ri = *sk[pairs[p].first];
    const Sketch& rj = *sk[pairs[p].second];
    MapParams mp = map_params_from_sketch(ri, cp, model);
    res[p].ref_id = pairs[p].first;
    res[p].query_id = pairs[p].second;
    res[p].r = chain_seeds(ri, rj, mp);  // triangle.rs:98
  }
  double t2 = now_s();
  for (auto& r : res) if (r.r.ani > 0.1f) out.push_back(r);  // triangle.rs:99 (NaN fails the compare)
  kmer_to_sketch_free(idx);
  if (n_chained) *n_chained = pairs.size();
  if (t_screen) *t_screen = t1 - t0;
  if (t_chain) *t_chain = t2 - t1;
  return out;
}

static std::vector<PairResult> query_ref_driver(const std::vector<const Sketch*>& refs, const std::vector<const Sketch*>& queries,
                                                const CommandParams& cp, bool use_index, int threads, bool is_search) {
  std::vector<PairResult> out;
  if (refs.empty() || queries.empty()) return out;
  double screen_val = cp.screen_val == 0. ? SEARCH_ANI_CUTOFF_DEFAULT : cp.screen_val;
  int model = get_model_id(refs[0]->c, cp.learned_ani);
  KmerToSketch* idx = use_index ? kmer_to_sketch_from_refs(refs) : nullptr;
  std::vector<std::pair<uint32_t, uint32_t>> pairs;  // (ref, query)
  for (size_t j = 0; j < queries.size(); j++) {
    const Sketch& q = *queries[j];
    if (!use_index) {
      for (size_t i = 0; i < refs.size(); i++) {
        // dist.rs:104-105 check_markers_quickly(query_sketch, ref_sketch, ..) / search.rs:127 (rescue_small = false)
        bool pass = check_markers_quickly(q, *refs[i], screen_val, is_search ? false : cp.rescue_small);
        if (pass) pairs.push_back({(uint32_t)i, (uint32_t)j});
      }
    } else {
      auto pass = is_search ? screen_refs_indices(screen_val, *idx, q, refs)            // search.rs:134-140
                            : screen_refs(screen_val, *idx, q, refs, cp.rescue_small);  // dist.rs:122-129
      for (uint32_t i : pass) pairs.push_back({i, (uint32_t)j});
    }
  }
  std::vector<PairResult> res(pairs.size());
  if (threads < 1) threads = 1;
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads)
  for (long p = 0; p < (long)pairs.size(); p++) {
    const Sketch& r = *refs[pairs[p].first];
    const Sketch& q = *queries[pairs[p].second];
    MapParams mp = map_params_from_sketch(r, cp, model);
    res[p].ref_id = pairs[p].first;
    res[p].query_id = pairs[p].second;
    res[p].r = chain_seeds(r, q, mp);
  }
  float keep = is_search ? 0.5f : 0.1f;  // search.rs:176 / dist.rs:115,139
  for (auto& r : res) if (r.r.ani > keep) out.push_back(r);
  if (idx) kmer_to_sketch_free(idx);
  return out;
}

std::vector<PairResult> dist(const std::vector<const Sketch*>& refs, const std::vector<const Sketch*>& queries,
                             const CommandParams& cp, bool use_index, int threads) {
  return query_ref_driver(refs, queries, cp, use_index, threads, false);
}
std::vector<PairResult> search(const std::vector<const Sketch*>& refs, const std::vector<const Sketch*>& queries,
                               const CommandParams& cp, bool use_index, int threads) {
  return query_ref_driver(refs, queries, cp, use_index, threads, true);
}

}  // namespace orc
